"""CPU restatement of multi-token (speculative-decode verification) GQA decode, checker only, never the product.

Query token i of request b attends to key positions [0, S_b - Q + i]: the end-aligned causal mask of the reference's
ref_paged_attn (tests/kernels/attention/test_flashinfer.py:29-80) with query_lens = [Q] * B.  Row (b, i) is therefore a
single-token decode over the first S_b - Q + 1 + i keys, and that is how it is computed here: through the oracle's
gqa_decode on the expanded batch (page-table row repeated, seq_len S_b - Q + 1 + i).  With q_len = 1 the expanded batch
is the batch itself.  Pinned to the reference by tests/golden/golden_gqa_spec.pt."""
from __future__ import annotations

import torch

from oracle import moe_oracle as O


def expand(seq_lens: torch.Tensor, page_table: torch.Tensor, q_len: int):
    """(seq_lens, page_table) of the expanded batch: one single-token request per query row (b, i), b * q_len + i,
    seeing S_b - q_len + 1 + i keys (0 when that is not positive)."""
    sl = seq_lens.reshape(-1).to(torch.int64)
    i = torch.arange(q_len, dtype=torch.int64)
    lens = (sl[:, None] - q_len + 1 + i[None, :]).clamp_min(0).reshape(-1).to(torch.int32)
    return lens, page_table.repeat_interleave(q_len, dim=0)


def gqa_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, seq_lens: torch.Tensor,
               page_table: torch.Tensor, sm_scale: float, q_len: int = 1):
    """q [B*Q, Hq, D] (request b's Q tokens contiguous, in draft order), caches [pages, page, Hkv, D], seq_lens [B] (all
    keys of request b, its Q new tokens included).  Returns out f32 [B*Q, Hq, D], lse f32 [B*Q, Hq]; a row with no
    visible key gives out = 0, lse = -inf."""
    B = seq_lens.numel()
    assert q.shape[0] == B * q_len and page_table.shape[0] == B
    lens, pt = expand(seq_lens, page_table, q_len)
    return O.gqa_decode(q, k_cache, v_cache, lens, pt, sm_scale)
