"""CPU restatement of multi-token (speculative-decode verification) MLA decode, checker only, never the product.

Query token i of request b attends to key positions [0, S_b - Q + i]: the end-aligned causal mask of the reference's FlashMLA
decode (causal=True; its test reference is scaled_dot_product_attention(..., is_causal=True) of
tests/kernels/attention/test_flashmla.py:138-155, mask tril(diagonal = s_k - s_q)).  Row (b, i) is therefore a single-token
decode over the first S_b - Q + 1 + i keys, and that is how it is computed here: through the oracle's mla_decode on the
expanded batch (page-table row repeated, seq_len S_b - Q + 1 + i).  With q_len = 1 the expanded batch is the batch itself.
Pinned to the reference by tests/golden/golden_mla_spec.pt."""
from __future__ import annotations

import torch

from gqa_spec_oracle import expand
from oracle import moe_oracle as O

__all__ = ["expand", "mla_decode"]


def mla_decode(q_nope: torch.Tensor, q_pe: torch.Tensor, kv_cache: torch.Tensor, seq_lens: torch.Tensor,
               page_table: torch.Tensor, sm_scale: float, q_len: int = 1):
    """q_nope [B*Q, Hq, 512], q_pe [B*Q, Hq, 64] (request b's Q tokens contiguous, in draft order), kv_cache
    [pages, page, 576], seq_lens [B] (all keys of request b, its Q new tokens included).  Returns out f32 [B*Q, Hq, 512],
    lse f32 [B*Q, Hq]; a row with no visible key gives out = 0, lse = -inf."""
    B = seq_lens.numel()
    assert q_nope.shape[0] == B * q_len and q_pe.shape[0] == B * q_len and page_table.shape[0] == B
    lens, pt = expand(seq_lens, page_table, q_len)
    return O.mla_decode(q_nope, q_pe, kv_cache, lens, pt, sm_scale)
