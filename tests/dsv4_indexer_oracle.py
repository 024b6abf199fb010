"""CPU restatement of the DeepSeek-V4 C4A indexer for decode and of V4's global key lists, checker only, never the product.

  q_quant        the fp8 path of _fused_indexer_q_rope_quant_kernel (vllm/models/deepseek_v4/common/ops/
                 fused_indexer_q.py:70-176): GPT-J pair RoPE of dims 64-127 (pair (64 + 2i, 65 + 2i), cos[i], sin[i] of an f32
                 cos | sin table) in fp32, each rotated value rounded to bf16; scale = 2^ceil(log2(fp32(max(amax, 1e-4) /
                 448))) over the 128 values; e4m3(clamp(x / scale, +-448)); weights_out = w * scale * softmax_scale *
                 head_scale in fp32.
  candidates     n_t = (p + 1) // ratio compressed rows for a token at position p (0 for p < 0).
  logits / topk  indexer_oracle.paged_logits / topk_rows with one row per token: seq_len n_t and page row
                 block_table[token_to_req[t]] (the reference's SparseAttnIndexer decode over the compressed cache).
  swa            _compute_swa_indices_and_lens_kernel (v1/attention/backends/mla/sparse_swa.py:744-800);
  c128a          the decode branch of _build_c128a_topk_metadata_kernel (models/deepseek_v4/sparse_mla.py:353-408);
  global_topk    _compute_global_topk_indices_and_lens_kernel (models/deepseek_v4/common/ops/cache_utils.py:477-525);
  slot_mapping   _compressed_slot_mapping_kernel (v1/attention/backends/mla/compressor_utils.py:8-50);
                 local index i -> block_table[req][i // bs] * bs + i % bs, and -1 where i // bs >= max_blocks (the
                 reference would read past the table's row there); -1 past a list's length; a token with slot_mapping < 0
                 gets length 0 and a row of -1 (the reference's rows of such tokens are unused).
  short_context  _fill_short_context_topk_indices (models/deepseek_v4/attention.py:72-86).
The decode over these lists is dsv4_sparse_oracle.decode.  Pinned to the reference by tests/golden/golden_dsv4_indexer.pt."""
from __future__ import annotations

import torch

import indexer_oracle as IX

__all__ = ["q_quant", "candidates", "logits", "topk", "swa", "c128a", "global_topk", "slot_mapping", "short_context"]

FP8 = torch.float8_e4m3fn


def q_quant(q: torch.Tensor, weights: torch.Tensor, positions: torch.Tensor, cos_sin: torch.Tensor, softmax_scale: float,
            head_scale: float):
    """q bf16 [T, H, 128], weights bf16 [T, H], cos_sin f32 [P, 64].  Returns (q_fp8 e4m3 [T, H, 128], weights_out f32)."""
    pos = positions.long().clamp(0, cos_sin.shape[0] - 1)
    cs = cos_sin.float()[pos]
    c, s = cs[:, None, :32], cs[:, None, 32:]
    x = q.float()
    x0, x1 = x[..., 64::2], x[..., 65::2]
    r0 = (x0 * c - x1 * s).bfloat16().float()
    r1 = (x1 * c + x0 * s).bfloat16().float()
    xr = torch.cat((x[..., :64], torch.stack((r0, r1), dim=-1).flatten(-2)), dim=-1)
    amax = xr.abs().amax(dim=-1)
    scale = IX.ue8m0_ceil(torch.clamp(amax, min=1e-4) / 448.0)
    q8 = (xr / scale[..., None]).clamp(-448.0, 448.0).to(FP8)
    w = weights.float() * scale * softmax_scale * head_scale
    return q8, w


def candidates(positions: torch.Tensor, ratio: int) -> torch.Tensor:
    p = positions.long()
    return torch.where(p < 0, torch.zeros_like(p), torch.div(p + 1, ratio, rounding_mode="floor")).int()


def logits(q_fp8, weights, k_cache, positions, token_to_req, block_table, ratio: int) -> torch.Tensor:
    """f64 [T, max_blocks * page]: the logits on [0, n_t), -inf elsewhere."""
    width = block_table.shape[1] * k_cache.shape[1]
    n = candidates(positions, ratio).clamp(max=width)
    return IX.paged_logits(q_fp8, weights, k_cache, n, block_table[token_to_req.long()], 1, width)


def topk(lg: torch.Tensor, positions: torch.Tensor, ratio: int, k: int) -> torch.Tensor:
    """int32 [T, k]: the k largest of [0, min(n_t, width)) ascending, ties to the lowest positions, -1 padding."""
    return IX.topk_rows(lg, candidates(positions, ratio), 1, k)


def short_context(positions: torch.Tensor, ratio: int, k: int) -> torch.Tensor:
    n = candidates(positions, ratio).long()
    j = torch.arange(k)
    return torch.where(j[None] < n[:, None], j[None], -1).int()


def _lookup(block_table: torch.Tensor, req: int, local: torch.Tensor, bs: int) -> torch.Tensor:
    col = torch.div(local, bs, rounding_mode="floor")
    ok = (local >= 0) & (col < block_table.shape[1])
    blk = block_table[req].long()[col.clamp(0, block_table.shape[1] - 1)]
    return torch.where(ok, blk * bs + local % bs, torch.full_like(local, -1))


def _lists(T, width, slot_map, token_to_req, block_table, bs, local_and_len):
    out = torch.full((T, width), -1, dtype=torch.int32)
    lens = torch.zeros(T, dtype=torch.int32)
    for t in range(T):
        if int(slot_map[t]) < 0:
            continue
        local, n = local_and_len(t)
        out[t] = _lookup(block_table, int(token_to_req[t]), local, bs).int()
        lens[t] = n
    return out, lens


def swa(positions, slot_map, token_to_req, block_table, bs: int, window: int):
    """(indices int32 [T, window], lens int32 [T])."""
    def f(t):
        p = int(positions[t])
        start = max(p - window + 1, 0)
        n = max(p + 1 - start, 0)
        j = torch.arange(window)
        return torch.where(j < n, start + j, torch.full_like(j, -1)), n
    return _lists(positions.numel(), window, slot_map, token_to_req, block_table, bs, f)


def c128a(positions, slot_map, token_to_req, block_table, bs: int, ratio: int, width: int):
    """(indices int32 [T, width], lens int32 [T])."""
    def f(t):
        p = int(positions[t])
        n = 0 if p < 0 else min((p + 1) // ratio, width)
        j = torch.arange(width)
        return torch.where(j < n, j, torch.full_like(j, -1)), n
    return _lists(positions.numel(), width, slot_map, token_to_req, block_table, bs, f)


def global_topk(local: torch.Tensor, slot_map, token_to_req, block_table, bs: int):
    """local int [T, k] -> (indices int32 [T, k], lens int32 [T] = entries >= 0)."""
    def f(t):
        row = local[t].long()
        return row, int((row >= 0).sum())
    return _lists(local.shape[0], local.shape[1], slot_map, token_to_req, block_table, bs, f)


def slot_mapping(positions, slot_map, token_to_req, block_table, bs: int, ratio: int) -> torch.Tensor:
    """int64 [T]: the slot of compressed row p // ratio for a token closing a window, else -1."""
    out = torch.full((positions.numel(),), -1, dtype=torch.int64)
    for t in range(positions.numel()):
        p = int(positions[t])
        if int(slot_map[t]) >= 0 and p >= 0 and (p + 1) % ratio == 0:
            out[t] = int(_lookup(block_table, int(token_to_req[t]), torch.tensor([p // ratio]), bs)[0])
    return out
