"""CPU restatement of the DeepSeek-V3.2 lightning indexer for decode, checker only, never the product.

  ue8m0_ceil         the power of two >= x, from the exponent bits: the reference's exp2(ceil(log2(x))) (the ue8m0 scale
                     format; sparse_attn_indexer.py:185, cache_kernels.cu:643-645) evaluated exactly.
  q_rope_quant       _fused_indexer_q_rope_quant_kernel (sparse_attn_indexer.py:127-251): RoPE of dims 0..63 in fp32, each
                     rotated value rounded to bf16; q_scale = ue8m0_ceil(max(amax, 1e-10) * (1 / 448)) over the 128 dims;
                     e4m3(clamp(x / q_scale, +-448)); weights_out = weight * q_scale * softmax_scale * head_scale in fp32.
  k_rope             RotaryEmbedding.forward_static on k[:, :64] in bf16 arithmetic (oracle.moe_oracle.apply_rotary_emb).
  k_quant_cache      indexer_k_quant_and_cache (csrc/libtorch_stable/cache_kernels.cu:599-659): scale = max(amax, 1e-4) / 448
                     (ue8m0_ceil of it when ue8m0), byte = e4m3(k / scale) saturating, into the [blocks, block_size, 132]
                     cache: block_size x 128 value bytes, then block_size fp32 scales; slot < 0 writes nothing.
  paged_logits       fp8_paged_mqa_logits_torch (rocm_aiter_mla_sparse.py:264-363) / the reference test's
                     _ref_fp8_fp4_paged_mqa_logits (tests/kernels/attention/test_deepgemm_attention.py:153-200):
                     logit[b*Q + i, j] = k_scale[j] * sum_h w[b*Q + i, h] * relu(q8 . k8_j) for j <= S_b - Q + i, in float64
                     over the exact e4m3 values, -inf elsewhere.
  topk_rows          top_k_per_row_decode (sampler.cu:567-614, 661-720): row_end = max(0, S_b - Q + i + 1); the topk largest
                     of [0, row_end) in ascending position order, ties (-0 equals +0) to the lowest positions, -1 padding;
                     row_end <= topk gives 0 .. row_end - 1.
Pinned to the reference by tests/golden/golden_indexer.pt."""
from __future__ import annotations

import math

import torch

from oracle import moe_oracle as O

__all__ = ["ue8m0_ceil", "q_rope_quant", "k_rope", "k_quant_cache", "k_cache_rows", "paged_logits", "topk_rows"]

FP8 = torch.float8_e4m3fn


def ue8m0_ceil(x: torch.Tensor) -> torch.Tensor:
    """Smallest power of two >= x for positive normal fp32 x, exactly (bit arithmetic on the exponent)."""
    b = x.float().contiguous().view(torch.int32).long()
    e = (b >> 23) + ((b & 0x7FFFFF) != 0).long()
    return (e << 23).int().view(torch.float32)


def _rope_pairs(x: torch.Tensor, is_neox: bool):
    return (x[..., :32], x[..., 32:64]) if is_neox else (x[..., 0:64:2], x[..., 1:64:2])


def _join(o1, o2, is_neox: bool):
    return torch.cat((o1, o2), dim=-1) if is_neox else torch.stack((o1, o2), dim=-1).flatten(-2)


def q_rope_quant(q: torch.Tensor, weights: torch.Tensor, positions: torch.Tensor, cos_sin: torch.Tensor, is_neox: bool,
                 softmax_scale: float, head_scale: float):
    """q bf16 [T,H,128], weights [T,H] (bf16), cos_sin bf16 [P, 64].  Returns (q_fp8 e4m3 [T,H,128], weights_out f32)."""
    pos = positions.long().clamp(0, cos_sin.shape[0] - 1)
    cs = cos_sin.float()[pos]
    c, s = cs[:, None, :32], cs[:, None, 32:]
    x = q.float()
    x0, x1 = _rope_pairs(x, is_neox)
    r0 = (x0 * c - x1 * s).bfloat16().float()
    r1 = (x1 * c + x0 * s).bfloat16().float()
    xr = torch.cat((_join(r0, r1, is_neox), x[..., 64:]), dim=-1)
    amax = xr.abs().amax(dim=-1)
    scale = ue8m0_ceil(torch.clamp(amax, min=1e-10) * (1.0 / 448.0))
    q8 = (xr / scale[..., None]).clamp(-448.0, 448.0).to(FP8)
    w = weights.float() * scale * softmax_scale * head_scale
    return q8, w


def k_rope(k: torch.Tensor, positions: torch.Tensor, cos_sin: torch.Tensor, is_neox: bool) -> torch.Tensor:
    """k bf16 [T,128] -> bf16 [T,128], dims 0..63 rotated in bf16 arithmetic (forward_static)."""
    pos = positions.long().clamp(0, cos_sin.shape[0] - 1)
    cos, sin = cos_sin[pos].chunk(2, dim=-1)
    rot = O.apply_rotary_emb(k[:, None, :64], cos, sin, is_neox)[:, 0]
    return torch.cat((rot, k[:, 64:]), dim=-1)


def k_quant(k: torch.Tensor, ue8m0: bool):
    """k bf16 [N,128] -> (e4m3 [N,128], fp32 scales [N])."""
    x = k.float()
    scale = torch.clamp(x.abs().amax(dim=-1), min=1e-4) / 448.0
    if ue8m0:
        scale = ue8m0_ceil(scale)
    return (x / scale[:, None]).clamp(-448.0, 448.0).to(FP8), scale


def k_quant_cache(k: torch.Tensor, slot_mapping: torch.Tensor, k_cache: torch.Tensor, ue8m0: bool) -> torch.Tensor:
    """Write rows of k (bf16 [T,128], already rotated) into k_cache uint8 [blocks, block_size, 132] in place; slots
    are distinct."""
    bs = k_cache.shape[1]
    flat = k_cache.view(-1)
    q8, scale = k_quant(k, ue8m0)
    keep = slot_mapping.reshape(-1) >= 0
    sl = slot_mapping.reshape(-1)[keep].long()
    base = torch.div(sl, bs, rounding_mode="floor") * (bs * 132)
    off = sl % bs
    flat[((base + off * 128)[:, None] + torch.arange(128)).reshape(-1)] = q8[keep].view(torch.uint8).reshape(-1)
    flat[((base + bs * 128 + off * 4)[:, None] + torch.arange(4)).reshape(-1)] = \
        scale[keep].contiguous().view(torch.uint8).reshape(-1)
    return k_cache


def k_cache_rows(k_cache: torch.Tensor):
    """uint8 [blocks, block_size, 132] -> (values f64 [blocks, block_size, 128], scales f64 [blocks, block_size])."""
    nb, bs, _ = k_cache.shape
    flat = k_cache.reshape(nb, bs * 132)
    vals = flat[:, :bs * 128].contiguous().view(FP8).double().reshape(nb, bs, 128)
    scales = flat[:, bs * 128:].contiguous().view(torch.float32).double().reshape(nb, bs)
    return vals, scales


def paged_logits(q_fp8: torch.Tensor, weights: torch.Tensor, k_cache: torch.Tensor, seq_lens: torch.Tensor,
                 page_table: torch.Tensor, q_len: int, width: int) -> torch.Tensor:
    """q_fp8 e4m3 [B*Q,H,128], weights [B*Q,H].  Returns f64 [B*Q, width]: the logits on [0, row_end), -inf elsewhere."""
    nb, bs, _ = k_cache.shape
    flat = k_cache.reshape(nb, bs * 132)
    B, Q = seq_lens.numel(), q_len
    out = torch.full((B * Q, width), -math.inf, dtype=torch.float64)
    q = q_fp8.double()
    w = weights.double()
    for b in range(B):
        S = int(seq_lens[b])
        npg = -(-S // bs)
        if npg == 0:
            continue
        rows = flat[page_table[b, :npg].long()]
        kv = rows[:, :bs * 128].contiguous().view(FP8).double().reshape(npg * bs, 128)
        ks = rows[:, bs * 128:].contiguous().view(torch.float32).double().reshape(npg * bs)
        for i in range(Q):
            r = b * Q + i
            end = max(0, S - Q + i + 1)
            if end == 0:
                continue
            s = torch.relu(q[r] @ kv[:end].T)                    # [H, end]
            out[r, :end] = (w[r][:, None] * s).sum(0) * ks[:end]
    return out


def topk_rows(logits: torch.Tensor, seq_lens: torch.Tensor, q_len: int, topk: int) -> torch.Tensor:
    """int32 [B*Q, topk]: per row the topk largest of [0, row_end) in ascending position order, ties to the lowest
    positions, -1 padding."""
    B, Q = seq_lens.numel(), q_len
    out = torch.full((B * Q, topk), -1, dtype=torch.int32)
    for r in range(B * Q):
        end = min(max(0, int(seq_lens[r // Q]) - Q + r % Q + 1), logits.shape[1])
        if end <= topk:
            out[r, :end] = torch.arange(end, dtype=torch.int32)
            continue
        # a stable descending sort keeps equal values in position order: the first topk are the lowest-position winners
        order = torch.sort(logits[r, :end], descending=True, stable=True).indices[:topk]
        out[r] = order.sort().values.int()
    return out
