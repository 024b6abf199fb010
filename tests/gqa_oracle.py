"""CPU restatements of the GQA attention-block ops around the decode kernel (checker only, never the product):
Qwen3's per-head q/k RMSNorm + RoPE and the paged cache write of the FlashInfer backend.  Built on the oracle's
rms_norm / rope_forward_static, which are pinned to the reference's own ops by golden fixtures."""
from __future__ import annotations

import torch

from oracle import moe_oracle as O


def qk_norm_rope(qkv: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor, num_heads: int,
                 num_kv_heads: int, head_dim: int, rotary_dim: int, q_weight: torch.Tensor | None,
                 k_weight: torch.Tensor | None, eps: float, is_neox: bool) -> torch.Tensor:
    """reference tests/kernels/core/test_fused_qk_norm_rope.py:21-47 (_apply_qk_norm_rope): split the packed qkv rows,
    per-head RMSNorm of q and k (skipped when the weight is None: no q/k norm, Mixtral), RoPE of q and k
    (RotaryEmbedding.forward_static), concatenation [q | k | v].  qkv [T, (Hq + 2 Hkv) * head_dim]."""
    q, k, v = qkv.split([num_heads * head_dim, num_kv_heads * head_dim, num_kv_heads * head_dim], dim=-1)
    if q_weight is not None:
        q = O.rms_norm(q.reshape(*q.shape[:-1], num_heads, head_dim), q_weight, eps).reshape(q.shape)
    if k_weight is not None:
        k = O.rms_norm(k.reshape(*k.shape[:-1], num_kv_heads, head_dim), k_weight, eps).reshape(k.shape)
    q, k = O.rope_forward_static(positions, q, k, head_dim, rotary_dim, cos_sin_cache, is_neox)
    return torch.cat([q, k, v], dim=-1)


def reshape_and_cache_flash(key: torch.Tensor, value: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
                            slot_mapping: torch.Tensor):
    """reference csrc/libtorch_stable/cache_kernels.cu:315-400 (bf16 cache, no scaling): key / value [T, Hkv, D] go to
    row slot_mapping[t] (block = slot // block_size, offset = slot % block_size; slot < 0 = padded token, skipped) of
    k_cache / v_cache, the [blocks, block_size, Hkv, D] views the FlashInfer backend passes (flashinfer.py:2276-2290), so
    that the NHD and HND packed caches are both written through their strides.  The rows are those of
    tests/kernels/attention/test_cache.py:406-414.  Writes in place; returns (k_cache, v_cache)."""
    bs = k_cache.shape[1]
    for t in range(key.shape[0]):
        s = int(slot_mapping[t])
        if s < 0:
            continue
        k_cache[s // bs, s % bs] = key[t]
        v_cache[s // bs, s % bs] = value[t]
    return k_cache, v_cache
