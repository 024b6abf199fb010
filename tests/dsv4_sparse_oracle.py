"""CPU restatement of DeepSeek-V4 sparse attention decode and its cache insert, float64 where it computes, checker only, never
the product.

  pack      kv bf16 [N, 512] -> the 584-byte-per-token cache, uint8 [blocks, block_size, 584] (a padded block stride is kept):
            the reference's quantize_and_insert_k_kernel (vllm/models/deepseek_v4/common/ops/cache_utils.py:37-160).  Per 64
            NoPE dims scale = 2^ceil(log2(max(amax, 1e-4) / 448)) (fp32 quotient; the ceiling is exact, see _ue8m0_byte),
            e4m3(x / scale) saturating, ue8m0 byte log2(scale) + 127, pad byte 0; rope dims stored as bf16.  Block layout of
            flashmla_sparse.py:76-85: block_size x 576 data bytes (448 e4m3 | 64 bf16) then block_size x 8 scale bytes.
  read      one slot back to 512 values: _read_fp8_ds_mla_cache (tests/kernels/attention/test_rocm_triton_attn_dsv4.py:125-147),
            float(e4m3) * 2^(s - 127) | rope.
  decode    _ref_sparse_decode_ragged with sinks (same file :150-190) over the lists the FlashMLA call passes
            (models/deepseek_v4/nvidia/flashmla.py:151-244): swa_indices[t, :swa_lens[t]] then extra_indices[t, :extra_lens[t]],
            a slot < 0 or past its cache skipped; a token with no valid key gets 0 (as _ref_sparse_prefill_ragged, :61-88).
  insert    fused_deepseek_v4_qnorm_rope_kv_rope_quant_insert (csrc/libtorch_stable/fused_deepseek_v4_qnorm_rope_kv_insert_kernel.cu
            :179-379; torch statements in tests/kernels/test_fused_deepseek_v4_qnorm_rope_kv_insert.py:51-124): q RMSNorm without
            weight then GPT-J RoPE of the last 64 dims, rounded to bf16 once, padded heads zero; kv RoPE, rounded to bf16,
            packed into slot_mapping[t] (< 0: nothing).
Pinned to the reference by tests/golden/golden_dsv4_sparse.pt."""
from __future__ import annotations

import torch

__all__ = ["pack", "read", "dequant_all", "decode", "insert", "rope_gptj", "bf16_ulp_distance", "HEAD_BYTES"]

NOPE, ROPE, HEAD_BYTES = 448, 64, 584
EPS_AMAX = float(torch.tensor(1e-4, dtype=torch.float32))   # the fp32 1e-4 of fmaxf(amax, 1e-4f)


def _ue8m0_byte(amax: torch.Tensor) -> torch.Tensor:
    """ceil(log2(fp32(max(amax, 1e-4) / 448))) + 127, exactly.  amax is a bf16 value (8-bit mantissa), so the fp32 quotient is a
    power of two only when it is exactly one; frexp gives the ceiling without rounding a log2."""
    r = (torch.clamp(amax.to(torch.float32), min=EPS_AMAX) / 448.0).double()
    m, e = torch.frexp(r)                       # r = m * 2^e, m in [0.5, 1)
    return (e - (m == 0.5).to(e.dtype) + 127).to(torch.int64)


def _block_bytes(cache: torch.Tensor, b: int) -> torch.Tensor:
    return cache[b].reshape(-1)   # [block_size * 584] bytes of block b (a view, also for a padded block stride)


def pack(kv: torch.Tensor, block_size: int, slots: torch.Tensor | None = None, cache: torch.Tensor | None = None,
         num_blocks: int | None = None) -> torch.Tensor:
    """Quantise kv bf16 [N, 512] into rows slots[i] (default 0..N-1) of cache (zeros [num_blocks, block_size, 584] if None)."""
    N = kv.shape[0]
    slots = torch.arange(N) if slots is None else slots.reshape(-1).long()
    if cache is None:
        nb = num_blocks or max(1, -(-(int(slots.max()) + 1) // block_size))
        cache = torch.zeros(nb, block_size, HEAD_BYTES, dtype=torch.uint8)
    x = kv.to(torch.bfloat16).float()
    for i in range(N):
        s = int(slots[i])
        if s < 0 or s >= cache.shape[0] * block_size:
            continue
        blk, pos = _block_bytes(cache, s // block_size), s % block_size
        g = x[i, :NOPE].reshape(7, 64)
        e = _ue8m0_byte(g.abs().amax(dim=-1))                       # [7]
        inv = torch.pow(2.0, (127 - e).double()).float()            # exact
        q8 = (g * inv[:, None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8).reshape(-1)
        blk[pos * 576:pos * 576 + NOPE] = q8
        blk[pos * 576 + NOPE:pos * 576 + 576] = x[i, NOPE:].bfloat16().view(torch.uint8)
        rec = block_size * 576 + pos * 8
        blk[rec:rec + 7] = e.to(torch.uint8)
        blk[rec + 7] = 0
    return cache


def read(cache: torch.Tensor, slot: int, block_size: int) -> torch.Tensor:
    """float64 [512] of one slot: float(e4m3) * 2^(s - 127) for the NoPE dims, then the bf16 rope dims."""
    blk, pos = _block_bytes(cache, slot // block_size), slot % block_size
    nope = blk[pos * 576:pos * 576 + NOPE].contiguous().view(torch.float8_e4m3fn).double()
    s = blk[block_size * 576 + pos * 8:block_size * 576 + pos * 8 + 7].double()
    nope = nope * torch.pow(2.0, s - 127.0).repeat_interleave(64)
    rope = blk[pos * 576 + NOPE:pos * 576 + 576].contiguous().view(torch.bfloat16).double()
    return torch.cat([nope, rope])


def dequant_all(cache: torch.Tensor) -> torch.Tensor:
    """float64 [blocks * block_size, 512]: every slot of the cache."""
    nb, bs, _ = cache.shape
    flat = torch.stack([_block_bytes(cache, b) for b in range(nb)])           # [nb, bs * 584]
    data = flat[:, :bs * 576].reshape(nb * bs, 576)
    s = flat[:, bs * 576:].reshape(nb * bs, 8)[:, :7].double()
    nope = data[:, :NOPE].contiguous().view(torch.float8_e4m3fn).double() * torch.pow(2.0, s - 127.0).repeat_interleave(64, 1)
    return torch.cat([nope, data[:, NOPE:].contiguous().view(torch.bfloat16).double()], dim=1)


def _valid(cache, idx_row, n):
    nslots = cache.shape[0] * cache.shape[1]
    return [int(s) for s in idx_row[:max(0, min(int(n), idx_row.numel()))] if 0 <= int(s) < nslots]


def decode(q, swa_cache, swa_indices, swa_lens, scale, attn_sink=None, extra_cache=None, extra_indices=None, extra_lens=None,
           swa_rows=None, extra_rows=None):
    """float64 out [T, Hq, 512].  swa_rows / extra_rows: dequant_all of the caches, if the caller has them already."""
    T, Hq, _ = q.shape
    qd = q.double()
    swa_rows = dequant_all(swa_cache) if swa_rows is None else swa_rows
    if extra_cache is not None and extra_rows is None:
        extra_rows = dequant_all(extra_cache)
    out = torch.zeros(T, Hq, 512, dtype=torch.float64)
    for t in range(T):
        kv = [swa_rows[_valid(swa_cache, swa_indices[t], swa_lens[t])]]
        if extra_cache is not None:
            kv.append(extra_rows[_valid(extra_cache, extra_indices[t], extra_lens[t])])
        kv = torch.cat(kv)
        if kv.shape[0] == 0:
            continue
        s = (qd[t] @ kv.T) * scale                                   # [Hq, n]
        if attn_sink is not None:
            s = torch.cat([s, attn_sink.double().reshape(Hq, 1)], dim=1)
            p = torch.softmax(s, dim=1)[:, :-1]
        else:
            p = torch.softmax(s, dim=1)
        out[t] = p @ kv
    return out


def rope_gptj(x: torch.Tensor, positions: torch.Tensor, cos_sin: torch.Tensor) -> torch.Tensor:
    """GPT-J pair RoPE of the last 64 dims of x [..., 512] (float64), (cos | sin)[position] of the f32 cache."""
    cs = cos_sin.double()[positions.long()]                           # [T, 64]
    c, s = cs[:, :32], cs[:, 32:]
    if x.dim() == 3:                                                  # [T, H, 512]: one position per token
        c, s = c[:, None], s[:, None]
    out = x.clone()
    e, o = x[..., NOPE::2], x[..., NOPE + 1::2]
    out[..., NOPE::2] = e * c - o * s
    out[..., NOPE + 1::2] = e * s + o * c
    return out


def insert(q, kv, positions, cos_sin, slot_mapping, cache, q_head_padded, eps):
    """Returns q_out bf16 [T, q_head_padded, 512]; writes the kv rows into cache in place."""
    T, Hq, _ = q.shape
    x = q.double()
    x = x * torch.rsqrt((x * x).mean(dim=-1, keepdim=True) + eps)
    q_out = torch.zeros(T, q_head_padded, 512, dtype=torch.bfloat16)
    q_out[:, :Hq] = rope_gptj(x, positions, cos_sin).bfloat16()
    kvr = rope_gptj(kv.double(), positions, cos_sin).bfloat16()
    pack(kvr, cache.shape[1], slot_mapping, cache)
    return q_out


def bf16_ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Distance in bf16 steps between two bf16 tensors of the same sign pattern (ordered-integer difference)."""
    def key(t):
        i = t.contiguous().view(torch.int16).to(torch.int64)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (key(a.bfloat16()) - key(b.bfloat16())).abs()

