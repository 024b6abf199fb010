"""CPU restatement of the DeepSeek-V4 KV compressor (ops.dsv4_compress), float64 where it computes, checker only, never the
product.

  state_write  _save_partial_states_kernel (vllm/models/deepseek_v4/common/ops/save_partial_states.py:48-101): token t with
               s = slot_mapping[t] >= 0 writes row s of the state = kv | score + ape[position % ratio] (one fp32 add).
  rows         the compression of _fused_kv_compress_norm_rope_insert_sparse_attn / _indexer_attn
               (common/ops/fused_compress_quant_cache.py:113-297, 657-828): tokens with s >= 0 and (p + 1) % ratio == 0 pool
               the state rows of positions p - (1 + overlap) ratio + 1 .. p of their request (positions < 0: no row; with
               overlap the older ratio rows use columns [0, D), the newer [D, 2D)) by a per-column softmax of the scores;
               RMSNorm with the bf16 weight; GPT-J RoPE of the last 64 dims at (p // ratio) * ratio.  float64 rows.
  compress     the rows stored at kv_slot_mapping[t] (< 0 or past the cache: nothing): D 512 by dsv4_sparse_oracle.pack
               (the 584-byte row), D 128 by indexer_oracle.k_quant_cache(ue8m0=True) (the 132-byte row), both rounding the
               row to bf16 first.
Pinned to the reference by tests/golden/golden_dsv4_compress.pt."""
from __future__ import annotations

import torch

import dsv4_sparse_oracle as V4
import indexer_oracle as IX

__all__ = ["state_write", "rows", "compress", "coff"]


def coff(ratio: int) -> int:
    return 2 if ratio == 4 else 1


def state_write(kv_score: torch.Tensor, ape: torch.Tensor, positions: torch.Tensor, slot_mapping: torch.Tensor,
                state: torch.Tensor) -> torch.Tensor:
    """kv_score f32 [T, 2 * half], ape f32 [ratio, half], state f32 [blocks, block_size, 2 * half], written in place."""
    half = ape.shape[1]
    ratio = ape.shape[0]
    flat = state.view(-1, 2 * half)
    for t in range(kv_score.shape[0]):
        s = int(slot_mapping[t])
        if s < 0:
            continue
        flat[s, :half] = kv_score[t, :half].float()
        flat[s, half:] = kv_score[t, half:2 * half].float() + ape[int(positions[t]) % ratio].float()
    return state


def rows(state: torch.Tensor, block_table: torch.Tensor, token_to_req: torch.Tensor, positions: torch.Tensor,
         slot_mapping: torch.Tensor, norm_weight: torch.Tensor, eps: float, cos_sin: torch.Tensor, ratio: int):
    """{token: float64 row [D]} for every token that compresses (the kv slot is not looked at)."""
    D = norm_weight.numel()
    half = coff(ratio) * D
    sbs = state.shape[1]
    W = coff(ratio) * ratio
    flat = state.view(-1, 2 * half).double()
    w = norm_weight.double()
    out = {}
    for t in range(positions.numel()):
        p = int(positions[t])
        if int(slot_mapping[t]) < 0 or p < 0 or (p + 1) % ratio != 0:
            continue
        kv = torch.zeros(W, D, dtype=torch.float64)
        sc = torch.full((W, D), -float("inf"), dtype=torch.float64)
        bt = block_table[int(token_to_req[t])]
        for i in range(W):
            q = p - W + 1 + i
            if q < 0:
                continue
            r = flat[int(bt[q // sbs]) * sbs + q % sbs]
            c0 = D if (W > ratio and i >= ratio) else 0
            kv[i], sc[i] = r[c0:c0 + D], r[half + c0:half + c0 + D]
        c = (torch.softmax(sc, dim=0) * kv).sum(0)
        x = c * torch.rsqrt((c * c).mean() + eps) * w
        cp = min((p // ratio) * ratio, cos_sin.shape[0] - 1)
        cs = cos_sin[cp].double()
        e, o = x[D - 64::2].clone(), x[D - 63::2].clone()
        x[D - 64::2] = e * cs[:32] - o * cs[32:]
        x[D - 63::2] = o * cs[:32] + e * cs[32:]
        out[t] = x
    return out


def compress(state, block_table, token_to_req, positions, slot_mapping, norm_weight, eps, cos_sin, ratio, kv_slot_mapping,
             kv_cache):
    """Writes the rows into kv_cache (uint8 [blocks, block_size, 584 or 132]) in place; returns rows()."""
    r = rows(state, block_table, token_to_req, positions, slot_mapping, norm_weight, eps, cos_sin, ratio)
    nslots = kv_cache.shape[0] * kv_cache.shape[1]
    for t, x in r.items():
        s = int(kv_slot_mapping[t])
        if s < 0 or s >= nslots:
            continue
        if kv_cache.shape[2] == 584:
            V4.pack(x.bfloat16()[None], kv_cache.shape[1], torch.tensor([s]), kv_cache)
        else:
            IX.k_quant_cache(x.bfloat16()[None], torch.tensor([s]), kv_cache, True)
    return r


def _scales(x: torch.Tensor, block: int) -> torch.Tensor:
    """The ue8m0 scale exponent of each quant block of the bf16-rounded rows x [n, D]."""
    a = x.bfloat16().float().abs().reshape(x.shape[0], -1, block).amax(-1)
    return torch.log2(IX.ue8m0_ceil(torch.clamp(a, min=V4.EPS_AMAX) / 448.0))


def _near_power_of_two(x: torch.Tensor, block: int) -> torch.Tensor:
    """Quant blocks of the bf16-rounded row x [D] whose max(amax, 1e-4) / 448 lies within 2^-20 of a power of two.  A bf16
    amax of 1.75 * 2^k makes it one exactly, and the reference's amax * fp32(1 / 448) then rounds above it: its ceiling,
    and so its scale, is one step larger than that of the exact quotient."""
    a = x.bfloat16().double().abs().reshape(-1, block).amax(-1).clamp(min=V4.EPS_AMAX) / 448.0
    return (a / torch.pow(2.0, torch.round(torch.log2(a))) - 1).abs() < 2.0 ** -20


def ambiguous_blocks(x: torch.Tensor, block: int) -> torch.Tensor:
    """Quant blocks of the float64 row x [D] whose scale an fp32 rounding decides: it changes when x is scaled by
    1 -+ 2^-20, or its amax / 448 is within 2^-20 of a power of two."""
    return (_scales(x[None] * (1 + 2 ** -20), block) != _scales(x[None] * (1 - 2 ** -20), block))[0] | \
        _near_power_of_two(x, block)


def _e4m3_key(b: torch.Tensor) -> torch.Tensor:
    """e4m3 codes as ordered integers (sign-magnitude; +0 and -0 both 0), so that one code step is a difference of 1."""
    i = b.to(torch.int64)
    return torch.where(i >= 128, -(i - 128), i)


def check_cache(got: torch.Tensor, ref: torch.Tensor, rows_: dict, kv_slot_mapping: torch.Tensor) -> int:
    """Compare a compressed cache with the oracle's (same initial bytes): bytes outside the rows the oracle wrote are
    equal; in a written row the scales are equal and the e4m3 codes within one code step, except in the quant blocks of
    ambiguous_blocks; rope dims within one bf16 ulp.  Returns the number of exempt blocks."""
    nb, bs, row = ref.shape
    D, block = (512, 64) if row == 584 else (128, 128)
    mask = torch.zeros(nb, bs * row, dtype=torch.bool)
    exempt = 0
    for t, x in rows_.items():
        s = int(kv_slot_mapping[t])
        if s < 0 or s >= nb * bs:
            continue
        b, p = s // bs, s % bs
        gb, rb = got[b].reshape(-1), ref[b].reshape(-1)
        amb = ambiguous_blocks(x, block)
        exempt += int(amb.sum())
        if row == 584:
            data, rec = slice(p * 576, p * 576 + 448), slice(bs * 576 + p * 8, bs * 576 + p * 8 + 8)
            rope = slice(p * 576 + 448, p * 576 + 576)
            keep = ~amb[:7].repeat_interleave(64)
            sg, sr = gb[rec], rb[rec]
            assert torch.equal(sg[:7][~amb[:7]], sr[:7][~amb[:7]]) and int(sg[7]) == int(sr[7]) == 0, (t, sg, sr)
            assert int(V4.bf16_ulp_distance(gb[rope].contiguous().view(torch.bfloat16),
                                            rb[rope].contiguous().view(torch.bfloat16)).max()) <= 1, t
            mask[b, rope] = True
        else:
            data, rec = slice(p * 128, p * 128 + 128), slice(bs * 128 + p * 4, bs * 128 + p * 4 + 4)
            keep = (~amb[0]).repeat(128)
            if not amb[0]:
                assert torch.equal(gb[rec], rb[rec]), t
        d = (_e4m3_key(gb[data]) - _e4m3_key(rb[data])).abs()
        assert int(d[keep].max()) <= 1 if keep.any() else True, (t, int(d[keep].max()))
        mask[b, data] = True
        mask[b, rec] = True
    g, r = got.reshape(nb, -1), ref.reshape(nb, -1)
    assert torch.equal(g[~mask], r[~mask])
    return exempt
