"""CPU restatement of sparse MLA decode (DeepSeek-V3.2 / GLM-5 layers with a lightning indexer), checker only, never the
product.

  convert          request-local top-k indices -> global cache slots: the reference's triton_convert_req_index_to_global_index
                   (v1/attention/backends/mla/sparse_utils.py:120-160) on its decode path: slot = page_table[req][idx // page]
                   * page + idx % page, -1 where idx < 0 or idx // page >= max_pages.
  ds_mla_quantize  the 656-byte fp8_ds_mla row of concat_and_cache_ds_mla_kernel (csrc/libtorch_stable/cache_kernels.cu:496-590):
                   per 128-dim tile scale = max(amax / 448, FLT_MIN) in fp32, e4m3(value / scale) (saturating), the four
                   fp32 scales at bytes 512-527, the 64 bf16 rope dims at bytes 528-655.
  ds_mla_dequantize  the row back to 576 bf16 values: bf16(float(e4m3) * scale), the fp32 product rounded once to bf16.
  mla_decode_sparse  gather of each token's valid slots and softmax attention in fp32, through oracle.moe_oracle.mla_decode.
Pinned to the reference by tests/golden/golden_mla_sparse.pt."""
from __future__ import annotations

import torch

from oracle import moe_oracle as O

__all__ = ["convert", "ds_mla_quantize", "ds_mla_dequantize", "mla_decode_sparse", "golden_w_uv"]

FLT_MIN = torch.finfo(torch.float32).tiny


def convert(req_id: torch.Tensor, page_table: torch.Tensor, topk_indices: torch.Tensor, page: int) -> torch.Tensor:
    """Global slot of every entry, int32 [T, topk]; -1 for an entry that names no key."""
    idx = topk_indices.long()
    blk = torch.div(idx, page, rounding_mode="floor")
    ok = (idx >= 0) & (blk < page_table.shape[1])
    rows = page_table.long()[req_id.long()]                       # [T, max_pages]
    base = torch.gather(rows, 1, torch.where(ok, blk, torch.zeros_like(blk)))
    return torch.where(ok, base * page + idx % page, torch.full_like(idx, -1)).int()


def ds_mla_quantize(kv_c: torch.Tensor, k_pe: torch.Tensor) -> torch.Tensor:
    """kv_c [N, 512], k_pe [N, 64] bf16 -> fp8_ds_mla rows uint8 [N, 656]."""
    N = kv_c.shape[0]
    x = kv_c.float().reshape(N, 4, 128)
    scale = torch.clamp(x.abs().amax(dim=-1) / 448.0, min=FLT_MIN)          # fp32 [N, 4]
    q8 = (x / scale[..., None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).reshape(N, 512)
    return torch.cat([q8.view(torch.uint8), scale.contiguous().view(torch.uint8).reshape(N, 16),
                      k_pe.to(torch.bfloat16).contiguous().view(torch.uint8).reshape(N, 128)], dim=1)


def ds_mla_dequantize(rows: torch.Tensor) -> torch.Tensor:
    """fp8_ds_mla rows uint8 [..., 656] -> bf16 [..., 576] (latent | rope)."""
    shp = rows.shape[:-1]
    r = rows.reshape(-1, 656).contiguous()
    scale = r[:, 512:528].contiguous().view(torch.float32)                   # [N, 4]
    lat = r[:, :512].contiguous().view(torch.float8_e4m3fn).float().reshape(-1, 4, 128) * scale[..., None]
    rope = r[:, 528:].contiguous().view(torch.bfloat16)
    return torch.cat([lat.reshape(-1, 512).bfloat16(), rope], dim=1).reshape(*shp, 576)


def mla_decode_sparse(q_nope: torch.Tensor, q_pe: torch.Tensor, kv_cache: torch.Tensor, topk_indices: torch.Tensor,
                      req_id: torch.Tensor, page_table: torch.Tensor, sm_scale: float):
    """q_nope [T,Hq,512], q_pe [T,Hq,64]; kv_cache bf16 [pages,page,576] or fp8_ds_mla uint8 [pages,page,656] (read through
    ds_mla_dequantize).  Token t attends to the cache rows convert() gives it (in index order, repeats included).  Returns
    out f32 [T,Hq,512], lse f32 [T,Hq]; a token with no valid entry gives out = 0, lse = -inf."""
    page = kv_cache.shape[1]
    flat = (ds_mla_dequantize(kv_cache) if kv_cache.dtype == torch.uint8 else kv_cache).reshape(-1, 576)
    slots = convert(req_id, page_table, topk_indices, page)
    T = q_nope.shape[0]
    out = torch.zeros(T, q_nope.shape[1], 512)
    lse = torch.zeros(T, q_nope.shape[1])
    for t in range(T):
        s = slots[t][slots[t] >= 0].long()
        # the token's keys as one page of a one-request paged cache
        kv = flat[s].float()[None] if s.numel() else torch.zeros(1, 1, 576)
        o, l = O.mla_decode(q_nope[t:t + 1].float(), q_pe[t:t + 1].float(), kv, torch.tensor([s.numel()]),
                            torch.zeros(1, 1, dtype=torch.int32), sm_scale)
        out[t], lse[t] = o[0], l[0]
    return out, lse


def golden_w_uv(hq: int) -> torch.Tensor:
    """The fixture's v up-projection W_UV [hq, 512, 128] bf16: a fixed integer pattern / 64 (exact in bf16), so that the
    fixture need not store 128 KB per head."""
    h = torch.arange(hq)[:, None, None]
    k = torch.arange(512)[None, :, None]
    n = torch.arange(128)[None, None, :]
    return (((h * 7 + k * 13 + n * 29 + (k * n) % 11) % 17) - 8).float().div(64.0).bfloat16()
