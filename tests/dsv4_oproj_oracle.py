"""Oracle of the DeepSeek-V4 attention output projection (ops.dsv4_inv_rope_quant, ops.dsv4_o_proj).

inv_rope_quant restates the C contract exactly: the inverse GPT-J rotation of dims 448-511 in fp32 with every product and
sum rounded on its own (no FMA), the block scale 2^ceil(log2(max(absmax, 1e-10) * fp32(1 / 448))) with the ceiling taken
from the fp32 bits, and e4m3 codes of x / scale, clamped to +-448.  Its bytes are the kernel's bytes.
wo_a is the float64 GEMM on given fp8 operands: per k-block the exact sum of code products, times both scales, summed
over k-blocks.  It also returns sum |a * w| * scales per output, which bounds the rounding of any fp32 / tensor-core
evaluation of the same sum.  Runs on whatever device its inputs are on."""
import torch

NOPE, ROT, HEAD = 448, 64, 512


def ue8m0_ceil(x: torch.Tensor) -> torch.Tensor:
    """Smallest power of two >= x (positive normal f32), from the exponent bits."""
    b = x.contiguous().view(torch.int32)
    e = (b >> 23) + ((b & 0x7FFFFF) != 0).to(torch.int32)
    return (e << 23).view(torch.float32)


def inv_rope(o: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor) -> torch.Tensor:
    """f32 [T, H, 512]: o with the inverse rotation of its last 64 dims, not rounded to bf16."""
    pos = positions.reshape(-1).long().clamp(0, cos_sin_cache.shape[0] - 1)
    cs = cos_sin_cache[pos]
    c, s = cs[:, None, :ROT // 2], cs[:, None, ROT // 2:]
    x = o.float().clone()
    xe, xo = x[..., NOPE::2].clone(), x[..., NOPE + 1::2].clone()
    x[..., NOPE::2] = (xe * c) + (xo * s)
    x[..., NOPE + 1::2] = (xo * c) - (xe * s)
    return x


def inv_rope_quant(o: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor, n_groups: int):
    """(o_fp8 e4m3 [T, G, D], o_scale f32 [T, G, D / 128]) as b200_dsv4_inv_rope_quant defines them."""
    T, H, _ = o.shape
    D = H // n_groups * HEAD
    x = inv_rope(o, positions, cos_sin_cache).reshape(T, n_groups, D // 128, 128)
    amax = x.abs().amax(-1).clamp(min=1e-10)
    scale = ue8m0_ceil(amax * torch.tensor(1.0 / 448.0, dtype=torch.float32, device=x.device))
    q = (x / scale[..., None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q.reshape(T, n_groups, D), scale


def wo_a(o_fp8: torch.Tensor, o_scale: torch.Tensor, w: torch.Tensor, w_scale: torch.Tensor):
    """(z float64 [T, G * R], bound float64 [T, G * R]) for o_fp8 [T, G, D], o_scale [T, G, D / 128], w e4m3 [G * R, D],
    w_scale f32 [G * R / 128, D / 128]."""
    T, G, D = o_fp8.shape
    KB = D // 128
    R = w.shape[0] // G
    z = torch.empty(T, G, R, dtype=torch.float64, device=o_fp8.device)
    bound = torch.empty_like(z)
    for g in range(G):
        a = o_fp8[:, g].double().reshape(T, KB, 128).permute(1, 0, 2)            # [KB, T, 128]
        wg = w[g * R:(g + 1) * R].double().reshape(R, KB, 128).permute(1, 2, 0)   # [KB, 128, R]
        sw = w_scale[g * R // 128:(g + 1) * R // 128].double().repeat_interleave(128, 0).t()   # [KB, R]
        sa = o_scale[:, g].double().t()                                        # [KB, T]
        f = sa[:, :, None] * sw[:, None, :]                                   # [KB, T, R]
        z[:, g] = (torch.bmm(a, wg) * f).sum(0)
        bound[:, g] = (torch.bmm(a.abs(), wg.abs()) * f.abs()).sum(0)
    return z.reshape(T, G * R), bound.reshape(T, G * R)


def calc_diff(x: torch.Tensor, y: torch.Tensor) -> float:
    """1 - cosine-like similarity (DeepGEMM's calc_diff, the reference test's metric)."""
    x, y = x.double(), y.double()
    return float(1 - 2 * (x * y).sum() / (x * x + y * y).sum())


def quant_weight(w: torch.Tensor):
    """A bf16/f32 weight [N, K] as e4m3 with block-128 f32 scales (ue8m0, as V4-Flash's checkpoint stores them)."""
    N, K = w.shape
    b = w.float().reshape(N // 128, 128, K // 128, 128)
    amax = b.abs().amax(dim=(1, 3)).clamp(min=1e-10)
    scale = ue8m0_ceil(amax / 448.0)
    q = (b / scale[:, None, :, None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q.reshape(N, K), scale
