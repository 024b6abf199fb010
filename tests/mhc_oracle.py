"""Float64 restatement of DeepSeek-V4's manifold hyper-connections (ops.mhc_pre / mhc_post / mhc_fused_post_pre / hc_head),
with bf16 roundings only where the kernels round:
  post     r'[t, j] = bf16(post[t, j] x[t] + sum_i comb[t, i, j] r[t, i])           (kernels/mhc/torch.py:94-106)
  pre      mixes = (r_flat . fn^T) * rsqrt(sum r_flat^2 / 4H + rms_eps); sigmoid gates; Sinkhorn of the 4 x 4 block;
           layer_input = bf16(sum_i pre_i r_i)                                       (torch.py:6-91)
  pre with norm_weight: the row o = sum_i pre_i r_i is rounded to bf16, the mean square is that of the unrounded o, and
           layer_input = bf16(float(bf16(o)) * rsqrt(ms + norm_eps) * w)            (tilelang_kernels.py:305-350)
  hc_head  bf16(sum_i (sigmoid(mixes_i s0 + base_i) + hc_eps) r_i), mixes from fn [4, 4H]
                                                                                     (tests/kernels/test_mhc_kernels.py:82-96)
A kernel accumulates in fp32, so where the terms of a sum cancel its result can be many bf16 ulps of a tiny value away from
the float64 one; the functions therefore also return `slack`, a per-element bound 2^-22 * (sum of |terms|) on that fp32
error, and bf16_close accepts a value within the given ulps or within its slack.  Nothing here is imported by the product."""
import torch

HC = 4
FP32_SLACK = 2.0 ** -22


def bf16_ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """|a - b| in bf16 units in the last place, as integers (sign-magnitude bit patterns made monotonic)."""
    def key(t):
        i = t.bfloat16().contiguous().view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (key(a) - key(b)).abs()


def bf16_close(got: torch.Tensor, ref: torch.Tensor, slack: torch.Tensor, ulps: int) -> bool:
    return bool(((bf16_ulp_distance(got, ref) <= ulps) | ((got.double() - ref.double()).abs() <= slack)).all())


def sinkhorn(logits: torch.Tensor, repeat: int, eps: float) -> torch.Tensor:
    """[..., 4, 4]: row softmax + eps, column normalisation, then repeat - 1 row / column normalisations (each dividing by
    the sum + eps) — sinkhorn_normalize_ref, tests/kernels/test_mhc_kernels.py:18-24; torch.py:76-82."""
    x = torch.softmax(logits.double(), -1) + eps
    x = x / (x.sum(-2, keepdim=True) + eps)
    for _ in range(repeat - 1):
        x = x / (x.sum(-1, keepdim=True) + eps)
        x = x / (x.sum(-2, keepdim=True) + eps)
    return x


def post(x, residual, post_layer_mix, comb_res_mix, with_slack=False):
    """bf16 [T, 4, H]: the einsum "...ij,...ih->...jh" of torch.py:94-106 plus post[j] x, in float64, rounded once."""
    T = residual.shape[0]
    c, r = comb_res_mix.double().reshape(T, HC, HC), residual.double()
    px = post_layer_mix.double().reshape(T, HC, 1) * x.double().reshape(T, 1, -1)
    out = (torch.einsum("tij,tih->tjh", c, r) + px).bfloat16()
    if not with_slack:
        return out
    return out, FP32_SLACK * (torch.einsum("tij,tih->tjh", c.abs(), r.abs()) + px.abs())


def _mixes(residual, fn, rms_eps):
    T, _, H = residual.shape
    r = residual.double().reshape(T, HC * H)
    return (r @ fn.double().t()) * torch.rsqrt((r * r).sum(-1, keepdim=True) / (HC * H) + rms_eps)


def _weighted(residual, pre, norm_weight, norm_eps):
    """(bf16 output, slack)"""
    o = (pre.unsqueeze(-1) * residual.double()).sum(1)
    slack = FP32_SLACK * (pre.unsqueeze(-1) * residual.double().abs()).sum(1)
    if norm_weight is None:
        return o.bfloat16(), slack
    f = torch.rsqrt((o * o).mean(-1, keepdim=True) + norm_eps) * norm_weight.bfloat16().double()
    return (o.bfloat16().double() * f).bfloat16(), slack * f.abs()


def pre(residual, fn, hc_scale, hc_base, rms_eps, hc_pre_eps, hc_sinkhorn_eps, hc_post_mult_value, sinkhorn_repeat,
        norm_weight=None, norm_eps=1e-6, with_slack=False):
    """(post_mix f64 [T, 4, 1], comb_mix f64 [T, 4, 4], layer_input bf16 [T, H]) — torch.py:6-91 (mhc_pre_torch), and with
    norm_weight the fused RMSNorm of mhc_pre_big_fuse_with_norm_tilelang (tilelang_kernels.py:305-350).  with_slack: the
    layer_input's slack is appended."""
    T = residual.shape[0]
    s, b = hc_scale.double(), hc_base.double()
    m = _mixes(residual, fn, rms_eps)
    pre_mix = torch.sigmoid(m[:, :HC] * s[0] + b[:HC]) + hc_pre_eps
    post_mix = torch.sigmoid(m[:, HC:2 * HC] * s[1] + b[HC:2 * HC]) * hc_post_mult_value
    comb = sinkhorn(m[:, 2 * HC:].reshape(T, HC, HC) * s[2] + b[2 * HC:].reshape(1, HC, HC), sinkhorn_repeat,
                    hc_sinkhorn_eps)
    li, slack = _weighted(residual, pre_mix, norm_weight, norm_eps)
    return (post_mix.reshape(T, HC, 1), comb, li) + ((slack,) if with_slack else ())


def fused_post_pre(x, residual, post_layer_mix, comb_res_mix, fn, hc_scale, hc_base, rms_eps, hc_pre_eps, hc_sinkhorn_eps,
                   hc_post_mult_value, sinkhorn_repeat, norm_weight=None, norm_eps=1e-6):
    """post, then pre on the bf16 streams that post returns (MHCFusedPostPreOp.forward_native's order)."""
    r = post(x, residual, post_layer_mix, comb_res_mix)
    return (r, *pre(r, fn, hc_scale, hc_base, rms_eps, hc_pre_eps, hc_sinkhorn_eps, hc_post_mult_value, sinkhorn_repeat,
                    norm_weight, norm_eps))


def hc_head(residual, fn, hc_scale, hc_base, rms_eps, hc_eps, with_slack=False):
    """bf16 [T, H] — hc_head_ref (tests/kernels/test_mhc_kernels.py:82-96), hc_head_fuse_tilelang
    (tilelang_kernels.py:884-977)."""
    m = _mixes(residual, fn, rms_eps)
    g = torch.sigmoid(m * hc_scale.double()[0] + hc_base.double()) + hc_eps
    out, slack = _weighted(residual, g, None, 0.0)
    return (out, slack) if with_slack else out
