"""Float64 mirror of the fused MoE decode kernel's arithmetic (lvllm_b200/csrc/moe_fused.cu), with fault injection.

The mirror accumulates in float64 and rounds only where the kernel rounds:
  * FP8: activations quantised per token and 128-column group (phase 0b, moe_fused.cu:624-648); every k-block's partial
    product promoted with its weight and activation scales (:934-979);
  * 4-bit formats: bf16 activations saturated to fp16 (:652-663), weights dequantised to the fp16 values the wgmma A
    fragments hold (:213-265); NVFP4 global scales applied after the reduction (:1128-1133, :1199-1205, :986);
  * gate and up rounded to the compute dtype (round_act, :1211-1214), SiLU * up, SwiGLU-OAI or relu^2 (:1215-1225),
    clamped to +-65504 and rounded to the compute dtype (:1226);
  * FP8: the intermediate requantised per token and 128-column group (:1228-1246);
  * y stored in fp32 (:1264-1274), the combine over the top-k slots in fixed order (:1315-1362), the output dtype.

The quantisers / dequantisers are those of oracle/moe_oracle.py.  GEMM partial products are kept per k-block (of the
kernel's k-block size) and per chunk, so a fault of the stream-K schedule — a k-block or a contributor's range dropped or
counted twice, a tile stored into its neighbour's columns, a k-block read at the wrong offset — can be injected into the
reduction of one (phase, chunk, tile) and its effect measured with the same metric the GPU tests use.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

import fused_schedule as FS
from oracle import moe_oracle as O

F64 = torch.float64
F32 = torch.float32


# ------------------------------------------------------------------------------------------ layers
@dataclass
class Layer:
    """A layer in two views: `ctor` are the checkpoint tensors the lk_moe class takes, the rest is what the kernel
    multiplies (float32 storage of values that are exact in it)."""
    geo: FS.Geometry
    act: torch.dtype          # activation dtype of the class (bf16 / fp16)
    act_type: int             # 0 SiLU, 1 SwiGLU-OAI (packed halves), 2 relu^2
    ctor: tuple               # (w13, w2, s13, s2, g13, g2), absent = None
    w13: torch.Tensor         # [E, N1, H] kernel operand values (FP8: e4m3 values, scales separate)
    w2: torch.Tensor          # [E, H, I]
    ws13: torch.Tensor | None = None   # FP8 block scales [E, N1/128, H/128]
    ws2: torch.Tensor | None = None
    g13: torch.Tensor | None = None    # NVFP4 global scales [E, 2]
    g2: torch.Tensor | None = None     # [E]
    alpha: float = 1.702
    limit: float = 7.0

    @property
    def cmp(self) -> torch.dtype:
        """Compute dtype of the intermediate (moe_fused.cu:1443): fp16 for fp16 activations and the 4-bit formats."""
        return torch.float16 if (self.act == torch.float16 or self.geo.wq) else torch.bfloat16

    @property
    def e8m0(self) -> bool:
        return self.geo.fmt == "fp8_e8m0"


def _fp16_mx_scale(e8: torch.Tensor) -> torch.Tensor:
    """e8m0 -> fp16 2^(E-127) as the kernel forms it: exponent field E-112 clamped to [0, 30] (moe_fused.cu:260-264)."""
    f = (e8.to(torch.int32) - 112).clamp(0, 30)
    return (f.to(torch.int16) << 10).view(torch.float16).to(F32)


def make_layer(fmt: str, E: int, H: int, I: int, g: torch.Generator, gated: bool = True, act=torch.bfloat16,
               act_type: int | None = None) -> Layer:
    geo = FS.Geometry(fmt, E, H, I, gated)
    if act_type is None:
        act_type = 0 if gated else 2
    N1 = 2 * I if gated else I
    w13f = torch.randn(E, N1, H, generator=g) / 10
    w2f = torch.randn(E, H, I, generator=g) / 10
    if fmt in ("bf16", "fp16"):
        dt = torch.bfloat16 if fmt == "bf16" else torch.float16
        w13, w2 = w13f.to(dt), w2f.to(dt)
        return Layer(geo, act, act_type, (w13, w2, None, None, None, None), w13.float(), w2.float())
    if fmt.startswith("fp8"):
        q13, s13 = O.quant_fp8_block(w13f)
        q2, s2 = O.quant_fp8_block(w2f)
        ctor = (q13, q2, s13, s2, None, None)
        if fmt == "fp8_e8m0":   # re-quantised at ingest to power-of-two block scales (repack.cu:268-277)
            q13, s13 = O.requant_weight_ue8m0(q13, s13)
            q2, s2 = O.requant_weight_ue8m0(q2, s2)
        return Layer(geo, act, act_type, ctor, q13.float(), q2.float(), s13.float(), s2.float())
    if fmt == "int4":
        sdt = torch.float16 if act == torch.float16 else torch.bfloat16
        p13, s13 = O.quant_int4_group(w13f, 32, scale_dtype=sdt)
        p2, s2 = O.quant_int4_group(w2f, 32, scale_dtype=sdt)
        return Layer(geo, act, act_type, (p13, p2, s13, s2, None, None),
                     O.dequant_int4_group(p13, s13, 32, torch.float16), O.dequant_int4_group(p2, s2, 32, torch.float16))
    if fmt == "nvfp4":
        p13, s13, g13 = O.quant_nvfp4(w13f.reshape(E * 2, I, H))   # separate global scales for gate and up
        g13 = g13.reshape(E, 2).contiguous()
        p13, s13 = p13.reshape(E, 2 * I, H // 2).contiguous(), s13.reshape(E, 2 * I, H // 16).contiguous()
        p2, s2, g2 = O.quant_nvfp4(w2f)
        g2 = g2.contiguous()
        v13 = O.unpack_e2m1(p13) * s13.float().repeat_interleave(16, -1)    # exact in fp16; global scale after the sum
        v2 = O.unpack_e2m1(p2) * s2.float().repeat_interleave(16, -1)
        return Layer(geo, act, act_type, (p13, p2, s13, s2, g13, g2), v13, v2, g13=g13.float(), g2=g2.float())
    if fmt == "mxfp4":
        p13, s13 = O.quant_mxfp4(w13f)
        p2, s2 = O.quant_mxfp4(w2f)
        v13 = O.unpack_e2m1(p13) * _fp16_mx_scale(s13).repeat_interleave(32, -1)
        v2 = O.unpack_e2m1(p2) * _fp16_mx_scale(s2).repeat_interleave(32, -1)
        return Layer(geo, act, act_type, (p13, p2, s13, s2, None, None), v13, v2)
    raise ValueError(fmt)


# ------------------------------------------------------------------------------------------ faults
@dataclass(frozen=True)
class Fault:
    """One schedule fault in the reduction of (phase ph, chunk q, schedule tile j).
    kind: "drop" / "double" the k-blocks `kbs`; "shift": k-block kbs[0] read at k-block kbs[1]'s offset;
    "neighbour": GEMM2 tile j stored into tile j + 1's columns."""
    ph: int
    q: int
    j: int
    kind: str
    kbs: tuple = ()


def _tile_cols(sch: FS.Schedule, ph: int, j: int) -> torch.Tensor:
    geo = sch.geo
    if ph == 0:
        cols = [torch.arange(128 * j, 128 * j + 128)]
        if geo.gated:
            cols.append(torch.arange(geo.I + 128 * j, geo.I + 128 * j + 128))
    else:
        cols = [torch.arange(128 * jt, 128 * jt + 128) for jt in sch.out_tiles(1, j)]
    return torch.cat(cols)


def _reduce(P: torch.Tensor, sch: FS.Schedule, ph: int, faults) -> torch.Tensor:
    acc = P.sum(0)
    moves = []
    for f in faults:
        cols = _tile_cols(sch, ph, f.j)
        if f.kind == "drop":
            acc[:, cols] -= P[list(f.kbs)][:, :, cols].sum(0)
        elif f.kind == "double":
            acc[:, cols] += P[list(f.kbs)][:, :, cols].sum(0)
        elif f.kind == "shift":
            acc[:, cols] += P[f.kbs[1]][:, cols] - P[f.kbs[0]][:, cols]
        elif f.kind == "neighbour":
            moves.append(f)
        else:
            raise ValueError(f.kind)
    for f in moves:
        src = _tile_cols(sch, 1, f.j)
        acc[:, src + 128] = acc[:, src].clone()
        acc[:, src] = 0.0
    return acc


def _round(x: torch.Tensor, dt: torch.dtype) -> torch.Tensor:
    """fp32 accumulator / value rounded to dt, back in float64."""
    return x.to(F32).to(dt).to(F64)


# ------------------------------------------------------------------------------------------ the mirror
class Mirror:
    """The kernel's launch for one routing, chunk by chunk; `out(faults)` recomputes only the chunks a fault touches."""

    def __init__(self, layer: Layer, sch: FS.Schedule, hidden: torch.Tensor, topk_w: torch.Tensor):
        assert sch.supported
        self.L, self.sch = layer, sch
        self.M, self.H = hidden.shape
        geo = layer.geo
        x = hidden.to(layer.act)
        if geo.fp8:
            xq, xs = O.per_token_group_quant_fp8(x.float(), 128, ue8m0=layer.e8m0)
            self.x, self.xs = xq.to(F64), xs.to(F64)
        elif geo.wq:
            self.x, self.xs = x.float().clamp(-65504, 65504).half().to(F64), None
        else:
            self.x, self.xs = x.to(F64), None
        self.topk_w = topk_w.to(F32)
        self._p1, self._y = {}, {}

    def _gemm(self, xr, xs, w, ws):
        """Partial products per k-block: [KB, rows, N] (FP8: promoted with the block scales)."""
        epk = self.L.geo.epk
        r, K = xr.shape
        N = w.shape[0]
        P = torch.einsum("rkc,nkc->krn", xr.reshape(r, K // epk, epk), w.to(F64).reshape(N, K // epk, epk))
        if xs is not None:
            wsx = ws.to(F64).repeat_interleave(128, 0)[:N].t()           # [KB, N]
            P = P * xs.t()[:, :, None] * wsx[:, None, :]
        return P

    def _p1_of(self, q):
        if q not in self._p1:
            ch = self.sch.chunks[q]
            tok = torch.tensor([s // self.sch.k for s in ch.slots])
            L = self.L
            xs = self.xs[tok] if self.xs is not None else None
            self._p1[q] = self._gemm(self.x[tok], xs, L.w13[ch.expert], L.ws13[ch.expert] if L.ws13 is not None else None)
        return self._p1[q]

    def _chunk_y(self, q, faults):
        L, geo, sch = self.L, self.L.geo, self.sch
        e = sch.chunks[q].expert
        h = _reduce(self._p1_of(q), sch, 0, [f for f in faults if f.ph == 0])
        I = geo.I
        if L.g13 is not None:
            h[:, :I] *= float(L.g13[e, 0])
            h[:, I:] *= float(L.g13[e, 1])
        g0 = _round(h[:, :I], L.cmp)
        if geo.gated:
            u0 = _round(h[:, I:], L.cmp)
            if L.act_type == 1:
                gg = g0.clamp(max=L.limit)
                uu = u0.clamp(-L.limit, L.limit)
                r = (uu + 1.0) * gg / (1.0 + torch.exp(-L.alpha * gg))
            else:
                r = g0 / (1.0 + torch.exp(-g0)) * u0
        else:
            r = g0.clamp(min=0) ** 2
        v = _round(r.clamp(-65504, 65504), L.cmp)
        if geo.fp8:
            iq, is_ = O.per_token_group_quant_fp8(v.to(F32), 128, ue8m0=L.e8m0)
            P2 = self._gemm(iq.to(F64), is_.to(F64), L.w2[e], L.ws2[e])
        else:
            P2 = self._gemm(v, None, L.w2[e], None)
        y = _reduce(P2, sch, 1, [f for f in faults if f.ph == 1])
        if L.g2 is not None:
            y = y * float(L.g2[e])
        return y.to(F32).to(F64)                                             # y is stored in fp32

    def out(self, faults=(), out_dtype=F32) -> torch.Tensor:
        sch = self.sch
        ys = {}
        for q in range(len(sch.chunks)):
            fq = [f for f in faults if f.q == q]
            if fq:
                ys[q] = self._chunk_y(q, fq)
            else:
                if q not in self._y:
                    self._y[q] = self._chunk_y(q, [])
                ys[q] = self._y[q]
        # row -> (chunk, index) and the fixed-order combine
        where = {}
        for q, ch in enumerate(sch.chunks):
            for i in range(ch.nrows):
                where[ch.row0 + i] = (q, i)
        out = torch.zeros(self.M, self.H, dtype=F64)
        k = sch.k
        for t in range(self.M):
            for j in range(k):
                row = sch.row_of_slot[t * k + j]
                if row < 0:
                    continue
                q, i = where[row]
                out[t] += float(self.topk_w[t, j]) * ys[q][i]
        return out.to(F32).to(out_dtype).to(F64)


def reference(layer: Layer, hidden, ids, topk_w, G: int, out_dtype=F32, align_g1: int = 60) -> torch.Tensor:
    """The mirror's output for a launch; rows of tokens without a local expert are zeros."""
    sch = FS.build(layer.geo, ids, G, align_g1)
    if not sch.chunks:
        return torch.zeros(hidden.shape, dtype=F64)
    return Mirror(layer, sch, hidden, topk_w).out(out_dtype=out_dtype)


# ------------------------------------------------------------------------------------------ the metric
def tile_errors(out: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """e(t, c) = ||out - ref||_2 / ||ref||_2 over token t and 128-column output tile c: [M, H / 128].  A tile whose
    reference is exactly zero scores 0 when the output is zero there too and inf otherwise."""
    M, H = ref.shape
    d = (out.to(F64) - ref.to(F64)).reshape(M, H // 128, 128).norm(dim=-1)
    n = ref.to(F64).reshape(M, H // 128, 128).norm(dim=-1)
    e = d / torch.where(n > 0, n, torch.ones_like(n))
    return torch.where((n == 0) & (d > 0), torch.full_like(e, float("inf")), e)


def max_tile_error(out, ref) -> float:
    return float(tile_errors(out, ref).max())
