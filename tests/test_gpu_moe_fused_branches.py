"""The fused MoE decode kernel (lvllm_b200/csrc/moe_fused.cu), branch by branch, against its float64 mirror.

Each case names the schedule branches it is there for (labels of tests/fused_schedule.py).  Before it launches, the case
asserts that the schedule model reaches them at the device's SM count, so coverage cannot disappear when a shape rule
changes.  Then it runs cpu_decode (fp32 output) twice and gpu_prefill (activation-dtype output) once.  It checks them
against the mirror (tests/fused_oracle.py) with the per-tile metric: e(t, c) = ||out - ref|| / ||ref|| over every token t
and 128-column output tile c, maximum over (t, c).  A stream-K fault stays inside one tile or one chunk's tokens, so it
moves the maximum, where a mean over the whole output would hide it.  Rows of tokens with no local expert must be exact
zeros, and two eager launches must be bit-identical.

Thresholds.  Noise floor = the largest max-tile error over the whole case matrix, per format and output dtype.  It was
measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit) and is listed in FLOOR.  The mirror rounds where the
kernel rounds, so what is left is fp32 accumulation order and the tensor cores' own accumulation: a gate / up value that
lands on the other side of a rounding point.  The 16-bit and 4-bit thresholds are about 3x their floor.
FP8 is different.  When the largest gate / up value of a token's 128-column group re-rounds, that group's requantisation
scale moves, and every e4m3 value of the group re-rounds with it.  The token's whole output then moves by up to 2 %,
the same amount in every column tile.  That floor is a property of the FP8 recipe, and a float64 mirror cannot follow
it.  The FP8 thresholds are therefore 1.4-1.7x their floor.  The kernel is deterministic, so each case's error is a fixed
number at a given SM count, not a sample.
tests/test_fused_schedule_cpu.py shows on CPU that every injected schedule fault, at the weakest point of every case,
scores at least 4x the threshold.
"""
from __future__ import annotations

from dataclasses import dataclass

import pytest
import torch

import fused_oracle as FO
import fused_schedule as FS

# largest max-tile error over the case matrix on an H100 80GB HBM3 (132 SMs, 700 W): (format, output) -> error;
# "f32" = cpu_decode, "act" = gpu_prefill in the activation dtype
FLOOR = {
    ("bf16", "f32"): 7.9e-5, ("bf16", "act"): 8.4e-4,
    ("fp16", "f32"): 7.8e-5, ("fp16", "act"): 2.8e-4,
    ("fp8", "f32"): 2.15e-2, ("fp8", "act"): 2.17e-2,
    ("fp8_e8m0", "f32"): 1.80e-2, ("fp8_e8m0", "act"): 1.79e-2,
    ("int4", "f32"): 2.5e-4, ("int4", "act"): 1.27e-3,
    ("nvfp4", "f32"): 7.6e-5, ("nvfp4", "act"): 1.12e-3,
    ("mxfp4", "f32"): 2.9e-5, ("mxfp4", "act"): 4.9e-4,
}
THRESH = {
    ("bf16", "f32"): 2.5e-4, ("bf16", "act"): 2.5e-3,
    ("fp16", "f32"): 2.5e-4, ("fp16", "act"): 1e-3,
    ("fp8", "f32"): 3e-2, ("fp8", "act"): 3e-2,
    ("fp8_e8m0", "f32"): 3e-2, ("fp8_e8m0", "act"): 3e-2,
    ("int4", "f32"): 8e-4, ("int4", "act"): 4e-3,
    ("nvfp4", "f32"): 2.5e-4, ("nvfp4", "act"): 3.5e-3,
    ("mxfp4", "f32"): 1e-4, ("mxfp4", "act"): 1.5e-3,
}

H100_SMS = 132


@dataclass(frozen=True)
class Case:
    fmt: str
    E: int
    H: int
    I: int
    M: int
    k: int
    routing: tuple = ("random",)     # ("random",) | ("counts", [rows per expert]) | ("ids", [[...]]) | ("none",)
    labels: tuple = ()
    gated: bool = True
    act: torch.dtype = torch.bfloat16
    align_g1: int = 60
    seed: int = 0


def routing(c: Case, g: torch.Generator):
    """ids [M, k] int32 and top-k weights [M, k] f32 in [0.5, 1.5) (no slot so light that its expert drops out)."""
    M, k, E = c.M, c.k, c.E
    kind = c.routing[0]
    if kind == "random":
        ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(M)]).int()
    elif kind == "counts":
        counts = c.routing[1]
        assert sum(counts) == M * k and max(counts) <= M
        flat = torch.cat([torch.full((n,), e, dtype=torch.int32) for e, n in enumerate(counts)])
        ids = flat.reshape(k, M).t()   # slot p = (token p % M, column p // M): no token gets an expert twice
    elif kind == "ids":
        ids = torch.tensor(c.routing[1], dtype=torch.int32)
    elif kind == "none":
        ids = torch.full((M, k), -1, dtype=torch.int32)
    else:
        raise ValueError(kind)
    w = torch.rand(M, k, generator=g) + 0.5
    return ids.contiguous(), w.float().contiguous()


def _fmt_cases():
    out = {}
    for fmt in ("bf16", "fp16", "fp8", "fp8_e8m0", "int4", "nvfp4", "mxfp4"):
        w4 = fmt in FS.W4
        act = torch.float16 if fmt == "fp16" else torch.bfloat16
        for M in (16, 17, 32, 33):
            tn = (16 if M <= 16 else 32 if M <= 32 else 64) if w4 else (16 if M <= 16 else 32)
            out[f"{fmt}_m{M}"] = Case(fmt, 8, 512, 256, M, 2, act=act, labels=(f"tnmax{tn}",), seed=M)
    return out


CASES = {
    # unpaired GEMM2 (H / 128 odd): J2e = J2, KI2 = (KB2 + 1) / 2, jt = j and the unpaired w2 addressing
    "unpaired_bf16": Case("bf16", 8, 1152, 256, 5, 2, labels=("g2_unpaired",)),
    "unpaired_fp16": Case("fp16", 8, 1152, 256, 5, 2, act=torch.float16, labels=("g2_unpaired",)),
    "unpaired_fp8": Case("fp8", 8, 1152, 256, 5, 2, labels=("g2_unpaired",)),
    # FP8 half iterations: non-gated relu^2 GEMM1 with H / 128 odd, unpaired GEMM2 with I / 128 odd
    "fp8_relu2_half_g1": Case("fp8", 8, 1152, 256, 3, 2, gated=False, labels=("g1_half_iter", "g2_unpaired")),
    "fp8_unpaired_half_g2": Case("fp8", 8, 1152, 384, 3, 2, labels=("g2_unpaired", "g2_half_iter")),
    # more than 16 contributors on a tile of <= 4 rows: GEMM1 (56 per tile) and GEMM2 (32 per tile)
    "fp8_g1_gt16_small": Case("fp8", 4, 7168, 256, 1, 1, routing=("ids", [[2]]), labels=("g1_fix_small_multi",)),
    "fp8_g2_gt16_small": Case("fp8", 4, 256, 4096, 1, 1, routing=("ids", [[1]]), labels=("g2_fix_small_multi",)),
    # more than 16 contributors on a tile of more than 4 rows (rounds of 4 contributors, one 16-column block)
    "fp8_g1_gt16_wide": Case("fp8", 2, 7168, 256, 8, 1, routing=("counts", [8, 0]),
                             labels=("g1_fix_wide_gt16", "g1_split_rows5_16")),
    # split tiles of 5-16 and of 17-32 rows (one and two 16-column fix-up blocks)
    "bf16_split_rows": Case("bf16", 4, 2048, 256, 32, 1, routing=("counts", [24, 8, 0, 0]),
                            labels=("g1_split_rows17_32", "g1_split_rows5_16", "ng1")),
    # 4-bit chunks of 57-64 rows: eight 8-column fix-up blocks
    "int4_rows64": Case("int4", 8, 512, 256, 64, 2, routing=("counts", [60, 30, 20, 10, 4, 2, 1, 1]),
                        labels=("w4_fix_8blocks", "tnmax64", "ng2")),
    # NG = 2 on a 16-bit layer
    "bf16_ng2": Case("bf16", 16, 512, 256, 24, 4, labels=("ng2",)),
    # GEMM1 cut at tile boundaries, and the same launch forced to stream-K
    "fp8_g1_aligned": Case("fp8", 64, 512, 384, 64, 2, labels=("g1_aligned", "ng2")),
    "fp8_g1_streamk": Case("fp8", 64, 512, 384, 64, 2, align_g1=0, labels=("g1_streamk", "ng2")),
    # E = 512 at an M that fused_supported still accepts with top-8 routing; empty batches
    "bf16_e512": Case("bf16", 512, 256, 128, 32, 8, labels=("fused", "ng2")),
    "bf16_no_rows": Case("bf16", 8, 512, 256, 4, 2, routing=("none",), labels=("no_rows",)),
    "fp8_no_rows": Case("fp8", 8, 512, 256, 4, 2, routing=("none",), labels=("no_rows",)),
    **_fmt_cases(),
}


def case_routing(c: Case):
    """(hidden, ids, topk weights) of a case: seeded, independent of the layer's weights."""
    g = torch.Generator().manual_seed(2000 + c.seed + 7 * c.M + c.H + c.E)
    ids, w = routing(c, g)
    return (torch.randn(c.M, c.H, generator=g) / 10).to(c.act), ids, w


def case_inputs(c: Case):
    layer = FO.make_layer(c.fmt, c.E, c.H, c.I, torch.Generator().manual_seed(1000 + c.seed + c.H + c.E),
                          gated=c.gated, act=c.act)
    return (layer, *case_routing(c))


# ------------------------------------------------------------------------------------------ GPU side
def _lk_class(fmt, act):
    import lk_moe
    base = {"bf16": "MOE_BF16", "fp16": "MOE_FP16", "fp8": "MOE_FP8", "fp8_e8m0": "MOE_FP8", "int4": "MOE_WNA16",
            "nvfp4": "MOE_NVFP4", "mxfp4": "MOE_MXFP4"}[fmt]
    if act == torch.float16 and fmt not in ("bf16", "fp16"):
        base += "_FP16"
    return getattr(lk_moe, base)


def _cfg(c: Case):
    import lk_moe
    cfg = lk_moe.MOEConfigV2()
    cfg.expert_num, cfg.top_k, cfg.hidden_size, cfg.intermediate_size = c.E, c.k, c.H, c.I
    cfg.max_batch_size = cfg.max_num_seqs = 256
    cfg.groupN, cfg.groupK = {"fp8": (128, 128), "fp8_e8m0": (128, 128), "int4": (1, 32), "nvfp4": (1, 16),
                              "mxfp4": (1, 32)}.get(c.fmt, (0, 0))
    cfg.has_gate_proj = c.gated
    cfg.activation_type = 0 if c.gated else 2
    return cfg


def build_moe(c: Case, layer, monkeypatch):
    if c.fmt == "fp8_e8m0":
        monkeypatch.setenv("B200MOE_FP8_E8M0", "1")
    else:
        monkeypatch.delenv("B200MOE_FP8_E8M0", raising=False)
    ptrs = [t.contiguous().data_ptr() if t is not None else 0 for t in layer.ctor]
    return _lk_class(c.fmt, c.act)(_cfg(c), *ptrs)


def decode(moe, hd, idd, wd, out):
    moe.cpu_decode(torch.cuda.current_stream().cuda_stream, hd.shape[0], idd.shape[1], hd.data_ptr(), idd.data_ptr(),
                   wd.data_ptr(), out.data_ptr())


def run_case(name: str, dev, monkeypatch):
    """Runs one case; returns (fp32 error, act-dtype error, schedule)."""
    c = CASES[name]
    G = torch.cuda.get_device_properties(dev).multi_processor_count
    layer, hidden, ids, w = case_inputs(c)
    sch = FS.build(layer.geo, ids, G, c.align_g1)
    FS.check_invariants(sch)
    missing = set(c.labels) - sch.labels
    assert not missing, f"{name}: at G = {G} the schedule does not reach {sorted(missing)} (reaches {sorted(sch.labels)})"
    assert "fused" in sch.labels, f"{name}: not a fused launch"
    monkeypatch.setenv("B200MOE_ALIGN_G1", str(c.align_g1))
    moe = build_moe(c, layer, monkeypatch)
    hd, idd, wd = hidden.to(dev), ids.to(dev), w.to(dev)
    o1 = torch.full((c.M, c.H), float("nan"), dtype=torch.float32, device=dev)
    o2 = torch.full_like(o1, float("nan"))
    op = torch.full((c.M, c.H), float("nan"), dtype=c.act, device=dev)
    decode(moe, hd, idd, wd, o1)
    decode(moe, hd, idd, wd, o2)
    moe.gpu_prefill(hd.data_ptr(), op.data_ptr(), idd.data_ptr(), wd.data_ptr(), c.M, c.k,
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    moe.close()
    assert torch.equal(o1, o2), f"{name}: two eager launches differ"
    o1, op = o1.cpu(), op.cpu()
    none_local = ((ids < 0) | (ids >= c.E)).all(dim=1)
    assert torch.equal(o1[none_local], torch.zeros_like(o1[none_local])), f"{name}: rows without a local expert"
    assert torch.equal(op[none_local].float(), torch.zeros_like(o1[none_local]))
    if sch.chunks:
        mirror = FO.Mirror(layer, sch, hidden, w)
        e32 = FO.max_tile_error(o1, mirror.out(out_dtype=torch.float32))
        ep = FO.max_tile_error(op, mirror.out(out_dtype=c.act))
    else:
        e32 = ep = 0.0
    return e32, ep, sch


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_fused_branch_case(dev, name, monkeypatch):
    c = CASES[name]
    e32, ep, _ = run_case(name, dev, monkeypatch)
    t32, tp = THRESH[(c.fmt, "f32")], THRESH[(c.fmt, "act")]
    assert e32 < t32, f"{name}: cpu_decode max tile error {e32:.3g} >= {t32:.3g}"
    assert ep < tp, f"{name}: gpu_prefill max tile error {ep:.3g} >= {tp:.3g}"


# ------------------------------------------------------------------------------------------ counter hygiene
HYGIENE = ("fp8_g1_gt16_small", "unpaired_bf16", "int4_rows64")   # A, B, C: different shape, format and chunk count


@pytest.mark.gpu
def test_counters_clean_across_layers_and_graph(dev, monkeypatch):
    """All layers of a device share one workspace and one set of cross-CTA counters, which carry no generation tag: a
    launch must hand them back at zero whatever shape ran before it.  Layers A, B, C run in the order A, B, C, A, C, B,
    eagerly and then captured in one CUDA graph replayed twice.  Every output is bit-identical to that layer's launch
    on its own."""
    monkeypatch.setenv("B200MOE_ALIGN_G1", "60")
    layers = []
    for name in HYGIENE:
        c = CASES[name]
        layer, hidden, ids, w = case_inputs(c)
        moe = build_moe(c, layer, monkeypatch)
        layers.append((moe, hidden.to(dev), ids.to(dev), w.to(dev), c))
    alone = []
    for moe, hd, idd, wd, c in layers:
        o = torch.empty(c.M, c.H, dtype=torch.float32, device=dev)
        decode(moe, hd, idd, wd, o)
        torch.cuda.synchronize()
        alone.append(o.clone())
    order = (0, 1, 2, 0, 2, 1)
    outs = [torch.full((layers[i][4].M, layers[i][4].H), float("nan"), device=dev) for i in order]
    for o, i in zip(outs, order):
        moe, hd, idd, wd, _ = layers[i]
        decode(moe, hd, idd, wd, o)
    torch.cuda.synchronize()
    for n, (o, i) in enumerate(zip(outs, order)):
        assert torch.equal(o, alone[i]), f"eager launch {n} (layer {'ABC'[i]}) differs from the layer run alone"
    st = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            for o, i in zip(outs, order):
                moe, hd, idd, wd, _ = layers[i]
                decode(moe, hd, idd, wd, o)
    st.wait_stream(side)
    for rep in range(2):
        for o in outs:
            o.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for n, (o, i) in enumerate(zip(outs, order)):
            assert torch.equal(o, alone[i]), f"replay {rep}, launch {n} (layer {'ABC'[i]}) differs from the layer run alone"
    del graph
    for moe, *_ in layers:
        moe.close()


# ------------------------------------------------------------------------------------------ construction refusal
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["int4", "nvfp4", "mxfp4"])
def test_w4_odd_hidden_tiles_refused_at_construction(dev, fmt):
    """The fused kernel streams 4-bit w2 in tile pairs, so a 4-bit layer with H / 128 odd could never run
    (fused_supported refuses it).  Both constructors refuse it up front and say why."""
    from lvllm_b200._lib import B200Error
    c = Case(fmt, 2, 1152, 256, 1, 1)
    layer = FO.make_layer(fmt, c.E, c.H, c.I, torch.Generator().manual_seed(0))
    cls = _lk_class(fmt, torch.bfloat16)
    ptrs = [t.contiguous().data_ptr() if t is not None else 0 for t in layer.ctor]
    with pytest.raises(B200Error, match="hidden_size % 256"):
        cls(_cfg(c), *ptrs)
    with pytest.raises(B200Error, match="hidden_size % 256"):
        cls.from_expert_shards(_cfg(c), iter(()))
