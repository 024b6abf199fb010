"""GPU (-m gpu): the fused GQA q/k-norm + RoPE + paged cache write, and GQA decode reading the FlashInfer backend's
packed KV cache in place.

Kernel vs the reference-generated golden fixture and vs the oracle (tests/gqa_oracle.py), cache bytes on the packed NHD /
HND layouts and on separate caches, decode on packed views vs contiguous copies, a three-step decode chain, the same chain
captured in a CUDA graph, the bench shapes, and the argument refusals of the C entry points."""
import os

import pytest
import torch

import gqa_oracle as GO
from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu

D = 128
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_gqa.pt")
SENTINEL = 0x7FA5   # a bf16 NaN pattern no kernel output can produce


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_diff(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return 1 - 2 * (a * b).sum() / max((a * a + b * b).sum(), 1e-12)


def make_cache(layout, blocks, page, hkv, fill):
    """(physical buffer, k view, v view).  NHD / HND: the FlashInfer backend's per-layer tensor (logical (blocks, Hkv,
    page, 2D), flashinfer.py:398-433) split as the backend splits it (:2276-2290); "separate": two contiguous caches."""
    if layout == "separate":
        phys = fill((2, blocks, page, hkv, D))
        return phys, phys[0], phys[1]
    if layout == "NHD":
        phys = fill((blocks, page, hkv, 2 * D))
        logical = phys.permute(0, 2, 1, 3)
    else:
        phys = fill((blocks, hkv, page, 2 * D))
        logical = phys
    k, v = logical.transpose(1, 2).split(D, dim=-1)
    return phys, k, v


def assert_ulps(got, ref, rot, neox, n=2):
    """|got - ref| <= n bf16 ulp at the magnitude of the rotated pair (|o1|^2 + |o2|^2 = |x1|^2 + |x2|^2 bounds the
    operands of the reference's bf16 products), or of the element itself outside the rotary dims."""
    got, ref = got.float().cpu().reshape(-1, D), ref.float().cpu().reshape(-1, D)
    idx = torch.arange(D)
    half = rot // 2
    partner = torch.where(idx < half, idx + half, idx - half) if neox else idx ^ 1
    partner = torch.where(idx < rot, partner, idx)
    scale = torch.maximum(ref.abs(), torch.sqrt(ref ** 2 + ref[:, partner] ** 2))
    ulp = torch.exp2(torch.floor(torch.log2(scale.clamp_min(2.0 ** -126))) - 7)
    err = (got - ref).abs()
    bad = err > n * ulp
    assert not bad.any(), f"{int(bad.sum())} elements beyond {n} ulp; worst {float((err / ulp).max()):.2f} ulp"


def _table(g, c, dev):
    t = torch.zeros(g["max_position"], c["rotary_dim"], dtype=torch.bfloat16)
    t[c["positions"]] = c["cos_sin_rows"]
    return t.to(dev)


def _golden():
    return torch.load(GOLDEN, weights_only=True)


@pytest.mark.parametrize("ci", range(11))
def test_kernel_vs_reference_golden(dev, ci):
    from lvllm_b200 import ops
    g = _golden()
    assert len(g["cases"]) == 11
    c = g["cases"][ci]
    hq, hkv, T, rot = c["num_heads"], c["num_kv_heads"], c["tokens"], c["rotary_dim"]
    qkv = g["qkv"][c["heads"]][:T]
    phys, kc, vc = make_cache("separate", 2, 16, hkv, lambda s: torch.zeros(*s, dtype=torch.bfloat16, device=dev))
    slots = torch.tensor([5, 16 + 9][:T], dtype=torch.int64)
    w = (c["q_weight"].to(dev), c["k_weight"].to(dev)) if c["norm"] else (None, None)
    q = ops.gqa_qknorm_rope_cache_write(qkv.to(dev), c["positions"].to(dev), _table(g, c, dev), slots.to(dev), kc, vc, hq,
                                        hkv, w[0], w[1], c["eps"], c["is_neox"])
    torch.cuda.synchronize()
    assert q.shape == (T, hq, D) and q.is_contiguous()
    assert_ulps(q, c["q_out"], rot, c["is_neox"])
    k_rows = kc.reshape(-1, hkv, D)[slots.to(dev)]
    v_rows = vc.reshape(-1, hkv, D)[slots.to(dev)]
    assert_ulps(k_rows, c["k_out"], rot, c["is_neox"])
    assert torch.equal(v_rows.cpu(), qkv[:, (hq + hkv) * D:].reshape(T, hkv, D))


def _inputs(gen, T, hq, hkv, max_pos, rot, norm):
    qkv = (torch.randn(T, (hq + 2 * hkv) * D, generator=gen) * 2).bfloat16()
    inv = 1.0 / (1e6 ** (torch.arange(0, rot, 2, dtype=torch.float) / rot))
    fr = torch.einsum("i,j->ij", torch.arange(max_pos, dtype=torch.float), inv)
    table = torch.cat((fr.cos(), fr.sin()), dim=-1).bfloat16()
    w = ((1 + 0.1 * torch.randn(D, generator=gen)).bfloat16(), (1 + 0.1 * torch.randn(D, generator=gen)).bfloat16()) \
        if norm else (None, None)
    return qkv, table, w


def _oracle_qk(qkv, pos, table, hq, hkv, rot, w, eps, neox):
    out = GO.qk_norm_rope(qkv, pos, table, hq, hkv, D, rot, w[0], w[1], eps, neox)
    q, k, v = out.split([hq * D, hkv * D, hkv * D], dim=-1)
    return q.reshape(-1, hq, D), k.reshape(-1, hkv, D), v.reshape(-1, hkv, D)


def _dev(w, dev):
    return tuple(x.to(dev) if x is not None else None for x in w)


@pytest.mark.parametrize("layout", ["NHD", "HND", "separate"])
def test_cache_bytes(dev, layout):
    """Every byte of the cache after the call == the sentinel-filled cache written by the oracle's reshape_and_cache_flash
    with the kernel's own k and the input v: padded slots and all other rows untouched."""
    from lvllm_b200 import ops
    gen = torch.Generator().manual_seed(3)
    T, hq, hkv, rot, blocks, page = 7, 16, 4, 64, 6, 16
    qkv, table, w = _inputs(gen, T, hq, hkv, 4096, rot, True)
    pos = torch.tensor([0, 1, 4095, 17, 900, 3, 2048])
    slots = torch.tensor([3, -1, 16 * 5 + 15, 16, 47, -1, 64], dtype=torch.int64)
    fill = lambda s: torch.full(s, SENTINEL, dtype=torch.int16, device=dev).view(torch.bfloat16)  # noqa: E731
    phys, kc, vc = make_cache(layout, blocks, page, hkv, fill)
    q = ops.gqa_qknorm_rope_cache_write(qkv.to(dev), pos.to(dev), table.to(dev), slots.to(dev), kc, vc, hq, hkv,
                                        *_dev(w, dev), 1e-6, True)
    torch.cuda.synchronize()
    q_ref, k_ref, v_in = _oracle_qk(qkv, pos, table, hq, hkv, rot, w, 1e-6, True)
    assert_ulps(q, q_ref, rot, True)
    valid = slots >= 0
    k_rows = torch.stack([kc[int(s) // page, int(s) % page] for s in slots[valid]]).cpu()
    assert_ulps(k_rows, k_ref[valid], rot, True)
    exp_phys, ek, ev = make_cache(layout, blocks, page, hkv,
                                  lambda s: torch.full(s, SENTINEL, dtype=torch.int16).view(torch.bfloat16))
    k_all = torch.zeros(T, hkv, D, dtype=torch.bfloat16)
    k_all[valid] = k_rows
    GO.reshape_and_cache_flash(k_all, v_in, ek, ev, slots)
    assert torch.equal(phys.cpu().view(torch.int16), exp_phys.view(torch.int16))


def _decode_case(dev, layout, B, S, page, hq, hkv, splits, seed):
    from lvllm_b200 import ops
    gen = torch.Generator(device=dev).manual_seed(seed)
    npg = -(-S // page)
    phys, kc, vc = make_cache(layout, B * npg, page, hkv,
                              lambda s: torch.randn(*s, generator=gen, device=dev).bfloat16())
    cpu_gen = torch.Generator().manual_seed(seed)
    pt = torch.randperm(B * npg, generator=cpu_gen).reshape(B, npg).int()
    lens = torch.tensor([max(1, S - 13 * (b % 5)) for b in range(B)], dtype=torch.int32)
    q = torch.randn(B, hq, D, generator=cpu_gen).bfloat16()
    scale = D ** -0.5
    out, lse = ops.gqa_decode(q.to(dev), kc, vc, lens.to(dev), pt.to(dev), scale, num_kv_splits=splits)
    out_c, lse_c = ops.gqa_decode(q.to(dev), kc.contiguous(), vc.contiguous(), lens.to(dev), pt.to(dev), scale,
                                  num_kv_splits=splits)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), out_c.view(torch.int16))
    assert torch.equal(lse, lse_c)
    sel = sorted({0, B - 1})
    ref, lse_ref = _oracle_decode(q[sel], kc, vc, lens[sel], pt[sel], scale)
    assert _cos_diff(out.cpu().float()[sel], ref) < 1e-5
    torch.testing.assert_close(lse.cpu()[sel], lse_ref, atol=1e-3, rtol=1e-3)


def _oracle_decode(q, kc, vc, lens, pt, scale):
    """O.gqa_decode on the pages the selected requests use (gathered to the CPU, page table renumbered)."""
    pages = pt.flatten().long()
    ks, vs = kc[pages.to(kc.device)].cpu(), vc[pages.to(vc.device)].cpu()
    return O.gqa_decode(q, ks, vs, lens, torch.arange(pages.numel(), dtype=torch.int32).reshape(pt.shape), scale)


@pytest.mark.parametrize("layout", ["NHD", "HND"])
@pytest.mark.parametrize("B,S,page,hq,hkv,splits", [
    (8, 700, 16, 32, 8, 0),      # tensor-core kernel (group 4)
    (5, 333, 32, 64, 4, 0),      # tensor-core kernel (group 16)
    (4, 500, 16, 48, 1, 0),      # group 48: split-KV CUDA-core kernel
    (6, 600, 16, 32, 8, 3),      # split count below the page table: CUDA-core kernel
])
def test_decode_reads_packed_cache_in_place(dev, layout, B, S, page, hq, hkv, splits):
    _decode_case(dev, layout, B, S, page, hq, hkv, splits, seed=11)


def _chain_setup(dev, layout, seed):
    gen = torch.Generator().manual_seed(seed)
    B, page, hq, hkv, rot = 3, 16, 16, 4, 128
    lens0 = torch.tensor([14, 31, 100], dtype=torch.int32)   # request 1 crosses into a new page at its second step
    npg = -(-(int(lens0.max()) + 3) // page)
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int()
    _, table, w = _inputs(gen, 1, hq, hkv, 8192, rot, True)
    steps = [(torch.randn(B, (hq + 2 * hkv) * D, generator=gen) * 2).bfloat16() for _ in range(3)]
    dgen = torch.Generator(device=dev).manual_seed(seed)
    phys, kc, vc = make_cache(layout, B * npg, page, hkv,
                              lambda s: torch.randn(*s, generator=dgen, device=dev).bfloat16())
    return dict(B=B, page=page, hq=hq, hkv=hkv, rot=rot, lens0=lens0, pt=pt, table=table, w=w, steps=steps, phys=phys,
                kc=kc, vc=vc)


def _slots(pt, pos, page):
    b = torch.arange(pt.shape[0])
    return (pt[b, (pos // page).long()].long() * page + (pos % page).long()).to(torch.int64)


def test_decode_step_chain(dev):
    """Three steps: write the new token (positions = seq_lens, slots from the page table) into the packed NHD cache, then
    decode with seq_lens + 1.  Each step matches the oracle on the updated cache."""
    from lvllm_b200 import ops
    s = _chain_setup(dev, "NHD", 5)
    lens = s["lens0"].clone()
    for qkv in s["steps"]:
        slots = _slots(s["pt"], lens, s["page"])
        q = ops.gqa_qknorm_rope_cache_write(qkv.to(dev), lens.to(dev), s["table"].to(dev), slots.to(dev), s["kc"], s["vc"],
                                            s["hq"], s["hkv"], *_dev(s["w"], dev), 1e-6, True)
        out, lse = ops.gqa_decode(q, s["kc"], s["vc"], (lens + 1).to(dev), s["pt"].to(dev), D ** -0.5)
        torch.cuda.synchronize()
        q_ref, k_ref, v_in = _oracle_qk(qkv, lens.long(), s["table"], s["hq"], s["hkv"], s["rot"], s["w"], 1e-6, True)
        assert_ulps(q, q_ref, s["rot"], True)
        k_rows = torch.stack([s["kc"][int(x) // s["page"], int(x) % s["page"]] for x in slots]).cpu()
        v_rows = torch.stack([s["vc"][int(x) // s["page"], int(x) % s["page"]] for x in slots]).cpu()
        assert_ulps(k_rows, k_ref, s["rot"], True)
        assert torch.equal(v_rows, v_in)
        ref, lse_ref = _oracle_decode(q.cpu(), s["kc"], s["vc"], lens + 1, s["pt"], D ** -0.5)
        assert _cos_diff(out.cpu().float(), ref) < 1e-5
        torch.testing.assert_close(lse.cpu(), lse_ref, atol=1e-3, rtol=1e-3)
        lens += 1


def test_cuda_graph_replay_matches_eager_chain(dev):
    """write + decode captured once on static buffers, replayed for three steps with positions, slots and seq_lens
    updated in place: outputs and cache bit-identical to the eager chain."""
    from lvllm_b200 import ops
    s = _chain_setup(dev, "NHD", 7)
    phys_g = s["phys"].clone()
    kc_g, vc_g = phys_g.permute(0, 2, 1, 3).transpose(1, 2).split(D, dim=-1)
    table, pt = s["table"].to(dev), s["pt"].to(dev)
    w = _dev(s["w"], dev)
    qkv_s = torch.zeros(s["B"], (s["hq"] + 2 * s["hkv"]) * D, dtype=torch.bfloat16, device=dev)
    pos_s = torch.zeros(s["B"], dtype=torch.int64, device=dev)
    slot_s = torch.full((s["B"],), -1, dtype=torch.int64, device=dev)
    lens_s = torch.ones(s["B"], dtype=torch.int32, device=dev)

    def step():
        q = ops.gqa_qknorm_rope_cache_write(qkv_s, pos_s, table, slot_s, kc_g, vc_g, s["hq"], s["hkv"], *w, 1e-6, True)
        return ops.gqa_decode(q, kc_g, vc_g, lens_s, pt, D ** -0.5)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()                      # warm-up with slot -1 and seq_len 1: writes nothing
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(phys_g.view(torch.int16), s["phys"].view(torch.int16))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_s, lse_s = step()
    lens = s["lens0"].clone()
    for qkv in s["steps"]:
        slots = _slots(s["pt"], lens, s["page"])
        qkv_s.copy_(qkv)
        pos_s.copy_(lens)
        slot_s.copy_(slots)
        lens_s.copy_(lens + 1)
        graph.replay()
        q = ops.gqa_qknorm_rope_cache_write(qkv.to(dev), lens.to(dev), table, slots.to(dev), s["kc"], s["vc"], s["hq"],
                                            s["hkv"], *w, 1e-6, True)
        out, lse = ops.gqa_decode(q, s["kc"], s["vc"], (lens + 1).to(dev), pt, D ** -0.5)
        torch.cuda.synchronize()
        assert torch.equal(out_s.view(torch.int16), out.view(torch.int16))
        assert torch.equal(lse_s, lse)
        assert torch.equal(phys_g.view(torch.int16), s["phys"].view(torch.int16))
        lens += 1


@pytest.mark.parametrize("B,S,hq,hkv,norm", [(64, 2048, 32, 8, False),    # Mixtral-8x7B bench shape
                                             (256, 512, 64, 4, True)])    # Qwen3-235B-A22B bench shape
def test_bench_shapes_on_packed_nhd_cache(dev, B, S, hq, hkv, norm):
    from lvllm_b200 import ops
    gen = torch.Generator().manual_seed(9)
    page, rot = 16, 128
    npg = -(-(S + 1) // page)
    qkv, table, w = _inputs(gen, B, hq, hkv, 32768, rot, norm)
    dgen = torch.Generator(device=dev).manual_seed(9)
    phys, kc, vc = make_cache("NHD", B * npg, page, hkv, lambda s: torch.randn(*s, generator=dgen, device=dev).bfloat16())
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int()
    lens = torch.tensor([S - 7 * (b % 9) for b in range(B)], dtype=torch.int32)
    slots = _slots(pt, lens, page)
    q = ops.gqa_qknorm_rope_cache_write(qkv.to(dev), lens.to(dev), table.to(dev), slots.to(dev), kc, vc, hq, hkv,
                                        *_dev(w, dev), 1e-6, True)
    out, lse = ops.gqa_decode(q, kc, vc, (lens + 1).to(dev), pt.to(dev), D ** -0.5)
    torch.cuda.synchronize()
    q_ref, k_ref, _ = _oracle_qk(qkv, lens.long(), table, hq, hkv, rot, w, 1e-6, True)
    assert_ulps(q, q_ref, rot, True)
    k_rows = torch.stack([kc[int(x) // page, int(x) % page] for x in slots]).cpu()
    assert_ulps(k_rows, k_ref, rot, True)
    sel = [0, B // 2, B - 1]
    ref, lse_ref = _oracle_decode(q.cpu()[sel], kc, vc, lens[sel] + 1, pt[sel], D ** -0.5)
    assert _cos_diff(out.cpu().float()[sel], ref) < 1e-5
    torch.testing.assert_close(lse.cpu()[sel], lse_ref, atol=1e-3, rtol=1e-3)


def test_argument_refusals(dev):
    """Each refused case of the C entry points returns B200_ERR_INVALID (-1) and launches nothing."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    T, hq, hkv, page, blocks = 2, 16, 4, 16, 2
    qkv = torch.zeros(T, (hq + 2 * hkv) * D, dtype=torch.bfloat16, device=dev)
    pos = torch.zeros(T, dtype=torch.int64, device=dev)
    table = torch.zeros(16, D, dtype=torch.bfloat16, device=dev)
    slots = torch.tensor([0, 1], dtype=torch.int64, device=dev)
    cache = torch.zeros(2, blocks, page, hkv, D, dtype=torch.bfloat16, device=dev)
    q_out = torch.empty(T, hq, D, dtype=torch.bfloat16, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    base = dict(qkv=qkv.data_ptr(), pos=pos.data_ptr(), cs=table.data_ptr(), max_pos=16, rot=D, slots=slots.data_ptr(),
                kc=cache[0].data_ptr(), vc=cache[1].data_ptr(), bs=page * hkv * D, ps=hkv * D, hs=D, q_out=q_out.data_ptr(),
                head_dim=D)

    def call(**kw):
        a = dict(base, **kw)
        return lib.b200_gqa_qknorm_rope_cache_write(stream, a["qkv"], a["pos"], a["cs"], a["max_pos"], a["rot"], 1, None,
                                                    None, 1e-6, a["slots"], a["kc"], a["vc"], a["bs"], a["ps"], a["hs"],
                                                    page, a["q_out"], T, hq, hkv, a["head_dim"])

    assert call() == 0
    torch.cuda.synchronize()
    refused = [dict(head_dim=64), dict(head_dim=256), dict(rot=63), dict(rot=1), dict(rot=130), dict(bs=page * hkv * D + 4),
               dict(ps=hkv * D - 2), dict(hs=D + 1), dict(qkv=None), dict(pos=None), dict(cs=None), dict(slots=None),
               dict(kc=None), dict(vc=None), dict(q_out=None)]
    n0 = lib.b200moe_launch_count()
    for kw in refused:
        assert call(**kw) == -1, kw
    assert lib.b200moe_launch_count() == n0
    # the strided decode entry refuses strides the 16-byte row loads cannot follow
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    sl = torch.ones(1, dtype=torch.int32, device=dev)
    ptab = torch.zeros(1, 1, dtype=torch.int32, device=dev)
    out = torch.empty(1, hq, D, dtype=torch.bfloat16, device=dev)
    qd = torch.zeros(1, hq, D, dtype=torch.bfloat16, device=dev)
    for bs, ps, hs in ((page * hkv * D, hkv * D, D + 4), (page * hkv * D, 4, D), (12, hkv * D, D)):
        rc = lib.b200_gqa_decode_ex(stream, qd.data_ptr(), cache[0].data_ptr(), cache[1].data_ptr(), bs, ps, hs,
                                    sl.data_ptr(), ptab.data_ptr(), 1, hq, hkv, D, page, 1, 0.1, 1, ws.data_ptr(),
                                    out.data_ptr(), None)
        assert rc == -1, (bs, ps, hs)
