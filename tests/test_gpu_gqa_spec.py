"""GPU (-m gpu): multi-token GQA decode (speculative-decode verification, ops.gqa_decode(q_len_per_req=Q)).

Kernel vs the oracle (tests/gqa_spec_oracle.py) on separate and packed NHD / HND caches for both kernels, vs the
reference-generated golden fixture, bit for bit vs today's single-token call on the expanded batch, Q = 1 through the new
entry point vs b200_gqa_decode_ex, a write + decode verification chain eagerly and in a CUDA graph, the bench shapes, and the
argument refusals."""
import math
import os

import pytest
import torch

import gqa_oracle as GO
import gqa_spec_oracle as SO

pytestmark = pytest.mark.gpu

D = 128
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_gqa_spec.pt")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_diff(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return 1 - 2 * (a * b).sum() / max((a * a + b * b).sum(), 1e-12)


def make_cache(layout, blocks, page, hkv, fill):
    """(physical buffer, k view, v view): separate contiguous caches, or the FlashInfer backend's packed NHD / HND tensor
    split as the backend splits it (flashinfer.py:398-433, :2276-2290)."""
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


def _oracle(q, kc, vc, lens, pt, scale, Q, reqs):
    """The oracle on requests `reqs` (their pages gathered to the CPU, page table renumbered); returns (rows, out, lse)."""
    reqs = list(reqs)
    rows = [b * Q + i for b in reqs for i in range(Q)]
    sub = pt[reqs]
    pages = sub.flatten().long()
    ks, vs = kc[pages.to(kc.device)].cpu(), vc[pages.to(vc.device)].cpu()
    out, lse = SO.gqa_decode(q[rows].cpu(), ks, vs, lens[reqs], torch.arange(pages.numel(), dtype=torch.int32)
                             .reshape(sub.shape), scale, q_len=Q)
    return rows, out, lse


def _check_blind_rows(out, lse, lens, Q):
    """Rows with no visible key are exact zeros with lse -inf; every other output is finite."""
    blind = torch.tensor([int(lens[r // Q]) - Q + 1 + r % Q <= 0 for r in range(out.shape[0])])
    o, ls = out.cpu(), lse.cpu()
    assert not torch.isnan(o.float()).any() and not torch.isnan(ls).any()
    assert torch.equal(o[blind].view(torch.int16), torch.zeros_like(o[blind]).view(torch.int16))
    assert (ls[blind] == -math.inf).all()
    assert torch.isfinite(o[~blind].float()).all() and torch.isfinite(ls[~blind]).all()
    return blind


def _lens(B, S, Q, special):
    lens = [max(Q, S - 13 * (b % 5)) for b in range(B)]
    for b, s in special.items():
        if b < B:
            lens[b] = s
    return torch.tensor(lens, dtype=torch.int32)


def _setup(dev, layout, B, S, page, hq, hkv, Q, seed, special):
    gen = torch.Generator().manual_seed(seed)
    lens = _lens(B, S, Q, special)
    npg = -(-int(lens.max()) // page)
    dgen = torch.Generator(device=dev).manual_seed(seed)
    phys, kc, vc = make_cache(layout, B * npg, page, hkv, lambda s: torch.randn(*s, generator=dgen, device=dev).bfloat16())
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int()
    q = torch.randn(B * Q, hq, D, generator=gen).bfloat16()
    return q, kc, vc, lens, pt


# (B, S, page, Hq, Hkv, Q, num_kv_splits); lens: request 0 has S = Q, request 1 has 129 keys, request 2 fewer keys than Q
MATRIX = [
    (5, 300, 16, 32, 8, 2, 0), (5, 300, 16, 32, 8, 4, 0), (5, 300, 16, 32, 8, 8, 0),   # tensor cores, group 4
    (4, 333, 16, 64, 4, 2, 0), (4, 333, 16, 64, 4, 3, 0), (4, 333, 16, 64, 4, 4, 0),   # group 16: 1 / 2 / 2 q-groups
    (3, 200, 32, 8, 8, 16, 0),                                                          # group 1, 16 draft tokens
    (4, 250, 16, 48, 1, 2, 0),                                                          # group 48: CUDA cores
    (5, 300, 16, 32, 8, 3, 3),                                                          # 3 splits: CUDA cores
    (40, 1000, 16, 64, 4, 3, 0),                                                        # ~20 work items per CTA
]


@pytest.mark.parametrize("layout", ["separate", "NHD", "HND"])
@pytest.mark.parametrize("B,S,page,hq,hkv,Q,splits", MATRIX)
def test_spec_decode_vs_oracle(dev, layout, B, S, page, hq, hkv, Q, splits):
    from lvllm_b200 import ops
    q, kc, vc, lens, pt = _setup(dev, layout, B, S, page, hq, hkv, Q, 11, {0: Q, 1: 129, 2: max(1, Q - 2)})
    scale = D ** -0.5
    out, lse = ops.gqa_decode(q.to(dev), kc, vc, lens.to(dev), pt.to(dev), scale, num_kv_splits=splits,
                              q_len_per_req=Q)
    torch.cuda.synchronize()
    assert out.shape == (B * Q, hq, D) and lse.shape == (B * Q, hq)
    blind = _check_blind_rows(out, lse, lens, Q)
    assert blind.any()   # request 2 has fewer keys than Q
    rows, ref, lse_ref = _oracle(q, kc, vc, lens, pt, scale, Q, sorted({0, 1, 2, B - 1}))
    assert _cos_diff(out.cpu().float()[rows], ref) < 1e-5
    # l is the sum of the bf16-rounded P that the PV product uses: over a handful of keys (request 0 has S = Q) its rounding
    # does not average out, and lse is only within the bf16 unit roundoff 2^-8 (a single key is exact: P = 1)
    few = torch.tensor([0 < int(lens[r // Q]) - Q + 1 + r % Q < 16 for r in rows])
    torch.testing.assert_close(lse.cpu()[rows][~few], lse_ref[~few], atol=1e-3, rtol=1e-3)
    torch.testing.assert_close(lse.cpu()[rows][few], lse_ref[few], atol=2 ** -8, rtol=0)


def test_golden(dev):
    from lvllm_b200 import ops
    g = torch.load(GOLDEN, weights_only=True)
    for c in g["cases"]:
        p = g["pools"][c["num_kv_heads"]]
        Q = c["q_len"]
        out, lse = ops.gqa_decode(c["q"].to(dev), p["k_cache"].to(dev), p["v_cache"].to(dev),
                                  torch.tensor(c["kv_lens"], dtype=torch.int32, device=dev), c["block_tables"].to(dev),
                                  g["scale"], q_len_per_req=Q)
        torch.cuda.synchronize()
        assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
        # fixture is fp32 (reference ref_paged_attn); bf16 inputs / outputs -> cos_diff threshold of the reference MLA test
        assert _cos_diff(out.cpu().float(), c["out"]) < 5e-5, (c["num_heads"], c["num_kv_heads"], Q)


@pytest.mark.parametrize("B,S,hq,hkv,Q,splits,exact", [
    (5, 300, 32, 8, 2, 0, True),     # tensor cores, N = 16 in both calls
    (5, 300, 32, 8, 4, 0, True),
    (3, 200, 8, 8, 16, 0, True),     # group 1: 16 draft tokens fill the 16 columns the expanded call also uses
    (4, 250, 48, 1, 3, 0, True),     # CUDA cores (group 48)
    (5, 300, 32, 8, 3, 3, True),     # CUDA cores (3 splits)
    (4, 333, 64, 4, 2, 0, False),    # group 16: N = 32 against 16 in the expanded call
])
def test_matches_expanded_batch(dev, B, S, hq, hkv, Q, splits, exact):
    """The spec call against today's single-token call on the expanded batch: each (request, draft token) a request of
    its own (page-table row repeated, seq_len S_b - Q + 1 + i), same split count."""
    from lvllm_b200 import ops
    page = 16
    q, kc, vc, lens, pt = _setup(dev, "NHD", B, S, page, hq, hkv, Q, 23, {0: Q, 1: 129, 2: max(1, Q - 2)})
    scale = D ** -0.5
    qd, ptd = q.to(dev), pt.to(dev)
    out, lse = ops.gqa_decode(qd, kc, vc, lens.to(dev), ptd, scale, num_kv_splits=splits, q_len_per_req=Q)
    lens_x, pt_x = SO.expand(lens, pt, Q)
    out_x, lse_x = ops.gqa_decode(qd, kc, vc, lens_x.to(dev), pt_x.to(dev), scale, num_kv_splits=splits)
    torch.cuda.synchronize()
    if exact:
        assert torch.equal(out.view(torch.int16), out_x.view(torch.int16))
        assert torch.equal(lse, lse_x)
    else:
        assert _cos_diff(out.cpu().float(), out_x.cpu().float()) < 1e-5
        torch.testing.assert_close(lse, lse_x, atol=1e-3, rtol=1e-3)


@pytest.mark.parametrize("hq,hkv,splits", [(32, 8, 0), (48, 1, 0), (32, 8, 3)])
def test_q_len_1_is_decode_ex(dev, hq, hkv, splits):
    """b200_gqa_decode_spec with q_len 1 == b200_gqa_decode_ex, bit for bit, on both kernels."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    B, S, page = 6, 400, 16
    q, kc, vc, lens, pt = _setup(dev, "NHD", B, S, page, hq, hkv, 1, 31, {})
    splits = splits or -(-(pt.shape[1] * page) // 128)
    qd, ld, ptd = q.to(dev), lens.to(dev), pt.to(dev)
    ws = torch.empty(lib.b200_gqa_decode_workspace_bytes(B, hq, D, splits), dtype=torch.uint8, device=dev)
    bs, ps, hs = kc.stride()[:3]
    stream = torch.cuda.current_stream().cuda_stream
    res = []
    for fn in ("ex", "spec"):
        out = torch.empty(B, hq, D, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(B, hq, dtype=torch.float32, device=dev)
        args = [stream, qd.data_ptr(), kc.data_ptr(), vc.data_ptr(), bs, ps, hs, ld.data_ptr(), ptd.data_ptr(), B]
        args += [1] if fn == "spec" else []
        args += [hq, hkv, D, page, pt.shape[1], D ** -0.5, splits, ws.data_ptr(), out.data_ptr(), lse.data_ptr()]
        assert getattr(lib, f"b200_gqa_decode_{fn}")(*args) == 0
        res.append((out, lse))
    torch.cuda.synchronize()
    assert torch.equal(res[0][0].view(torch.int16), res[1][0].view(torch.int16))
    assert torch.equal(res[0][1], res[1][1])


def _slots(pt, pos, page, Q):
    b = torch.arange(pt.shape[0]).repeat_interleave(Q)
    return (pt[b, (pos // page).long()].long() * page + (pos % page).long()).to(torch.int64)


def _chain_setup(dev, seed, Q):
    gen = torch.Generator().manual_seed(seed)
    B, page, hq, hkv, rot = 3, 16, 16, 4, 128
    lens0 = torch.tensor([13, 30, 126], dtype=torch.int32)   # drafts cross pages and, for request 2, a 128-token split
    npg = -(-(int(lens0.max()) + 4 * Q) // page)
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int()
    inv = 1.0 / (1e6 ** (torch.arange(0, rot, 2, dtype=torch.float) / rot))
    fr = torch.einsum("i,j->ij", torch.arange(4096, dtype=torch.float), inv)
    table = torch.cat((fr.cos(), fr.sin()), dim=-1).bfloat16()
    w = ((1 + 0.1 * torch.randn(D, generator=gen)).bfloat16(), (1 + 0.1 * torch.randn(D, generator=gen)).bfloat16())
    steps = [(torch.randn(B * Q, (hq + 2 * hkv) * D, generator=gen) * 2).bfloat16() for _ in range(3)]
    accepted = [torch.tensor([1, Q, 2]), torch.tensor([Q, 1, 3]), torch.tensor([2, 3, 1])]
    dgen = torch.Generator(device=dev).manual_seed(seed)
    phys, kc, vc = make_cache("NHD", B * npg, page, hkv, lambda s: torch.randn(*s, generator=dgen, device=dev).bfloat16())
    return dict(B=B, page=page, hq=hq, hkv=hkv, rot=rot, lens0=lens0, pt=pt, table=table, w=w, steps=steps,
                accepted=accepted, phys=phys, kc=kc, vc=vc)


def _positions(lens, Q):
    return (lens.long().repeat_interleave(Q) + torch.arange(Q).repeat(lens.numel()))


def test_verification_chain_eager_and_graph(dev):
    """A verification step: the fused q/k-norm + RoPE + cache write puts Q tokens per request at positions S_b .. S_b+Q-1,
    then the spec decode runs with seq_lens S_b + Q.  Eagerly each step matches the oracle; captured once in a CUDA graph
    and replayed for three steps (qkv, positions, slots and seq_lens updated in place, requests advanced by different
    accepted counts), out, lse and the cache are bit-identical to the eager chain."""
    from lvllm_b200 import ops
    Q = 3
    s = _chain_setup(dev, 5, Q)
    B, page, hq, hkv = s["B"], s["page"], s["hq"], s["hkv"]
    table, pt = s["table"].to(dev), s["pt"].to(dev)
    w = tuple(x.to(dev) for x in s["w"])
    phys_g = s["phys"].clone()
    kc_g, vc_g = phys_g.permute(0, 2, 1, 3).transpose(1, 2).split(D, dim=-1)
    qkv_s = torch.zeros(B * Q, (hq + 2 * hkv) * D, dtype=torch.bfloat16, device=dev)
    pos_s = torch.zeros(B * Q, dtype=torch.int64, device=dev)
    slot_s = torch.full((B * Q,), -1, dtype=torch.int64, device=dev)
    lens_s = torch.full((B,), Q, dtype=torch.int32, device=dev)

    def step(qkv, pos, slots, lens, kc, vc):
        q = ops.gqa_qknorm_rope_cache_write(qkv, pos, table, slots, kc, vc, hq, hkv, *w, 1e-6, True)
        return (q,) + ops.gqa_decode(q, kc, vc, lens, pt, D ** -0.5, q_len_per_req=Q)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(qkv_s, pos_s, slot_s, lens_s, kc_g, vc_g)       # warm-up with slots -1: writes nothing
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(phys_g.view(torch.int16), s["phys"].view(torch.int16))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _, out_s, lse_s = step(qkv_s, pos_s, slot_s, lens_s, kc_g, vc_g)
    lens = s["lens0"].clone()
    for qkv, acc in zip(s["steps"], s["accepted"]):
        pos = _positions(lens, Q)
        slots = _slots(s["pt"], pos, page, Q)
        q, out, lse = step(qkv.to(dev), pos.to(dev), slots.to(dev), (lens + Q).to(dev), s["kc"], s["vc"])
        qkv_s.copy_(qkv)
        pos_s.copy_(pos)
        slot_s.copy_(slots)
        lens_s.copy_(lens + Q)
        graph.replay()
        torch.cuda.synchronize()
        # eager step vs the oracle: the kernel's own q, on the cache the kernel wrote
        q_ref = GO.qk_norm_rope(qkv, pos, s["table"], hq, hkv, D, s["rot"], s["w"][0], s["w"][1], 1e-6, True)
        q_ref = q_ref[:, :hq * D].reshape(B * Q, hq, D)
        assert _cos_diff(q.cpu().float(), q_ref.float()) < 1e-5
        rows, ref, lse_ref = _oracle(q.cpu(), s["kc"], s["vc"], lens + Q, s["pt"], D ** -0.5, Q, range(B))
        assert _cos_diff(out.cpu().float()[rows], ref) < 1e-5
        torch.testing.assert_close(lse.cpu()[rows], lse_ref, atol=1e-3, rtol=1e-3)
        # graph replay vs the eager chain
        assert torch.equal(out_s.view(torch.int16), out.view(torch.int16))
        assert torch.equal(lse_s, lse)
        assert torch.equal(phys_g.view(torch.int16), s["phys"].view(torch.int16))
        lens += acc.to(torch.int32)


@pytest.mark.parametrize("B,S,hq,hkv,Q", [(64, 2048, 32, 8, 2), (64, 2048, 32, 8, 4),   # Mixtral-8x7B bench shape
                                          (256, 512, 64, 4, 2)])                         # Qwen3-235B-A22B bench shape
def test_bench_shapes_on_packed_nhd_cache(dev, B, S, hq, hkv, Q):
    from lvllm_b200 import ops
    page = 16
    gen = torch.Generator().manual_seed(9)
    lens = torch.tensor([S + Q - 7 * (b % 9) for b in range(B)], dtype=torch.int32)
    npg = -(-int(lens.max()) // page)
    dgen = torch.Generator(device=dev).manual_seed(9)
    _, kc, vc = make_cache("NHD", B * npg, page, hkv, lambda s: torch.randn(*s, generator=dgen, device=dev).bfloat16())
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int()
    q = torch.randn(B * Q, hq, D, generator=gen).bfloat16()
    out, lse = ops.gqa_decode(q.to(dev), kc, vc, lens.to(dev), pt.to(dev), D ** -0.5, q_len_per_req=Q)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    rows, ref, lse_ref = _oracle(q, kc, vc, lens, pt, D ** -0.5, Q, [0, B // 2, B - 1])
    assert _cos_diff(out.cpu().float()[rows], ref) < 1e-5
    torch.testing.assert_close(lse.cpu()[rows], lse_ref, atol=1e-3, rtol=1e-3)


def test_refusals(dev):
    """q_len outside [1, 16] returns B200_ERR_INVALID (-1) and launches nothing; ops.gqa_decode refuses a q that does not
    hold q_len_per_req rows per request and a page table without one row per request."""
    from lvllm_b200 import _lib as L
    from lvllm_b200 import ops
    lib = L.lib()
    B, hq, hkv, page = 2, 16, 4, 16
    cache = torch.zeros(2, 2, page, hkv, D, dtype=torch.bfloat16, device=dev)
    ws = torch.empty(1 << 22, dtype=torch.uint8, device=dev)
    sl = torch.full((B,), 4, dtype=torch.int32, device=dev)
    ptab = torch.zeros(B, 1, dtype=torch.int32, device=dev)
    out = torch.empty(B * 17, hq, D, dtype=torch.bfloat16, device=dev)
    qd = torch.zeros(B * 17, hq, D, dtype=torch.bfloat16, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def call(q_len):
        return lib.b200_gqa_decode_spec(stream, qd.data_ptr(), cache[0].data_ptr(), cache[1].data_ptr(), page * hkv * D,
                                        hkv * D, D, sl.data_ptr(), ptab.data_ptr(), B, q_len, hq, hkv, D, page, 1, 0.1, 1,
                                        ws.data_ptr(), out.data_ptr(), None)

    n0 = lib.b200moe_launch_count()
    for q_len in (0, 17):
        assert call(q_len) == -1, q_len
        assert b"q_len" in lib.b200moe_last_error()
    assert lib.b200moe_launch_count() == n0
    assert call(16) == 0
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        ops.gqa_decode(qd[:B * 3 - 1], cache[0], cache[1], sl, ptab, 0.1, q_len_per_req=3)
    with pytest.raises(ValueError):
        ops.gqa_decode(qd[:B * 3], cache[0], cache[1], sl, ptab, 0.1, q_len_per_req=2)
    with pytest.raises(ValueError):
        ops.gqa_decode(qd[:B * 3], cache[0], cache[1], sl, torch.zeros(B + 1, 1, dtype=torch.int32, device=dev), 0.1,
                       q_len_per_req=3)
