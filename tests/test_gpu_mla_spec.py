"""GPU (-m gpu): multi-token MLA decode (verification of multi-token-prediction drafts, ops.mla_decode(q_len_per_req=Q)).

Kernel vs the oracle (tests/mla_spec_oracle.py) over head counts, draft lengths, split counts and edge-case lengths, on the
bf16 and the e4m3 cache; vs the reference-generated golden fixture; bit for bit vs today's single-token call on the
expanded batch; Q = 1 through the new entry point vs b200_mla_decode_ex / b200_mla_decode_vup; a rope + cache write ->
q absorb -> decode + v up-projection verification chain, eagerly and in a CUDA graph; and the argument refusals."""
import math
import os

import pytest
import torch

import mla_spec_oracle as SO
from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu

F8 = torch.float8_e4m3fn
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_mla_spec.pt")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_diff(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return 1 - 2 * (a * b).sum() / max((a * a + b * b).sum(), 1e-12)


def _visible(lens, Q, rows):
    """Keys seen by query rows `rows` (b * Q + i): S_b - Q + 1 + i."""
    return torch.tensor([int(lens[r // Q]) - Q + 1 + r % Q for r in rows])


def _check_blind_rows(out, lse, lens, Q):
    """Rows with no visible key are exact zeros with lse -inf; every other output is finite."""
    blind = _visible(lens, Q, range(out.shape[0])) <= 0
    o, ls = out.cpu(), lse.cpu()
    assert not torch.isnan(o.float()).any() and not torch.isnan(ls).any()
    assert torch.equal(o[blind].view(torch.int16), torch.zeros_like(o[blind]).view(torch.int16))
    assert (ls[blind] == -math.inf).all()
    assert torch.isfinite(o[~blind].float()).all() and torch.isfinite(ls[~blind]).all()
    return blind


def _check_lse(lse, lse_ref, lens, Q, rows):
    """The reference's lse bound (1e-3), except for rows that see fewer than 16 keys: l is the sum of the bf16-rounded P
    the PV product uses, and over a handful of keys that rounding does not average out (bf16 unit roundoff 2^-8; a single
    key is exact, P = 1).  Blind rows are -inf on both sides."""
    vis = _visible(lens, Q, rows)
    few, blind = (vis > 0) & (vis < 16), vis <= 0
    ls = lse.cpu()[rows]
    torch.testing.assert_close(ls[~few & ~blind], lse_ref[~few & ~blind], atol=1e-3, rtol=1e-3)
    torch.testing.assert_close(ls[few], lse_ref[few], atol=2 ** -8, rtol=0)
    assert (ls[blind] == -math.inf).all() and (lse_ref[blind] == -math.inf).all()


def _oracle(qn, qp, cache, lens, pt, scale, Q, reqs):
    """The oracle on requests `reqs` (their pages gathered to the CPU, page table renumbered); returns (rows, out, lse)."""
    reqs = list(reqs)
    rows = [b * Q + i for b in reqs for i in range(Q)]
    sub = pt[reqs]
    pages = sub.flatten().long()
    out, lse = SO.mla_decode(qn[rows].cpu(), qp[rows].cpu(), cache[pages.to(cache.device)].cpu(), lens[reqs],
                             torch.arange(pages.numel(), dtype=torch.int32).reshape(sub.shape), scale, q_len=Q)
    return rows, out, lse


def _lens(B, S, Q, special):
    lens = [max(Q, S - 13 * (b % 5)) for b in range(B)]
    for b, s in special.items():
        if b < B:
            lens[b] = s
    return torch.tensor(lens, dtype=torch.int32)


def _setup(dev, B, S, page, hq, Q, seed, special, kv_dtype=torch.bfloat16, q8=False):
    gen = torch.Generator().manual_seed(seed)
    lens = _lens(B, S, Q, special)
    npg = -(-int(lens.max()) // page)
    dgen = torch.Generator(device=dev).manual_seed(seed)
    cache = torch.randn(B * npg + 2, page, 576, generator=dgen, device=dev).to(kv_dtype)
    pt = torch.randperm(B * npg + 2, generator=gen)[:B * npg].reshape(B, npg).int()   # shuffled pages
    qn = torch.randn(B * Q, hq, 512, generator=gen).bfloat16()
    qp = torch.randn(B * Q, hq, 64, generator=gen).bfloat16()
    if q8:
        qn, qp = qn.to(F8), qp.to(F8)
    return qn, qp, cache, lens, pt


def _special(Q):
    """Request lengths of the edge cases, beside request 0, which keeps the row's S: S = Q, 129 (the draft crosses a
    128-token tile), S < Q (blind rows)."""
    return {1: Q, 2: 129, 3: max(1, Q - 2)}


# (B, S, page, Hq, Q, num_kv_splits)
MATRIX = [
    (1, 4096, 64, 128, 2, 0), (1, 4096, 64, 128, 4, 0),   # bench shape (DeepSeek-V3, Hq 128): one draft token per q-group
    (4, 4096, 64, 128, 3, 8),                             # Hq 128, CTAs walking 4 tiles, the edge cases beside S = 4096
    (5, 300, 16, 16, 4, 0), (5, 300, 16, 16, 8, 0),       # TP8 shard: one q-group, and an exactly full one
    (4, 333, 16, 64, 3, 0),                               # two q-groups, the second partial (2 + 1 draft tokens)
    (4, 250, 16, 20, 3, 0),                               # 20 heads: 6 draft tokens fit, 8 rows unused
    (4, 200, 32, 8, 16, 0), (4, 200, 32, 20, 16, 0),      # 16 draft tokens: one full q-group / three of 6, 6, 4
    (5, 700, 16, 16, 4, 2),                               # 2 splits: CTAs walk 3 tiles, the causal limit in the last one
    (2, 700, 16, 16, 4, 600),                             # more than 512 splits: decode_merge_kernel<512>
]


@pytest.mark.parametrize("B,S,page,hq,Q,splits", MATRIX)
def test_spec_decode_vs_oracle(dev, B, S, page, hq, Q, splits):
    from lvllm_b200 import ops
    qn, qp, cache, lens, pt = _setup(dev, B, S, page, hq, Q, 11, _special(Q))
    scale = 1.0 / math.sqrt(576)
    out, lse = ops.mla_decode(qn.to(dev), qp.to(dev), cache, lens.to(dev), pt.to(dev), scale, num_kv_splits=splits,
                              q_len_per_req=Q)
    torch.cuda.synchronize()
    assert out.shape == (B * Q, hq, 512) and lse.shape == (B * Q, hq)
    blind = _check_blind_rows(out, lse, lens, Q)
    assert int(lens[0]) == S and blind.any() == (B > 3)   # request 3 has fewer keys than Q
    rows, ref, lse_ref = _oracle(qn, qp, cache, lens, pt, scale, Q, sorted({0, 1, 2, 3, B - 1} & set(range(B))))
    # metric + thresholds of reference tests/kernels/attention/test_cutlass_mla_decode.py:15-32
    assert _cos_diff(out.cpu().float()[rows], ref) < 1e-5
    _check_lse(lse, lse_ref, lens, Q, rows)


@pytest.mark.parametrize("B,S,page,hq,Q,q8", [(4, 300, 16, 16, 4, False), (4, 300, 16, 16, 4, True),
                                              (1, 4096, 64, 128, 2, True), (4, 4096, 64, 128, 3, False),
                                              (4, 333, 16, 64, 3, False)])
def test_spec_decode_fp8_cache_vs_oracle(dev, B, S, page, hq, Q, q8):
    """The e4m3 latent cache with bf16 or e4m3 queries against the oracle on the descaled inputs (as the single-token
    test_mla_decode_fp8_cache_vs_oracle; reference fp8 mode of test_cutlass_mla_decode.py:101-110, cos_diff < 1e-4)."""
    from lvllm_b200 import ops
    qn, qp, cache, lens, pt = _setup(dev, B, S, page, hq, Q, 13, _special(Q), kv_dtype=F8, q8=q8)
    scale = 1.0 / math.sqrt(576)
    dq_k, dq_q = 0.5, 2.0
    out, lse = ops.mla_decode(qn.to(dev), qp.to(dev), cache, lens.to(dev), pt.to(dev), scale, max_seq_len=int(lens.max()),
                              q_scale=dq_q, k_scale=dq_k, q_len_per_req=Q)
    torch.cuda.synchronize()
    blind = _check_blind_rows(out, lse, lens, Q)
    assert int(lens[0]) == S and blind.any() == (B > 3)
    f = dq_q if q8 else 1.0
    rows, ref, lse_ref = _oracle((qn.float() * f).bfloat16(), (qp.float() * f).bfloat16(), (cache.float() * dq_k).bfloat16(),
                                 lens, pt, scale, Q, sorted({0, 1, 2, 3, B - 1} & set(range(B))))
    assert _cos_diff(out.cpu().float()[rows], ref) < 1e-4
    _check_lse(lse, lse_ref, lens, Q, rows)


def test_golden(dev):
    from lvllm_b200 import ops
    g = torch.load(GOLDEN, weights_only=True)
    for c in g["cases"]:
        Q, B, hq = c["q_len"], len(c["kv_lens"]), c["num_heads"]
        q = g["q_pool"][:c["q_rows"]].reshape(B * Q, hq, 576)
        lens = torch.tensor(c["kv_lens"], dtype=torch.int32)
        out, lse = ops.mla_decode(q[..., :512].contiguous().to(dev), q[..., 512:].contiguous().to(dev), g["kv_cache"].to(dev),
                                  lens.to(dev), c["block_tables"].to(dev), g["scale"], q_len_per_req=Q)
        torch.cuda.synchronize()
        assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
        # the fixture is fp32 (the reference's causal SDPA) and keeps every fourth value dim
        assert _cos_diff(out.cpu().float()[..., g["out_dims"]], c["out"]) < 1e-5, (hq, Q)
        _check_lse(lse, c["lse"], lens, Q, list(range(B * Q)))


@pytest.mark.parametrize("B,S,page,hq,Q,splits,kv8", [
    (5, 300, 16, 16, 4, 3, False),     # one q-group: four draft tokens share each KV tile
    (4, 333, 16, 64, 3, 3, False),     # two q-groups
    (1, 4096, 64, 128, 2, 8, False),   # bench shape, CTAs walking 4 tiles
    (4, 4096, 64, 128, 3, 8, True),    # Hq 128 on the e4m3 cache, the edge cases beside S = 4096
    (4, 700, 16, 20, 16, 2, True),     # e4m3 cache, three q-groups, CTAs walking several tiles
    (2, 700, 16, 16, 4, 600, False),   # more than 512 splits
])
def test_matches_expanded_batch(dev, B, S, page, hq, Q, splits, kv8):
    """The spec call against today's single-token call on the expanded batch (each (request, draft token) a request of its
    own: page-table row repeated, seq_len S_b - Q + 1 + i), with the same split count and page-table width.  A row's
    arithmetic does not depend on the other MMA rows and masked tiles add exact zeros: bit-identical."""
    from lvllm_b200 import ops
    qn, qp, cache, lens, pt = _setup(dev, B, S, page, hq, Q, 23, _special(Q), kv_dtype=F8 if kv8 else torch.bfloat16)
    assert int(lens[0]) == S
    scale = 1.0 / math.sqrt(576)
    qnd, qpd = qn.to(dev), qp.to(dev)
    out, lse = ops.mla_decode(qnd, qpd, cache, lens.to(dev), pt.to(dev), scale, num_kv_splits=splits, k_scale=0.5,
                              q_len_per_req=Q)
    lens_x, pt_x = SO.expand(lens, pt, Q)
    out_x, lse_x = ops.mla_decode(qnd, qpd, cache, lens_x.to(dev), pt_x.to(dev), scale, num_kv_splits=splits, k_scale=0.5)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), out_x.view(torch.int16))
    assert torch.equal(lse, lse_x)


@pytest.mark.parametrize("kv8,q8", [(False, False), (True, False), (True, True)])
def test_q_len_1_is_decode_ex_and_vup(dev, kv8, q8):
    """b200_mla_decode_spec with q_len 1 == b200_mla_decode_ex (w_uv NULL) and == b200_mla_decode_vup (w_uv given), bit for
    bit."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    B, S, page, hq, splits = 4, 900, 32, 32, 5
    qn, qp, cache, lens, pt = _setup(dev, B, S, page, hq, 1, 31, {}, kv_dtype=F8 if kv8 else torch.bfloat16, q8=q8)
    gen = torch.Generator().manual_seed(3)
    w_uv = (torch.randn(hq, 512, 128, generator=gen) / math.sqrt(512)).bfloat16().to(dev)
    qnd, qpd, ld, ptd = qn.to(dev), qp.to(dev), lens.to(dev), pt.to(dev)
    ws = torch.empty(lib.b200_mla_decode_workspace_bytes(B, hq, splits), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    head = [stream, qnd.data_ptr(), qpd.data_ptr(), int(q8), cache.data_ptr(), int(kv8), 2.0, 0.5, ld.data_ptr(),
            ptd.data_ptr(), B]
    tail = [hq, page, pt.shape[1], 1.0 / math.sqrt(576), splits, ws.data_ptr()]

    def bufs():
        return (torch.empty(B, hq, 512, dtype=torch.bfloat16, device=dev), torch.empty(B, hq, dtype=torch.float32, device=dev),
                torch.empty(B, hq, 128, dtype=torch.bfloat16, device=dev))

    o0, l0, _ = bufs()
    assert lib.b200_mla_decode_ex(*head, *tail, o0.data_ptr(), l0.data_ptr()) == 0
    o1, l1, _ = bufs()
    assert lib.b200_mla_decode_spec(*head, 1, *tail, o1.data_ptr(), l1.data_ptr(), None, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(o0.view(torch.int16), o1.view(torch.int16)) and torch.equal(l0, l1)
    o2, l2, v2 = bufs()
    assert lib.b200_mla_decode_vup(*head, *tail, w_uv.data_ptr(), v2.data_ptr(), o2.data_ptr(), l2.data_ptr()) == 0
    o3, l3, v3 = bufs()
    assert lib.b200_mla_decode_spec(*head, 1, *tail, o3.data_ptr(), l3.data_ptr(), w_uv.data_ptr(), v3.data_ptr()) == 0
    torch.cuda.synchronize()
    assert torch.equal(v2.view(torch.int16), v3.view(torch.int16)) and torch.equal(o2.view(torch.int16), o3.view(torch.int16))
    assert torch.equal(l2, l3)


def _chain_setup(dev, seed, Q):
    gen = torch.Generator().manual_seed(seed)
    B, page, hq = 3, 64, 16
    lens0 = torch.tensor([62, 10, 126], dtype=torch.int32)   # request 0's draft crosses a page, request 2's a 128-token tile
    npg = -(-(int(lens0.max()) + 4 * Q) // page)
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int()
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.float) / 64))
    fr = torch.einsum("i,j->ij", torch.arange(4096, dtype=torch.float), inv)
    table = torch.cat((fr.cos(), fr.sin()), dim=-1).bfloat16()
    w_uk_t = (torch.randn(hq, 128, 512, generator=gen) / math.sqrt(128)).bfloat16()
    w_uv = (torch.randn(hq, 512, 128, generator=gen) / math.sqrt(512)).bfloat16()
    steps = [dict(q_nope=torch.randn(B * Q, hq, 128, generator=gen).bfloat16(),
                  q_pe=torch.randn(B * Q, hq, 64, generator=gen).bfloat16(),
                  k_pe=torch.randn(B * Q, 64, generator=gen).bfloat16(),
                  kv_c=torch.randn(B * Q, 512, generator=gen).bfloat16()) for _ in range(3)]
    accepted = [torch.tensor([1, Q, 2]), torch.tensor([Q, 1, 3]), torch.tensor([2, 3, 1])]
    dgen = torch.Generator(device=dev).manual_seed(seed)
    cache = torch.randn(B * npg, page, 576, generator=dgen, device=dev).bfloat16()
    return dict(B=B, page=page, hq=hq, lens0=lens0, pt=pt, table=table, w_uk_t=w_uk_t, w_uv=w_uv, steps=steps,
                accepted=accepted, cache=cache)


def test_verification_chain_eager_and_graph(dev):
    """A verification step: RoPE + latent cache write of Q draft tokens per request at positions S_b .. S_b+Q-1 (slots
    crossing a 64-token page), q absorb, then the spec decode with seq_lens S_b + Q and the fused merge + v up-projection.
    Eagerly each step matches the oracle chain; captured once in a CUDA graph and replayed for three steps (inputs,
    positions, slots and seq_lens updated in place, requests advanced by different accepted counts), out_v, out, lse and
    the cache are bit-identical to the eager chain."""
    from lvllm_b200 import ops
    Q = 3
    s = _chain_setup(dev, 5, Q)
    B, page, hq = s["B"], s["page"], s["hq"]
    table, pt = s["table"].to(dev), s["pt"].to(dev)
    w_uk_t, w_uv = s["w_uk_t"].to(dev), s["w_uv"].to(dev)
    scale = 1.0 / math.sqrt(192)
    cache_g = s["cache"].clone()
    st = {k: torch.zeros_like(v, device=dev) for k, v in s["steps"][0].items()}
    pos_s = torch.zeros(B * Q, dtype=torch.int64, device=dev)
    slot_s = torch.full((B * Q,), -1, dtype=torch.int64, device=dev)
    lens_s = torch.full((B,), Q, dtype=torch.int32, device=dev)

    def step(x, pos, slots, lens, cache):
        ops.mla_rope_cache_write(x["q_pe"], x["k_pe"], x["kv_c"], pos, table, slots, cache)   # q_pe, k_pe rotated in place
        ql = ops.mla_q_absorb(x["q_nope"], w_uk_t)
        return (ql,) + ops.mla_decode(ql, x["q_pe"], cache, lens, pt, scale, w_uv=w_uv, q_len_per_req=Q)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(st, pos_s, slot_s, lens_s, cache_g)       # warm-up with slots -1: writes nothing
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(cache_g.view(torch.int16), s["cache"].view(torch.int16))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _, v_s, o_s, lse_s = step(st, pos_s, slot_s, lens_s, cache_g)
    lens = s["lens0"].clone()
    for x, acc in zip(s["steps"], s["accepted"]):
        pos = lens.long().repeat_interleave(Q) + torch.arange(Q).repeat(B)
        b = torch.arange(B).repeat_interleave(Q)
        slots = (s["pt"][b, (pos // page)].long() * page + pos % page).to(torch.int64)
        if torch.equal(lens, s["lens0"]):   # the first step: request 0's draft crosses a page
            assert (pos[:Q] // page).unique().numel() == 2
        cache_before = s["cache"].cpu()
        xd = {k: v.to(dev) for k, v in x.items()}
        ql, out_v, o, lse = step(xd, pos.to(dev), slots.to(dev), (lens + Q).to(dev), s["cache"])
        for k in st:
            st[k].copy_(x[k])
        pos_s.copy_(pos)
        slot_s.copy_(slots)
        lens_s.copy_(lens + Q)
        graph.replay()
        torch.cuda.synchronize()
        # eager step vs the oracle chain: rope (the kernel rounds once, the reference after every bf16 op: <= 2 ulp)
        qp_ref, kp_ref = O.rope_forward_static(pos, x["q_pe"].reshape(B * Q, hq * 64), x["k_pe"], 64, 64, s["table"], False)
        torch.testing.assert_close(xd["q_pe"].cpu().float(), qp_ref.reshape(B * Q, hq, 64).float(), atol=3e-2, rtol=2e-2)
        torch.testing.assert_close(xd["k_pe"].cpu().float(), kp_ref.float(), atol=3e-2, rtol=2e-2)
        # cache write of the kernel's own rotated k_pe, bit for bit
        ref_cache = O.concat_and_cache_mla(x["kv_c"], xd["k_pe"].cpu(), cache_before.clone(), slots)
        assert torch.equal(s["cache"].cpu().view(torch.int16), ref_cache.view(torch.int16))
        ql_ref = O.mla_q_absorb(x["q_nope"], s["w_uk_t"])
        torch.testing.assert_close(ql.cpu().float(), ql_ref.float(), atol=2e-2, rtol=2e-2)
        # decode + v up-projection on the kernel's own ql / q_pe and cache
        rows, o_ref, lse_ref = _oracle(ql.cpu(), xd["q_pe"].cpu(), s["cache"], lens + Q, s["pt"], scale, Q, range(B))
        v_ref = O.mla_v_up(o_ref.bfloat16(), s["w_uv"])
        assert _cos_diff(o.cpu().float(), o_ref) < 1e-5
        assert _cos_diff(out_v.cpu().float(), v_ref.float()) < 2e-5
        _check_lse(lse, lse_ref, lens + Q, Q, rows)
        # graph replay vs the eager chain
        for a, e in ((v_s, out_v), (o_s, o)):
            assert torch.equal(a.view(torch.int16), e.view(torch.int16))
        assert torch.equal(lse_s, lse)
        assert torch.equal(cache_g.view(torch.int16), s["cache"].view(torch.int16))
        lens += acc.to(torch.int32)


def test_refusals(dev):
    """q_len outside [1, 16] returns B200_ERR_INVALID (-1) and launches nothing; ops.mla_decode refuses a q that does not
    hold q_len_per_req rows per request, a page table with fewer rows than requests, and more than 128 heads."""
    from lvllm_b200 import _lib as L
    from lvllm_b200 import ops
    from lvllm_b200._lib import B200Error
    lib = L.lib()
    B, hq, page = 2, 16, 16
    cache = torch.zeros(2, page, 576, dtype=torch.bfloat16, device=dev)
    ws = torch.empty(lib.b200_mla_decode_workspace_bytes(B * 17, hq, 1), dtype=torch.uint8, device=dev)
    sl = torch.full((B,), 4, dtype=torch.int32, device=dev)
    ptab = torch.zeros(B, 1, dtype=torch.int32, device=dev)
    out = torch.empty(B * 17, hq, 512, dtype=torch.bfloat16, device=dev)
    qn = torch.zeros(B * 17, hq, 512, dtype=torch.bfloat16, device=dev)
    qp = torch.zeros(B * 17, hq, 64, dtype=torch.bfloat16, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def call(q_len):
        return lib.b200_mla_decode_spec(stream, qn.data_ptr(), qp.data_ptr(), 0, cache.data_ptr(), 0, 1.0, 1.0, sl.data_ptr(),
                                        ptab.data_ptr(), B, q_len, hq, page, 1, 0.1, 1, ws.data_ptr(), out.data_ptr(), None,
                                        None, None)

    n0 = lib.b200moe_launch_count()
    for q_len in (0, 17):
        assert call(q_len) == -1, q_len
        assert b"q_len" in lib.b200moe_last_error()
    assert lib.b200moe_launch_count() == n0
    assert call(16) == 0
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        ops.mla_decode(qn[:B * 3 - 1], qp[:B * 3 - 1], cache, sl, ptab, 0.1, q_len_per_req=3)
    with pytest.raises(ValueError):
        ops.mla_decode(qn[:B * 3], qp[:B * 3], cache, sl, ptab, 0.1, q_len_per_req=2)
    with pytest.raises(ValueError):   # fewer page-table rows than requests: the kernel would read past the table
        ops.mla_decode(qn[:B * 3], qp[:B * 3], cache, sl, ptab[:1], 0.1, q_len_per_req=3)
    with pytest.raises(B200Error, match="num_heads <= 128"):
        ops.mla_decode(torch.zeros(B * 2, 129, 512, dtype=torch.bfloat16, device=dev),
                       torch.zeros(B * 2, 129, 64, dtype=torch.bfloat16, device=dev), cache, sl, ptab, 0.1, q_len_per_req=2)
