"""GPU (-m gpu): the lightning indexer for decode (ops.indexer_qk_rope_quant_cache_write, indexer_logits, indexer_topk,
indexer_decode).

The q/k write byte for byte against the oracle (tests/indexer_oracle.py); the logits against the float64 oracle over head
counts, draft-token counts, page sizes and short or ragged sequences, and against the reference-generated golden
(golden_indexer.pt) at the reference test's threshold; the top-k exactly against the oracle (order included, forced ties
included), by the reference's comparison on kernel-made logits, and on 160K-token rows in the cluster and one-CTA forms;
the chain into sparse MLA decode eagerly and as a CUDA-graph replay; the argument refusals."""
import math
import os

import pytest
import torch

import indexer_oracle as IX

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_indexer.pt")
SENT = 12345.0
INVALID = -1   # B200_ERR_INVALID


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


# Hopper's e4m3 wgmma accumulates its products with fewer mantissa bits than fp32 (the reason DeepGEMM promotes its fp8
# accumulators), so the kernel's logits are compared with the float64 oracle against the magnitude of the summed terms,
# k_scale * sum_h |w_h| * (|q_h| . |k|), not against the logit itself, which cancellation can make small.  Observed on an
# H100: up to 2e-4 of the logit where the two are alike.
ACC_TOL = 2 ** -10


def _abs_bound(q8, w, cache, sl, pt, Q, width):
    return IX.paged_logits(q8.float().abs().to(torch.float8_e4m3fn), w.abs(), _abs_cache(cache), sl, pt, Q, width)


def _abs_cache(cache):
    """The cache with every e4m3 value byte replaced by its magnitude (sign bit cleared); scales are positive."""
    nb, page, _ = cache.shape
    flat = cache.reshape(nb, page * 132).clone()
    flat[:, :page * 128] &= 0x7F
    return flat.reshape(nb, page, 132)


def _calc_diff(x, y):
    x, y = x.double(), y.double()
    return 1 - 2 * (x * y).sum() / (x * x + y * y).sum()


def _qk_inputs(gen, T, H, P=300):
    q = (torch.randn(T, H, 128, generator=gen) * torch.logspace(-2, 1, H)[None, :, None]).bfloat16()
    fused = torch.randn(T, H + 128 + 8, generator=gen).bfloat16()       # [k | weights | pad], weights a column slice
    k = fused[:, :128].contiguous()
    w = fused[:, 128:128 + H]
    cs = torch.randn(P, 64, generator=gen).bfloat16()
    pos = torch.randint(-3, P + 3, (T,), generator=gen)                 # clamped to the table
    return q, w, k, cs, pos


def _cache(gen, R, npg, page, H, Q, lens, ue8m0=True):
    """An indexer cache written by the oracle for R requests of `lens` keys over a random page table, with the q side of
    B*Q draft tokens."""
    nb = R * npg + 3
    pt = torch.randperm(nb, generator=gen)[:R * npg].reshape(R, npg).int()
    cache = torch.zeros(nb, page, 132, dtype=torch.uint8)
    k = torch.randn(R * npg * page, 128, generator=gen).bfloat16()
    slots = (pt.long()[:, :, None] * page + torch.arange(page)).reshape(-1)
    IX.k_quant_cache(k, slots, cache, ue8m0)
    q = torch.randn(R * Q, H, 128, generator=gen).bfloat16()
    wt = torch.randn(R * Q, H, generator=gen).bfloat16()
    q8, w = IX.q_rope_quant(q, wt, torch.zeros(R * Q, dtype=torch.long), torch.ones(1, 64).bfloat16(), True,
                            128 ** -0.5, H ** -0.5)
    return q8, w, cache, torch.tensor(lens, dtype=torch.int32), pt


@pytest.mark.parametrize("neox", [True, False], ids=["neox", "interleaved"])
@pytest.mark.parametrize("ue8m0", [True, False], ids=["ue8m0", "fp32_scale"])
def test_qk_write_bit_exact(dev, neox, ue8m0):
    from lvllm_b200 import ops
    T, H, page, nb = 37, 64, 16, 5
    gen = torch.Generator().manual_seed(int(neox) * 2 + int(ue8m0))
    q, w, k, cs, pos = _qk_inputs(gen, T, H)
    slots = torch.randperm(nb * page, generator=gen)[:T]
    slots[[3, 20]] = -1
    cache = torch.full((nb, page, 132), 0xAB, dtype=torch.uint8)
    wd = torch.cat([k, w, torch.zeros(T, 8).bfloat16()], 1).to(dev)[:, 128:128 + H]
    cache_d = cache.to(dev)
    q8, wo = ops.indexer_qk_rope_quant_cache_write(q.to(dev), wd, k.to(dev), pos.to(dev), cs.to(dev), slots.to(dev),
                                                   cache_d, 128 ** -0.5, H ** -0.5, neox, ue8m0)
    torch.cuda.synchronize()
    rq8, rwo = IX.q_rope_quant(q, w, pos, cs, neox, 128 ** -0.5, H ** -0.5)
    assert torch.equal(q8.cpu().view(torch.uint8), rq8.view(torch.uint8))
    assert torch.equal(wo.cpu().view(torch.int32), rwo.view(torch.int32))
    IX.k_quant_cache(IX.k_rope(k, pos, cs, neox), slots, cache, ue8m0)
    assert torch.equal(cache_d.cpu(), cache)                          # slot -1 rows keep their 0xAB sentinels
    assert (cache == 0xAB).any()


LOGIT_CASES = [(H, Q, page) for H in (32, 64) for Q in (1, 2, 3, 4, 16) for page in (16, 64)]


@pytest.mark.parametrize("H,Q,page", LOGIT_CASES)
def test_logits_vs_oracle(dev, H, Q, page):
    from lvllm_b200 import ops
    npg = 6 if page == 64 else 20
    cap = npg * page
    lens = [0, 1, max(1, Q - 1), cap, cap - 7, 2 * page + 3, 97]
    gen = torch.Generator().manual_seed(H * 100 + Q * 10 + page)
    q8, w, cache, sl, pt = _cache(gen, len(lens), npg, page, H, Q, lens)
    width = cap + 40
    lg = torch.full((len(lens) * Q, width), SENT, device=dev)
    ops.indexer_logits(q8.to(dev), w.to(dev), cache.to(dev), sl.to(dev), pt.to(dev), Q, logits=lg)
    torch.cuda.synchronize()
    got = lg.cpu().double()
    ref = IX.paged_logits(q8, w, cache, sl, pt, Q, cap)
    bound = _abs_bound(q8, w, cache, sl, pt, Q, cap)
    for r in range(len(lens) * Q):
        S = lens[r // Q]
        end = max(0, S - Q + r % Q + 1)
        limit = -(-S // page) * page
        if end:
            assert ((got[r, :end] - ref[r, :end]).abs() <= ACC_TOL * bound[r, :end]).all(), r
        assert (got[r, end:limit] == -math.inf).all(), r
        assert (got[r, limit:] == SENT).all(), r                      # nothing past the request's pages


@pytest.mark.parametrize("Q,table_pages", [(1, 128), (2, 128), (1, 2560)], ids=["q1", "q2", "wide_table"])
def test_logits_steady_state_vs_oracle(dev, Q, table_pages):
    """Many more work items than CTAs and more tiles per item than pipeline stages: 64 requests of up to 8192 keys (page 64),
    so every CTA takes several items (the q tile and weights are reloaded between them) and its stage ring wraps (the
    producer waits on stages the MMA warpgroup has not yet released).  Contexts are ragged; in the wide_table case the
    page table is 20 times wider than the longest context, as an engine's max_model_len-wide table is, and the kernel
    still sizes its work from the contexts."""
    from lvllm_b200 import ops
    H, page, B = 64, 64, 64
    gen = torch.Generator().manual_seed(40 + Q + table_pages)
    lens = [8192] * 48 + torch.randint(1, 8192, (16,), generator=gen).tolist()
    npg = 8192 // page
    q8, w, cache, sl, pt = _cache(gen, B, npg, page, H, Q, lens)
    if table_pages > npg:    # the extra entries name blocks that are never read
        pt = torch.cat([pt, torch.zeros(B, table_pages - npg, dtype=torch.int32)], 1)
    lg = ops.indexer_logits(q8.to(dev), w.to(dev), cache.to(dev), sl.to(dev), pt.to(dev), Q)
    torch.cuda.synchronize()
    got = lg[:, :npg * page].cpu().double()
    ref = IX.paged_logits(q8, w, cache, sl, pt, Q, npg * page)
    bound = _abs_bound(q8, w, cache, sl, pt, Q, npg * page)
    fin = torch.isfinite(ref)
    assert ((got[fin] - ref[fin]).abs() <= ACC_TOL * bound[fin]).all()
    for r in range(B * Q):                                            # -inf from row_end to the end of the last page
        S = lens[r // Q]
        assert (got[r, S - Q + r % Q + 1:-(-S // page) * page] == -math.inf).all(), r


def test_logits_golden(dev):
    from lvllm_b200 import ops
    g = torch.load(GOLDEN, weights_only=True)
    for name in ("logits_q1", "logits_q2", "logits_q3"):
        c = g[name]
        ref = c["logits"]
        lg = ops.indexer_logits(c["q_fp8"].view(torch.float8_e4m3fn).to(dev), c["weights"].to(dev), c["k_cache"].to(dev),
                                c["seq_lens"].to(dev), c["page_table"].to(dev), c["q_len"]).cpu()
        fin = torch.isfinite(ref)
        assert _calc_diff(lg.masked_fill(~fin, 0), ref.masked_fill(~fin, 0)) < 1e-3, name
        assert torch.isfinite(lg[fin]).all()


def _topk(dev, logits, lens, Q, topk):
    from lvllm_b200 import ops
    return ops.indexer_topk(logits.to(dev), torch.tensor(lens, dtype=torch.int32).to(dev), topk, Q).cpu()


@pytest.mark.parametrize("rows_per_req,topk", [(1, 2048), (2, 2048), (3, 100), (1, 1)])
def test_topk_exact_vs_oracle(dev, rows_per_req, topk):
    gen = torch.Generator().manual_seed(topk + rows_per_req)
    W = 9000
    lens = [0, 1, topk, topk + 1, 5000, W, 3 * topk + 17, 2]
    x = torch.randn(len(lens) * rows_per_req, W, generator=gen)
    got = _topk(dev, x, lens, rows_per_req, topk)
    assert torch.equal(got, IX.topk_rows(x, torch.tensor(lens), rows_per_req, topk))


def test_topk_on_a_column_slice(dev):
    """logits as the first W columns of a wider buffer: rows are read through the buffer's row stride and never past
    column W, even where seq_lens runs beyond it."""
    from lvllm_b200 import ops
    gen = torch.Generator().manual_seed(8)
    W, pad, topk = 6000, 37, 512
    buf = torch.full((6, W + pad), math.inf)                          # the padding would win every selection
    buf[:, :W] = torch.randn(6, W, generator=gen)
    lens = torch.tensor([W, 4000, W + 30], dtype=torch.int32)         # the last runs past the slice: clamped to W
    got = ops.indexer_topk(buf.to(dev)[:, :W], lens.to(dev), topk, 2).cpu()
    assert torch.equal(got, IX.topk_rows(buf[:, :W], lens, 2, topk))
    assert int(got.max()) < W


def test_topk_forced_ties(dev):
    gen = torch.Generator().manual_seed(5)
    W = 20000
    x = (torch.randn(12, W, generator=gen) * 2).round() / 2           # few distinct values: ties at every threshold
    x[3] = 1.0
    x[4, ::3] = -math.inf
    x[6, ::2] = -0.0                                                  # -0 ties with +0
    lens = [W, W, 3000, W, W, 2049, W, 12345, W, 2100, 4097, W]
    for topk in (2048, 700):
        got = _topk(dev, x, lens, 1, topk)
        assert torch.equal(got, IX.topk_rows(x, torch.tensor(lens), 1, topk)), topk


def _reference_compare(logits, got, want, ends, topk, tol=1e-5):
    """The reference's compare_top_k_results (tests/kernels/test_top_k_per_row.py:132-183): equal sets, or the values at
    the indices only one side picked agree within tol."""
    for r in range(got.shape[0]):
        n = min(topk, int(ends[r]))
        a, b = got[r][:n].tolist(), want[r][:n].tolist()
        if set(a) == set(b):
            continue
        oa = sorted(logits[r, i].item() for i in set(a) - set(b))
        ob = sorted(logits[r, i].item() for i in set(b) - set(a))
        if len(oa) != len(ob) or not torch.allclose(torch.tensor(oa), torch.tensor(ob), rtol=tol, atol=tol):
            return False
    return True


def test_topk_on_kernel_logits_reference_criterion(dev):
    from lvllm_b200 import ops
    H, Q, page, npg, topk = 64, 2, 64, 80, 2048
    lens = [5000, 2048, 4097, 700]
    gen = torch.Generator().manual_seed(11)
    q8, w, cache, sl, pt = _cache(gen, len(lens), npg, page, H, Q, lens)
    lg = ops.indexer_logits(q8.to(dev), w.to(dev), cache.to(dev), sl.to(dev), pt.to(dev), Q)
    got = ops.indexer_topk(lg, sl.to(dev), topk, Q).cpu()
    lgc = lg.cpu()
    ends = [max(0, lens[r // Q] - Q + r % Q + 1) for r in range(len(lens) * Q)]
    want = torch.full((len(ends), topk), -1, dtype=torch.int32)
    for r, e in enumerate(ends):
        want[r, :min(topk, e)] = torch.topk(lgc[r, :e], min(topk, e)).indices.int()
    assert _reference_compare(lgc, got, want, ends, topk)
    assert torch.equal(got, IX.topk_rows(lgc, sl, Q, topk))          # and exactly the oracle's rule on these logits


@pytest.mark.parametrize("rows", [1, 140], ids=["cluster", "one_cta"])
def test_topk_160k_rows(dev, rows):
    """160K-token rows: batch 1 runs as one cluster of CTAs per row, 140 rows as one CTA per row."""
    W = 160 * 1024
    gen = torch.Generator(device=dev).manual_seed(rows)
    x = torch.randn(rows, W, device=dev, generator=gen)
    x[:, ::7] = x[:, ::7].round()                                       # ties among the large values too
    lens = torch.full((rows,), W, dtype=torch.int32)
    lens[rows // 2] = W - 12345
    got = _topk(dev, x, lens.tolist(), 1, 2048)
    again = _topk(dev, x, lens.tolist(), 1, 2048)
    assert torch.equal(got, again)
    assert torch.equal(got, IX.topk_rows(x.cpu(), lens, 1, 2048))


def test_chain_into_sparse_decode_eager_and_graph(dev):
    """q/k write -> indexer_decode -> mla_decode_sparse.  Every S_b <= topk: the indices are 0 .. S_b - 1 then -1 (the
    oracle's), and the sparse decode is bit-identical to the dense decode on the same latent cache; a CUDA-graph replay
    gives the same bits."""
    from lvllm_b200 import _lib as L
    from lvllm_b200 import ops
    B, H, page, npg, topk, hq = 3, 64, 64, 32, 2048, 16
    gen = torch.Generator().manual_seed(21)
    lens = torch.tensor([5, 700, 2048], dtype=torch.int32)
    nb = B * npg
    pt = torch.randperm(nb, generator=gen).reshape(B, npg).int().to(dev)
    icache = torch.zeros(nb, page, 132, dtype=torch.uint8, device=dev)
    lat = torch.randn(nb, page, 576, generator=gen).bfloat16().to(dev)
    cs = torch.randn(4096, 64, generator=gen).bfloat16().to(dev)
    # fill the indexer cache for every key, then the decode step writes the new tokens' rows again
    for b in range(B):
        S = int(lens[b])
        pos = torch.arange(S)
        slots = (pt.cpu()[b, pos // page].long() * page + pos % page).to(dev)
        kb = torch.randn(S, 128, generator=gen).bfloat16().to(dev)
        ops.indexer_qk_rope_quant_cache_write(torch.zeros(S, H, 128, dtype=torch.bfloat16, device=dev),
                                              torch.zeros(S, H, dtype=torch.bfloat16, device=dev), kb, pos.to(dev), cs,
                                              slots, icache, 128 ** -0.5, H ** -0.5)
    q = torch.randn(B, H, 128, generator=gen).bfloat16().to(dev)
    wts = torch.randn(B, H, generator=gen).bfloat16().to(dev)
    kn = torch.randn(B, 128, generator=gen).bfloat16().to(dev)
    pos = (lens - 1).long().to(dev)
    slots = (pt.cpu()[torch.arange(B), (lens - 1) // page].long() * page + (lens - 1) % page).to(dev)
    qn = torch.randn(B, hq, 512, generator=gen).bfloat16().to(dev)
    qp = torch.randn(B, hq, 64, generator=gen).bfloat16().to(dev)
    sl = lens.to(dev)
    rid = torch.arange(B, dtype=torch.int32, device=dev)
    scale = 1.0 / math.sqrt(576)

    def step():
        q8, w = ops.indexer_qk_rope_quant_cache_write(q, wts, kn, pos, cs, slots, icache, 128 ** -0.5, H ** -0.5)
        idx = ops.indexer_decode(q8, w, icache, sl, pt, 1, topk)
        out, lse = ops.mla_decode_sparse(qn, qp, lat, idx, rid, pt, scale, num_kv_splits=2)
        return idx, out, lse

    idx, out, lse = step()
    torch.cuda.synchronize()
    want = torch.full((B, topk), -1, dtype=torch.int32)
    for b in range(B):
        want[b, :lens[b]] = torch.arange(int(lens[b]), dtype=torch.int32)
    assert torch.equal(idx.cpu(), want)
    lib = L.lib()
    ws = torch.empty(lib.b200_mla_decode_workspace_bytes(B, hq, 2), dtype=torch.uint8, device=dev)
    d_out = torch.empty(B, hq, 512, dtype=torch.bfloat16, device=dev)
    d_lse = torch.empty(B, hq, dtype=torch.float32, device=dev)
    L.check(lib.b200_mla_decode_ex(torch.cuda.current_stream().cuda_stream, qn.data_ptr(), qp.data_ptr(), 0, lat.data_ptr(),
                                   0, 1.0, 1.0, sl.data_ptr(), pt.data_ptr(), B, hq, page, npg, scale, 2, ws.data_ptr(),
                                   d_out.data_ptr(), d_lse.data_ptr()), "b200_mla_decode_ex")
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), d_out.view(torch.int16)) and torch.equal(lse, d_lse)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_idx, g_out, g_lse = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_idx, idx) and torch.equal(g_out.view(torch.int16), out.view(torch.int16))
    assert torch.equal(g_lse, lse)


def test_chain_indices_match_oracle_past_topk(dev):
    """Contexts longer than topk: the kernel chain's indices against the oracle's top-k of the oracle's logits, by the
    reference's comparison with its tolerance widened to the kernel's accumulation error."""
    from lvllm_b200 import ops
    H, Q, page, npg, topk = 64, 2, 64, 64, 2048
    lens = [4096, 2500, 3001]
    gen = torch.Generator().manual_seed(33)
    q8, w, cache, sl, pt = _cache(gen, len(lens), npg, page, H, Q, lens)
    idx = ops.indexer_decode(q8.to(dev), w.to(dev), cache.to(dev), sl.to(dev), pt.to(dev), Q, topk).cpu()
    ref = IX.paged_logits(q8, w, cache, sl, pt, Q, npg * page)
    bound = _abs_bound(q8, w, cache, sl, pt, Q, npg * page)
    want = IX.topk_rows(ref, sl, Q, topk)
    ends = [max(0, lens[r // Q] - Q + r % Q + 1) for r in range(len(lens) * Q)]
    tol = 2 * ACC_TOL * float(bound[torch.isfinite(bound)].max())   # two logits within the kernel's error may swap
    assert _reference_compare(ref.float(), idx, want, ends, topk, tol=tol)
    for r in range(idx.shape[0]):                                     # and swaps are rare
        assert len(set(idx[r].tolist()) & set(want[r].tolist())) >= 0.99 * topk


def test_refusals(dev):
    from lvllm_b200 import _lib as L
    lib = L.lib()
    st = torch.cuda.current_stream().cuda_stream
    B, H, page, npg = 2, 64, 64, 4
    q8 = torch.zeros(B * 16 + 1, 64, 128 + 16, dtype=torch.uint8, device=dev)
    w = torch.zeros(B * 17, 64, dtype=torch.float32, device=dev)
    cache = torch.zeros(16, 128, 132, dtype=torch.uint8, device=dev)
    sl = torch.ones(B, dtype=torch.int32, device=dev)
    pt = torch.zeros(B, npg, dtype=torch.int32, device=dev)
    lg = torch.zeros(B * 17, npg * 128 + 4, dtype=torch.float32, device=dev)
    out = torch.zeros(B * 17, 4096, dtype=torch.int32, device=dev)
    n0 = lib.b200moe_launch_count()

    def logits(q_ptr=q8.data_ptr(), heads=H, q_len=1, pg=page, stride=npg * page, nb=16):
        return lib.b200_indexer_logits(st, q_ptr, w.data_ptr(), cache.data_ptr(), nb, pg, sl.data_ptr(), pt.data_ptr(), B,
                                       q_len, heads, npg, lg.data_ptr(), stride)

    assert logits() == 0
    n1 = lib.b200moe_launch_count()
    assert logits(heads=48) == INVALID
    assert logits(q_len=17) == INVALID and logits(pg=128) == INVALID
    assert logits(stride=npg * page - 1) == INVALID and logits(q_ptr=q8.data_ptr() + 8) == INVALID
    tk = lambda k, p=lg.data_ptr(), width=lg.shape[1]: lib.b200_indexer_topk(st, p, lg.shape[1], width, sl.data_ptr(), B, 1,
                                                                           k, out.data_ptr())
    assert tk(4096) == INVALID and tk(0) == INVALID and tk(16, lg.data_ptr() + 2) == INVALID
    assert tk(16, width=lg.shape[1] + 1) == INVALID and tk(16, width=0) == INVALID
    qb = torch.zeros(3, H, 128 + 8, dtype=torch.bfloat16, device=dev)
    kb = torch.zeros(3, 128 + 8, dtype=torch.bfloat16, device=dev)
    pos = torch.zeros(3, dtype=torch.int64, device=dev)
    cs = torch.zeros(8, 64, dtype=torch.bfloat16, device=dev)
    rc = lib.b200_indexer_qk_rope_quant_cache_write(st, qb.data_ptr() + 8, qb.data_ptr(), H, kb.data_ptr(), pos.data_ptr(),
                                                    cs.data_ptr(), 8, 1, pos.data_ptr(), cache.data_ptr(), 128, 1, 1.0, 1.0,
                                                    q8.data_ptr(), w.data_ptr(), 3, H)
    assert rc == INVALID
    torch.cuda.synchronize()
    assert lib.b200moe_launch_count() == n1 == n0 + 1                 # the refusals launched nothing
