"""GPU (-m gpu): DeepSeek-V4 key selection for decode: the C4A indexer's q side (ops.dsv4_indexer_q_quant), its logits and
top-k over the compressed indexer cache with one row per token (ops.dsv4_indexer_decode), and the global key lists
(ops.dsv4_swa_indices, dsv4_c128a_indices, dsv4_global_topk_indices, dsv4_compressed_slot_mapping).

Against the oracle (tests/dsv4_indexer_oracle.py): the q side and the lists bit for bit; the logits within the e4m3
wgmma's accumulation error (test_gpu_indexer.py's criterion); the top-k exactly the oracle's top-k of the kernel's own
logits, the same bits with and without the short-context hint, and per-token candidate counts for multi-token rows of one
request, which the V3.2 per-request mask gets wrong.  End to end through library calls only, for a C4A and a C128A layer
over decode steps that cross compression boundaries: q-norm + RoPE + SWA insert, compressor fed by the new slot mapping,
q side, indexer, lists and sparse decode, against the oracle composition; CUDA-graph replay bit-identical to eager calls;
a token's lists and output the same bits alone and in a batch of 32."""
import math

import pytest
import torch

import dsv4_compress_oracle as C
import dsv4_indexer_oracle as O
import dsv4_sparse_oracle as V4
import indexer_oracle as IX
from lvllm_b200 import ops

pytestmark = pytest.mark.gpu

SENT = 12345.0
ACC_TOL = 2 ** -10   # the e4m3 wgmma's accumulation error against the summed magnitudes (see test_gpu_indexer.py)
EPS, MAX_POS = 1e-6, 4096


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_sin(n=MAX_POS):
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(n, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


@pytest.mark.parametrize("H", [32, 64])
def test_q_quant_bit_exact(dev, H):
    T = 41
    gen = torch.Generator().manual_seed(H)
    q = (torch.randn(T, H, 128, generator=gen) * torch.logspace(-3, 1, H)[None, :, None]).bfloat16()
    q[0, 0] = 0.0                                                          # under the 1e-4 clamp
    q[1, 1, 7] = 3.5                                                       # amax 448 * 2^-7 on some heads
    fused = torch.randn(T, H + 40, generator=gen).bfloat16()
    cs = _cos_sin(300)
    pos = torch.randint(-3, 303, (T,), generator=gen)                     # clamped to the table
    wd = fused.to(dev)[:, 24:24 + H]                                       # strided rows
    q8, wo = ops.dsv4_indexer_q_quant(q.to(dev), wd, pos.to(dev), cs.to(dev), 128 ** -0.5, H ** -0.5)
    rq8, rwo = O.q_quant(q, fused[:, 24:24 + H], pos, cs, 128 ** -0.5, H ** -0.5)
    assert torch.equal(q8.cpu().view(torch.uint8), rq8.view(torch.uint8))
    assert torch.equal(wo.cpu().view(torch.int32), rwo.view(torch.int32))


def _list_inputs(gen, T, R, maxb, max_pos):
    pos = torch.randint(0, max_pos, (T,), generator=gen)
    req = torch.randint(0, R, (T,), generator=gen).int()
    sm = torch.arange(T)
    sm[10 + torch.randperm(T - 10, generator=gen)[:3]] = -1                # invalid tokens, past the edge cases
    bt = torch.randperm(R * maxb + 5, generator=gen)[:R * maxb].reshape(R, maxb).int()
    return pos, req, sm, bt


def test_lists_bit_exact(dev):
    gen = torch.Generator().manual_seed(3)
    T, R = 64, 5
    # SWA: window 128 on blocks of 64; positions cross blocks, p < W, and windows reaching a block column at the width
    pos, req, sm, bt = _list_inputs(gen, T, R, 8, 8 * 64)
    pos[:6] = torch.tensor([0, 5, 127, 128, 63, 64])
    pos[6:9] = torch.tensor([8 * 64 - 1, 8 * 64, 8 * 64 + 70])              # last column, at the width, past it
    d = [x.to(dev) for x in (pos, sm, req, bt)]
    si, sl = ops.dsv4_swa_indices(d[0], d[1], d[2], d[3], 64, 128)
    ri, rl = O.swa(pos, sm, req, bt, 64, 128)
    assert torch.equal(si.cpu(), ri) and torch.equal(sl.cpu(), rl)
    assert (ri[7] == -1).sum() > 0 and (ri[8] == -1).sum() > (ri[7] == -1).sum()
    # C128A: ratio 128 on compressed blocks of 2, width 6 below some counts; ratio 4 on blocks of 64
    for ratio, cbs, maxb, width in ((128, 2, 4, 6), (128, 2, 2, 8), (4, 64, 3, 200)):
        pos, req, sm, bt = _list_inputs(gen, T, R, maxb, 1200)
        pos[:5] = torch.tensor([126, 127, 128, 255, 767 + 128 * 3])
        d = [x.to(dev) for x in (pos, sm, req, bt)]
        ci, cl = ops.dsv4_c128a_indices(d[0], d[1], d[2], d[3], cbs, ratio, width)
        ri, rl = O.c128a(pos, sm, req, bt, cbs, ratio, width)
        assert torch.equal(ci.cpu(), ri) and torch.equal(cl.cpu(), rl), (ratio, width)
        # compressor slot mapping: just below, at and after a boundary
        pos[5:8] = torch.tensor([ratio - 2, ratio - 1, ratio])
        d[0] = pos.to(dev)
        ks = ops.dsv4_compressed_slot_mapping(d[0], d[1], d[2], d[3], cbs, ratio)
        assert torch.equal(ks.cpu(), O.slot_mapping(pos, sm, req, bt, cbs, ratio)), ratio
        assert int((ks >= 0).sum()) >= 1
    # top-k -> global, local lists with -1 padding and entries at and past the table's width
    pos, req, sm, bt = _list_inputs(gen, T, R, 4, 1)
    loc = torch.full((T, 512), -1, dtype=torch.int32)
    for t in range(T):
        n = int(torch.randint(0, 4 * 64 + 41, (1,), generator=gen))
        loc[t, :n] = torch.randperm(4 * 64 + 40, generator=gen)[:n].sort().values.int()
    gi, gl = ops.dsv4_global_topk_indices(loc.to(dev), sm.to(dev), req.to(dev), bt.to(dev), 64)
    ri, rl = O.global_topk(loc, sm, req, bt, 64)
    assert torch.equal(gi.cpu(), ri) and torch.equal(gl.cpu(), rl)


def _indexer_case(gen, positions, req, R, maxb, H=64, page=64):
    """An indexer cache written by the oracle over every slot of R requests' pages, and the q side of the tokens."""
    nb = R * maxb + 3
    bt = torch.randperm(nb, generator=gen)[:R * maxb].reshape(R, maxb).int()
    cache = torch.zeros(nb, page, 132, dtype=torch.uint8)
    slots = (bt.long()[:, :, None] * page + torch.arange(page)).reshape(-1)
    IX.k_quant_cache(torch.randn(slots.numel(), 128, generator=gen).bfloat16(), slots, cache, True)
    T = positions.numel()
    q8, w = O.q_quant(torch.randn(T, H, 128, generator=gen).bfloat16(), torch.randn(T, H, generator=gen).bfloat16(),
                      positions, _cos_sin(8), 128 ** -0.5, H ** -0.5)
    return q8, w, cache, bt


@pytest.mark.parametrize("H", [32, 64])
def test_topk_logits_and_hint(dev, H):
    gen = torch.Generator().manual_seed(40 + H)
    topk, ratio, page, maxb, R = 512, 4, 64, 40, 4
    pos = torch.tensor([0, 3, 4, 2047, 2048, 2051, 4095, 8191, 9000, 10239, 10300, -1])   # counts past the width too
    req = torch.tensor([0, 1, 2, 3, 0, 1, 2, 3, 0, 1, 2, 3], dtype=torch.int32)
    q8, w, cache, bt = _indexer_case(gen, pos, req, R, maxb, H, page)
    width = maxb * page
    lg = torch.full((pos.numel(), width + 16), SENT, device=dev)
    d = dict(q_fp8=q8.to(dev), weights=w.to(dev), k_cache=cache.to(dev), positions=pos.to(dev), token_to_req=req.to(dev),
             block_table=bt.to(dev), compress_ratio=ratio, topk=topk)
    idx = ops.dsv4_indexer_decode(**d, logits=lg).cpu()
    got = lg.cpu().double()
    n = O.candidates(pos, ratio).clamp(max=width)
    ref = IX.paged_logits(q8, w, cache, n, bt[req.long()], 1, width)
    bound = IX.paged_logits(q8.float().abs().to(torch.float8_e4m3fn), w.abs(), _abs_cache(cache), n, bt[req.long()], 1,
                            width)
    for r in range(pos.numel()):
        e, limit = int(n[r]), -(-int(n[r]) // page) * page
        assert ((got[r, :e] - ref[r, :e]).abs() <= ACC_TOL * bound[r, :e]).all(), r
        assert (got[r, e:limit] == -math.inf).all() and (got[r, limit:] == SENT).all(), r
    assert torch.equal(idx, O.topk(lg.cpu()[:, :width], pos, ratio, topk))
    assert torch.equal(idx, ops.dsv4_indexer_decode(**d, max_seq_len=10301).cpu())        # hint too long to skip
    # short contexts: the hint skips the logits and gives the same bits
    short = torch.tensor([0, 3, 4, 100, 2046, 2047, 7, -1])
    sd = dict(d, positions=short.to(dev), token_to_req=req[:8].to(dev), q_fp8=q8[:8].to(dev), weights=w[:8].to(dev))
    lg2 = torch.full((8, width), SENT, device=dev)
    a = ops.dsv4_indexer_decode(**sd)
    b = ops.dsv4_indexer_decode(**sd, max_seq_len=2048, logits=lg2)
    assert torch.equal(a, b) and torch.equal(a.cpu(), O.short_context(short, ratio, topk))
    assert bool((lg2 == SENT).all())                                                     # no logit computed


def _abs_cache(cache):
    nb, page, _ = cache.shape
    flat = cache.reshape(nb, page * 132).clone()
    flat[:, :page * 128] &= 0x7F
    return flat.reshape(nb, page, 132)


@pytest.mark.parametrize("topk", [64, 2048])
def test_topk_mtp_rows(dev, topk):
    """2-4 tokens of one request: each gets its own (p + 1) // 4 candidates.  The V3.2 path's per-request mask
    (S - Q + i + 1 with S the last token's count) lists other candidates: with every candidate selected (topk 2048) its
    lists differ."""
    gen = torch.Generator().manual_seed(topk)
    for p0, Q in ((402, 4), (399, 2), (1203, 3)):
        pos = torch.arange(p0, p0 + Q)
        req = torch.zeros(Q, dtype=torch.int32)
        q8, w, cache, bt = _indexer_case(gen, pos, req, 1, 8)
        d = [x.to(dev) for x in (q8, w, cache)]
        lg = torch.empty(Q, 8 * 64, device=dev)
        idx = ops.dsv4_indexer_decode(d[0], d[1], d[2], pos.to(dev), req.to(dev), bt.to(dev), 4, topk, logits=lg).cpu()
        assert torch.equal(idx, O.topk(lg.cpu(), pos, 4, topk)), (p0, Q)
        counts = O.candidates(pos, 4)
        if topk == 2048:
            assert torch.equal((idx >= 0).sum(1).int(), counts)
            v32 = ops.indexer_decode(d[0], d[1], d[2], counts[-1:].to(dev), bt.to(dev), Q, topk).cpu()
            assert not torch.equal(v32, idx), (p0, Q)


class Layer:
    """One V4 attention layer's caches for decode: the SWA cache (block size 64, window 128), the compressed attention
    cache and, for C4A, the indexer cache (64 compressed rows per block at ratio 4, 2 at ratio 128), the compressor
    states, and per-request block tables over shuffled pools."""

    def __init__(self, gen, dev, ratio, R, max_pos, Hq=64, Hi=64, topk=32):
        self.dev, self.ratio, self.R, self.Hq, self.Hi, self.topk = dev, ratio, R, Hq, Hi, topk
        self.cbs = 64 if ratio == 4 else 2
        self.sbs = 16

        def table(per, pad=3):
            return torch.randperm(R * per + pad, generator=gen)[:R * per].reshape(R, per).int(), R * per + pad

        self.swa_bt, swa_nb = table(-(-max_pos // 64))
        self.c_bt, c_nb = table(-(-(max_pos // ratio) // self.cbs) + 1)       # one column past the last row used
        self.st_bt, st_nb = table(-(-max_pos // self.sbs))
        self.swa_btd, self.c_btd, self.st_btd = (b.to(dev) for b in (self.swa_bt, self.c_bt, self.st_bt))
        self.swa = torch.zeros(swa_nb, 64, 584, dtype=torch.uint8, device=dev)
        self.comp = torch.zeros(c_nb, self.cbs, 584, dtype=torch.uint8, device=dev)
        coff = C.coff(ratio)
        self.state = torch.zeros(st_nb, self.sbs, 2 * coff * 512, device=dev)
        self.ape = torch.randn(ratio, coff * 512, generator=gen).to(dev)
        self.norm = (1 + 0.25 * torch.randn(512, generator=gen)).bfloat16().to(dev)
        if ratio == 4:
            self.icache = torch.zeros(c_nb, self.cbs, 132, dtype=torch.uint8, device=dev)
            self.istate = torch.zeros(st_nb, self.sbs, 2 * 2 * 128, device=dev)
            self.iape = torch.randn(4, 2 * 128, generator=gen).to(dev)
            self.inorm = (1 + 0.25 * torch.randn(128, generator=gen)).bfloat16().to(dev)
        self.cs = _cos_sin().to(dev)
        self.sink = torch.randn(Hq, generator=gen).to(dev)

    def inputs(self, gen, items):
        """items: (request, position) per token, or None for a padded token.  Random activations of the step (device)."""
        T = len(items)
        pos = torch.tensor([it[1] if it else 0 for it in items])
        req = torch.tensor([it[0] if it else 0 for it in items], dtype=torch.int32)
        sm = torch.tensor([int(self.swa_bt[r, p // 64]) * 64 + p % 64 if it else -1 for it in items
                           for r, p in [it or (0, 0)]])
        coff = C.coff(self.ratio)
        x = dict(positions=pos, token_to_req=req, slot_mapping=sm,
                 q=torch.randn(T, self.Hq, 512, generator=gen).bfloat16(), kv=torch.randn(T, 512, generator=gen).bfloat16(),
                 kv_score=torch.randn(T, 2 * coff * 512, generator=gen),
                 state_slots=torch.tensor([int(self.st_bt[r, p // self.sbs]) * self.sbs + p % self.sbs if it else -1
                                           for it in items for r, p in [it or (0, 0)]]))
        if self.ratio == 4:
            x.update(ikv_score=torch.randn(T, 4 * 128, generator=gen), iq=torch.randn(T, self.Hi, 128, generator=gen).bfloat16(),
                     iw=torch.randn(T, self.Hi + 8, generator=gen).bfloat16())
        return {k: v.to(self.dev) for k, v in x.items()}

    def step(self, x, logits=None):
        """One layer step through library calls only.  Returns every output the step makes."""
        pos, req, sm = x["positions"], x["token_to_req"], x["slot_mapping"]
        q = ops.dsv4_qnorm_rope_kv_insert(x["q"], x["kv"], pos, self.cs, sm, self.swa, self.Hq, EPS)
        ksm = ops.dsv4_compressed_slot_mapping(pos, sm, req, self.c_btd, self.cbs, self.ratio)
        ops.dsv4_compress(x["kv_score"], self.ape, pos, self.state, x["state_slots"], req, self.st_btd, self.norm, EPS,
                          self.cs, self.comp, ksm, self.ratio)
        out = dict(q=q, kv_slots=ksm)
        if self.ratio == 4:
            ops.dsv4_compress(x["ikv_score"], self.iape, pos, self.istate, x["state_slots"], req, self.st_btd, self.inorm,
                              EPS, self.cs, self.icache, ksm, 4)
            q8, w = ops.dsv4_indexer_q_quant(x["iq"], x["iw"][:, 4:4 + self.Hi], pos, self.cs, 128 ** -0.5,
                                             self.Hi ** -0.5)
            local = ops.dsv4_indexer_decode(q8, w, self.icache, pos, req, self.c_btd, 4, self.topk, logits=logits)
            ei, el = ops.dsv4_global_topk_indices(local, sm, req, self.c_btd, self.cbs)
            out.update(q8=q8, w=w, local=local)
        else:
            ei, el = ops.dsv4_c128a_indices(pos, sm, req, self.c_btd, self.cbs, 128, 8)
        si, sl = ops.dsv4_swa_indices(pos, sm, req, self.swa_btd, 64, 128)
        o = ops.dsv4_sparse_decode(q, self.swa, si, sl, 512 ** -0.5, self.sink, self.comp, ei, el, num_kv_splits=2)
        out.update(si=si, sl=sl, ei=ei, el=el, out=o)
        return out

    def check(self, x, got, logits):
        """The oracle composition of the step over the caches the kernels wrote."""
        pos, req, sm = (x[k].cpu() for k in ("positions", "token_to_req", "slot_mapping"))
        assert torch.equal(got["kv_slots"].cpu(), O.slot_mapping(pos, sm, req, self.c_bt, self.cbs, self.ratio))
        si, sl = O.swa(pos, sm, req, self.swa_bt, 64, 128)
        assert torch.equal(got["si"].cpu(), si) and torch.equal(got["sl"].cpu(), sl)
        if self.ratio == 4:
            q8, w = O.q_quant(x["iq"].cpu(), x["iw"].cpu()[:, 4:4 + self.Hi], pos, self.cs.cpu(), 128 ** -0.5,
                              self.Hi ** -0.5)
            assert torch.equal(got["q8"].cpu().view(torch.uint8), q8.view(torch.uint8))
            assert torch.equal(got["w"].cpu(), w)
            width = self.c_bt.shape[1] * self.cbs
            local = O.topk(logits.cpu()[:, :width], pos, 4, self.topk)
            assert torch.equal(got["local"].cpu(), local)
            ei, el = O.global_topk(local, sm, req, self.c_bt, self.cbs)
        else:
            ei, el = O.c128a(pos, sm, req, self.c_bt, self.cbs, 128, 8)
        assert torch.equal(got["ei"].cpu(), ei) and torch.equal(got["el"].cpu(), el)
        want = V4.decode(got["q"].cpu(), self.swa.cpu(), si, sl, 512 ** -0.5, self.sink.cpu(), self.comp.cpu(), ei, el)
        torch.testing.assert_close(got["out"].cpu().double(), want, atol=2e-2, rtol=2e-2)


def _logits(L, T):
    return torch.full((T, L.c_bt.shape[1] * L.cbs), SENT, device=L.dev)


@pytest.mark.parametrize("ratio,starts", [(4, [130, 61, 9, 200]), (128, [250, 126, 380, 60])], ids=["c4a", "c128a"])
def test_end_to_end_steps_and_graph(dev, ratio, starts):
    gen = torch.Generator().manual_seed(ratio)
    R, steps = len(starts), 6
    L = Layer(gen, dev, ratio, R, max(starts) + steps + 8)
    # the prompts in one call per request
    for r, s in enumerate(starts):
        x = L.inputs(gen, [(r, p) for p in range(s)])
        L.step(x, _logits(L, s))
    boundaries = 0
    for k in range(steps):
        items = [(r, s + k) for r, s in enumerate(starts)] + [None]
        boundaries += sum((s + k + 1) % ratio == 0 for s in starts)
        x = L.inputs(gen, items)
        lg = _logits(L, len(items))
        got = L.step(x, lg)
        torch.cuda.synchronize()
        L.check(x, got, lg)
        assert int(got["el"][-1]) == 0 and int(got["sl"][-1]) == 0          # the padded token
    assert boundaries >= 2
    # the last step again as a CUDA-graph replay: the same bits (the step rewrites the same cache bytes)
    lg = _logits(L, len(items))
    eager = L.step(x, lg)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        L.step(x, lg)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g = L.step(x, lg)
    graph.replay()
    torch.cuda.synchronize()
    for k, v in eager.items():
        assert torch.equal(g[k].view(torch.uint8) if v.dtype == torch.float8_e4m3fn else g[k],
                           v.view(torch.uint8) if v.dtype == torch.float8_e4m3fn else v), k


def test_batch_of_32_invariance(dev):
    gen = torch.Generator().manual_seed(32)
    R = 32
    starts = [int(s) for s in torch.randint(40, 400, (R,), generator=gen)]
    L = Layer(gen, dev, 4, R, max(starts) + 8)
    for r, s in enumerate(starts):
        L.step(L.inputs(gen, [(r, p) for p in range(s)]), _logits(L, s))
    x = L.inputs(gen, [(r, s) for r, s in enumerate(starts)])
    batch = L.step(x, _logits(L, R))
    for t in (0, 17):
        one = L.step({k: v[t:t + 1] for k, v in x.items()}, _logits(L, 1))
        for k in ("local", "si", "sl", "ei", "el", "out"):
            assert torch.equal(one[k], batch[k][t:t + 1]), (t, k)
