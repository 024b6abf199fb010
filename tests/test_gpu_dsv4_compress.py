"""GPU (-m gpu): the DeepSeek-V4 KV compressor (ops.dsv4_compress) at its three shapes: (D 512, ratio 4) and (D 512, ratio
128) into the 584-byte attention cache, (D 128, ratio 4) into the indexer's 132-byte cache.

Against the float64 oracle (tests/dsv4_compress_oracle.py): the state bit for bit; the compressed rows by
dsv4_compress_oracle.check_cache (scales equal and e4m3 codes within one step except where an fp32 rounding decides the
scale, rope dims within one bf16 ulp), on caches and states filled with canary bytes, so that nothing is written for
non-boundary tokens, state slot -1, cache slot -1 or a cache slot past the end.  Bit relations: a 300-token prompt in one
call against 300 one-token calls, a batch against its requests one by one, CUDA-graph replay of a decode step against eager
calls.  Chains: the compressed cache read by ops.dsv4_sparse_decode and by ops.indexer_logits."""
import pytest
import torch

import dsv4_compress_oracle as C
import dsv4_sparse_oracle as V4
import indexer_oracle as IX
from lvllm_b200 import ops

pytestmark = pytest.mark.gpu

SHAPES = [(512, 4), (512, 128), (128, 4)]
IDS = ["c4a_512", "c128a_512", "c4a_indexer_128"]
EPS, MAX_POS = 1e-6, 4096


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_sin():
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(MAX_POS, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


class Layer:
    """One compressor's weights and caches: state blocks of sbs rows spread over a shuffled pool, one block table row per
    request; the output cache of kv_nb blocks of kv_bs rows; canary bytes everywhere."""

    def __init__(self, gen, D, ratio, n_req=3, max_pos=512, sbs=16, kv_bs=16, kv_nb=None):
        self.D, self.ratio, self.half = D, ratio, C.coff(ratio) * D
        self.sbs, self.kv_bs = sbs, kv_bs
        per = -(-max_pos // sbs)
        self.block_table = torch.randperm(n_req * per + 3, generator=gen)[:n_req * per].reshape(n_req, per).int()
        self.state = torch.randn(n_req * per + 3, sbs, 2 * self.half, generator=gen)
        self.kv_nb = kv_nb or -(-n_req * (max_pos // ratio) // kv_bs)
        self.row = 584 if D == 512 else 132
        self.cache = torch.randint(0, 256, (self.kv_nb, kv_bs, self.row), generator=gen, dtype=torch.uint8)
        self.ape = torch.randn(ratio, self.half, generator=gen)
        self.w = (1 + 0.25 * torch.randn(D, generator=gen)).bfloat16()
        self.cs = _cos_sin()
        # compressed row j of request r goes to slot kv_base[r] + j
        self.kv_base = [r * (max_pos // ratio) for r in range(n_req)]

    def tokens(self, gen, items):
        """items: (request, position) per token, or None for a padded token.  Returns the call's inputs (CPU)."""
        T = len(items)
        buf = torch.randn(T, 2 * self.half + 8, generator=gen)                  # rows with a stride
        kv_score = buf[:, :2 * self.half]
        pos = torch.tensor([p if it else 0 for it in items for p in [it[1] if it else 0]], dtype=torch.int64)
        req = torch.tensor([it[0] if it else 0 for it in items], dtype=torch.int32)
        slot = torch.tensor([int(self.block_table[r, p // self.sbs]) * self.sbs + p % self.sbs if it else -1
                             for it in items for r, p in [it or (0, 0)]], dtype=torch.int64)
        kslot = torch.tensor([self.kv_base[r] + p // self.ratio if it else -1 for it in items for r, p in [it or (0, 0)]],
                             dtype=torch.int64)
        return dict(kv_score=kv_score, positions=pos, slot_mapping=slot, token_to_req=req, kv_slot_mapping=kslot)

    def run(self, dev, state, cache, t):
        ops.dsv4_compress(t["kv_score"].to(dev), self.ape.to(dev), t["positions"].to(dev), state, t["slot_mapping"].to(dev),
                          t["token_to_req"].to(dev), self.block_table.to(dev), self.w.to(dev), EPS, self.cs.to(dev), cache,
                          t["kv_slot_mapping"].to(dev), self.ratio)

    def oracle(self, state, cache, t):
        C.state_write(t["kv_score"], self.ape, t["positions"], t["slot_mapping"], state)
        return C.compress(state, self.block_table, t["token_to_req"], t["positions"], t["slot_mapping"], self.w, EPS,
                          self.cs, self.ratio, t["kv_slot_mapping"], cache)


@pytest.mark.parametrize("D,ratio", SHAPES, ids=IDS)
def test_matches_oracle_and_writes_nothing_else(dev, D, ratio):
    gen = torch.Generator().manual_seed(D + ratio)
    L = Layer(gen, D, ratio, max_pos=512)
    R = ratio
    # request 0: a prompt chunk from position 0 (windows reaching below 0 at ratio 4); request 1: decode tokens whose
    # windows read rows of earlier calls; request 2: a non-boundary token; padded tokens
    items = [(0, p) for p in range(0, 3 * R + 3)] + [(1, 3 * R - 1), None, (1, 3 * R), (2, R + 1), (2, 2 * R - 1), None]
    t = L.tokens(gen, items)
    t["kv_slot_mapping"][2 * R - 1] = -1                                       # a boundary token with cache slot -1
    t["kv_slot_mapping"][R - 1] = L.kv_nb * L.kv_bs + 2                        # and one past the cache
    t["slot_mapping"][len(items) - 2] = -1                                     # state slot -1 at a boundary: nothing
    state_d, cache_d = L.state.to(dev), L.cache.to(dev)
    L.run(dev, state_d, cache_d, t)
    state, cache = L.state.clone(), L.cache.clone()
    rows = L.oracle(state, cache, t)
    assert len(rows) >= 2
    assert torch.equal(state_d.cpu(), state)
    C.check_cache(cache_d.cpu(), cache, rows, t["kv_slot_mapping"])


@pytest.mark.parametrize("D,ratio", SHAPES, ids=IDS)
def test_split_and_batch_invariance(dev, D, ratio):
    gen = torch.Generator().manual_seed(3 * D + ratio)
    L = Layer(gen, D, ratio, n_req=2, max_pos=512)
    prompt = L.tokens(gen, [(0, p) for p in range(300)])
    other = L.tokens(gen, [(1, p) for p in range(40, 40 + 2 * ratio + 1)])
    a_state, a_cache = L.state.to(dev), L.cache.to(dev)
    L.run(dev, a_state, a_cache, prompt)
    b_state, b_cache = L.state.to(dev), L.cache.to(dev)
    for i in range(300):
        L.run(dev, b_state, b_cache, {k: v[i:i + 1] for k, v in prompt.items()})
    assert torch.equal(a_state, b_state) and torch.equal(a_cache, b_cache)
    # both requests in one call == one request after the other
    both = {k: torch.cat([prompt[k], other[k]]) for k in prompt}
    c_state, c_cache = L.state.to(dev), L.cache.to(dev)
    L.run(dev, c_state, c_cache, both)
    L.run(dev, a_state, a_cache, other)
    assert torch.equal(a_state, c_state) and torch.equal(a_cache, c_cache)


@pytest.mark.parametrize("D,ratio", SHAPES, ids=IDS)
def test_graph_replay_matches_eager(dev, D, ratio):
    """A decode step of 3 requests, captured once and replayed for 12 steps: positions cross 3 boundaries at ratio 4 and
    one at ratio 128."""
    gen = torch.Generator().manual_seed(7 * D + ratio)
    L = Layer(gen, D, ratio, max_pos=512)
    start = [120, 250, 300] if ratio == 128 else [0, 5, 33]
    steps = [L.tokens(gen, [(r, start[r] + s) for r in range(3)]) for s in range(12)]
    e_state, e_cache = L.state.to(dev), L.cache.to(dev)
    for t in steps:
        L.run(dev, e_state, e_cache, t)
    g_state, g_cache = L.state.to(dev), L.cache.to(dev)
    static = {k: v.to(dev) for k, v in steps[0].items()}
    ape, bt, w, cs = L.ape.to(dev), L.block_table.to(dev), L.w.to(dev), L.cs.to(dev)

    def step():
        ops.dsv4_compress(static["kv_score"], ape, static["positions"], g_state, static["slot_mapping"],
                          static["token_to_req"], bt, w, EPS, cs, g_cache, static["kv_slot_mapping"], ratio)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                                                 # warm-up, then back to the start state
    torch.cuda.current_stream().wait_stream(s)
    g_state.copy_(L.state.to(dev))
    g_cache.copy_(L.cache.to(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    g_state.copy_(L.state.to(dev))
    g_cache.copy_(L.cache.to(dev))
    for t in steps:
        for k, v in t.items():
            static[k].copy_(v)
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_state, e_state) and torch.equal(g_cache, e_cache)


def _decode_loop(dev, L, gen, n_req, n_steps):
    """n_steps one-token steps for every request from position 0, on the GPU and in the oracle."""
    state_d, cache_d = L.state.to(dev), L.cache.to(dev)
    state, cache = L.state.clone(), L.cache.clone()
    rows = {}
    for s in range(n_steps):
        t = L.tokens(gen, [(r, s) for r in range(n_req)])
        L.run(dev, state_d, cache_d, t)
        rows.update({(s, k): v for k, v in L.oracle(state, cache, t).items()})
    return cache_d, cache


def test_chain_into_sparse_decode(dev):
    gen = torch.Generator().manual_seed(21)
    n_req, n_steps, Hq = 2, 64, 64
    L = Layer(gen, 512, 4, n_req=n_req, max_pos=256, kv_bs=16)
    got, ref = _decode_loop(dev, L, gen, n_req, n_steps)
    swa = V4.pack((torch.randn(128, 512, generator=gen)).bfloat16(), 64, num_blocks=2)
    si = torch.stack([torch.randperm(128, generator=gen)[:32] for _ in range(n_req)]).int()
    sl = torch.full((n_req,), 32, dtype=torch.int32)
    ei = torch.stack([torch.tensor([L.kv_base[r] + j for j in range(n_steps // 4)]) for r in range(n_req)]).int()
    el = torch.full((n_req,), n_steps // 4, dtype=torch.int32)
    q = torch.randn(n_req, Hq, 512, generator=gen).bfloat16()
    scale = 512 ** -0.5
    out = ops.dsv4_sparse_decode(q.to(dev), swa.to(dev), si.to(dev), sl.to(dev), scale, extra_cache=got,
                                 extra_indices=ei.to(dev), extra_lens=el.to(dev))
    want = V4.decode(q, swa, si, sl, scale, None, ref, ei, el)
    torch.testing.assert_close(out.cpu().double(), want, atol=2e-2, rtol=2e-2)


def test_chain_into_indexer_logits(dev):
    gen = torch.Generator().manual_seed(22)
    n_req, n_steps, H = 2, 128, 64
    L = Layer(gen, 128, 4, n_req=n_req, max_pos=512, kv_bs=16)
    got, ref = _decode_loop(dev, L, gen, n_req, n_steps)
    n = n_steps // 4
    pt = torch.stack([torch.arange(L.kv_base[r] // 16, L.kv_base[r] // 16 + n // 16) for r in range(n_req)]).int()
    sl = torch.full((n_req,), n, dtype=torch.int32)
    q8 = (torch.randn(n_req, H, 128, generator=gen) * 8).to(torch.float8_e4m3fn)
    w = torch.randn(n_req, H, generator=gen)
    logits = ops.indexer_logits(q8.to(dev), w.to(dev), got, sl.to(dev), pt.to(dev)).cpu().double()
    want = IX.paged_logits(q8, w, ref, sl, pt, 1, n)
    # the accumulation tolerance of the indexer tests, plus what the (at most one-code) differences between the kernel's
    # and the oracle's cache bytes move a logit
    acc = 2 ** -10 * IX.paged_logits(q8.float().abs().to(torch.float8_e4m3fn), w.abs(), _abs_cache(ref), sl, pt, 1, n)
    moved = (IX.paged_logits(q8, w, got.cpu(), sl, pt, 1, n) - want).abs()
    assert ((logits[:, :n] - want).abs() <= acc + moved + 1e-12).all()


def _abs_cache(cache):
    nb, page, _ = cache.shape
    flat = cache.reshape(nb, page * 132).clone()
    flat[:, :page * 128] &= 0x7F
    return flat.reshape(nb, page, 132)


def test_python_refusals(dev):
    L = Layer(torch.Generator().manual_seed(1), 512, 4, n_req=1, max_pos=64)
    t = L.tokens(torch.Generator().manual_seed(2), [(0, 3)])
    with pytest.raises(ValueError):
        ops.dsv4_compress(t["kv_score"].to(dev), L.ape.to(dev), t["positions"].to(dev), L.state.to(dev),
                          t["slot_mapping"].to(dev), t["token_to_req"].to(dev), L.block_table.to(dev), L.w.to(dev), EPS,
                          L.cs.to(dev), L.cache.to(dev)[..., :132].contiguous(), t["kv_slot_mapping"].to(dev), 4)
