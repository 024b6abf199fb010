"""GPU (-m gpu): DeepSeek-V4 sparse attention decode (ops.dsv4_sparse_decode) and its q-norm + RoPE + cache insert
(ops.dsv4_qnorm_rope_kv_insert).

The insert byte for byte (e4m3 and scale bytes) and within one bf16 ulp (rope dims, q) against the float64 oracle
(tests/dsv4_sparse_oracle.py); the decode against the oracle on the dequantised caches over SWA-only, SWA + C4A-like and
SWA + C128A-like lists, block sizes 64 / 16 / 2, head counts 64, 128, 16 and 20, invalid entries anywhere, a token without
keys and with / without a sink; bit relations between calls; insert -> decode eagerly and in a CUDA graph."""
import math

import pytest
import torch

import dsv4_sparse_oracle as V4
from lvllm_b200 import ops

pytestmark = pytest.mark.gpu

SCALE = 512 ** -0.5


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _kv(gen, n):
    """n bf16 rows [n, 512] whose 64-dim groups span magnitudes (so the ue8m0 scales differ between groups)."""
    x = torch.randn(n, 512, generator=gen)
    x[:, :448] *= torch.pow(2.0, torch.randint(-6, 2, (n, 7), generator=gen).float()).repeat_interleave(64, 1)
    return x.bfloat16()


def _cache(gen, blocks, bs, pad=0):
    """A packed cache of blocks * bs random rows, uint8 [blocks, bs, 584]; pad > 0: a view with a padded block stride."""
    c = V4.pack(_kv(gen, blocks * bs), bs, num_blocks=blocks)
    if not pad:
        return c
    buf = torch.zeros(blocks, bs * 584 + pad, dtype=torch.uint8)
    buf[:, :bs * 584] = c.reshape(blocks, -1)
    return buf, buf.as_strided((blocks, bs, 584), (bs * 584 + pad, 584, 1))


def _rows(gen, T, width, n_valid, n_slots):
    """int32 [T, width]: n_valid[t] distinct valid slots per row at random places, the rest -1 or out of range."""
    r = torch.full((T, width), -1, dtype=torch.int32)
    for t in range(T):
        r[t, torch.randperm(width, generator=gen)[:width // 5]] = n_slots + int(torch.randint(0, 1000, (1,), generator=gen))
        k = min(n_valid[t], width)
        r[t, torch.randperm(width, generator=gen)[:k]] = torch.randperm(n_slots, generator=gen)[:k].int()
    return r


def _to(dev, *xs):
    return [x.to(dev) if isinstance(x, torch.Tensor) else x for x in xs]


# (name, Hq, T, swa: (block size, blocks, width), extra: (block size, blocks, width) or None)
CASES = [
    ("swa", 64, 4, (64, 8, 128), None),
    ("c4a", 128, 3, (64, 8, 128), (16, 64, 512)),
    ("c4a_h20", 20, 5, (64, 8, 128), (16, 48, 384)),
    ("c128a", 16, 6, (64, 4, 128), (2, 40, 64)),
]


def _decode_case(gen, Hq, T, swa, extra):
    sbs, snb, sw = swa
    sc = _cache(gen, snb, sbs, pad=64)
    si = _rows(gen, T, sw, [sw] + [int(x) for x in torch.randint(1, sw, (T - 1,), generator=gen)], snb * sbs)
    sl = torch.randint(sw // 2, sw + 1, (T,), generator=gen, dtype=torch.int32)
    sl[0] = sw
    ex = None
    if extra:
        ebs, enb, ew = extra
        ec = _cache(gen, enb, ebs)
        ei = _rows(gen, T, ew, [int(x) for x in torch.randint(ew // 2, ew + 1, (T,), generator=gen)], enb * ebs)
        el = torch.randint(ew // 2, ew + 1, (T,), generator=gen, dtype=torch.int32)
        ex = (ec, ei, el)
    # token 1: one valid key; the last token: none in either list
    si[1] = -1
    si[1, 37 % sw] = 3
    sl[1] = sw
    si[T - 1] = -1
    if ex:
        ex[1][1] = -1
        ex[1][T - 1] = -1
    q = torch.randn(T, Hq, 512, generator=gen).bfloat16()
    sink = torch.randn(Hq, generator=gen).float() * 2
    return q, sc, si, sl, ex, sink


@pytest.mark.parametrize("with_sink", [False, True])
@pytest.mark.parametrize("name,Hq,T,swa,extra", CASES, ids=[c[0] for c in CASES])
def test_decode_matches_oracle(dev, name, Hq, T, swa, extra, with_sink):
    gen = torch.Generator().manual_seed(sum(map(ord, name)) + 7 * with_sink)
    q, (sbuf, sc), si, sl, ex, sink = _decode_case(gen, Hq, T, swa, extra)
    sink = sink if with_sink else None
    ref = V4.decode(q, sc, si, sl, SCALE, sink, *(ex or (None, None, None)))
    sbuf_d = sbuf.to(dev)
    sc_d = sbuf_d.as_strided(sc.shape, sc.stride())
    kw = {}
    if ex:
        kw = dict(extra_cache=ex[0].to(dev), extra_indices=ex[1].to(dev), extra_lens=ex[2].to(dev))
    out = ops.dsv4_sparse_decode(*_to(dev, q), sc_d, *_to(dev, si, sl), SCALE,
                                 attn_sink=sink.to(dev) if sink is not None else None, **kw)
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.equal(out[T - 1], torch.zeros_like(out[T - 1]))          # no valid key: 0, with or without a sink
    torch.testing.assert_close(out.double(), ref, atol=2e-2, rtol=2e-2)


def test_bit_relations(dev):
    gen = torch.Generator().manual_seed(11)
    q, (_, sc), si, sl, (ec, ei, el), sink = _decode_case(gen, 64, 4, (64, 8, 128), (16, 64, 512))
    q, sc, si, sl, ec, ei, el, sink = _to(dev, q, sc.contiguous(), si, sl, ec, ei, el, sink)
    ext = dict(extra_cache=ec, extra_indices=ei, extra_lens=el)
    a = ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, attn_sink=sink, **ext)
    b = ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, attn_sink=sink, **ext)
    assert torch.equal(a, b)                                                  # repeated calls
    ninf = torch.full_like(sink, -math.inf)
    assert torch.equal(ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, attn_sink=ninf, **ext),
                       ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, **ext))   # sink -inf == no sink
    # extra_lens = 0 == no extra list (one split: the same tiles in the same CTA)
    z = dict(extra_cache=ec, extra_indices=ei, extra_lens=torch.zeros_like(el))
    assert torch.equal(ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, attn_sink=sink, num_kv_splits=1, **z),
                       ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, attn_sink=sink, num_kv_splits=1))
    # other split counts: the merge order and each split's running maximum (the base of the bf16 P) change, nothing else
    for splits in (1, 2, 5, 16):
        o = ops.dsv4_sparse_decode(q, sc, si, sl, SCALE, attn_sink=sink, num_kv_splits=splits, **ext)
        torch.testing.assert_close(o.float(), a.float(), atol=1e-2, rtol=1e-2)


@pytest.mark.parametrize("Hq,Hp,bs,pad", [(64, 128, 64, 0), (20, 64, 16, 32)])
def test_insert_matches_oracle(dev, Hq, Hp, bs, pad):
    gen = torch.Generator().manual_seed(Hq)
    T, nb, max_pos = 37, 3, 4096
    q = (torch.randn(T, Hq, 512, generator=gen) * 3).bfloat16()
    kv = _kv(gen, T)
    kv[5, 64:128] *= 1e-6                                                     # below the 1e-4 clamp
    pos = torch.randint(0, max_pos, (T,), generator=gen)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(max_pos, dtype=torch.float64)[:, None] * inv[None]
    cs = torch.cat([f.cos(), f.sin()], dim=1).float()
    slots = torch.randperm(nb * bs, generator=gen)[:T]
    slots[[0, 9, 30]] = -1
    slots[17] = nb * bs + 3                                                   # past the cache: nothing written
    init = torch.randint(0, 256, (nb, bs * 584 + pad), generator=gen, dtype=torch.uint8)
    ref_cache = init.as_strided((nb, bs, 584), (bs * 584 + pad, 584, 1)).clone()
    q_ref = V4.insert(q, kv, pos, cs, slots, ref_cache, Hp, 1e-6)
    buf = init.to(dev)
    cache = buf.as_strided((nb, bs, 584), (bs * 584 + pad, 584, 1))
    q_out = ops.dsv4_qnorm_rope_kv_insert(*_to(dev, q, kv, pos, cs, slots), cache, Hp, 1e-6).cpu()
    got = buf.cpu()
    assert torch.equal(q_out[:, Hq:], torch.zeros_like(q_out[:, Hq:]))
    assert int(V4.bf16_ulp_distance(q_out[:, :Hq], q_ref[:, :Hq]).max()) <= 1
    assert torch.equal(got[:, bs * 584:], init[:, bs * 584:])                 # the block padding is never written
    # every row, written or not (rows no slot names keep their initial bytes in both)
    g3 = got.as_strided((nb, bs, 584), (bs * 584 + pad, 584, 1))
    rope_dist = 0
    for b in range(nb):
        gb, rb = g3[b].reshape(-1), ref_cache[b].reshape(-1)
        for p in range(bs):
            d = slice(p * 576, p * 576 + 448)
            r = slice(p * 576 + 448, p * 576 + 576)
            s = slice(bs * 576 + p * 8, bs * 576 + p * 8 + 8)
            assert torch.equal(gb[d], rb[d]) and torch.equal(gb[s], rb[s]), (b, p)
            rope_dist = max(rope_dist, int(V4.bf16_ulp_distance(gb[r].contiguous().view(torch.bfloat16),
                                                                rb[r].contiguous().view(torch.bfloat16)).max()))
    assert rope_dist <= 1


def test_insert_then_decode_eager_and_graph(dev):
    """insert writes T tokens' rows, decode reads them (plus older rows) through index lists; then the same two calls are
    captured in one CUDA graph and replayed with new inputs and new index contents."""
    gen = torch.Generator().manual_seed(5)
    T, Hq, Hp, bs, nb, W = 8, 64, 64, 64, 4, 128
    max_pos = 2048
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(max_pos, dtype=torch.float64)[:, None] * inv[None]
    cs = torch.cat([f.cos(), f.sin()], dim=1).float().to(dev)
    cache = V4.pack(_kv(gen, nb * bs), bs, num_blocks=nb).to(dev)
    sink = (torch.randn(Hq, generator=gen) * 2).to(dev)
    q_in = torch.empty(T, Hq, 512, dtype=torch.bfloat16, device=dev)
    kv_in = torch.empty(T, 512, dtype=torch.bfloat16, device=dev)
    pos = torch.empty(T, dtype=torch.int64, device=dev)
    slots = torch.empty(T, dtype=torch.int64, device=dev)
    idx = torch.empty(T, W, dtype=torch.int32, device=dev)
    lens = torch.empty(T, dtype=torch.int32, device=dev)

    def fill(step):
        g = torch.Generator().manual_seed(100 + step)
        q_in.copy_((torch.randn(T, Hq, 512, generator=g) * 2).bfloat16())
        kv_in.copy_(_kv(g, T))
        p = torch.randint(0, max_pos, (T,), generator=g)
        s = torch.randperm(nb * bs, generator=g)[:T]
        pos.copy_(p)
        slots.copy_(s)
        rows = _rows(g, T, W, [int(x) for x in torch.randint(20, W, (T,), generator=g)], nb * bs)
        rows[:, 0] = s.int()                                                 # each token sees its own new row
        idx.copy_(rows)
        lens.copy_(torch.randint(W // 2, W + 1, (T,), generator=g, dtype=torch.int32))

    def step():
        qo = ops.dsv4_qnorm_rope_kv_insert(q_in, kv_in, pos, cs, slots, cache, Hp, 1e-6)
        return ops.dsv4_sparse_decode(qo, cache, idx, lens, SCALE, attn_sink=sink, num_kv_splits=2), qo

    def check(out, qo):
        ref = V4.decode(qo.cpu(), cache.cpu(), idx.cpu(), lens.cpu(), SCALE, sink.cpu())
        torch.testing.assert_close(out.cpu().double(), ref, atol=2e-2, rtol=2e-2)

    fill(0)
    out, qo = step()
    check(out, qo)
    eager_cache = cache.clone()
    fill(1)
    out1_eager, _ = step()
    cache.copy_(eager_cache)                                                 # replay step 1 from the same cache state
    fill(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                                               # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    cache.copy_(eager_cache)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_qo = step()
    fill(1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_out, out1_eager)
    check(g_out, g_qo)


def test_python_refusals(dev):
    q = torch.zeros(2, 64, 512, dtype=torch.bfloat16, device=dev)
    c = torch.zeros(2, 64, 584, dtype=torch.uint8, device=dev)
    i = torch.zeros(2, 128, dtype=torch.int32, device=dev)
    n = torch.zeros(2, dtype=torch.int32, device=dev)
    with pytest.raises(ValueError):
        ops.dsv4_sparse_decode(q.float(), c, i, n, SCALE)
    with pytest.raises(ValueError):
        ops.dsv4_sparse_decode(q, c[..., :576], i, n, SCALE)
    with pytest.raises(ValueError):
        ops.dsv4_sparse_decode(q, c, i[:1], n, SCALE)
    with pytest.raises(ValueError):
        ops.dsv4_sparse_decode(q, c, i, n, SCALE, extra_cache=c)
    with pytest.raises(ValueError):
        ops.dsv4_sparse_decode(q, c, i, n, SCALE, attn_sink=torch.zeros(3, device=dev))
    with pytest.raises(ValueError):
        ops.dsv4_qnorm_rope_kv_insert(q, q[:, 0], n.long(), torch.zeros(8, 64, device=dev), n.long(), c, 32, 1e-6)
