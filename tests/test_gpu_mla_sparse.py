"""GPU (-m gpu): sparse MLA decode (ops.mla_decode_sparse, attention over each query token's top-k keys) and the
fp8_ds_mla cache write.

Kernel vs the oracle (tests/mla_sparse_oracle.py) on the bf16 and fp8_ds_mla caches over head counts, top-k widths and split
counts, with invalid entries anywhere; vs the reference-generated golden fixture; bit for bit vs the dense decode on in-order
indices and vs one-token calls; the v up-projection form; the cache write byte for byte; a cache write -> sparse decode
chain eagerly and in a CUDA graph; and the argument refusals."""
import math
import os

import pytest
import torch

import mla_sparse_oracle as SP
from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_mla_sparse.pt")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_diff(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return 1 - 2 * (a * b).sum() / max((a * a + b * b).sum(), 1e-12)


def _cache(gen, pages, page, ds_mla):
    """A random latent cache: bf16 [pages, page, 576], or its fp8_ds_mla rows uint8 [pages, page, 656]."""
    c = torch.randn(pages, page, 576, generator=gen).bfloat16()
    if not ds_mla:
        return c
    return SP.ds_mla_quantize(c[..., :512].reshape(-1, 512), c[..., 512:].reshape(-1, 64)).reshape(pages, page, 656)


def _setup(T, R, npg, page, hq, topk, seed, ds_mla, special=True):
    """T query tokens of R requests over a page table [R, npg] (a permutation of R * npg + 2 pages: two pages no request
    owns).  Index rows: random request-local positions, with -1 runs and entries one page past the table; with `special`,
    token 0 has no valid entry, token 1 only -1 in its first half (masked tiles before valid ones) and token 2 holds a
    single key repeated."""
    gen = torch.Generator().manual_seed(seed)
    cache = _cache(gen, R * npg + 2, page, ds_mla)
    pt = torch.randperm(R * npg + 2, generator=gen)[:R * npg].reshape(R, npg).int()
    rid = torch.randint(0, R, (T,), generator=gen, dtype=torch.int32)
    idx = torch.randint(0, npg * page, (T, topk), generator=gen, dtype=torch.int32)
    for t in range(T):
        a = int(torch.randint(0, topk, (1,), generator=gen))
        idx[t, a:a + topk // 8] = -1
        idx[t, topk - topk // 16:] = -1
        b = int(torch.randint(0, topk, (1,), generator=gen))
        idx[t, b:b + 5] = npg * page + 3          # past the page table
    if special and T >= 3:
        idx[0] = -1
        idx[0, :7] = npg * page
        idx[1, :topk // 2] = -1
        idx[2] = -1
        idx[2, topk // 3::max(1, topk // 5)] = 11
    qn = torch.randn(T, hq, 512, generator=gen).bfloat16()
    qp = torch.randn(T, hq, 64, generator=gen).bfloat16()
    return qn, qp, cache, idx, rid, pt


def _valid_count(idx, npg, page):
    return ((idx >= 0) & (idx // page < npg)).sum(-1)


def _check(out, lse, ref_o, ref_l, idx, npg, page):
    """cos_diff < 1e-5 and lse within 1e-3 (the MLA tests' thresholds) on tokens with valid entries; tokens without one
    are exact zeros with lse -inf; no NaN anywhere."""
    o, ls = out.cpu(), lse.cpu()
    assert not torch.isnan(o.float()).any() and not torch.isnan(ls).any()
    blind = _valid_count(idx, npg, page) == 0
    assert torch.equal(o[blind].view(torch.int16), torch.zeros_like(o[blind]).view(torch.int16))
    assert (ls[blind] == -math.inf).all() and (ref_l[blind] == -math.inf).all()
    assert _cos_diff(o[~blind].float(), ref_o[~blind]) < 1e-5
    torch.testing.assert_close(ls[~blind], ref_l[~blind], atol=1e-3, rtol=1e-3)


def _run(dev, qn, qp, cache, idx, rid, pt, scale, splits=0, w_uv=None):
    from lvllm_b200 import ops
    return ops.mla_decode_sparse(qn.to(dev), qp.to(dev), cache.to(dev), idx.to(dev), rid.to(dev), pt.to(dev), scale,
                                 num_kv_splits=splits, w_uv=None if w_uv is None else w_uv.to(dev))


@pytest.mark.parametrize("ds_mla", [False, True], ids=["bf16", "fp8_ds_mla"])
@pytest.mark.parametrize("T,hq,topk,page,splits", [
    (3, 128, 2048, 64, 0),     # DeepSeek-V3.2: Hq 128, index_topk 2048
    (4, 128, 2048, 64, 3),     # uneven tiles per split
    (5, 16, 2048, 64, 0),      # a TP8 shard
    (4, 20, 300, 16, 2),       # a head count that does not divide 128, a partial last tile
    (3, 16, 1, 16, 1),         # a single entry
    (3, 64, 640, 64, 9),       # more splits than tiles: empty splits
])
def test_sparse_decode_vs_oracle(dev, ds_mla, T, hq, topk, page, splits):
    npg = 24
    qn, qp, cache, idx, rid, pt = _setup(T, 3, npg, page, hq, topk, 1 + hq + topk, ds_mla, special=topk > 1)
    if topk == 1:   # token 0 past the table, tokens 1 and 2 one valid key each
        idx[:, 0] = torch.tensor([npg * page, 5, 200], dtype=torch.int32)
    scale = 1.0 / math.sqrt(576)
    out, lse = _run(dev, qn, qp, cache, idx, rid, pt, scale, splits)
    torch.cuda.synchronize()
    ref_o, ref_l = SP.mla_decode_sparse(qn, qp, cache, idx, rid, pt, scale)   # fp8_ds_mla: on the dequantised cache
    _check(out, lse, ref_o, ref_l, idx, npg, page)


@pytest.mark.parametrize("ds_mla", [False, True], ids=["bf16", "fp8_ds_mla"])
def test_golden(dev, ds_mla):
    """Against the reference's sparse SDPA on the unquantised keys (golden_mla_sparse.pt), after the W_UV projection as the
    reference test compares.  bf16 cache: the latent output within cos_diff 1e-5, out_v within the reference's bf16
    tolerance (rtol 0.01, atol 0.01).  fp8_ds_mla cache: out_v within the reference's fp8 tolerance (rtol 0.065, atol 0.05)
    of the oracle run on the dequantised cache, which is what the reference test compares against.  Against the unquantised
    keys that tolerance does not hold everywhere: it does for the Hq 128 and Hq 16 cases (max |diff| 0.009 on an H100), but
    in the Hq 20 case 1.4 % of out_v exceeds it, by up to 0.071 absolute, from the token whose only key is one row: its output
    is that row's quantised latent, so no e4m3 error averages out.  All of it is quantisation error (the kernel matches the
    dequantised oracle); the bound asserted against the unquantised keys is atol 0.1."""
    g = torch.load(GOLDEN, weights_only=True)
    page = 16
    for c in g["attention"]:
        hq, S, idx = c["num_heads"], c["kv_len"], c["topk_indices"]
        T = idx.shape[0]
        q = g["q_pool"][:c["q_rows"]].reshape(T, hq, 576)
        npg = -(-S // page)
        keys = torch.zeros(npg * page, 576, dtype=torch.bfloat16)
        keys[:S] = g["keys"][:S]
        pt = torch.randperm(npg, generator=torch.Generator().manual_seed(S)).int()
        cache = torch.zeros(npg, page, 576, dtype=torch.bfloat16)
        cache[pt.long()] = keys.reshape(npg, page, 576)
        if ds_mla:
            cache = SP.ds_mla_quantize(cache[..., :512].reshape(-1, 512), cache[..., 512:].reshape(-1, 64)).reshape(npg, page, 656)
        w_uv = SP.golden_w_uv(hq)
        out_v, out, lse = _run(dev, q[..., :512].contiguous(), q[..., 512:].contiguous(), cache, idx,
                               torch.zeros(T, dtype=torch.int32), pt[None], g["scale"], w_uv=w_uv)
        torch.cuda.synchronize()
        v = out_v.cpu().float()
        if ds_mla:
            o_dq, _ = SP.mla_decode_sparse(q[..., :512], q[..., 512:], cache, idx, torch.zeros(T, dtype=torch.int32), pt[None],
                                           g["scale"])
            v_dq = torch.einsum("tnl,nlv->tnv", o_dq, w_uv.float())
            torch.testing.assert_close(v, v_dq, rtol=0.065, atol=0.05)
            excess = ((v - c["out_v"]).abs() - 0.065 * c["out_v"].abs()).clamp(min=0)
            print(f"fp8_ds_mla vs unquantised golden, Hq {hq}: max |diff| {(v - c['out_v']).abs().max():.4f}, "
                  f"{(excess > 0.05).float().mean() * 100:.2f} % beyond rtol 0.065 + atol 0.05")
            torch.testing.assert_close(v, c["out_v"], rtol=0.065, atol=0.1)
        else:
            assert _cos_diff(out.cpu().float()[..., g["out_dims"]], c["out"]) < 1e-5, hq
            torch.testing.assert_close(v, c["out_v"], rtol=0.01, atol=0.01)


@pytest.mark.parametrize("splits", [1, 4, 5, 16])
def test_in_order_indices_are_dense_decode(dev, splits):
    """Indices 0 .. S_b - 1 in order, padded with -1 to topk = max_pages * page: bit-identical out and lse to
    b200_mla_decode_ex at the same split count (the same 128-token tiles per CTA)."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    B, hq, page, npg = 4, 128, 64, 32
    topk = npg * page
    gen = torch.Generator().manual_seed(splits)
    cache = _cache(gen, B * npg, page, False).to(dev)
    pt = torch.randperm(B * npg, generator=gen).reshape(B, npg).int().to(dev)
    lens = torch.tensor([1, 130, 1500, 2048], dtype=torch.int32)
    lens_d = lens.to(dev)
    qn = torch.randn(B, hq, 512, generator=gen).bfloat16().to(dev)
    qp = torch.randn(B, hq, 64, generator=gen).bfloat16().to(dev)
    idx = torch.full((B, topk), -1, dtype=torch.int32)
    for b in range(B):
        idx[b, :lens[b]] = torch.arange(int(lens[b]), dtype=torch.int32)
    scale = 1.0 / math.sqrt(192)
    ws = torch.empty(lib.b200_mla_decode_workspace_bytes(B, hq, splits), dtype=torch.uint8, device=dev)
    out = torch.empty(B, hq, 512, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(B, hq, dtype=torch.float32, device=dev)
    L.check(lib.b200_mla_decode_ex(torch.cuda.current_stream().cuda_stream, qn.data_ptr(), qp.data_ptr(), 0, cache.data_ptr(),
                                   0, 1.0, 1.0, lens_d.data_ptr(), pt.data_ptr(), B, hq, page, npg, scale, splits,
                                   ws.data_ptr(), out.data_ptr(), lse.data_ptr()), "b200_mla_decode_ex")
    s_out, s_lse = _run(dev, qn, qp, cache, idx, torch.arange(B, dtype=torch.int32), pt, scale, splits)
    torch.cuda.synchronize()
    assert torch.equal(s_out.view(torch.int16), out.view(torch.int16))
    assert torch.equal(s_lse, lse)


@pytest.mark.parametrize("ds_mla", [False, True], ids=["bf16", "fp8_ds_mla"])
def test_tokens_in_one_call_are_one_token_calls(dev, ds_mla):
    """T tokens (several of them draft tokens of one request) in one call: bit-identical to T one-token calls."""
    T, hq, topk, page, npg = 6, 32, 512, 64, 12
    qn, qp, cache, idx, rid, pt = _setup(T, 2, npg, page, hq, topk, 7, ds_mla)
    rid[3:] = 1
    scale = 1.0 / math.sqrt(576)
    out, lse = _run(dev, qn, qp, cache, idx, rid, pt, scale, 2)
    for t in range(T):
        o1, l1 = _run(dev, qn[t:t + 1], qp[t:t + 1], cache, idx[t:t + 1], rid[t:t + 1], pt, scale, 2)
        assert torch.equal(o1.view(torch.int16), out[t:t + 1].view(torch.int16)), t
        assert torch.equal(l1, lse[t:t + 1]), t


@pytest.mark.parametrize("ds_mla", [False, True], ids=["bf16", "fp8_ds_mla"])
def test_permuted_index_row(dev, ds_mla):
    """The key set, not the order of the index row, decides the result (within the oracle thresholds)."""
    T, hq, topk, page, npg = 3, 128, 2048, 64, 40
    qn, qp, cache, idx, rid, pt = _setup(T, 2, npg, page, hq, topk, 11, ds_mla, special=False)
    perm = torch.stack([torch.randperm(topk, generator=torch.Generator().manual_seed(t)) for t in range(T)])
    scale = 1.0 / math.sqrt(576)
    out, lse = _run(dev, qn, qp, cache, idx, rid, pt, scale)
    out_p, lse_p = _run(dev, qn, qp, cache, torch.gather(idx, 1, perm), rid, pt, scale)
    torch.cuda.synchronize()
    assert _cos_diff(out_p.cpu().float(), out.cpu().float()) < 1e-5
    torch.testing.assert_close(lse_p.cpu(), lse.cpu(), atol=1e-3, rtol=1e-3)


def test_invalid_tokens_and_masked_leading_tiles(dev):
    """A token with no valid entry (all -1, or every entry past the page table) gives out 0 and lse -inf; tokens whose first
    tiles are fully masked, at every split count, give no NaN and match the oracle."""
    T, hq, topk, page, npg = 4, 64, 1024, 64, 8
    gen = torch.Generator().manual_seed(3)
    cache = _cache(gen, npg, page, False)
    pt = torch.randperm(npg, generator=gen)[None].int()
    idx = torch.full((T, topk), -1, dtype=torch.int32)
    idx[1] = npg * page + torch.arange(topk, dtype=torch.int32)         # all past the table
    idx[2, 7 * 128 + 5:7 * 128 + 40] = torch.arange(35, dtype=torch.int32)   # only the last tile holds keys
    idx[3, 3 * 128:5 * 128] = torch.randint(0, npg * page, (256,), generator=gen, dtype=torch.int32)
    qn = torch.randn(T, hq, 512, generator=gen).bfloat16() * 4
    qp = torch.randn(T, hq, 64, generator=gen).bfloat16()
    rid = torch.zeros(T, dtype=torch.int32)
    scale = 1.0 / math.sqrt(192)
    ref_o, ref_l = SP.mla_decode_sparse(qn, qp, cache, idx, rid, pt, scale)
    for splits in (1, 2, 3, 8):
        out, lse = _run(dev, qn, qp, cache, idx, rid, pt, scale, splits)
        torch.cuda.synchronize()
        _check(out, lse, ref_o, ref_l, idx, npg, page)
        assert (lse.cpu()[:2] == -math.inf).all()


def test_w_uv_form(dev):
    """With w_uv: out_v matches the oracle's o . W_UV and the optional latent output and lse match the call without w_uv."""
    T, hq, topk, page, npg = 4, 128, 2048, 64, 40
    for ds_mla in (False, True):
        qn, qp, cache, idx, rid, pt = _setup(T, 2, npg, page, hq, topk, 21, ds_mla)
        w_uv = (torch.randn(hq, 512, 128, generator=torch.Generator().manual_seed(2)) / math.sqrt(512)).bfloat16()
        scale = 1.0 / math.sqrt(576)
        out_v, o_lat, lse = _run(dev, qn, qp, cache, idx, rid, pt, scale, w_uv=w_uv)
        out, lse0 = _run(dev, qn, qp, cache, idx, rid, pt, scale)
        torch.cuda.synchronize()
        ref_o, ref_l = SP.mla_decode_sparse(qn, qp, cache, idx, rid, pt, scale)
        v_ref = O.mla_v_up(ref_o.bfloat16(), w_uv)
        live = _valid_count(idx, npg, page) > 0
        assert _cos_diff(out_v.cpu().float()[live], v_ref.float()[live]) < 2e-5
        assert torch.equal(out_v.cpu()[~live].view(torch.int16), torch.zeros_like(out_v.cpu()[~live]).view(torch.int16))
        assert _cos_diff(o_lat.cpu().float(), out.cpu().float()) < 1e-5
        torch.testing.assert_close(lse.cpu(), lse0.cpu(), atol=1e-3, rtol=1e-3)
        _check(o_lat, lse, ref_o, ref_l, idx, npg, page)


def _rope_table():
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.float) / 64))
    fr = torch.einsum("i,j->ij", torch.arange(4096, dtype=torch.float), inv)
    return torch.cat((fr.cos(), fr.sin()), dim=-1).bfloat16()


def test_ds_mla_cache_write_byte_exact(dev):
    """ops.mla_rope_cache_write on a 656-byte cache: the row of concat_and_cache_ds_mla_kernel, byte for byte (the oracle's
    quantisation of kv_c and of the kernel's own rotated k_pe), every other byte untouched (padded slots included)."""
    from lvllm_b200 import ops
    gen = torch.Generator().manual_seed(4)
    T, hq, page, pages = 9, 16, 16, 4
    kv_c = torch.randn(T, 512, generator=gen) * torch.tensor([1e-3, 1.0, 200.0, 0.0]).repeat_interleave(128)
    kv_c[1] = 0
    kv_c[2, :128] = 1e-37                                      # amax / 448 below FLT_MIN: the FLT_MIN scale
    kv_c = kv_c.bfloat16()
    k_pe = torch.randn(T, 64, generator=gen).bfloat16()
    q_pe = torch.randn(T, hq, 64, generator=gen).bfloat16()
    pos = torch.randint(0, 4096, (T,), generator=gen)
    slots = torch.randperm(pages * page, generator=gen)[:T]
    slots[4] = -1
    slots[7] = -1
    cache0 = torch.randint(0, 256, (pages, page, 656), generator=gen, dtype=torch.uint8)
    cache = cache0.to(dev)
    kp, qp = k_pe.to(dev), q_pe.to(dev)
    ops.mla_rope_cache_write(qp, kp, kv_c.to(dev), pos.to(dev), _rope_table().to(dev), slots.to(dev), cache)
    torch.cuda.synchronize()
    want = cache0.clone().reshape(-1, 656)
    rows = SP.ds_mla_quantize(kv_c, kp.cpu())
    for t in range(T):
        if slots[t] >= 0:
            want[slots[t]] = rows[t]
    assert torch.equal(cache.cpu().reshape(-1, 656), want)
    # the rope of k_pe is the one the bf16 cache path applies
    kp2, qp2 = k_pe.to(dev), q_pe.to(dev)
    bf_cache = torch.zeros(pages, page, 576, dtype=torch.bfloat16, device=dev)
    ops.mla_rope_cache_write(qp2, kp2, kv_c.to(dev), pos.to(dev), _rope_table().to(dev), slots.to(dev), bf_cache)
    assert torch.equal(kp2.view(torch.int16), kp.view(torch.int16)) and torch.equal(qp2.view(torch.int16), qp.view(torch.int16))


def test_step_chain_eager_and_graph(dev):
    """cache write (fp8_ds_mla) -> sparse decode with the v up-projection, for three steps: captured once in a CUDA graph
    and replayed with inputs updated in place, out_v, out, lse and the cache are bit-identical to the eager chain."""
    from lvllm_b200 import ops
    T, hq, topk, page, npg = 4, 16, 512, 64, 10
    gen = torch.Generator().manual_seed(9)
    table = _rope_table().to(dev)
    pt = torch.randperm(2 * npg, generator=gen).reshape(2, npg).int().to(dev)
    rid = torch.tensor([0, 0, 1, 1], dtype=torch.int32, device=dev)
    w_uv = (torch.randn(hq, 512, 128, generator=gen) / math.sqrt(512)).bfloat16().to(dev)
    cache0 = _cache(gen, 2 * npg, page, True).to(dev)
    cache_e, cache_g = cache0.clone(), cache0.clone()
    scale = 1.0 / math.sqrt(576)

    def inputs(step):
        g = torch.Generator().manual_seed(100 + step)
        pos = torch.tensor([300, 301, 90, 91]) + 2 * step
        slots = (pt.cpu()[rid.cpu().long(), pos // page].long() * page + pos % page)
        idx = torch.randint(0, int(pos.max()) + 1, (T, topk), generator=g, dtype=torch.int32)
        idx[:, topk - 40:] = -1
        return dict(q_nope=torch.randn(T, hq, 512, generator=g).bfloat16(), q_pe=torch.randn(T, hq, 64, generator=g).bfloat16(),
                    k_pe=torch.randn(T, 64, generator=g).bfloat16(), kv_c=torch.randn(T, 512, generator=g).bfloat16(),
                    pos=pos, slots=slots, idx=idx)

    def step(x, cache):
        ops.mla_rope_cache_write(x["q_pe"], x["k_pe"], x["kv_c"], x["pos"], table, x["slots"], cache)
        return ops.mla_decode_sparse(x["q_nope"], x["q_pe"], cache, x["idx"], rid, pt, scale, num_kv_splits=2, w_uv=w_uv)

    st = {k: torch.zeros_like(v).to(dev) for k, v in inputs(0).items()}
    st["slots"].fill_(-1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(st, cache_g)   # warm-up with slots -1: writes nothing
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(cache_g, cache0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        v_g, o_g, l_g = step(st, cache_g)
    for s in range(3):
        x = inputs(s)
        xd = {k: v.to(dev) for k, v in x.items()}
        v_e, o_e, l_e = step(xd, cache_e)
        for k in st:
            st[k].copy_(x[k])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(v_g.view(torch.int16), v_e.view(torch.int16))
        assert torch.equal(o_g.view(torch.int16), o_e.view(torch.int16))
        assert torch.equal(l_g, l_e)
        assert torch.equal(cache_g, cache_e)
        assert torch.isfinite(l_e).all()


def test_refusals(dev):
    """B200_ERR_INVALID (-1) with nothing launched: kv_dtype 1, more than 128 heads, topk < 1, a NULL required pointer,
    num_splits <= 0, num_splits > 512 with w_uv; ops.mla_decode_sparse refuses e4m3 queries and a cache of another layout."""
    from lvllm_b200 import _lib as L
    from lvllm_b200 import ops
    lib = L.lib()
    T, hq, page, topk = 2, 16, 16, 64
    cache = torch.zeros(2, page, 656, dtype=torch.uint8, device=dev)
    ws = torch.empty(lib.b200_mla_decode_workspace_bytes(T, 129, 600), dtype=torch.uint8, device=dev)
    idx = torch.zeros(T, topk, dtype=torch.int32, device=dev)
    rid = torch.zeros(T, dtype=torch.int32, device=dev)
    ptab = torch.zeros(1, 2, dtype=torch.int32, device=dev)
    out = torch.empty(T, 129, 512, dtype=torch.bfloat16, device=dev)
    out_v = torch.empty(T, 129, 128, dtype=torch.bfloat16, device=dev)
    w_uv = torch.zeros(129, 512, 128, dtype=torch.bfloat16, device=dev)
    qn = torch.zeros(T, 129, 512, dtype=torch.bfloat16, device=dev)
    qp = torch.zeros(T, 129, 64, dtype=torch.bfloat16, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def call(**kw):
        a = dict(q_nope=qn.data_ptr(), q_pe=qp.data_ptr(), kv=cache.data_ptr(), kv_dtype=2, idx=idx.data_ptr(), topk=topk,
                 rid=rid.data_ptr(), pt=ptab.data_ptr(), max_pages=2, T=T, hq=hq, page=page, scale=0.1, splits=1,
                 ws=ws.data_ptr(), out=out.data_ptr(), lse=None, w_uv=None, out_v=None)
        a.update(kw)
        return lib.b200_mla_decode_sparse(stream, *a.values())

    n0 = lib.b200moe_launch_count()
    bad = [dict(kv_dtype=1), dict(kv_dtype=3), dict(hq=129), dict(hq=0), dict(topk=0), dict(splits=0), dict(splits=-1),
           dict(splits=513, w_uv=w_uv.data_ptr(), out_v=out_v.data_ptr()), dict(w_uv=w_uv.data_ptr()), dict(out=None)]
    bad += [{k: None} for k in ("q_nope", "q_pe", "kv", "idx", "rid", "pt", "ws")]
    for kw in bad:
        assert call(**kw) == -1, kw
        assert b"b200_mla_decode_sparse" in lib.b200moe_last_error()
    assert lib.b200moe_launch_count() == n0
    assert call(hq=128, splits=513) == 0          # above 512 splits without w_uv: decode_merge_kernel
    assert call(hq=128, splits=512, w_uv=w_uv.data_ptr(), out_v=out_v.data_ptr()) == 0
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="bf16 queries"):
        ops.mla_decode_sparse(qn[:, :hq].to(torch.float8_e4m3fn), qp[:, :hq].to(torch.float8_e4m3fn), cache, idx, rid, ptab, 0.1)
    with pytest.raises(ValueError, match="kv_cache"):
        ops.mla_decode_sparse(qn[:, :hq], qp[:, :hq], torch.zeros(2, page, 576, dtype=torch.float8_e4m3fn, device=dev),
                              idx, rid, ptab, 0.1)
