"""GPU (-m gpu): DeepSeek-V4 manifold hyper-connections (ops.mhc_pre / mhc_post / mhc_fused_post_pre / hc_head).

Each op against the float64 oracle (tests/mhc_oracle.py) at H in {1280, 4096, 7168} and T in {1, 2, 7, 16, 64, 256}, with and
without the fused norm: r' within 1 bf16 ulp, post_mix and comb_mix within 2e-6, layer_input within 1 ulp (2 with the norm)
and hc_head within 1 ulp, each or within the fp32 accumulation bound where the stream terms cancel.  The fused op bit-identical
to mhc_pre(mhc_post(...)); batch invariance; determinism and CUDA-graph replay; all-zero padding rows; a layer chain."""
import pytest
import torch

import mhc_oracle as M
from lvllm_b200 import ops

pytestmark = pytest.mark.gpu

EPS, REPEAT, POST_MULT = 1e-6, 20, 2.0
HS, TS = (1280, 4096, 7168), (1, 2, 7, 16, 64, 256)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _weights(gen, H, big=False):
    """fn, hc_scale, hc_base, norm_weight, head fn, head scale, head base as the reference test draws them; big: a large
    hc_scale, so the comb logits span several units."""
    fn = (torch.randn(24, 4, H, generator=gen) * 1e-4 * (1 + torch.arange(4).mul(0.01).view(1, -1, 1))).flatten(1, 2)
    sc = torch.tensor([30.0, 30.0, 500.0]) if big else torch.randn(3, generator=gen) * 0.1
    return dict(fn=fn, hc_scale=sc, hc_base=torch.randn(24, generator=gen) * 0.1,
                norm_weight=(1 + 0.1 * torch.randn(H, generator=gen)).bfloat16(),
                head_fn=torch.randn(4, 4 * H, generator=gen) * 1e-4, head_scale=torch.randn(1, generator=gen) * 0.1,
                head_base=torch.randn(4, generator=gen) * 0.1)


def _inputs(gen, T, H, pad=()):
    residual = torch.randn(T, 4, H, generator=gen).bfloat16()
    x = torch.randn(T, H, generator=gen).bfloat16()
    plm = torch.rand(T, 4, 1, generator=gen) * 2
    crm = torch.rand(T, 4, 4, generator=gen)
    crm = crm / crm.sum(-2, keepdim=True)
    for t in pad:
        residual[t], x[t] = 0, 0
    return residual, x, plm, crm


def _g(t, d):
    return t.to(d) if t is not None else None


def _pre_args(w, norm):
    return (w["fn"], w["hc_scale"], w["hc_base"], EPS, EPS, EPS, POST_MULT, REPEAT), \
        dict(norm_weight=w["norm_weight"] if norm else None, norm_eps=EPS)


def _check_pre(got, residual, w, norm):
    args, kw = _pre_args(w, norm)
    pm, cm, li, slack = M.pre(residual, *args, **kw, with_slack=True)
    assert got[0].shape == (residual.shape[0], 4, 1) and got[1].shape == (residual.shape[0], 4, 4)
    assert (got[0].cpu().double() - pm).abs().max() <= 2e-6
    assert (got[1].cpu().double() - cm).abs().max() <= 2e-6
    assert M.bf16_close(got[2].cpu(), li, slack, 2 if norm else 1)


def _dev_args(w, norm, d):
    args, kw = _pre_args(w, norm)
    return tuple(_g(a, d) if torch.is_tensor(a) else a for a in args), {k: _g(v, d) if torch.is_tensor(v) else v
                                                                        for k, v in kw.items()}


@pytest.mark.parametrize("H", HS)
@pytest.mark.parametrize("T", TS)
def test_ops_against_oracle(dev, H, T):
    gen = torch.Generator().manual_seed(1000 * T + H)
    w = _weights(gen, H, big=T == 7)
    residual, x, plm, crm = _inputs(gen, T, H, pad=(T // 2,) if T > 1 else ())
    rd, xd, pd, cd = (t.to(dev) for t in (residual, x, plm, crm))
    r_post, slack = M.post(x, residual, plm, crm, with_slack=True)
    got_post = ops.mhc_post(xd, rd, pd, cd)
    assert M.bf16_close(got_post.cpu(), r_post, slack, 1)
    for norm in (False, True):
        args, kw = _dev_args(w, norm, dev)
        _check_pre(ops.mhc_pre(rd, *args, **kw), residual, w, norm)
        f = ops.mhc_fused_post_pre(xd, rd, pd, cd, *args, **kw)
        assert M.bf16_close(f[0].cpu(), r_post, slack, 1)
        _check_pre(f[1:], f[0].cpu(), w, norm)
    head, hslack = M.hc_head(residual, w["head_fn"], w["head_scale"], w["head_base"], EPS, EPS, with_slack=True)
    got = ops.hc_head(rd, w["head_fn"].to(dev), w["head_scale"].to(dev), w["head_base"].to(dev), EPS, EPS)
    assert M.bf16_close(got.cpu(), head, hslack, 1)
    if T > 1:   # the padding row
        t = T // 2
        assert torch.isfinite(f[1][t]).all() and torch.isfinite(f[2][t]).all() and (got[t] == 0).all()


@pytest.mark.parametrize("H", HS)
@pytest.mark.parametrize("T", (1, 7, 64))
def test_fused_is_post_then_pre_bit_exact(dev, H, T):
    gen = torch.Generator().manual_seed(7 * T + H)
    w = _weights(gen, H)
    rd, xd, pd, cd = (t.to(dev) for t in _inputs(gen, T, H))
    for norm in (False, True):
        args, kw = _dev_args(w, norm, dev)
        f = ops.mhc_fused_post_pre(xd, rd, pd, cd, *args, **kw)
        r = ops.mhc_post(xd, rd, pd, cd)
        p = ops.mhc_pre(r, *args, **kw)
        for a, b in zip(f, (r, *p)):
            assert torch.equal(a, b)


@pytest.mark.parametrize("H", (4096, 7168))
def test_batch_invariance(dev, H):
    """A token's outputs are the same bits alone, in batches of 16 and 64, and at any position in a batch of 256."""
    gen = torch.Generator().manual_seed(H)
    w = _weights(gen, H)
    args, kw = _dev_args(w, True, dev)
    rd, xd, pd, cd = (t.to(dev) for t in _inputs(gen, 256, H))

    def run(idx):
        return ops.mhc_fused_post_pre(xd[idx], rd[idx], pd[idx], cd[idx], *args, **kw)

    full = run(torch.arange(256, device=dev))
    for n in (1, 16, 64):
        for start in (0, 3, 256 - n):
            idx = torch.arange(start, start + n, device=dev)
            part = run(idx)
            for a, b in zip(part, full):
                assert torch.equal(a, b[idx])
    perm = torch.randperm(256, generator=gen).to(dev)
    for a, b in zip(run(perm), full):
        assert torch.equal(a, b[perm])
    hd = ops.hc_head(rd, w["head_fn"].to(dev), w["head_scale"].to(dev), w["head_base"].to(dev), EPS, EPS)
    one = ops.hc_head(rd[37:38], w["head_fn"].to(dev), w["head_scale"].to(dev), w["head_base"].to(dev), EPS, EPS)
    assert torch.equal(one, hd[37:38])


def test_deterministic_and_graph_replay(dev):
    H, T = 7168, 64
    gen = torch.Generator().manual_seed(5)
    w = _weights(gen, H)
    args, kw = _dev_args(w, True, dev)
    res, x, plm, crm = _inputs(gen, T, H)
    bufs = [t.to(dev) for t in (x, res, plm, crm)]
    eager = ops.mhc_fused_post_pre(*bufs, *args, **kw)
    for _ in range(3):
        again = ops.mhc_fused_post_pre(*bufs, *args, **kw)
        assert all(torch.equal(a, b) for a, b in zip(again, eager))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.mhc_fused_post_pre(*bufs, *args, **kw)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.mhc_fused_post_pre(*bufs, *args, **kw)
    res, x, plm, crm = _inputs(gen, T, H, pad=(3,))
    for b, n in zip(bufs, (x, res, plm, crm)):
        b.copy_(n.to(dev))
    g.replay()
    ref = ops.mhc_fused_post_pre(*bufs, *args, **kw)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(out, ref))
    assert not torch.equal(out[3], eager[3])


def test_empty_batch(dev):
    w = _weights(torch.Generator().manual_seed(0), 1280)
    args, kw = _dev_args(w, True, dev)
    r = torch.empty(0, 4, 1280, dtype=torch.bfloat16, device=dev)
    pm, cm, li = ops.mhc_pre(r, *args, **kw)
    assert pm.shape == (0, 4, 1) and cm.shape == (0, 4, 4) and li.shape == (0, 1280)


@pytest.mark.parametrize("H", HS)
def test_layer_chain(dev, H):
    """mhc_pre (first layer), two fused post + pre calls around stand-in sublayers, then hc_head, against the oracle chain
    fed with the library's own sublayer inputs (so that each step is compared on the same inputs)."""
    T = 16
    gen = torch.Generator().manual_seed(H + 1)
    ws = [_weights(gen, H) for _ in range(3)]
    residual = torch.randn(T, 4, H, generator=gen).bfloat16()
    residual[5] = 0
    mats = [torch.randn(H, H, generator=gen) / H ** 0.5 for _ in range(2)]
    args0, kw0 = _dev_args(ws[0], True, dev)
    r = residual.to(dev)
    pm, cm, li = ops.mhc_pre(r, *args0, **kw0)
    _check_pre((pm, cm, li), residual, ws[0], True)
    for k in range(2):
        x = (li.float() @ mats[k].to(dev)).bfloat16()       # stand-in sublayer
        args, kw = _dev_args(ws[k + 1], True, dev)
        r_prev = r
        r, pm_n, cm_n, li = ops.mhc_fused_post_pre(x, r, pm, cm, *args, **kw)
        ref_r, slack = M.post(x.cpu(), r_prev.cpu(), pm.cpu(), cm.cpu(), with_slack=True)
        assert M.bf16_close(r.cpu(), ref_r, slack, 1)
        _check_pre((pm_n, cm_n, li), r.cpu(), ws[k + 1], True)
        pm, cm = pm_n, cm_n
    w = ws[0]
    out = ops.hc_head(r, w["head_fn"].to(dev), w["head_scale"].to(dev), w["head_base"].to(dev), EPS, EPS)
    ref, slack = M.hc_head(r.cpu(), w["head_fn"], w["head_scale"], w["head_base"], EPS, EPS, with_slack=True)
    assert M.bf16_close(out.cpu(), ref, slack, 1)
    assert torch.isfinite(out.float()).all()
