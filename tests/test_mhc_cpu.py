"""CPU: the mHC oracle (tests/mhc_oracle.py) against the reference's own functions, stored in tests/golden/golden_mhc.pt —
post within 1 bf16 ulp, post_mix and comb_mix within 1e-6, layer_input and hc_head within 1 ulp (or, where the stream terms
cancel, within the fp32 accumulation bound of mhc_oracle.bf16_close), the normed pre against
the reference's unfused composition (mhc_pre_torch then rms_norm) at the reference test's atol = rtol = 1e-2 — and the C ABI's
refusals of bad arguments."""
import os

import torch

import mhc_oracle as M

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_mhc.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def _args(g, c):
    return (g["fn"], c["hc_scale"], c["hc_base"], g["eps"], g["eps"], g["eps"], g["post_mult"], g["repeat"])


def test_post_matches_reference():
    g = _load()
    for c in g["cases"]:
        out = M.post(c["x"], c["residual"], c["post_layer_mix"], c["comb_res_mix"])
        for ref in (c["post_torch"], c["post_ref"]):
            assert int(M.bf16_ulp_distance(out, ref).max()) <= 1, c["name"]


def test_pre_matches_reference():
    g = _load()
    for c in g["cases"]:
        for src, key in ((c["residual"], "pre_torch"), (c["post_torch"], "pre_torch_on_post"), (c["residual"], "pre_ref")):
            post_mix, comb_mix, layer_input, slack = M.pre(src, *_args(g, c), with_slack=True)
            ref = c[key]
            assert (post_mix - ref[0].double()).abs().max() <= 1e-6, (c["name"], key)
            assert (comb_mix - ref[1].double()).abs().max() <= 1e-6, (c["name"], key)
            assert M.bf16_close(layer_input, ref[2], slack, 1), (c["name"], key)


def test_large_scale_case_exercises_sinkhorn():
    """With hc_scale[2] = 500 the softmax rows are far from uniform and the 20 iterations move the matrix to near doubly
    stochastic; the oracle follows."""
    g = _load()
    c = next(c for c in g["cases"] if c["name"] == "t2_big")
    comb = M.pre(c["residual"], *_args(g, c))[1]
    assert comb.amax() > 0.5 and comb.amin() < 0.05
    assert (comb.sum(-1) - 1).abs().max() < 1e-2 and (comb.sum(-2) - 1).abs().max() < 1e-5


def test_sinkhorn_matches_reference():
    g = _load()
    for c in g["cases"]:
        got = M.sinkhorn(c["sinkhorn_logits"], g["repeat"], g["eps"])
        assert (got - c["sinkhorn"].double()).abs().max() <= 1e-6


def test_padding_row_is_finite_and_zero():
    g = _load()
    c = next(c for c in g["cases"] if c["name"] == "t5_pad")
    post_mix, comb_mix, layer_input = M.pre(c["residual"], *_args(g, c), norm_weight=g["norm_weight"],
                                            norm_eps=g["norm_eps"])
    assert torch.isfinite(post_mix[3]).all() and torch.isfinite(comb_mix[3]).all()
    assert (layer_input[3] == 0).all()
    assert (M.hc_head(c["residual"], g["head_fn"], g["head_scale"], g["head_base"], g["eps"], g["eps"])[3] == 0).all()


def test_normed_pre_matches_reference_composition():
    g = _load()
    for c in g["cases"]:
        li = M.pre(c["residual"], *_args(g, c), norm_weight=g["norm_weight"], norm_eps=g["norm_eps"])[2]
        torch.testing.assert_close(li.float(), c["pre_torch_normed"].float(), atol=1e-2, rtol=1e-2)


def test_hc_head_matches_reference():
    g = _load()
    for c in g["cases"]:
        out, slack = M.hc_head(c["residual"], g["head_fn"], g["head_scale"], g["head_base"], g["eps"], g["eps"],
                               with_slack=True)
        assert M.bf16_close(out, c["hc_head"], slack, 1), c["name"]


def test_c_abi_refuses_bad_arguments():
    """Refusals happen before any launch, so they are checked without a GPU: each call differs from a well-formed one in one
    argument, and the pointers (never dereferenced) are only checked for NULL and alignment."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    P = 1 << 20   # a 16-byte aligned stand-in address

    def post_pre(**kw):
        a = dict(x=P, res=P, plm=P, crm=P, fn=P, sc=P, base=P, w=None, T=2, H=4096, rms=1e-6, pre_eps=1e-6, sk_eps=1e-6,
                 mult=2.0, rep=20, neps=1e-6, ws=P, rout=P, pm=P, cm=P, li=P)
        a.update(kw)
        return lib.b200_mhc_post_pre(None, *a.values())

    def post(**kw):
        a = dict(x=P, res=P, plm=P, crm=P, T=2, H=4096, out=P)
        a.update(kw)
        return lib.b200_mhc_post(None, *a.values())

    def head(**kw):
        a = dict(res=P, fn=P, sc=P, base=P, T=2, H=4096, rms=1e-6, eps=1e-6, ws=P, out=P)
        a.update(kw)
        return lib.b200_hc_head(None, *a.values())

    for bad in (dict(res=None), dict(res=P + 2), dict(x=P + 8), dict(fn=None), dict(fn=P + 4), dict(sc=None),
                dict(base=P + 2), dict(w=P + 2), dict(T=0), dict(T=-1), dict(T=(1 << 20) + 1), dict(H=1000), dict(H=192),
                dict(H=16448), dict(rep=0), dict(rms=-1e-6), dict(pre_eps=-1.0), dict(sk_eps=float("nan")),
                dict(neps=-1e-6), dict(ws=None), dict(ws=P + 4), dict(rout=None), dict(rout=P + 2), dict(pm=None),
                dict(cm=P + 1), dict(li=None), dict(plm=None), dict(x=None), dict(x=None, plm=None, crm=None)):
        assert post_pre(**bad) == -1, bad
    for bad in (dict(x=None), dict(res=P + 2), dict(plm=None), dict(crm=P + 2), dict(out=None), dict(T=0),
                dict(H=1280 + 32), dict(H=128)):
        assert post(**bad) == -1, bad
    for bad in (dict(res=None), dict(fn=P + 8), dict(sc=None), dict(base=P + 1), dict(T=0), dict(H=4100), dict(rms=-1.0),
                dict(eps=-1e-6), dict(ws=None), dict(out=P + 2)):
        assert head(**bad) == -1, bad
    # the supported sizes, and the workspace rule
    for H in (1280, 4096, 7168):
        assert lib.b200_mhc_workspace_bytes(64, H) == 64 * (H // 64) * 25 * 4
