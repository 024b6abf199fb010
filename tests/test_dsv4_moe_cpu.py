"""CPU: DeepSeek-V4 MoE routing and the clamped SwiGLU.  The float32 oracle (tests/dsv4_moe_oracle.py) against the
reference's own functions stored in tests/golden/golden_dsv4_moe.pt (equal id sets, weights within 1e-6 relative, the
activation bit for bit), the C ABI's refusals of bad arguments, lk_moe.MOEConfigV2's mapping of an assigned swiglu_limit
to activation_type 3, and the Router's argument checks."""
import ctypes
import os

import numpy as np
import pytest
import torch

import dsv4_moe_oracle as D

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_dsv4_moe.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def _check_rows(w, ids, ref_w, ref_ids, rows):
    for t in rows:
        assert set(ids[t].tolist()) == set(ref_ids[t].tolist()), t
        # compare weight by expert id: tied scores may come out in another order
        mine = dict(zip(ids[t].tolist(), w[t].tolist()))
        for e, rw in zip(ref_ids[t].tolist(), ref_w[t].tolist()):
            assert abs(mine[e] - rw) <= 1e-6 * abs(rw) + 1e-30, (t, e, mine[e], rw)


def test_topk_matches_reference():
    g = _load()
    assert {c["E"] for c in g["topk"]} == {256, 384}
    for c in g["topk"]:
        w, ids = D.topk_sqrtsoftplus(c["logits"], g["k"], c["renorm"], c["bias"], g["rsf"])
        rows = [t for t in range(g["M"]) if not torch.isnan(c["logits"][t]).any()]
        for key in ("test", "torch"):
            _check_rows(w, ids, c[f"{key}_w"], c[f"{key}_ids"], rows)


def test_v4flash_bias_selects_but_does_not_weight():
    """With biases all about 8.08 the selection follows score + bias, and the weights are still the unbiased scores:
    weighting by the biased values would flatten them towards 1/k."""
    g = _load()
    c = next(c for c in g["topk"] if c["bias_kind"] == "v4flash")
    w, ids = D.topk_sqrtsoftplus(c["logits"], g["k"], True, c["bias"], g["rsf"])
    s = D.sqrt_softplus(c["logits"].numpy())
    t = 0
    raw = s[t, ids[t].numpy()]
    np.testing.assert_allclose(w[t].numpy(), raw / raw.sum() * g["rsf"], rtol=1e-6)
    assert w[t].max() / w[t].min() > 1.5


def test_nan_rows_become_zero_scores():
    """A non-finite score counts as 0 (the reference's torch paths propagate NaN instead): an all-NaN row selects the
    experts with the largest bias, with weight 0."""
    g = _load()
    for c in g["topk"]:
        if not torch.isnan(c["logits"]).any():
            continue
        w, ids = D.topk_sqrtsoftplus(c["logits"], g["k"], c["renorm"], c["bias"], g["rsf"])
        for t in g["nan_rows"]:
            assert torch.isnan(c["torch_w"][t]).all()
            assert set(ids[t].tolist()) == set(torch.topk(c["bias"], g["k"]).indices.tolist())
            assert (w[t] == 0).all()


def test_hash_matches_reference():
    g = _load()
    for c in g["hash"]:
        w, ids = D.topk_sqrtsoftplus(c["logits"], g["k"], c["renorm"], None, g["rsf"], c["input_ids"], g["hash_table"])
        assert torch.equal(ids, g["hash_table"][c["input_ids"].long()])   # table order
        for key in ("test", "torch"):
            assert torch.equal(ids, c[f"{key}_ids"].int())
            torch.testing.assert_close(w, c[f"{key}_w"], rtol=1e-6, atol=0)


def test_hash_out_of_range_gives_minus_one():
    g = _load()
    c = g["hash"][0]
    ids_in = c["input_ids"].clone()
    ids_in[0], ids_in[1] = -1, g["vocab"]
    table = g["hash_table"].clone()
    table[ids_in[2], 1] = 256
    table[ids_in[2], 4] = -5
    w, ids = D.topk_sqrtsoftplus(c["logits"], g["k"], True, None, g["rsf"], ids_in, table)
    assert (ids[:2] == -1).all() and (w[:2] == 0).all()
    assert ids[2, 1] == -1 and ids[2, 4] == -1 and w[2, 1] == 0 and w[2, 4] == 0
    assert torch.isclose(w[2].sum(), torch.tensor(g["rsf"]), rtol=1e-6)


def test_clamped_activation_matches_reference():
    a = _load()["act"]
    x = a["x"]
    d = x.shape[1] // 2
    assert (x[:, :d] > a["limit"]).float().mean() > 0.1 and (x[:, d:].abs() > a["limit"]).float().mean() > 0.1
    out = D.silu_clamp(x, a["limit"])
    assert torch.equal(out, a["forward_native"])
    torch.testing.assert_close(out, a["swiglu_limit_torch"], rtol=1e-6, atol=1e-6)


def test_clamped_activation_reaches_expert_oracles():
    from oracle import moe_oracle as O
    h = torch.linspace(-30, 30, 64).reshape(1, 64)
    with D.clamped_activation(10.0):
        assert torch.equal(O.apply_activation(h, 3), D.silu_clamp(h, 10.0))
        assert torch.equal(O.apply_activation(h, 0), torch.nn.functional.silu(h[:, :32]) * h[:, 32:])
    with pytest.raises(ValueError):
        O.apply_activation(h, 3)


# ---------------------------------------------------------------------------------------------- C ABI refusals
P = 1 << 20   # a 16-byte aligned stand-in address; refusals happen before any pointer is dereferenced


def test_routing_refusals():
    from lvllm_b200 import _lib as L
    lib = L.lib()

    def gating(scoring):
        return lib.b200_topk_gating(None, P, 0, None, 4, 256, 6, scoring, 1, 1.5, P, P, None)

    assert gating(3) == L.lib().b200_topk_gating(None, P, 0, None, 4, 256, 6, -1, 1, 1.5, P, P, None) != 0
    assert b"scoring" in lib.b200moe_last_error()

    def hash_topk(**kw):
        a = dict(lg=P, dt=0, ids=P, tab=P, vocab=64, M=4, E=256, k=6, renorm=1, rsf=1.5, w=P, out=P)
        a.update(kw)
        return lib.b200_hash_topk(None, *a.values())

    for kw in (dict(tab=None), dict(ids=None), dict(vocab=0), dict(vocab=-3), dict(k=33, E=512), dict(k=0)):
        assert hash_topk(**kw) != 0, kw

    def router(fn, **kw):
        a = dict(h=P, dt=0, wg=P, M=4, E=256, H=4096, bias=None, mode=3, scoring=0, k=6, renorm=1, ng=0, tg=0, rsf=1.5,
                 emap=None, ns=0, slb=-1, sw=1.0, ws=P, wsb=1 << 30, w=P, ids=P, loc=None, lg=None)
        extra = dict(inp=kw.pop("inp", P), tab=kw.pop("tab", P), vocab=kw.pop("vocab", 64))
        a.update(kw)
        if fn == "hash":
            return lib.b200_router_hash_topk(None, *a.values(), *extra.values())
        return lib.b200_router_topk(None, *a.values())

    assert router("topk", mode=4) != 0 and router("topk", mode=-1) != 0
    for kw in (dict(tab=None), dict(inp=None), dict(vocab=0), dict(mode=1), dict(mode=4), dict(k=33)):
        assert router("hash", **kw) != 0, kw


def _cfg(act, limit=None):
    from lvllm_b200 import _lib as L
    c = L.B200Config()
    c.expert_num, c.top_k, c.hidden_size, c.intermediate_size = 8, 2, 512, 256
    c.has_gate_proj, c.activation_type = 1, act
    if limit is not None:
        c.swiglu_limit = limit
    return c


@pytest.mark.parametrize("act,limit", [(4, 7.0), (-1, 7.0), (3, 0.0), (3, -1.0), (3, float("nan"))])
def test_create_refuses_bad_activation(act, limit):
    from lvllm_b200 import _lib as L
    h = ctypes.c_void_p()
    c = _cfg(act, limit)
    assert L.lib().b200moe_create_empty(ctypes.byref(c), L.FMT_16BIT, L.ACT_BF16, ctypes.byref(h)) != 0
    assert b"activation_type" in L.lib().b200moe_last_error()
    assert not h.value


# ---------------------------------------------------------------------------------------------- Python surface
def test_config_maps_assigned_limit_to_clamp():
    import lk_moe
    c = lk_moe.MOEConfigV2()
    assert c._to_c().activation_type == 0   # the default 7.0 alone changes nothing
    c.swiglu_limit = 10.0
    cc = c._to_c()
    assert cc.activation_type == 3 and cc.swiglu_limit == 10.0
    c2 = lk_moe.MOEConfigV2()
    c2.activation_type = 1
    c2.swiglu_limit = 7.0
    assert c2._to_c().activation_type == 1
    c3 = lk_moe.MOEConfigV2()
    c3.activation_type = 2
    c3.has_gate_proj = False
    c3.swiglu_limit = 10.0
    assert c3._to_c().activation_type == 2


def test_router_validation():
    from lvllm_b200 import router as R
    table = torch.zeros(64, 6, dtype=torch.int64)
    with pytest.raises(ValueError):
        R.Router(6, 256, scoring_func="sqrtsoftplus", num_expert_group=8, topk_group=4)
    with pytest.raises(ValueError):
        R.Router(6, 256, scoring_func="softmax", hash_indices_table=table)
    with pytest.raises(ValueError):
        R.Router(6, 256, scoring_func="sqrtsoftplus", hash_indices_table=torch.zeros(64, 5, dtype=torch.int32))
    r = R.Router(6, 256, scoring_func="sqrtsoftplus", hash_indices_table=table)
    assert r.hash_indices_table.dtype == torch.int32
    with pytest.raises(ValueError, match="input_ids"):
        r.select_experts(torch.zeros(1, 64), torch.zeros(1, 256))
    with pytest.raises(ValueError, match="input_ids"):
        r.select_experts(torch.zeros(1, 64), gate_weight=torch.zeros(256, 64))
    R.Router(6, 256, scoring_func="sqrtsoftplus", e_score_correction_bias=torch.zeros(256))
