"""CPU: the multi-token GQA decode oracle (tests/gqa_spec_oracle.py) against the reference.

With q_len = Q it matches the reference's ref_paged_attn (query_lens = [Q] * B, end-aligned causal mask) stored in
tests/golden/golden_gqa_spec.pt; with q_len = 1 it is the oracle's single-token decode bit for bit; the fixture's generator
reproduces it where the reference tree is present."""
import math
import os
import subprocess
import sys

import pytest
import torch

import gqa_spec_oracle as SO
from oracle import moe_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_gqa_spec.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def test_oracle_matches_reference_golden():
    g = _load()
    seen = set()
    for c in g["cases"]:
        p = g["pools"][c["num_kv_heads"]]
        Q, B = c["q_len"], len(c["kv_lens"])
        out, lse = SO.gqa_decode(c["q"].float(), p["k_cache"].float(), p["v_cache"].float(),
                                 torch.tensor(c["kv_lens"], dtype=torch.int32), c["block_tables"], g["scale"], q_len=Q)
        assert out.shape == (B * Q, c["num_heads"], g["head_dim"]) and lse.shape == (B * Q, c["num_heads"])
        torch.testing.assert_close(out, c["out"], atol=1e-5, rtol=1e-5)
        assert torch.isfinite(lse).all()
        seen.add((c["num_heads"] // c["num_kv_heads"], Q))
        assert min(c["kv_lens"]) >= Q   # every row sees a key (ref_paged_attn gives NaN otherwise)
    # the groups and draft lengths the fixture is meant to cover, and its edge cases
    assert {(4, 2), (4, 4), (16, 3), (1, 5), (48, 2)} <= seen
    assert any(c["q_len"] in c["kv_lens"] for c in g["cases"])
    assert any(c["q_len"] == 4 and 129 in c["kv_lens"] for c in g["cases"])
    assert os.path.getsize(GOLDEN) < 1 << 20


def test_q_len_1_is_the_single_token_oracle(golden):
    c = golden["gqa_decode"]
    lens = torch.tensor(c["kv_lens"])
    out1, lse1 = SO.gqa_decode(c["q"], c["k_cache"], c["v_cache"], lens, c["block_tables"], c["scale"], q_len=1)
    out0, lse0 = O.gqa_decode(c["q"], c["k_cache"], c["v_cache"], lens, c["block_tables"], c["scale"])
    assert torch.equal(out1, out0) and torch.equal(lse1, lse0)


def test_rows_without_a_visible_key():
    """S_b < Q: the first Q - S_b rows of request b see no key: out 0, lse -inf; the rest are ordinary rows."""
    gen = torch.Generator().manual_seed(2)
    Q, hq, hkv, D = 4, 8, 2, 128
    kc, vc = torch.randn(2, 16, hkv, D, generator=gen), torch.randn(2, 16, hkv, D, generator=gen)
    q = torch.randn(2 * Q, hq, D, generator=gen)
    lens = torch.tensor([2, 20], dtype=torch.int32)
    pt = torch.tensor([[1, 0], [0, 1]], dtype=torch.int32)
    out, lse = SO.gqa_decode(q, kc, vc, lens, pt, D ** -0.5, q_len=Q)
    assert torch.equal(out[:2], torch.zeros(2, hq, D)) and (lse[:2] == -math.inf).all()
    assert torch.isfinite(lse[2:]).all() and not torch.isnan(out).any()
    ref, ref_lse = O.gqa_decode(q[2:3], kc, vc, torch.tensor([1], dtype=torch.int32), pt[:1], D ** -0.5)
    assert torch.equal(out[2:3], ref) and torch.equal(lse[2:3], ref_lse)


def _reference_dir():
    d = os.environ.get("LVLLM_REFERENCE_DIR", "/root/reference")
    return d if os.path.isdir(os.path.join(d, "vllm", "model_executor")) else None


@pytest.mark.skipif(_reference_dir() is None, reason="needs the reference tree (LVLLM_REFERENCE_DIR)")
def test_make_golden_gqa_spec_reproduces_the_fixture(tmp_path):
    out = tmp_path / "golden_gqa_spec.pt"
    env = dict(os.environ, PYTHONPATH=_reference_dir())
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_golden_gqa_spec.py"), str(out)],
                       cwd=str(tmp_path), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    a, b = torch.load(str(out), weights_only=True), _load()
    assert a.keys() == b.keys() and len(a["cases"]) == len(b["cases"])
    for key in ("head_dim", "page_size", "scale"):
        assert a[key] == b[key], key
    assert a["pools"].keys() == b["pools"].keys()
    for h in a["pools"]:
        for key in ("k_cache", "v_cache"):
            assert torch.equal(a["pools"][h][key], b["pools"][h][key]), (h, key)
    for ca, cb in zip(a["cases"], b["cases"]):
        assert ca.keys() == cb.keys()
        for key in ca:
            if isinstance(ca[key], torch.Tensor):
                assert torch.equal(ca[key], cb[key]), key
            else:
                assert ca[key] == cb[key], key
