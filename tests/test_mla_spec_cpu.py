"""CPU: the multi-token MLA decode oracle (tests/mla_spec_oracle.py) against the reference.

With q_len = Q it matches the reference's causal attention (scaled_dot_product_attention(..., is_causal=True) of
tests/kernels/attention/test_flashmla.py:138-155) stored in tests/golden/golden_mla_spec.pt; with q_len = 1 it is the
oracle's single-token decode bit for bit; the fixture's generator reproduces it where the reference tree is present."""
import math
import os
import subprocess
import sys

import pytest
import torch

import mla_spec_oracle as SO
from oracle import moe_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_mla_spec.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def case_inputs(g, c):
    """(q_nope, q_pe, seq_lens) of a fixture case: its queries are the first rows of the fixture's query pool."""
    Q, B, hq = c["q_len"], len(c["kv_lens"]), c["num_heads"]
    q = g["q_pool"][:c["q_rows"]].reshape(B * Q, hq, 576)
    return q[..., :512].contiguous(), q[..., 512:].contiguous(), torch.tensor(c["kv_lens"], dtype=torch.int32)


def test_oracle_matches_reference_golden():
    g = _load()
    seen = set()
    for c in g["cases"]:
        Q, B, hq = c["q_len"], len(c["kv_lens"]), c["num_heads"]
        qn, qp, lens = case_inputs(g, c)
        out, lse = SO.mla_decode(qn.float(), qp.float(), g["kv_cache"].float(), lens, c["block_tables"], g["scale"], q_len=Q)
        assert out.shape == (B * Q, hq, 512) and lse.shape == (B * Q, hq)
        torch.testing.assert_close(out[..., g["out_dims"]], c["out"], atol=1e-5, rtol=1e-5)
        torch.testing.assert_close(lse, c["lse"], atol=1e-5, rtol=1e-5)
        assert torch.isfinite(lse).all()
        seen.add((hq, Q))
        assert min(c["kv_lens"]) >= Q   # every row sees a key (the reference gives NaN otherwise)
    # the head counts and draft lengths the fixture is meant to cover, and its edge cases
    assert {(128, 2), (16, 4), (16, 8), (64, 3), (20, 3)} <= seen
    assert any(c["q_len"] in c["kv_lens"] for c in g["cases"])
    assert any(c["q_len"] == 4 and 129 in c["kv_lens"] for c in g["cases"])
    # the stored value dims reach every 128-dim quarter (one CTA part each) and every 64-dim block of V
    assert set((g["out_dims"] // 64).tolist()) == set(range(8))
    assert os.path.getsize(GOLDEN) < 1 << 20


def test_q_len_1_is_the_single_token_oracle():
    gen = torch.Generator().manual_seed(4)
    B, hq, page = 3, 16, 16
    cache = torch.randn(8, page, 576, generator=gen).bfloat16()
    pt = torch.randperm(8, generator=gen)[:6].reshape(B, 2).int()
    lens = torch.tensor([1, 17, 32], dtype=torch.int32)
    qn, qp = torch.randn(B, hq, 512, generator=gen).bfloat16(), torch.randn(B, hq, 64, generator=gen).bfloat16()
    out1, lse1 = SO.mla_decode(qn, qp, cache, lens, pt, 0.05, q_len=1)
    out0, lse0 = O.mla_decode(qn, qp, cache, lens, pt, 0.05)
    assert torch.equal(out1, out0) and torch.equal(lse1, lse0)


def test_rows_without_a_visible_key():
    """S_b < Q: the first Q - S_b rows of request b see no key: out 0, lse -inf; the rest are ordinary rows."""
    gen = torch.Generator().manual_seed(2)
    Q, hq = 4, 8
    cache = torch.randn(2, 16, 576, generator=gen)
    qn, qp = torch.randn(2 * Q, hq, 512, generator=gen), torch.randn(2 * Q, hq, 64, generator=gen)
    lens = torch.tensor([2, 20], dtype=torch.int32)
    pt = torch.tensor([[1, 0], [0, 1]], dtype=torch.int32)
    scale = 1 / math.sqrt(576)
    out, lse = SO.mla_decode(qn, qp, cache, lens, pt, scale, q_len=Q)
    assert torch.equal(out[:2], torch.zeros(2, hq, 512)) and (lse[:2] == -math.inf).all()
    assert torch.isfinite(lse[2:]).all() and not torch.isnan(out).any()
    ref, ref_lse = O.mla_decode(qn[2:3], qp[2:3], cache, torch.tensor([1], dtype=torch.int32), pt[:1], scale)
    assert torch.equal(out[2:3], ref) and torch.equal(lse[2:3], ref_lse)


def _reference_dir():
    d = os.environ.get("LVLLM_REFERENCE_DIR", "/root/reference")
    return d if os.path.isfile(os.path.join(d, "tests", "kernels", "attention", "test_flashmla.py")) else None


@pytest.mark.skipif(_reference_dir() is None, reason="needs the reference tree (LVLLM_REFERENCE_DIR)")
def test_make_golden_mla_spec_reproduces_the_fixture(tmp_path):
    out = tmp_path / "golden_mla_spec.pt"
    env = dict(os.environ, PYTHONPATH=_reference_dir())
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_golden_mla_spec.py"), str(out)],
                       cwd=str(tmp_path), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    a, b = torch.load(str(out), weights_only=True), _load()
    assert a.keys() == b.keys() and len(a["cases"]) == len(b["cases"])
    for key in ("page_size", "scale"):
        assert a[key] == b[key], key
    for key in ("kv_cache", "q_pool", "out_dims"):
        assert torch.equal(a[key], b[key]), key
    for ca, cb in zip(a["cases"], b["cases"]):
        assert ca.keys() == cb.keys()
        for key in ca:
            if isinstance(ca[key], torch.Tensor):
                assert torch.equal(ca[key], cb[key]), key
            else:
                assert ca[key] == cb[key], key
