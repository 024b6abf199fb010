"""CPU: the GQA attention-block oracle (tests/gqa_oracle.py) against the reference.

qk_norm_rope is pinned bit for bit to tests/golden/golden_gqa.pt (the reference's own RMSNorm / RotaryEmbedding, composed as
its fused_qk_norm_rope test does); reshape_and_cache_flash is checked on the FlashInfer backend's packed NHD and HND caches
against the rows the reference's cache test expects."""
import os
import subprocess
import sys

import pytest
import torch

import gqa_oracle as GO

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_gqa.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def cos_sin_table(g, c):
    """The reference's cos | sin table at the rows the case uses (the fixture stores only those rows)."""
    t = torch.zeros(g["max_position"], c["rotary_dim"], dtype=torch.bfloat16)
    t[c["positions"]] = c["cos_sin_rows"]
    return t


def test_qk_norm_rope_matches_reference_golden():
    g = _load()
    D = g["head_dim"]
    seen = set()
    for c in g["cases"]:
        hq, hkv, T = c["num_heads"], c["num_kv_heads"], c["tokens"]
        qkv = g["qkv"][c["heads"]][:T]
        out = GO.qk_norm_rope(qkv, c["positions"], cos_sin_table(g, c), hq, hkv, D, c["rotary_dim"], c["q_weight"],
                              c["k_weight"], c["eps"], c["is_neox"])
        q, k, v = out.split([hq * D, hkv * D, hkv * D], dim=-1)
        assert torch.equal(q.reshape(T, hq, D), c["q_out"]), c
        assert torch.equal(k.reshape(T, hkv, D), c["k_out"]), c
        assert torch.equal(v, qkv[:, (hq + hkv) * D:])
        seen.add((c["is_neox"], c["rotary_dim"], c["norm"], c["eps"]))
    assert {r for _, r, _, _ in seen} == {128, 64, 32} and {n for *_, n, _ in seen} == {True, False}
    assert any(int(c["positions"].max()) >= 20000 for c in g["cases"])


def _packed(layout, blocks, page, hkv, D, fill):
    """The FlashInfer backend's per-layer cache (flashinfer.py:398-433) and its K / V views (:2276-2290)."""
    if layout == "NHD":
        phys = fill((blocks, page, hkv, 2 * D))
        logical = phys.permute(0, 2, 1, 3)            # (blocks, Hkv, page, 2D), stride order (0, 2, 1, 3)
    else:
        phys = fill((blocks, hkv, page, 2 * D))
        logical = phys
    k, v = logical.transpose(1, 2).split(D, dim=-1)
    return phys, k, v


@pytest.mark.parametrize("layout", ["NHD", "HND"])
def test_reshape_and_cache_flash_writes_the_reference_rows(layout):
    gen = torch.Generator().manual_seed(1)
    T, blocks, page, hkv, D = 6, 5, 16, 4, 128
    phys, kc, vc = _packed(layout, blocks, page, hkv, D, lambda s: torch.randn(*s, generator=gen).bfloat16())
    before = phys.clone()
    key = torch.randn(T, hkv, D, generator=gen).bfloat16()
    value = torch.randn(T, hkv, D, generator=gen).bfloat16()
    slots = torch.tensor([3, 17, -1, 79, 40, 0], dtype=torch.int64)
    GO.reshape_and_cache_flash(key, value, kc, vc, slots)
    # expected: tests/kernels/attention/test_cache.py:406-414 on the physical layout, K in [..., :D], V in [..., D:]
    exp = before.clone()
    for i in range(T):
        s = int(slots[i])
        if s < 0:
            continue
        b, o = s // page, s % page
        if layout == "NHD":
            exp[b, o, :, :D], exp[b, o, :, D:] = key[i], value[i]
        else:
            exp[b, :, o, :D], exp[b, :, o, D:] = key[i], value[i]
    assert torch.equal(phys.view(torch.int16), exp.view(torch.int16))
    written = sum(int(s) >= 0 for s in slots)
    assert int((phys.view(torch.int16) != before.view(torch.int16)).sum()) <= written * hkv * 2 * D


def _reference_dir():
    d = os.environ.get("LVLLM_REFERENCE_DIR", "/root/reference")
    return d if os.path.isdir(os.path.join(d, "vllm", "model_executor")) else None


@pytest.mark.skipif(_reference_dir() is None, reason="needs the reference tree (LVLLM_REFERENCE_DIR)")
def test_make_golden_gqa_reproduces_the_fixture(tmp_path):
    out = tmp_path / "golden_gqa.pt"
    env = dict(os.environ, PYTHONPATH=_reference_dir())
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_golden_gqa.py"), str(out)], cwd=str(tmp_path),
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    a, b = torch.load(str(out), weights_only=True), _load()
    assert a["max_position"] == b["max_position"] and len(a["cases"]) == len(b["cases"])
    for x, y in zip(a["qkv"], b["qkv"]):
        assert torch.equal(x, y)
    for ca, cb in zip(a["cases"], b["cases"]):
        assert ca.keys() == cb.keys()
        for key in ca:
            if isinstance(ca[key], torch.Tensor):
                assert torch.equal(ca[key], cb[key]), key
            else:
                assert ca[key] == cb[key], key
