"""CPU: the lightning-indexer oracle (tests/indexer_oracle.py) against the reference.

The logits match the reference's fp8_paged_mqa_logits_torch (both its branches), the k quantisation its
kv_cache_cast_to_fp8 / per_custom_dims_cast_to_fp8, the top-k torch.topk, all stored in tests/golden/golden_indexer.pt;
plus the cache row layout, the exact ue8m0 ceiling and the top-k rules."""
import math
import os

import torch

import indexer_oracle as IX

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_indexer.pt")
CASES = ("logits_q1", "logits_q2", "logits_q3")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def test_logits_match_reference_golden():
    g = _load()
    for name in CASES:
        c = g[name]
        ref = c["logits"]
        got = IX.paged_logits(c["q_fp8"].view(torch.float8_e4m3fn), c["weights"], c["k_cache"], c["seq_lens"],
                              c["page_table"], c["q_len"], ref.shape[1])
        fin = torch.isfinite(ref)
        assert torch.equal(fin, torch.isfinite(got)), name
        # the reference sums in fp32, the oracle in float64 over the same e4m3 values
        torch.testing.assert_close(got[fin].float(), ref[fin], rtol=1e-5, atol=1e-4)
    assert not torch.isfinite(g["logits_q1"]["logits"][0]).any()      # the empty request


def test_topk_matches_reference_golden():
    g = _load()
    k = g["topk"]["k"]
    for name in CASES:
        c = g[name]
        got = IX.topk_rows(c["logits"], c["seq_lens"], c["q_len"], k)
        for r, want in enumerate(g["topk"]["indices"][name]):
            row = got[r][got[r] >= 0]
            assert set(row.tolist()) == set(want.tolist()), (name, r)
            assert torch.equal(row, row.sort().values)


def test_k_quant_matches_reference_casts():
    g = _load()["kquant"]
    k = g["k"]
    v8, sc = IX.k_quant(k, ue8m0=True)
    assert torch.equal(v8.view(torch.uint8), g["ue8m0_values"]) and torch.equal(sc, g["ue8m0_scales"])
    cache = torch.zeros(1, 64, 132, dtype=torch.uint8)
    IX.k_quant_cache(k, torch.arange(64), cache, ue8m0=False)
    ref = g["plain_cache"]
    # the scales bit for bit; the reference test multiplies by 1 / scale where the cache kernel divides, so a value
    # byte may differ by one e4m3 step where the two roundings straddle a rounding boundary
    assert torch.equal(cache.reshape(-1)[64 * 128:], ref.reshape(-1)[64 * 128:])
    a = cache.reshape(-1)[:64 * 128].view(torch.float8_e4m3fn).float()
    b = ref.reshape(-1)[:64 * 128].view(torch.float8_e4m3fn).float()
    diff = a != b
    assert diff.float().mean() < 0.01
    assert ((a - b).abs()[diff] <= b.abs()[diff] * 2 ** -3 + 2 ** -9).all()


def test_ue8m0_ceil_is_the_reference_formula():
    """exp2(ceil(log2(x))) evaluated exactly (float64) on random scales, exact powers of two and their fp32
    neighbours.  In fp32 the formula's log2 can round to an integer just above a power of two (and give a scale below
    x); the bit form never does."""
    gen = torch.Generator().manual_seed(0)
    x = torch.exp2(torch.rand(4096, generator=gen) * 60 - 40)
    p2 = torch.exp2(torch.arange(-40, 21).float())
    up = torch.nextafter(p2, torch.full_like(p2, math.inf))
    down = torch.nextafter(p2, torch.zeros_like(p2))
    for v in (x, p2, up, down):
        want = torch.exp2(torch.ceil(torch.log2(v.double()))).float()
        assert torch.equal(IX.ue8m0_ceil(v), want)
    assert torch.equal(IX.ue8m0_ceil(p2), p2)
    assert (IX.ue8m0_ceil(up) == 2 * p2).all()


def test_cache_row_layout():
    """Block b of a [blocks, 16, 132] cache: 16 x 128 value bytes, then 16 fp32 scales; slot = block * 16 + offset."""
    cache = torch.full((3, 16, 132), 0xAB, dtype=torch.uint8)
    k = torch.zeros(3, 128).bfloat16()
    k[0, 0], k[1, 127], k[2, 5] = 448.0, -2.0, 1.0
    IX.k_quant_cache(k, torch.tensor([17, -1, 47]), cache, ue8m0=False)
    flat = cache.reshape(3, 16 * 132)
    assert flat[1, 128] == torch.tensor([448.0]).to(torch.float8_e4m3fn).view(torch.uint8)[0]   # amax / scale = 448
    assert flat[1, 16 * 128 + 4:16 * 128 + 8].view(torch.float32).item() == 1.0
    assert flat[2, 15 * 128 + 5] == torch.tensor([448.0]).to(torch.float8_e4m3fn).view(torch.uint8)[0]
    assert flat[2, 16 * 128 + 60:16 * 128 + 64].view(torch.float32).item() == torch.tensor(1.0 / 448).item()
    assert (flat[0] == 0xAB).all()                                  # slot -1 wrote nothing
    vals, scales = IX.k_cache_rows(cache)
    assert vals[1, 1, 0] == 448.0 and scales[2, 15] == torch.tensor(1.0 / 448).item()


def test_topk_rules():
    lg = torch.tensor([[3., 1., 3., 5., 3., -math.inf, 2., 3.]])
    # ties at the threshold go to the lowest positions; output ascending
    assert IX.topk_rows(lg, torch.tensor([8]), 1, 3).tolist() == [[0, 2, 3]]
    assert IX.topk_rows(lg, torch.tensor([8]), 1, 5).tolist() == [[0, 2, 3, 4, 7]]
    # row_end <= topk: every position, then -1
    assert IX.topk_rows(lg, torch.tensor([3]), 1, 4).tolist() == [[0, 1, 2, -1]]
    # row_end = 0 (a request shorter than its draft tokens): all -1
    got = IX.topk_rows(lg.repeat(2, 1), torch.tensor([1]), 2, 2)
    assert got.tolist() == [[-1, -1], [0, -1]]
    # distinct values: exactly torch.topk's set
    x = torch.randn(1, 5000, generator=torch.Generator().manual_seed(3))
    got = IX.topk_rows(x, torch.tensor([5000]), 1, 100)[0]
    assert torch.equal(got, torch.topk(x[0], 100).indices.sort().values.int())


def test_q_rope_quant_rules():
    gen = torch.Generator().manual_seed(2)
    q = torch.randn(3, 4, 128, generator=gen).bfloat16()
    w = torch.randn(3, 4, generator=gen).bfloat16()
    cs = torch.randn(10, 64, generator=gen).bfloat16()
    pos = torch.tensor([0, 9, 4])
    for neox in (True, False):
        q8, wo = IX.q_rope_quant(q, w, pos, cs, neox, 128 ** -0.5, 64 ** -0.5)
        x = q8.float()
        # the scale is the power of two at or above amax / 448: the largest byte lands in [224, 448]
        assert (x.abs().amax(-1) >= 224).all() and (x.abs().amax(-1) <= 448).all()
        scale = wo / (w.float() * (128 ** -0.5) * (64 ** -0.5))
        assert torch.allclose(torch.log2(scale), torch.log2(scale).round(), atol=1e-5)
