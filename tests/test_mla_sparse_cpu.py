"""CPU: the sparse MLA decode oracle (tests/mla_sparse_oracle.py) against the reference.

The index conversion matches the reference's _triton_convert_reference_impl bit for bit and the attention its sparse SDPA,
both stored in tests/golden/golden_mla_sparse.pt; the fp8_ds_mla row layout is the one flashmla_sparse.py:63-72 documents."""
import math
import os

import torch

import mla_sparse_oracle as SP

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_mla_sparse.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def attention_inputs(g, c):
    """(q_nope, q_pe, kv_cache [1, S, 576], topk_indices, req_id, page_table) of a fixture case: the request's S keys as
    one page, so request-local positions are cache rows."""
    T, hq = c["topk_indices"].shape[0], c["num_heads"]
    q = g["q_pool"][:c["q_rows"]].reshape(T, hq, 576)
    kv = g["keys"][:c["kv_len"]][None].contiguous()
    return (q[..., :512].contiguous(), q[..., 512:].contiguous(), kv, c["topk_indices"],
            torch.zeros(T, dtype=torch.int32), torch.zeros(1, 1, dtype=torch.int32))


def test_conversion_matches_reference_bit_exact():
    g = _load()
    for c in g["conversion"]:
        got = SP.convert(c["req_id"], c["block_table"], c["indices"], c["page"])
        assert got.dtype == torch.int32
        assert torch.equal(got, c["slots"])
        assert (got == -1).sum() > 0 and (c["indices"] >= c["page"] * c["block_table"].shape[1]).any()


def test_oracle_matches_reference_golden():
    g = _load()
    for c in g["attention"]:
        qn, qp, kv, idx, rid, pt = attention_inputs(g, c)
        out, lse = SP.mla_decode_sparse(qn, qp, kv, idx, rid, pt, g["scale"])
        torch.testing.assert_close(out[..., g["out_dims"]], c["out"], atol=1e-5, rtol=1e-5)
        out_v = torch.einsum("tnl,nlv->tnv", out, SP.golden_w_uv(c["num_heads"]).float())
        torch.testing.assert_close(out_v, c["out_v"], atol=1e-4, rtol=1e-5)
        assert torch.isfinite(lse).all()


def test_oracle_all_invalid_token():
    qn, qp = torch.randn(1, 4, 512), torch.randn(1, 4, 64)
    kv = torch.randn(2, 16, 576).bfloat16()
    out, lse = SP.mla_decode_sparse(qn, qp, kv, torch.tensor([[-1, 40, -1]], dtype=torch.int32),
                                    torch.zeros(1, dtype=torch.int32), torch.tensor([[1, 0]], dtype=torch.int32), 0.1)
    assert torch.equal(out, torch.zeros_like(out)) and (lse == -math.inf).all()


def test_ds_mla_row_layout():
    """A hand-built 656-byte row: bytes 0-511 e4m3 (one scale per 128), 512-527 four fp32 scales, 528-655 64 bf16 rope."""
    vals = torch.tensor([1.0, -2.0, 0.5, 448.0, -0.015625, 3.0, 0.0, 7.5])
    e4 = vals.repeat(64).to(torch.float8_e4m3fn)                       # 512 values
    scales = torch.tensor([0.25, 2.0, 1.0, 0.125])
    rope = torch.linspace(-4, 4, 64).bfloat16()
    row = torch.zeros(656, dtype=torch.uint8)
    row[:512] = e4.view(torch.uint8)
    row[512:528] = scales.view(torch.uint8)
    row[528:] = rope.view(torch.uint8)
    assert row[512:516].view(torch.float32).item() == 0.25 and row[524:528].view(torch.float32).item() == 0.125
    dq = SP.ds_mla_dequantize(row[None])[0]
    assert dq.dtype == torch.bfloat16 and dq.shape == (576,)
    want = (vals.repeat(64).reshape(4, 128) * scales[:, None]).reshape(512).bfloat16()
    assert torch.equal(dq[:512], want)
    assert torch.equal(dq[512:], rope)


def test_ds_mla_quantize_layout_and_round_trip():
    gen = torch.Generator().manual_seed(1)
    kv_c = (torch.randn(33, 512, generator=gen) * torch.tensor([0.01, 1.0, 30.0, 0.0]).repeat_interleave(128)).bfloat16()
    k_pe = torch.randn(33, 64, generator=gen).bfloat16()
    rows = SP.ds_mla_quantize(kv_c, k_pe)
    assert rows.dtype == torch.uint8 and rows.shape == (33, 656)
    scale = rows[:, 512:528].contiguous().view(torch.float32)
    amax = kv_c.float().reshape(33, 4, 128).abs().amax(-1)
    assert torch.equal(scale, torch.clamp(amax / 448.0, min=torch.finfo(torch.float32).tiny))
    assert torch.equal(rows[:, 528:].contiguous().view(torch.bfloat16), k_pe)
    dq = SP.ds_mla_dequantize(rows)
    assert torch.equal(dq[:, 384:512], torch.zeros(33, 128, dtype=torch.bfloat16))     # the all-zero tile
    # e4m3 keeps 3 mantissa bits: relative error <= 2^-4 on normals, absolute <= 2^-10 * scale on subnormals,
    # plus the bf16 rounding of the product
    err = (dq[:, :512].float() - kv_c.float()).abs()
    bound = kv_c.float().abs() * (2 ** -4 + 2 ** -8) + scale.repeat_interleave(128, dim=1) * 2 ** -9
    assert (err <= bound).all()
