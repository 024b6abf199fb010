"""CPU: the DeepSeek-V4 sparse decode oracle (tests/dsv4_sparse_oracle.py) against the reference's own functions, stored in
tests/golden/golden_dsv4_sparse.pt: the packer's bytes and the reader's rows bit for bit, the decode within the reference
test's tolerance (atol = rtol = 2e-2, tests/kernels/attention/test_rocm_triton_attn_dsv4.py), and the insert's e4m3 and scale
bytes exactly, its rope dims and q within one bf16 ulp (the reference test notes that its fp32 FMA form can round either way)."""
import os

import torch

import dsv4_sparse_oracle as V4

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_dsv4_sparse.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def test_pack_and_read_match_reference_bit_exact():
    p = _load()["pack"]
    cache = V4.pack(p["kv"], p["block_size"], p["slots"], num_blocks=p["cache"].shape[0])
    assert torch.equal(cache, p["cache"])
    rows = torch.stack([V4.read(p["cache"], int(s), p["block_size"]) for s in p["read_slots"]])
    assert torch.equal(rows.float(), p["read_rows"])
    # the clamped (1e-4) block and a block near the e4m3 limit are in the fixture
    rec = lambda s: p["cache"][s // 16].reshape(-1)[16 * 576 + (s % 16) * 8:][:8]   # noqa: E731
    s3, s7 = int(p["slots"][3]), int(p["slots"][7])
    assert int(rec(s3)[1]) == 127 + (-22) and int(rec(s7)[7]) == 0


def test_decode_matches_reference():
    g = _load()
    for c in g["decode"]:
        extra = c["extra_indices"] is not None
        out = V4.decode(c["q"], g["main_cache"], c["swa_indices"], c["swa_lens"], g["scale"], c["attn_sink"],
                        g["extra_cache"] if extra else None, c["extra_indices"], c["extra_lens"])
        torch.testing.assert_close(out.bfloat16().float(), c["out"].float(), atol=2e-2, rtol=2e-2)
        empty = (c["out"].float().abs().amax(dim=(1, 2)) == 0)
        assert torch.equal(out.abs().amax(dim=(1, 2)) == 0, empty) and empty.any() == (c["num_heads"] != 16)


def test_decode_sink_minus_inf_is_no_sink():
    g = _load()
    c = g["decode"][1]
    args = (c["q"], g["main_cache"], c["swa_indices"], c["swa_lens"], g["scale"])
    ext = dict(extra_cache=g["extra_cache"], extra_indices=c["extra_indices"], extra_lens=c["extra_lens"])
    a = V4.decode(*args, attn_sink=torch.full((c["num_heads"],), -float("inf")), **ext)
    assert torch.equal(a, V4.decode(*args, **ext))


def test_insert_matches_reference():
    i = _load()["insert"]
    T, hq, _ = i["q"].shape
    cache = torch.zeros_like(i["cache"])
    q_out = V4.insert(i["q"], i["kv"], torch.arange(T), i["cos_sin_rows"], i["slots"], cache, hq + 3, i["eps"])
    assert torch.equal(q_out[:, hq:], torch.zeros_like(q_out[:, hq:]))
    assert int(V4.bf16_ulp_distance(q_out[:, :hq], i["q_ref"].bfloat16()).max()) <= 1
    bs = i["block_size"]
    for s in i["slots"].tolist():
        if s < 0:
            continue
        got, ref = cache[s // bs].reshape(-1), i["cache"][s // bs].reshape(-1)
        p = s % bs
        assert torch.equal(got[p * 576:p * 576 + 448], ref[p * 576:p * 576 + 448])                  # e4m3 bytes
        assert torch.equal(got[bs * 576 + p * 8:][:8], ref[bs * 576 + p * 8:][:8])                  # scale bytes
        rope = lambda b: b[p * 576 + 448:p * 576 + 576].contiguous().view(torch.bfloat16)   # noqa: E731
        assert int(V4.bf16_ulp_distance(rope(got), rope(ref)).max()) <= 1
    # untouched outside the written rows (slot -1 writes nothing)
    written = torch.zeros_like(cache, dtype=torch.bool)
    for s in i["slots"].tolist():
        if s >= 0:
            blk = written[s // bs].reshape(-1)
            blk[(s % bs) * 576:(s % bs + 1) * 576] = True
            blk[bs * 576 + (s % bs) * 8:][:8] = True
    assert (cache[~written] == 0).all()
    t = [k for k, s in enumerate(i["slots"].tolist()) if s >= 0]
    e = torch.stack([cache[s // bs].reshape(-1)[bs * 576 + (s % bs) * 8:][:7] for s in i["slots"].tolist() if s >= 0])
    assert torch.equal(torch.pow(2.0, e.double() - 127).float(), i["scales"][t])


def test_dequant_all_is_read_of_every_slot():
    g = _load()
    c = g["extra_cache"]
    rows = V4.dequant_all(c)
    assert torch.equal(rows, torch.stack([V4.read(c, s, c.shape[1]) for s in range(c.shape[0] * c.shape[1])]))


def test_c_abi_refuses_bad_arguments():
    """Refusals happen before any launch, so they are checked without a GPU: each call differs from a well-formed one in one
    argument, and the pointers (never dereferenced) are only checked for NULL and alignment."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    P = 1 << 20   # a 16-byte aligned stand-in address

    def dec(**kw):
        a = dict(q=P, T=2, H=64, swa=P, sbs=64, snb=4, sstr=64 * 584, si=P, sk=128, sl=P, ex=None, ebs=0, enb=0, estr=0,
                 ei=None, ek=0, el=None, sink=None, scale=512 ** -0.5,
                 splits=4, ws=P, out=P)
        a.update(kw)
        return lib.b200_dsv4_sparse_decode(None, *a.values())

    def ins(**kw):
        a = dict(q=P, kv=P, pos=P, cs=P, maxpos=4096, slots=P, cache=P, bs=64, nb=4, stride=64 * 584, q_out=P, T=2, H=64,
                 Hp=128, eps=1e-6)
        a.update(kw)
        return lib.b200_dsv4_qnorm_rope_kv_insert(None, *a.values())

    for bad in (dict(q=P + 2), dict(q=None), dict(H=129), dict(T=0), dict(T=65536), dict(sbs=0), dict(sstr=64 * 584 - 16),
                dict(sstr=64 * 584 + 8), dict(swa=P + 8), dict(si=P + 2), dict(sk=0), dict(sl=None), dict(splits=0),
                dict(splits=513), dict(ws=P + 4), dict(out=None), dict(ex=P, ebs=16, enb=8, estr=16 * 584, ei=P, ek=0, el=P),
                dict(ex=P, ebs=16, enb=8, estr=16 * 584, ei=None, ek=64, el=P), dict(sink=P + 1)):
        assert dec(**bad) == -1, bad
    for bad in (dict(q=P + 2), dict(kv=None), dict(cache=P + 4), dict(stride=64 * 584 - 16), dict(Hp=63), dict(H=0),
                dict(maxpos=0), dict(slots=None), dict(q_out=P + 8), dict(eps=-1.0)):
        assert ins(**bad) == -1, bad
