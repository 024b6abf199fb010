"""CPU: the DeepSeek-V4 indexer oracle (tests/dsv4_indexer_oracle.py) against the reference's own kernels stored in
tests/golden/golden_dsv4_indexer.pt (the q side's bytes and weights, the four key lists, the short-context top-k), and the
C ABI and Python refusals of dsv4_indexer_q_quant, dsv4_indexer_decode and the key-list ops."""
import os

import pytest
import torch

import dsv4_indexer_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_dsv4_indexer.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def test_q_quant_matches_reference():
    g = _load()
    q = g["q"]
    c0, c1 = q["weights_cols"]
    q8, w = O.q_quant(q["q"], q["weights"][:, c0:c1], q["positions"], g["cos_sin"], q["softmax_scale"], q["head_scale"])
    assert torch.equal(q8.view(torch.uint8), q["q_fp8"])
    assert torch.equal(w.view(torch.int32), q["weights_out"].view(torch.int32))
    assert torch.equal(w.view(torch.int32), q["w_interp"].view(torch.int32))
    # head (0, 0): amax 3.5 = 448 * 2^-7 gives scale 2^-7 (the V3.2 kernel's amax * (1 / 448) would give 2^-6)
    scale = w[0, 0] / (q["weights"][0, c0].float() * q["softmax_scale"] * q["head_scale"])
    assert abs(float(scale) / 2 ** -7 - 1) < 1e-6
    assert int(q["q_fp8"][1, 1].sum()) == 0                                  # all-zero head: zero bytes


def test_lists_match_reference():
    L = _load()["lists"]
    pos, sm, req, bt = L["positions"], L["slot_mapping"], L["token_to_req"], L["block_table"]
    v = sm >= 0
    assert not bool(v.all())                                                  # a padded token is in the case
    i, n = O.swa(pos, sm, req, bt, L["swa_block_size"], L["window"])
    assert torch.equal(i[v], L["swa_indices"][v]) and torch.equal(n, L["swa_lens"])
    assert 0 < int(n[0]) < L["window"]                                       # p < W
    i, n = O.c128a(pos, sm, req, bt, L["c_block_size"], L["ratio"], L["width"])
    assert torch.equal(i[v], L["c128a_indices"][v]) and torch.equal(n, L["c128a_lens"])
    assert int(n.max()) == L["width"] < int(O.candidates(pos, L["ratio"]).max())   # width below the count
    i, n = O.global_topk(L["local_topk"], sm, req, bt, L["c_block_size"])
    assert torch.equal(i[v], L["global_indices"][v]) and torch.equal(n, L["global_lens"])
    s = O.slot_mapping(pos, sm, req, bt, L["c_block_size"], L["ratio"])
    assert torch.equal(s, L["kv_slot_mapping"]) and int((s >= 0).sum()) == 2
    assert torch.equal(O.short_context(pos, L["ratio"], L["topk"]), L["short_topk"])
    assert torch.equal(O.topk(torch.zeros(pos.numel(), 64, dtype=torch.float64), pos, L["ratio"], L["topk"]),
                       L["short_topk"])                                       # n_t <= topk: the top-k's own rule


def test_block_column_past_table_is_no_key():
    bt = torch.tensor([[5, 6]], dtype=torch.int32)
    pos = torch.tensor([9])
    one = torch.zeros(1, dtype=torch.long)
    i, n = O.swa(pos, one, one.int(), bt, 4, 4)                               # keys 6..9; 8, 9 in column 2 = width
    assert i.tolist() == [[26, 27, -1, -1]] and n.tolist() == [4]
    assert O.slot_mapping(torch.tensor([11]), one, one.int(), bt, 1, 4).tolist() == [-1]   # row 2, column 2


P = 1 << 20   # a 16-byte aligned stand-in address: refusals happen before anything is dereferenced


def _q_abi(lib, **kw):
    a = dict(q=P, w=P, ws=64, pos=P, cs=P, maxpos=64, ss=0.1, hs=0.1, q8=P, wo=P, T=2, H=64)
    a.update(kw)
    return lib.b200_dsv4_indexer_q_quant(None, *a.values())


def _dec_abi(lib, **kw):
    a = dict(q8=P, w=P, kc=P, nb=4, page=64, pos=P, req=P, bt=P, maxb=8, ratio=4, T=2, H=64, msl=0, lg=P, lgs=512,
             topk=512, out=P)
    a.update(kw)
    return lib.b200_dsv4_indexer_decode(None, *a.values())


def _ix_abi(lib, **kw):
    a = dict(kind=0, pos=P, sm=P, req=P, bt=P, bts=8, maxb=8, bs=64, param=128, loc=None, locs=0, out=P, outs=128,
             width=128, lens=P, T=2)
    a.update(kw)
    return lib.b200_dsv4_indices(None, *a.values())


def test_c_abi_refuses_bad_arguments():
    from lvllm_b200 import _lib as L
    lib = L.lib()
    assert _q_abi(lib, T=0) == 0 and _dec_abi(lib, T=0) == 0
    for bad in (dict(q=None), dict(q=P + 8), dict(w=None), dict(w=P + 1), dict(ws=63), dict(pos=None), dict(pos=P + 4),
                dict(cs=None), dict(cs=P + 2), dict(maxpos=0), dict(q8=P + 4), dict(wo=None), dict(wo=P + 2), dict(T=-1),
                dict(T=(1 << 20) + 1), dict(H=0), dict(H=129)):
        assert _q_abi(lib, **bad) == -1, bad
    assert _q_abi(lib, H=128, ws=128, T=0) == 0
    for bad in (dict(q8=None), dict(q8=P + 4), dict(w=P + 2), dict(kc=None), dict(kc=P + 8), dict(nb=0), dict(page=8),
                dict(page=128), dict(pos=P + 4), dict(req=None), dict(req=P + 2), dict(bt=None), dict(bt=P + 1),
                dict(maxb=0), dict(ratio=2), dict(ratio=0), dict(H=16), dict(H=128), dict(lg=None), dict(lg=P + 2),
                dict(lgs=511), dict(lgs=1 << 31), dict(topk=0), dict(topk=2049), dict(out=None), dict(out=P + 2),
                dict(T=-1), dict(T=(1 << 20) + 1)):
        assert _dec_abi(lib, **bad) == -1, bad
    assert _dec_abi(lib, page=16, H=32, ratio=128, lgs=128, topk=1, T=0) == 0
    for ok in (dict(), dict(kind=1, param=4), dict(kind=1, param=128), dict(kind=2, param=0, loc=P, locs=128),
               dict(kind=2, pos=None, loc=P, locs=128),
               dict(kind=3, param=4, lens=None, width=0, outs=0)):
        assert _ix_abi(lib, **ok, T=0) == 0, ok
    for bad in (dict(kind=-1), dict(kind=4), dict(pos=None), dict(pos=P + 4), dict(sm=P + 4), dict(req=None),
                dict(req=P + 2), dict(bt=P + 2), dict(bts=7), dict(maxb=0), dict(bs=0), dict(T=-1), dict(T=(1 << 20) + 1),
                dict(out=None), dict(out=P + 2), dict(lens=None), dict(lens=P + 2), dict(width=0), dict(outs=127),
                dict(width=(1 << 20) + 1, outs=1 << 21), dict(param=0), dict(param=129), dict(kind=1, param=8),
                dict(kind=2, loc=None, locs=128), dict(kind=2, loc=P + 2, locs=128), dict(kind=2, loc=P, locs=127),
                dict(kind=3, param=2), dict(kind=3, out=P + 4)):
        assert _ix_abi(lib, **bad) == -1, bad


def test_python_refusals():
    """The ops check dtypes and shapes before anything touches a device; well-formed calls on CPU tensors stop at the
    CUDA check."""
    from lvllm_b200 import ops
    T, H = 3, 64
    qa = dict(q=torch.zeros(T, H, 128, dtype=torch.bfloat16), weights=torch.zeros(T, H, dtype=torch.bfloat16),
              positions=torch.zeros(T, dtype=torch.long), cos_sin_cache=torch.zeros(16, 64), softmax_scale=0.1,
              head_scale=0.1)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_indexer_q_quant(**qa)
    da = dict(q_fp8=torch.zeros(T, H, 128, dtype=torch.float8_e4m3fn), weights=torch.zeros(T, H),
              k_cache=torch.zeros(4, 64, 132, dtype=torch.uint8), positions=torch.zeros(T, dtype=torch.long),
              token_to_req=torch.zeros(T, dtype=torch.int32), block_table=torch.zeros(2, 4, dtype=torch.int32),
              compress_ratio=4, topk=512)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_indexer_decode(**da)
    la = dict(positions=torch.zeros(T, dtype=torch.long), slot_mapping=torch.zeros(T, dtype=torch.long),
              token_to_req=torch.zeros(T, dtype=torch.int32), block_table=torch.zeros(2, 4, dtype=torch.int32),
              block_size=64)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_swa_indices(**la, window=128)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_c128a_indices(**la, compress_ratio=128, width=64)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_compressed_slot_mapping(**la, compress_ratio=4)
    ga = dict(topk_indices=torch.zeros(T, 8, dtype=torch.int32), slot_mapping=la["slot_mapping"],
              token_to_req=la["token_to_req"], block_table=la["block_table"], block_size=64)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_global_topk_indices(**ga)
    bad_q = [(dict(q=torch.zeros(T, H, 128)), "q must"), (dict(q=torch.zeros(T, H, 64, dtype=torch.bfloat16)), "q must"),
             (dict(q=torch.zeros(T, 129, 128, dtype=torch.bfloat16)), "q must"),
             (dict(weights=torch.zeros(T, H)), "weights"), (dict(weights=torch.zeros(T, H + 1, dtype=torch.bfloat16)),
                                                            "weights"),
             (dict(weights=torch.zeros(H, T, dtype=torch.bfloat16).t()), "weights"),
             (dict(cos_sin_cache=torch.zeros(16, 64, dtype=torch.bfloat16)), "cos_sin_cache"),
             (dict(cos_sin_cache=torch.zeros(16, 32)), "cos_sin_cache"),
             (dict(positions=torch.zeros(T + 1, dtype=torch.long)), "positions")]
    for kw, what in bad_q:
        with pytest.raises(ValueError, match=what):
            ops.dsv4_indexer_q_quant(**dict(qa, **kw))
    bad_d = [(dict(q_fp8=torch.zeros(T, H, 128, dtype=torch.bfloat16)), "q_fp8"),
             (dict(q_fp8=torch.zeros(T, 16, 128, dtype=torch.float8_e4m3fn)), "q_fp8"),
             (dict(weights=torch.zeros(T, H, dtype=torch.bfloat16)), "weights"), (dict(weights=torch.zeros(T, 32)), "weights"),
             (dict(k_cache=torch.zeros(4, 64, 584, dtype=torch.uint8)), "k_cache"),
             (dict(block_table=torch.zeros(8, dtype=torch.int32)), "block_table"),
             (dict(block_table=torch.zeros(2, 4)), "block_table"), (dict(compress_ratio=8), "compress_ratio"),
             (dict(topk=0), "topk"), (dict(topk=2049), "topk"), (dict(positions=torch.zeros(2, dtype=torch.long)), "positions"),
             (dict(token_to_req=torch.zeros(4, dtype=torch.int32)), "token_to_req")]
    for kw, what in bad_d:
        with pytest.raises(ValueError, match=what):
            ops.dsv4_indexer_decode(**dict(da, **kw))
    bad_l = [(dict(block_table=torch.zeros(4, dtype=torch.int32)), "block_table"),
             (dict(block_table=torch.zeros(2, 4)), "block_table"), (dict(block_table=torch.zeros(2, 0, dtype=torch.int32)),
                                                                   "block_table"),
             (dict(block_size=0), "block_size"), (dict(slot_mapping=torch.zeros(2, dtype=torch.long)), "slot_mapping"),
             (dict(token_to_req=torch.zeros(4, dtype=torch.int32)), "token_to_req")]
    for kw, what in bad_l:
        with pytest.raises(ValueError, match=what):
            ops.dsv4_swa_indices(**dict(la, **kw), window=128)
    with pytest.raises(ValueError, match="window"):
        ops.dsv4_swa_indices(**la, window=0)
    for kw in (dict(compress_ratio=8, width=64), dict(compress_ratio=128, width=0)):
        with pytest.raises(ValueError, match="compress_ratio"):
            ops.dsv4_c128a_indices(**la, **kw)
    with pytest.raises(ValueError, match="compress_ratio"):
        ops.dsv4_compressed_slot_mapping(**la, compress_ratio=2)
    for bad in (torch.zeros(T, 8), torch.zeros(T, dtype=torch.int32), torch.zeros(T, 0, dtype=torch.int32)):
        with pytest.raises(ValueError, match="topk_indices"):
            ops.dsv4_global_topk_indices(**dict(ga, topk_indices=bad))
    with pytest.raises(ValueError, match="slot_mapping"):
        ops.dsv4_global_topk_indices(**dict(ga, slot_mapping=torch.zeros(2, dtype=torch.long)))
