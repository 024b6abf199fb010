"""CPU: the DeepSeek-V4 KV compressor oracle (tests/dsv4_compress_oracle.py) against the reference's own kernels and torch
statement, stored in tests/golden/golden_dsv4_compress.pt: the state rows bit for bit, the compressed caches by
dsv4_compress_oracle.check_cache (scales equal, e4m3 codes within one step, rope dims within one bf16 ulp, nothing written
elsewhere), the rows within one bf16 ulp of the torch statement's; and the C ABI and Python refusals of dsv4_compress."""
import os

import pytest
import torch

import dsv4_compress_oracle as C
import dsv4_sparse_oracle as V4

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_dsv4_compress.pt")
IDS = ["c4a_512", "c128a_512", "c4a_indexer_128"]


def _load():
    return torch.load(GOLDEN, weights_only=True)


def _state(c):
    half = C.coff(c["ratio"]) * c["head_dim"]
    st = torch.zeros(c["state_blocks"], c["state_block_size"], 2 * half)
    st.view(-1, 2 * half)[c["early_slots"]] = c["early_rows"].float()
    return st


@pytest.mark.parametrize("i", range(3), ids=IDS)
def test_state_write_matches_reference_bit_exact(i):
    c = _load()["cases"][i]
    half = C.coff(c["ratio"]) * c["head_dim"]
    st = C.state_write(c["kv_score"].float(), c["ape"], c["positions"], c["slot_mapping"], _state(c))
    flat = st.view(-1, 2 * half)
    assert torch.equal(flat[c["written_slots"], half:], c["state_score"])
    ws = c["slot_mapping"] >= 0
    assert torch.equal(flat[c["slot_mapping"][ws], :half], c["kv_score"][ws, :half].float())
    assert c["slot_mapping"][-1] == -1 and int((flat.abs().sum(1) != 0).sum()) == int(ws.sum()) + len(c["early_slots"])


@pytest.mark.parametrize("i", range(3), ids=IDS)
def test_compress_matches_reference(i):
    g = _load()
    c = g["cases"][i]
    st = C.state_write(c["kv_score"].float(), c["ape"], c["positions"], c["slot_mapping"], _state(c))
    cache = torch.zeros_like(c["cache"])
    rows = C.compress(st, c["block_table"], c["token_to_req"], c["positions"], c["slot_mapping"], c["norm_weight"],
                      g["eps"], g["cos_sin"], c["ratio"], c["kv_slot_mapping"], cache)
    assert sorted(rows) == c["boundary_tokens"].tolist()
    C.check_cache(c["cache"], cache, rows, c["kv_slot_mapping"])
    got = torch.stack([rows[int(t)] for t in c["boundary_tokens"]]).bfloat16()
    assert int(V4.bf16_ulp_distance(got, c["torch_rows"]).max()) <= 1
    written = [int(c["kv_slot_mapping"][int(t)]) for t in c["boundary_tokens"]]
    assert -1 in written or c["ratio"] == 128                  # a boundary token with kv slot -1 writes nothing
    assert int((cache.reshape(cache.shape[0], -1) != 0).any(1).sum()) >= 1
    if c["head_dim"] == 512 and c["ratio"] == 4:               # request 1's second quant block is under the 1e-4 clamp
        t = next(int(t) for t in c["boundary_tokens"] if int(c["token_to_req"][int(t)]) == 1
                 and int(c["kv_slot_mapping"][int(t)]) >= 0)
        s = int(c["kv_slot_mapping"][t])
        bs = cache.shape[1]
        rec = c["cache"][s // bs].reshape(-1)[bs * 576 + (s % bs) * 8:][:8]
        assert int(rec[1]) == 127 - 22 and rows[t][64:128].abs().max() < 1e-4


def _abi(lib, **kw):
    P = 1 << 20   # a 16-byte aligned stand-in address
    a = dict(kvs=P, kvs_stride=2048, ape=P, pos=P, slots=P, req=P, bt=P, bt_stride=64, state=P, sbs=8, sstride=8 * 2048,
             w=P, eps=1e-6, cs=P, maxpos=4096, kslots=P, cache=P, bs=64, nb=4, stride=64 * 584, D=512, ratio=4, T=2)
    a.update(kw)
    return lib.b200_dsv4_compress(None, *a.values())


def test_c_abi_refuses_bad_arguments():
    """Refusals happen before any launch: each call differs from a well-formed one in one argument; pointers are only
    checked for NULL and alignment, never dereferenced."""
    from lvllm_b200 import _lib as L
    lib = L.lib()
    P = 1 << 20
    assert _abi(lib, T=0) == 0                                            # well-formed, nothing to do
    for bad in (dict(D=512, ratio=8), dict(D=128, ratio=128), dict(D=256), dict(ratio=1), dict(kvs=None),
                dict(kvs=P + 4), dict(kvs_stride=2047), dict(kvs_stride=2044), dict(ape=P + 8), dict(pos=P + 4),
                dict(slots=None), dict(req=P + 2), dict(bt=None), dict(bt_stride=0), dict(state=P + 4), dict(sbs=0),
                dict(sstride=8 * 2048 - 4), dict(sstride=8 * 2048 + 2), dict(w=None), dict(w=P + 2), dict(eps=-1.0),
                dict(eps=float("nan")), dict(cs=P + 1), dict(maxpos=0), dict(kslots=P + 4), dict(cache=P + 8), dict(bs=0),
                dict(nb=0), dict(stride=64 * 584 - 16), dict(stride=64 * 584 + 8), dict(T=-1), dict(T=(1 << 20) + 1),
                dict(D=128, kvs_stride=512, sstride=8 * 512, stride=64 * 132 - 4),
                dict(D=128, kvs_stride=512, sstride=8 * 512, stride=64 * 132 + 2),
                dict(ratio=128, sstride=8 * 1024 - 4)):
        assert _abi(lib, **bad) == -1, bad
    assert _abi(lib, D=128, kvs_stride=512, sstride=8 * 512, stride=64 * 132, T=0) == 0
    assert _abi(lib, ratio=128, kvs_stride=1024, sstride=8 * 1024, T=0) == 0


def _py_args(D=512, ratio=4, T=3, row=None):
    half = C.coff(ratio) * D
    row = row or (584 if D == 512 else 132)
    return dict(kv_score=torch.zeros(T, 2 * half), ape=torch.zeros(ratio, half), positions=torch.zeros(T, dtype=torch.long),
                state_cache=torch.zeros(4, 8, 2 * half), slot_mapping=torch.zeros(T, dtype=torch.long),
                token_to_req=torch.zeros(T, dtype=torch.int32), block_table=torch.zeros(2, 8, dtype=torch.int32),
                norm_weight=torch.ones(D, dtype=torch.bfloat16), eps=1e-6, cos_sin_cache=torch.zeros(16, 64),
                kv_cache=torch.zeros(2, 16, row, dtype=torch.uint8), kv_slot_mapping=torch.zeros(T, dtype=torch.long),
                compress_ratio=ratio)


def test_python_refusals():
    """ops.dsv4_compress checks dtypes and shapes before anything touches a device; a well-formed call on CPU tensors
    stops only at the CUDA check."""
    from lvllm_b200 import ops
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_compress(**_py_args())
    ops.dsv4_compress(**_py_args(T=0))                                    # T = 0: returns without a launch
    bad = [
        (dict(norm_weight=torch.ones(512)), "norm_weight"),
        (dict(norm_weight=torch.ones(256, dtype=torch.bfloat16)), "head_dim"),
        (dict(compress_ratio=8), "head_dim"),
        (dict(kv_cache=torch.zeros(2, 16, 132, dtype=torch.uint8)), "head_dim"),
        (dict(kv_cache=torch.zeros(2, 16, 584)), "kv_cache"),
        (dict(kv_cache=torch.zeros(2, 584, 16, dtype=torch.uint8).transpose(1, 2)), "kv_cache"),
        (dict(kv_score=torch.zeros(3, 2048, dtype=torch.bfloat16)), "kv_score"),
        (dict(kv_score=torch.zeros(3, 1024)), "kv_score"),
        (dict(kv_score=torch.zeros(2048, 3).t()), "kv_score"),
        (dict(ape=torch.zeros(4, 512)), "ape"),
        (dict(ape=torch.zeros(4, 1024, dtype=torch.bfloat16)), "ape"),
        (dict(state_cache=torch.zeros(4, 8, 1024)), "state_cache"),
        (dict(state_cache=torch.zeros(4, 8, 2048, dtype=torch.bfloat16)), "state_cache"),
        (dict(block_table=torch.zeros(8, dtype=torch.int32)), "block_table"),
        (dict(block_table=torch.zeros(2, 8)), "block_table"),
        (dict(cos_sin_cache=torch.zeros(16, 32)), "cos_sin_cache"),
        (dict(cos_sin_cache=torch.zeros(16, 64, dtype=torch.bfloat16)), "cos_sin_cache"),
        (dict(positions=torch.zeros(2, dtype=torch.long)), "positions"),
        (dict(slot_mapping=torch.zeros(4, dtype=torch.long)), "slot_mapping"),
        (dict(token_to_req=torch.zeros(2, dtype=torch.int32)), "token_to_req"),
        (dict(kv_slot_mapping=torch.zeros(2, dtype=torch.long)), "kv_slot_mapping"),
    ]
    for kw, what in bad:
        a = _py_args()
        a.update(kw)
        with pytest.raises(ValueError, match=what):
            ops.dsv4_compress(**a)
    a = _py_args(D=128, ratio=4)
    a["kv_cache"] = torch.zeros(2, 16, 584, dtype=torch.uint8)
    with pytest.raises(ValueError, match="head_dim"):
        ops.dsv4_compress(**a)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_compress(**_py_args(D=128, ratio=4))
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_compress(**_py_args(D=512, ratio=128))
