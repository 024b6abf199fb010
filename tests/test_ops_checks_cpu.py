"""The argument checks of the Python ops and of EpGroup.  The C ABI sees only pointers and sizes, so these checks are what
keeps a mis-shaped tensor from being read or written out of bounds: every public op refuses a malformed call with a
ValueError naming the argument before it touches a device or the library, a well-formed call on CPU tensors stops at
the CUDA check, and the ctypes prototypes agree with the C header."""
import ast
import ctypes as C
import inspect
import os
import re

import pytest
import torch

from lvllm_b200 import _lib, ops
from lvllm_b200.ep import EpGroup

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bf, f8, u8, i32, i64 = torch.bfloat16, torch.float8_e4m3fn, torch.uint8, torch.int32, torch.int64
T, E, K, H = 3, 8, 2, 64


def _z(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype)


@pytest.fixture
def no_library(monkeypatch):
    """Every check must run before the library is loaded."""
    def refuse():
        raise RuntimeError("the library was reached")
    monkeypatch.setattr(_lib, "lib", refuse)


def _well_formed():
    """Well-formed arguments of every public op, as CPU tensors."""
    mhc = dict(fn=_z(24, 4 * 256), hc_scale=_z(3), hc_base=_z(24), rms_eps=1e-6, hc_pre_eps=1e-6, hc_sinkhorn_eps=1e-6,
               hc_post_mult_value=2.0, sinkhorn_repeat=3)
    mhc_post = dict(x=_z(T, 256, dtype=bf), residual=_z(T, 4, 256, dtype=bf), post_layer_mix=_z(T, 4),
                    comb_res_mix=_z(T, 4, 4))
    mla_q = dict(q_nope=_z(T, 16, 512, dtype=bf), q_pe=_z(T, 16, 64, dtype=bf))
    kv = dict(k_cache=_z(4, 16, 2, 128, dtype=bf), v_cache=_z(4, 16, 2, 128, dtype=bf))
    lists = dict(positions=_z(T, dtype=i64), slot_mapping=_z(T, dtype=i64), token_to_req=_z(T, dtype=i32),
                 block_table=_z(2, 4, dtype=i32), block_size=64)
    idx8 = dict(q_fp8=_z(T, 32, 128, dtype=f8), weights=_z(T, 32), k_cache=_z(4, 64, 132, dtype=u8))
    o = dict(o=_z(T, 16, 512, dtype=bf), positions=_z(T, dtype=i64), cos_sin_cache=_z(16, 64), n_groups=2)
    return {
        "fused_topk": dict(gating_output=_z(T, E), topk=K, renormalize=True, e_score_correction_bias=_z(E)),
        "grouped_topk": dict(gating_output=_z(T, E), topk=K, renormalize=True, num_expert_group=4, topk_group=2,
                             e_score_correction_bias=_z(E)),
        "hash_topk": dict(gating_output=_z(T, E), topk=K, renormalize=True, input_ids=_z(T, dtype=i64),
                          hash_indices_table=_z(16, K, dtype=i32)),
        "router_topk": dict(hidden_states=_z(T, H, dtype=bf), gate_weight=_z(E, H, dtype=bf), topk=K, renormalize=True,
                            e_score_correction_bias=_z(E), expert_map=_z(E, dtype=i32)),
        "global_to_local_expert_ids": dict(topk_ids=_z(T, K, dtype=i32), expert_map=_z(E, dtype=i32)),
        "moe_permute": dict(hidden_states=_z(T, H, dtype=bf), topk_ids=_z(T, K, dtype=i32), n_local_expert=E),
        "moe_unpermute": dict(permuted=_z(T * K, H, dtype=bf), topk_weights=_z(T, K), inv_permuted_idx=_z(T, K, dtype=i32)),
        "rmsnorm_cast": dict(x_f32=_z(T, H), out=_z(T, H, dtype=bf)),
        "mla_decode": dict(**mla_q, kv_c_and_k_pe_cache=_z(4, 64, 576, dtype=bf), seq_lens=_z(T, dtype=i32),
                           page_table=_z(T, 2, dtype=i32), sm_scale=0.1, w_uv=_z(16, 512, 128, dtype=bf)),
        "mla_decode_sparse": dict(**mla_q, kv_cache=_z(4, 64, 656, dtype=u8), topk_indices=_z(T, 8, dtype=i32),
                                  req_id=_z(T, dtype=i32), page_table=_z(2, 2, dtype=i32), sm_scale=0.1,
                                  w_uv=_z(16, 512, 128, dtype=bf)),
        "dsv4_sparse_decode": dict(q=_z(T, 16, 512, dtype=bf), swa_cache=_z(4, 64, 584, dtype=u8),
                                   swa_indices=_z(T, 8, dtype=i32), swa_lens=_z(T, dtype=i32), sm_scale=0.1,
                                   attn_sink=_z(16), extra_cache=_z(4, 64, 584, dtype=u8),
                                   extra_indices=_z(T, 8, dtype=i32), extra_lens=_z(T, dtype=i32)),
        "dsv4_qnorm_rope_kv_insert": dict(q=_z(T, 16, 512, dtype=bf), kv=_z(T, 512, dtype=bf), positions=_z(T, dtype=i64),
                                          cos_sin_cache=_z(16, 64), slot_mapping=_z(T, dtype=i64),
                                          swa_cache=_z(4, 64, 584, dtype=u8), q_head_padded=16, eps=1e-6),
        "dsv4_compress": dict(kv_score=_z(T, 2048), ape=_z(4, 1024), positions=_z(T, dtype=i64),
                              state_cache=_z(4, 8, 2048), slot_mapping=_z(T, dtype=i64), token_to_req=_z(T, dtype=i32),
                              block_table=_z(2, 8, dtype=i32), norm_weight=_z(512, dtype=bf), eps=1e-6,
                              cos_sin_cache=_z(16, 64), kv_cache=_z(2, 16, 584, dtype=u8),
                              kv_slot_mapping=_z(T, dtype=i64), compress_ratio=4),
        "mhc_pre": dict(residual=_z(T, 4, 256, dtype=bf), **mhc, norm_weight=_z(256, dtype=bf)),
        "mhc_post": mhc_post,
        "mhc_fused_post_pre": dict(**mhc_post, **mhc, norm_weight=_z(256, dtype=bf)),
        "hc_head": dict(hidden_states=_z(T, 4, 256, dtype=bf), hc_fn=_z(4, 4 * 256), hc_scale=_z(1), hc_base=_z(4),
                        rms_norm_eps=1e-6, hc_eps=1e-6),
        "mla_rope_cache_write": dict(q_pe=_z(T, 16, 64, dtype=bf), k_pe=_z(T, 64, dtype=bf), kv_c=_z(T, 512, dtype=bf),
                                     positions=_z(T, dtype=i64), cos_sin_cache=_z(16, 64, dtype=bf),
                                     slot_mapping=_z(T, dtype=i64), kv_cache=_z(4, 16, 576, dtype=bf)),
        "mla_q_absorb": dict(q_nope=_z(T, 16, 128, dtype=bf), w_uk_t=_z(16, 128, 512, dtype=bf)),
        "gqa_decode": dict(q=_z(T, 8, 128, dtype=bf), **kv, seq_lens=_z(T, dtype=i32), page_table=_z(T, 2, dtype=i32),
                           sm_scale=0.1),
        "gqa_qknorm_rope_cache_write": dict(qkv=_z(T, 12 * 128, dtype=bf), positions=_z(T, dtype=i64),
                                            cos_sin_cache=_z(16, 64, dtype=bf), slot_mapping=_z(T, dtype=i64), **kv,
                                            num_heads=8, num_kv_heads=2, q_norm_weight=_z(128, dtype=bf),
                                            k_norm_weight=_z(128, dtype=bf)),
        "indexer_qk_rope_quant_cache_write": dict(q=_z(T, 32, 128, dtype=bf), weights=_z(T, 32, dtype=bf),
                                                  k=_z(T, 128, dtype=bf), positions=_z(T, dtype=i64),
                                                  cos_sin_cache=_z(16, 64, dtype=bf), slot_mapping=_z(T, dtype=i64),
                                                  k_cache=_z(4, 64, 132, dtype=u8), softmax_scale=0.1, head_scale=0.1),
        "indexer_logits": dict(**idx8, seq_lens=_z(T, dtype=i32), page_table=_z(T, 2, dtype=i32), logits=_z(T, 128)),
        "indexer_topk": dict(logits=_z(T, 128), seq_lens=_z(T, dtype=i32), topk=16),
        "indexer_decode": dict(**idx8, seq_lens=_z(T, dtype=i32), page_table=_z(T, 2, dtype=i32), q_len=1, topk=16),
        "dsv4_indexer_q_quant": dict(q=_z(T, 32, 128, dtype=bf), weights=_z(T, 32, dtype=bf), positions=_z(T, dtype=i64),
                                     cos_sin_cache=_z(16, 64), softmax_scale=0.1, head_scale=0.1),
        "dsv4_indexer_decode": dict(**idx8, positions=_z(T, dtype=i64), token_to_req=_z(T, dtype=i32),
                                    block_table=_z(2, 2, dtype=i32), compress_ratio=4, topk=16, logits=_z(T, 128)),
        "dsv4_swa_indices": dict(**lists, window=128),
        "dsv4_c128a_indices": dict(**lists, compress_ratio=128, width=64),
        "dsv4_global_topk_indices": dict(topk_indices=_z(T, 8, dtype=i32), slot_mapping=lists["slot_mapping"],
                                         token_to_req=lists["token_to_req"], block_table=lists["block_table"],
                                         block_size=64),
        "dsv4_compressed_slot_mapping": dict(**lists, compress_ratio=4),
        "dsv4_inv_rope_quant": o,
        "dsv4_o_proj": dict(**o, wo_a_weight=_z(256, 4096, dtype=f8), wo_a_scale=_z(2, 32)),
    }


def _public_ops():
    return sorted(n for n, f in inspect.getmembers(ops, inspect.isfunction)
                  if not n.startswith("_") and f.__module__ == ops.__name__)


def test_every_public_op_is_covered():
    """A new op must be added to the table of well-formed calls (and so to the CUDA-check test below)."""
    assert sorted(_well_formed()) == _public_ops()


@pytest.mark.parametrize("name", _public_ops())
def test_well_formed_cpu_call_stops_at_the_cuda_check(name, no_library):
    with pytest.raises(ValueError, match="CUDA"):
        getattr(ops, name)(**_well_formed()[name])


def _refused(call, argument: str):
    with pytest.raises(ValueError) as e:
        call()
    assert argument in str(e.value) and "CUDA" not in str(e.value), str(e.value)


_T = lambda t: t.t().contiguous().t()   # noqa: E731  (the same shape, column-major strides)

MALFORMED = [
    ("router_topk", dict(gate_weight=_z(E, H // 2, dtype=bf)), "gate_weight"),
    ("router_topk", dict(gate_weight=_z(E, H, dtype=torch.float16)), "gate_weight"),
    ("router_topk", dict(e_score_correction_bias=_z(E - 1)), "e_score_correction_bias"),
    ("router_topk", dict(expert_map=_z(E - 1, dtype=i32)), "expert_map"),
    ("router_topk", dict(scoring_func="softmax", num_expert_group=4, topk_group=2), "grouped routing"),
    ("fused_topk", dict(e_score_correction_bias=_z(E + 1)), "e_score_correction_bias"),
    ("fused_topk", dict(gating_output=_z(T, E, dtype=torch.float64)), "gating_output"),
    ("grouped_topk", dict(e_score_correction_bias=_z(E - 1)), "e_score_correction_bias"),
    ("grouped_topk", dict(gating_output=_z(T, E, dtype=torch.float64)), "gating_output"),
    ("moe_permute", dict(hidden_states=_z(T + 1, H, dtype=bf)), "hidden_states"),
    ("moe_unpermute", dict(topk_weights=_z(T, K + 1)), "topk_weights"),
    ("moe_unpermute", dict(topk_weights=_z(T + 1, K)), "topk_weights"),
    ("rmsnorm_cast", dict(out=_z(T, H // 2, dtype=bf)), "out"),
    ("rmsnorm_cast", dict(out=_z(T + 1, H, dtype=bf)), "out"),
    ("rmsnorm_cast", dict(out=_z(T, H)), "out"),
    ("rmsnorm_cast", dict(out=_T(_z(T, H, dtype=bf))), "out"),
    ("mla_decode", dict(q_nope=_z(T, 16, 256, dtype=bf)), "q_nope"),
    ("mla_decode", dict(q_nope=_z(T, 16, 512, dtype=f8), q_pe=_z(T, 16, 64, dtype=f8)), "q_nope"),   # bf16 cache
    ("mla_decode", dict(q_pe=_z(T, 16, 32, dtype=bf)), "q_pe"),
    ("mla_decode", dict(q_pe=_z(T, 8, 64, dtype=bf)), "q_pe"),
    ("mla_decode", dict(kv_c_and_k_pe_cache=_z(256, 576, dtype=bf)), "kv_cache"),
    ("mla_decode", dict(kv_c_and_k_pe_cache=_z(4, 64, 576, dtype=u8)), "kv_cache"),
    ("mla_decode", dict(w_uv=_z(16, 512, 64, dtype=bf)), "w_uv"),
    ("mla_decode", dict(w_uv=_z(16, 512, 128)), "w_uv"),
    ("mla_decode_sparse", dict(q_nope=_z(T, 16, 256, dtype=bf)), "q_nope"),
    ("mla_decode_sparse", dict(q_pe=_z(T, 16, 128, dtype=bf)), "q_pe"),
    ("mla_decode_sparse", dict(w_uv=_z(8, 512, 128, dtype=bf)), "w_uv"),
    ("mla_rope_cache_write", dict(k_pe=_z(T, 32, dtype=bf)), "k_pe"),
    ("mla_rope_cache_write", dict(k_pe=_z(T + 1, 64, dtype=bf)), "k_pe"),
    ("mla_rope_cache_write", dict(kv_c=_z(T, 256, dtype=bf)), "kv_c"),
    ("mla_rope_cache_write", dict(positions=_z(T + 1, dtype=i64)), "positions"),
    ("mla_rope_cache_write", dict(slot_mapping=_z(T - 1, dtype=i64)), "slot_mapping"),
    ("mla_rope_cache_write", dict(q_pe=_z(T, 16, 128, dtype=bf)[..., :64]), "q_pe"),   # rotated in place: no copy
    ("mla_rope_cache_write", dict(k_pe=_T(_z(T, 64, dtype=bf))), "k_pe"),
    ("mla_rope_cache_write", dict(cos_sin_cache=_z(16, 64)), "cos_sin_cache"),
    ("mla_rope_cache_write", dict(kv_cache=_z(4, 16, 576, dtype=u8)), "kv_cache"),
    ("mla_q_absorb", dict(q_nope=_z(T, 16, 64, dtype=bf)), "q_nope"),
    ("mla_q_absorb", dict(w_uk_t=_z(16, 128, 256, dtype=bf)), "w_uk_t"),
    ("mla_q_absorb", dict(w_uk_t=_z(8, 128, 512, dtype=bf)), "w_uk_t"),
    ("gqa_decode", dict(q=_z(T, 8, 128, dtype=torch.float16)), "q"),
    ("gqa_decode", dict(q=_z(T, 8, 64, dtype=bf)), "q"),
    ("indexer_qk_rope_quant_cache_write", dict(k_cache=_z(4, 64, 584, dtype=u8)), "k_cache"),
    ("indexer_logits", dict(logits=_z(T, 64)), "logits"),
]


@pytest.mark.parametrize("name,override,argument", MALFORMED, ids=[f"{n}-{i}" for i, (n, _, _) in enumerate(MALFORMED)])
def test_malformed_call_names_the_argument(name, override, argument, no_library):
    args = _well_formed()[name]
    args.update(override)
    _refused(lambda: getattr(ops, name)(**args), argument)


def _ep():
    ep = object.__new__(EpGroup)
    ep.world, ep.rank, ep.slot_elems = 1, 0, 64
    ep.m_local, ep.a2a_h, ep.a2a_k, ep.epr = 2, 16, 2, 4
    ep._out = _z(64)
    return ep


def test_ep_group_refusals(no_library):
    ep = _ep()
    ids, w = _z(2, 2, dtype=i32), _z(2, 2)
    _refused(lambda: ep.allreduce(_z(80)), "x_f32")                                   # past the peer slot
    _refused(lambda: ep.allreduce(_z(6)), "x_f32")
    _refused(lambda: ep.allreduce(_z(8, dtype=bf)), "x_f32")
    _refused(lambda: ep.allreduce(_z(8), _z(4, dtype=bf)), "out")
    _refused(lambda: ep.allreduce(_z(8), _z(8, dtype=i32)), "out")
    _refused(lambda: ep.allreduce_norm(_z(8, 16), _z(8, 16, dtype=bf)), "x_f32")       # 128 > 64 slot elements
    _refused(lambda: ep.allreduce_norm(_z(2, 16), _z(2, 8, dtype=bf)), "out")
    _refused(lambda: ep.allreduce_norm(_z(2, 16), _z(2, 16)), "out")
    _refused(lambda: ep.allreduce_norm(_z(2, 16), _z(2, 16, dtype=bf), residual=_z(1, 16, dtype=bf)), "residual")
    _refused(lambda: ep.allreduce_norm(_z(2, 16), _z(2, 16, dtype=bf), gamma=_z(8, dtype=bf)), "gamma")
    _refused(lambda: ep.allreduce_norm(_z(2, 16), _z(2, 16, dtype=bf), gamma=_z(16)), "gamma")
    _refused(lambda: ep.allreduce_norm(_z(2, 16), _z(2, 16, dtype=bf), sum_out=_z(2, 8)), "sum_out")
    _refused(lambda: ep.dispatch(_z(3, 16, dtype=bf), ids, w), "hidden_local")
    _refused(lambda: ep.dispatch(_z(2, 16, dtype=bf), ids.long(), w), "ids_global")
    _refused(lambda: ep.dispatch(_z(2, 16, dtype=bf), ids, w[:, :1]), "weights")
    for bad in (_z(2, 3, dtype=i32), _z(2, 2, dtype=i64), _z(4, dtype=i32), _T(_z(2, 2, dtype=i32))):
        _refused(lambda: ep.combine(bad, _z(2, 16)), "ids_global")
        _refused(lambda: ep.combine_norm(bad, _z(2, 16, dtype=bf)), "ids_global")
    _refused(lambda: ep.combine(ids, _z(3, 16)), "out")
    _refused(lambda: ep.combine(ids, _z(2, 16, dtype=i32)), "out")
    _refused(lambda: ep.combine_norm(ids, _z(2, 16)), "out")
    _refused(lambda: ep.combine_norm(ids, _z(2, 16, dtype=bf), residual=_z(2, 8, dtype=bf)), "residual")
    _refused(lambda: ep.combine_norm(ids, _z(2, 16, dtype=bf), residual=_z(2, 16, dtype=torch.float16)), "residual")
    _refused(lambda: ep.combine_norm(ids, _z(2, 16, dtype=bf), gamma=_z(2, 16, dtype=bf)), "gamma")
    _refused(lambda: ep.a2a_init(0, 16, 2, 4), "m_local")
    with pytest.raises(ValueError, match="world"):
        EpGroup(0, 9, torch.device("cpu"), 64)


def test_ep_group_well_formed_calls_reach_the_library(no_library):
    ep = _ep()
    ids, x16 = _z(2, 2, dtype=i32), _z(2, 16, dtype=bf)
    for call in (lambda: ep.allreduce(_z(64)), lambda: ep.allreduce(_z(4, 8), _z(4, 8, dtype=bf)),
                 lambda: ep.allreduce_norm(_z(2, 16), x16, residual=x16.clone(), gamma=_z(16, dtype=bf), sum_out=_z(2, 16)),
                 lambda: ep.dispatch(x16, ids, _z(2, 2)), lambda: ep.combine(ids, _z(2, 16)),
                 lambda: ep.combine_norm(ids, x16, residual=x16.clone(), gamma=_z(16, dtype=bf))):
        with pytest.raises(RuntimeError, match="library was reached"):
            call()


@pytest.mark.parametrize("module", ["ops.py", "ep.py"])
def test_no_assert_statements(module):
    """python -O strips assert statements: the argument checks must be raises."""
    tree = ast.parse(open(os.path.join(ROOT, "lvllm_b200", module)).read())
    assert not [n.lineno for n in ast.walk(tree) if isinstance(n, ast.Assert)]


def _header_kind(param: str) -> str:
    if "*" in param or param.split()[0] == "b200moe_handle":
        return "pointer"
    return {"int": "int32", "int32_t": "int32", "int64_t": "int64", "float": "float"}[param.replace("const", "").split()[0]]


def _ctypes_kind(t) -> str:
    if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
        return "pointer"
    return {C.c_int32: "int32", C.c_int64: "int64", C.c_float: "float"}[t]


def test_prototypes_match_the_header():
    """Every ctypes prototype has the parameter count and kinds (pointer / int32 / int64 / float) of its declaration in
    include/b200moe.h: an int64 stride declared as int32 would be passed truncated."""
    src = open(os.path.join(ROOT, "include", "b200moe.h")).read()
    src = re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", src, flags=re.S))
    decls = {}
    for ret, name, params in re.findall(r"(int64_t|int|const\s+char\s*\*)\s+(b200\w*)\s*\(([^)]*)\)\s*;", src):
        ps = [p.strip() for p in params.split(",") if p.strip() not in ("", "void")]
        decls[name] = (_header_kind(ret), [_header_kind(p) for p in ps])
    assert sorted(decls) == sorted(_lib.PROTOTYPES)
    for name, (res, args) in _lib.PROTOTYPES.items():
        assert decls[name] == (_ctypes_kind(res), [_ctypes_kind(a) for a in args]), name


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_router_workspace_outlives_growth():
    """A CUDA graph captured against the router's workspace keeps its buffer when a later, larger eager call on the same
    stream grows the workspace (a prefill batch after decode capture): the graph still replays to the eager result."""
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(0)
    E_, H_, k = 256, 7168, 8                                                              # DeepSeek-V3's router
    gate = (torch.randn(E_, H_, device=dev, generator=g) / 64).bfloat16()
    x1 = torch.randn(1, H_, device=dev, generator=g).bfloat16()
    x512 = torch.randn(512, H_, device=dev, generator=g).bfloat16()
    lib = _lib.lib()
    assert lib.b200_router_workspace_bytes(1, E_, H_) <= 1 << 20 < lib.b200_router_workspace_bytes(512, E_, H_)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ref = ops.router_topk(x1, gate, k, True)
        held = ops._workspaces[("router", dev.index, s.cuda_stream)]
        captured = held[-1]
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = ops.router_topk(x1, gate, k, True)
        ops.router_topk(x512, gate, k, True)
        assert held[-1] is not captured and any(b is captured for b in held)
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
