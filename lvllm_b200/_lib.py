"""ctypes binding of libb200moe.so (the C ABI declared in include/b200moe.h).

There is no CPU or PyTorch fallback: if the library cannot be loaded every wrapper raises.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# B200MOE_LIB_PATH: A/B-test an alternative build of the same library (bring-up aid)
LIB_PATH = os.environ.get("B200MOE_LIB_PATH") or os.path.join(_PKG, "libb200moe.so")


class B200Config(C.Structure):
    """b200moe_config == lk_moe.MOEConfigV2 (reference routed_experts.py:1490-1511)."""
    _fields_ = [
        ("num_processes", C.c_int32), ("process_id", C.c_int32), ("gpu_id", C.c_int32),
        ("has_gate_proj", C.c_int32), ("expert_num", C.c_int32), ("top_k", C.c_int32),
        ("hidden_size", C.c_int32), ("intermediate_size", C.c_int32), ("max_batch_size", C.c_int32),
        ("max_num_seqs", C.c_int32), ("stride", C.c_int32), ("group_min_len", C.c_int32),
        ("group_max_len", C.c_int32), ("groupN", C.c_int32), ("groupK", C.c_int32),
        ("activation_type", C.c_int32), ("swiglu_alpha", C.c_float), ("swiglu_limit", C.c_float),
        ("use_gpu_prefill", C.c_int32),
    ]


FMT_16BIT, FMT_FP8, FMT_WNA16, FMT_NVFP4, FMT_MXFP4 = 0, 1, 2, 3, 4
ACT_BF16, ACT_FP16 = 0, 1

_vp, _i32, _i64, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float

# name -> (restype, argtypes); every symbol declared in include/b200moe.h
PROTOTYPES = {
    "b200moe_last_error": (C.c_char_p, []),
    "b200moe_version": (C.c_char_p, []),
    "b200moe_launch_count": (_i64, []),
    "b200moe_debug_read": (_i32, [_i32, _vp, _i64]),
    "b200moe_profile": (_i32, [_i32]),
    "b200moe_profile_read": (_i32, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(_i64)]),
    "b200moe_create": (_i32, [C.POINTER(B200Config), _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32,
                              C.POINTER(_vp)]),
    "b200moe_create_empty": (_i32, [C.POINTER(B200Config), _i32, _i32, C.POINTER(_vp)]),
    "b200moe_load_experts": (_i32, [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200moe_finalize": (_i32, [_vp]),
    "b200moe_destroy": (_i32, [_vp]),
    "b200moe_device_bytes": (_i64, [_vp]),
    "b200moe_query": (_i32, [_vp, _i32]),
    "b200moe_cpu_decode": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b200moe_cpu_prefill": (_i32, [_vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b200moe_gpu_prefill": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp]),
    "b200_topk_gating": (_i32, [_vp, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp]),
    "b200_hash_topk": (_i32, [_vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "b200_grouped_topk": (_i32, [_vp, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "b200_global_to_local_ids": (_i32, [_vp, _vp, _vp, _i32, _i64, _vp]),
    "b200_router_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "b200_router_topk": (_i32, [_vp, _vp, _i32, _vp, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _f32, _vp,
                                _i32, _i32, _f32, _vp, _i64, _vp, _vp, _vp, _vp]),
    "b200_router_hash_topk": (_i32, [_vp, _vp, _i32, _vp, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _f32,
                                     _vp, _i32, _i32, _f32, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200_moe_permute": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b200_moe_unpermute": (_i32, [_vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _vp, _i32]),
    "b200_rmsnorm_cast": (_i32, [_vp, _vp, _vp, _i32, _i32, _f32, _f32, _i32]),
    "b200_mla_decode_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "b200_mla_decode": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32, _vp, _vp, _vp]),
    "b200_mla_decode_ex": (_i32, [_vp, _vp, _vp, _i32, _vp, _i32, _f32, _f32, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32,
                                  _vp, _vp, _vp]),
    "b200_mla_decode_spec": (_i32, [_vp, _vp, _vp, _i32, _vp, _i32, _f32, _f32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32,
                                    _i32, _vp, _vp, _vp, _vp, _vp]),
    "b200_mla_decode_sparse": (_i32, [_vp, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32,
                                      _vp, _vp, _vp, _vp, _vp]),
    "b200_dsv4_sparse_decode": (_i32, [_vp, _vp, _i32, _i32, _vp, _i32, _i32, _i64, _vp, _i32, _vp, _vp, _i32, _i32, _i64,
                                       _vp, _i32, _vp, _vp, _f32, _i32, _vp, _vp]),
    "b200_dsv4_qnorm_rope_kv_insert": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _i64, _vp, _i32, _i32, _i32,
                                              _f32]),
    "b200_dsv4_compress": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _i64, _vp, _f32, _vp, _i32, _vp,
                                  _vp, _i32, _i32, _i64, _i32, _i32, _i32]),
    "b200_mla_rope_cache_write": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _f32, _i32, _i32]),
    "b200_mla_q_absorb": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32]),
    "b200_mla_decode_vup": (_i32, [_vp, _vp, _vp, _i32, _vp, _i32, _f32, _f32, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32,
                                   _vp, _vp, _vp, _vp, _vp]),
    "b200_indexer_qk_rope_quant_cache_write": (_i32, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _i32,
                                                      _f32, _f32, _vp, _vp, _i32, _i32]),
    "b200_indexer_logits": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i64]),
    "b200_indexer_topk": (_i32, [_vp, _vp, _i64, _i64, _vp, _i32, _i32, _i32, _vp]),
    "b200_dsv4_indexer_q_quant": (_i32, [_vp, _vp, _vp, _i64, _vp, _vp, _i32, _f32, _f32, _vp, _vp, _i32, _i32]),
    "b200_dsv4_indexer_decode": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i64, _vp,
                                        _i64, _i32, _vp]),
    "b200_dsv4_indices": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _i32, _vp,
                                 _i32]),
    "b200_dsv4_inv_rope_quant": (_i32, [_vp, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200_dsv4_wo_a_workspace_bytes": (_i64, [_i32, _i32, _i32, _i32]),
    "b200_dsv4_wo_a": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp]),
    "b200_gqa_decode_workspace_bytes": (_i64, [_i32, _i32, _i32, _i32]),
    "b200_gqa_decode": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _f32, _i32,
                               _vp, _vp, _vp]),
    "b200_gqa_decode_ex": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _f32,
                                  _i32, _vp, _vp, _vp]),
    "b200_gqa_decode_spec": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32,
                                    _f32, _i32, _vp, _vp, _vp]),
    "b200_gqa_qknorm_rope_cache_write": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _vp, _vp, _i64,
                                                _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32]),
    "b200_mhc_workspace_bytes": (_i64, [_i32, _i32]),
    "b200_mhc_post_pre": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _f32, _f32, _f32, _i32, _f32,
                                 _vp, _vp, _vp, _vp, _vp]),
    "b200_mhc_post": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp]),
    "b200_hc_head": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _f32, _vp, _vp]),
    "b200_ep_flag_bytes": (_i64, []),
    "b200_ep_buffer_create": (_i32, [_i64, C.POINTER(_vp), _vp]),
    "b200_ep_buffer_open": (_i32, [_vp, C.POINTER(_vp)]),
    "b200_ep_buffer_close": (_i32, [_vp, _i32]),
    "b200_ep_allreduce": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _i64, _i64, _vp, _i32]),
    "b200_ep_allreduce_norm": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _i32, _i32, _i64, _vp, _vp, _f32,
                                      _f32, _vp, _vp, _i32]),
    "b200_ep_a2a_layout": (_i64, [_i32, _i32, _i32, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "b200_ep_dispatch": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32]),
    "b200_ep_combine_norm": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp,
                                    _f32, _f32, _vp, _i32]),
    "b200_ep_combine": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32]),
}

_lib = None


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it is missing — there is no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m lvllm_b200.build` (nvcc, sm_90a). "
                "lvllm_b200 has no CPU / PyTorch fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class B200Error(RuntimeError):
    pass


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().b200moe_last_error()
        raise B200Error(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
