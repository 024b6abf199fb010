"""Drop-in `lk_moe` module surface backed by libb200moe.so.

Mirrors exactly what Lvllm's call site uses (reference
vllm/model_executor/layers/fused_moe/routed_experts.py:1490-1899): `MOEConfigV2` (attribute bag), the ten
`MOE_*` classes constructed as ``MOE_X(cfg, w13_ptr, w2_ptr, w13_scale_ptr, w2_scale_ptr, w13_gscale_ptr,
w2_gscale_ptr)`` from raw ``tensor.data_ptr()`` integers of contiguous CPU tensors (absent = 0), and the
three methods ``cpu_decode / cpu_prefill / gpu_prefill`` with the reference's positional signatures.
Errors raise (the reference logs ctor failures, routed_experts.py:1415-1418).
"""
from __future__ import annotations

import ctypes as C

from . import _lib as L


class MOEConfigV2:
    """Plain attribute bag; field list of reference routed_experts.py:1490-1511.

    The reference assigns ``swiglu_limit`` explicitly only for models whose SiLU experts clamp (DeepSeek-V4,
    routed_experts.py:1506-1510), while every config carries the default 7.0.  So the bag records whether the caller
    assigned the limit, and ``activation_type 0`` with an assigned limit is sent to the library as type 3 (SiLU with
    the clamp).  Other types are sent as they are."""

    def __init__(self):
        self.num_processes = 1
        self.process_id = 0
        self.gpu_id = 0
        self.has_gate_proj = True
        self.expert_num = 0
        self.top_k = 0
        self.hidden_size = 0
        self.intermediate_size = 0
        self.max_batch_size = 0
        self.max_num_seqs = 0
        self.stride = 32
        self.group_min_len = 10
        self.group_max_len = 0
        self.groupN = 0
        self.groupK = 0
        self.activation_type = 0
        self.swiglu_alpha = 1.702
        self.swiglu_limit = 7.0
        self.use_gpu_prefill = False
        self.swiglu_limit_assigned = False

    def __setattr__(self, name, value):
        if name == "swiglu_limit" and "swiglu_limit" in self.__dict__:
            object.__setattr__(self, "swiglu_limit_assigned", True)
        object.__setattr__(self, name, value)

    def _to_c(self) -> L.B200Config:
        c = L.B200Config()
        for name, _ in L.B200Config._fields_:
            v = getattr(self, name)
            setattr(c, name, float(v) if name.startswith("swiglu") else int(v))
        if c.activation_type == 0 and self.swiglu_limit_assigned:
            c.activation_type = 3
        return c


class _MOEBase:
    _format = None
    _act = L.ACT_BF16
    #: set by loaders that already hold the checkpoint in HBM (b200moe_create weights_on_device=1)
    weights_on_device = False

    def __init__(self, cfg: MOEConfigV2, w13_ptr: int, w2_ptr: int, w13_scale_ptr: int = 0, w2_scale_ptr: int = 0,
                 w13_global_scale_ptr: int = 0, w2_global_scale_ptr: int = 0, weights_on_device: bool | None = None):
        self._h = C.c_void_p()
        self.cfg = cfg
        on_dev = self.weights_on_device if weights_on_device is None else weights_on_device
        c = cfg._to_c()
        rc = L.lib().b200moe_create(C.byref(c), w13_ptr or None, w2_ptr or None, w13_scale_ptr or None,
                                    w2_scale_ptr or None, w13_global_scale_ptr or None,
                                    w2_global_scale_ptr or None, self._format, self._act, int(bool(on_dev)),
                                    C.byref(self._h))
        L.check(rc, f"{type(self).__name__}()")

    @classmethod
    def from_expert_shards(cls, cfg: MOEConfigV2, shards, weights_on_device: bool = False):
        """Build the layer from per-expert (or per-range) checkpoint tensors without ever stacking them into one
        [E, ...] host tensor (SURVEY.md 8f row 4).  ``shards`` yields ``(first_expert, num_experts, w13_ptr, w2_ptr,
        w13_scale_ptr, w2_scale_ptr, w13_gscale_ptr, w2_gscale_ptr)`` with raw ``data_ptr()`` integers of contiguous
        tensors holding just those experts; each may be freed as soon as the generator is advanced."""
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self.cfg = cfg
        c = cfg._to_c()
        L.check(L.lib().b200moe_create_empty(C.byref(c), cls._format, cls._act, C.byref(self._h)), f"{cls.__name__}.from_expert_shards")
        for (e0, ne, w13, w2, s13, s2, g13, g2) in shards:
            L.check(L.lib().b200moe_load_experts(self._h, int(e0), int(ne), w13 or None, w2 or None, s13 or None, s2 or None,
                                                 g13 or None, g2 or None, int(bool(weights_on_device))), "load_experts")
        L.check(L.lib().b200moe_finalize(self._h), "finalize")
        return self

    # reference routed_experts.py:1842-1850
    def cpu_decode(self, stream_ptr: int, num_tokens: int, top_k: int, hidden_ptr: int, topk_ids_ptr: int,
                   topk_weights_ptr: int, out_f32_ptr: int) -> None:
        L.check(L.lib().b200moe_cpu_decode(self._h, stream_ptr or None, num_tokens, top_k, hidden_ptr, topk_ids_ptr,
                                           topk_weights_ptr, out_f32_ptr), "cpu_decode")

    # reference routed_experts.py:1868-1875
    def cpu_prefill(self, num_tokens: int, top_k: int, ids_host_ptr: int, weights_host_ptr: int,
                    hidden_host_ptr: int, out_f32_host_ptr: int) -> None:
        L.check(L.lib().b200moe_cpu_prefill(self._h, num_tokens, top_k, ids_host_ptr, weights_host_ptr,
                                            hidden_host_ptr, out_f32_host_ptr), "cpu_prefill")

    # reference routed_experts.py:1886-1894
    def gpu_prefill(self, hidden_ptr: int, out_ptr: int, topk_ids_ptr: int, topk_weights_ptr: int, num_tokens: int,
                    top_k: int, stream_ptr: int) -> None:
        L.check(L.lib().b200moe_gpu_prefill(self._h, hidden_ptr, out_ptr, topk_ids_ptr, topk_weights_ptr, num_tokens,
                                            top_k, stream_ptr or None), "gpu_prefill")

    def query(self, what: int) -> int:
        """b200moe_query: 0 native MXFP4 kernel in use, 1 tokens per pass, 2 interleaved w13, 3 4-bit flavour."""
        return int(L.lib().b200moe_query(self._h, what))

    def device_bytes(self) -> int:
        return int(L.lib().b200moe_device_bytes(self._h))

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            L.lib().b200moe_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _mk(name, fmt, act):
    return type(name, (_MOEBase,), {"_format": fmt, "_act": act, "__doc__": f"lk_moe.{name} in GPU HBM"})


MOE_BF16 = _mk("MOE_BF16", L.FMT_16BIT, L.ACT_BF16)
MOE_FP16 = _mk("MOE_FP16", L.FMT_16BIT, L.ACT_FP16)
MOE_FP8 = _mk("MOE_FP8", L.FMT_FP8, L.ACT_BF16)
MOE_FP8_FP16 = _mk("MOE_FP8_FP16", L.FMT_FP8, L.ACT_FP16)
MOE_WNA16 = _mk("MOE_WNA16", L.FMT_WNA16, L.ACT_BF16)
MOE_WNA16_FP16 = _mk("MOE_WNA16_FP16", L.FMT_WNA16, L.ACT_FP16)
MOE_NVFP4 = _mk("MOE_NVFP4", L.FMT_NVFP4, L.ACT_BF16)
MOE_NVFP4_FP16 = _mk("MOE_NVFP4_FP16", L.FMT_NVFP4, L.ACT_FP16)
MOE_MXFP4 = _mk("MOE_MXFP4", L.FMT_MXFP4, L.ACT_BF16)
MOE_MXFP4_FP16 = _mk("MOE_MXFP4_FP16", L.FMT_MXFP4, L.ACT_FP16)

__all__ = ["MOEConfigV2", "MOE_BF16", "MOE_FP16", "MOE_FP8", "MOE_FP8_FP16", "MOE_WNA16", "MOE_WNA16_FP16",
           "MOE_NVFP4", "MOE_NVFP4_FP16", "MOE_MXFP4", "MOE_MXFP4_FP16"]
