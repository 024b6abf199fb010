"""Expert-parallel group over NVLink peer memory (one process per GPU).

lk_moe's EP/TP contract is "tokens replicated, local experts, sum over ranks" (reference
vllm/model_executor/layers/fused_moe/runner/moe_runner.py:488-494).  NCCL (torch.distributed) is used only
to bootstrap: the 64-byte CUDA-IPC handles of every rank's staging/flag buffers are exchanged once with
all_gather_object; the data path is hand-written in csrc/ep.cu: a one-shot all-reduce (peer loads over NVLink,
release/acquire flags, fixed-order sum => bit-identical on all ranks) for replicated tokens, and a
dispatch / combine all-to-all for token-sharded callers (DP attention + EP experts, SURVEY.md 8e).
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.distributed as dist

from . import _lib as L

_OUT = {torch.bfloat16: 0, torch.float16: 1, torch.float32: 2}


def _norm_args(out: torch.Tensor, M: int, H: int, residual: torch.Tensor | None, gamma: torch.Tensor | None) -> None:
    """out bf16 / fp16 [M, H] of a fused residual add + RMSNorm, residual [M, H] and gamma [H] in its dtype."""
    if out.dtype not in (torch.bfloat16, torch.float16) or tuple(out.shape) != (M, H) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous bf16 / fp16 [{M}, {H}] tensor, got {out.dtype} {tuple(out.shape)}")
    for t, name, shape in ((residual, "residual", (M, H)), (gamma, "gamma", (H,))):
        if t is not None and (t.dtype != out.dtype or tuple(t.shape) != shape or not t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous {out.dtype} {list(shape)} tensor, got {t.dtype} "
                             f"{tuple(t.shape)}")


def exchange_handles(local: bytes, group=None) -> list[bytes]:
    """all-gather one opaque handle per rank (works on gloo and nccl groups)."""
    world = dist.get_world_size(group)
    out: list = [None] * world
    dist.all_gather_object(out, local, group=group)
    return out


class EpGroup:
    def __init__(self, rank: int, world: int, device: torch.device, max_elems: int, group=None):
        if not 1 <= world <= 8:
            raise ValueError(f"world must be 1-8, got {world}")
        self.rank, self.world, self.device = rank, world, device
        self.slot_elems = (max_elems + 3) // 4 * 4
        lib = L.lib()
        self._data = C.c_void_p()
        self._flags = C.c_void_p()
        hd = (C.c_ubyte * 64)()
        hf = (C.c_ubyte * 64)()
        # slots: [2] pull all-reduce (parity), then [2 parities][world] push all-reduce + norm
        L.check(lib.b200_ep_buffer_create((2 + 2 * world) * self.slot_elems * 4, C.byref(self._data), hd), "ep data buffer")
        L.check(lib.b200_ep_buffer_create(lib.b200_ep_flag_bytes(), C.byref(self._flags), hf), "ep flag buffer")
        handles = exchange_handles(bytes(hd) + bytes(hf), group)
        self._peer_data = (C.c_void_p * 8)()
        self._peer_flags = (C.c_void_p * 8)()
        for r, h in enumerate(handles):
            if r == rank:
                self._peer_data[r], self._peer_flags[r] = self._data.value, self._flags.value
                continue
            pd, pf = C.c_void_p(), C.c_void_p()
            L.check(lib.b200_ep_buffer_open((C.c_ubyte * 64).from_buffer_copy(h[:64]), C.byref(pd)), "open peer data")
            L.check(lib.b200_ep_buffer_open((C.c_ubyte * 64).from_buffer_copy(h[64:]), C.byref(pf)), "open peer flags")
            self._peer_data[r], self._peer_flags[r] = pd.value, pf.value
        self._out = torch.empty(self.slot_elems, dtype=torch.float32, device=device)
        dist.barrier(group)

    def allreduce(self, x_f32: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """sum over ranks of x (fp32), returns fp32 (internal buffer) or writes `out` (bf16/fp16/f32)."""
        n = x_f32.numel()
        if x_f32.dtype != torch.float32 or not x_f32.is_contiguous() or n % 4 or n > self.slot_elems:
            raise ValueError(f"x_f32 must be a contiguous f32 tensor of a multiple of 4 and at most {self.slot_elems} "
                             f"elements, got {x_f32.dtype} {tuple(x_f32.shape)}")
        if out is not None and (out.dtype not in _OUT or out.numel() != n or not out.is_contiguous()):
            raise ValueError(f"out must be a contiguous bf16 / fp16 / f32 tensor of {n} elements, got {out.dtype} "
                             f"{tuple(out.shape)}")
        if out is None:
            out = self._out[:n].view(x_f32.shape)
        od = _OUT[out.dtype]
        rc = L.lib().b200_ep_allreduce(torch.cuda.current_stream().cuda_stream, self._peer_data, self._peer_flags,
                                       self.world, self.rank, x_f32.data_ptr(), n, self.slot_elems, out.data_ptr(), od)
        L.check(rc, "b200_ep_allreduce")
        return out

    def allreduce_norm(self, x_f32: torch.Tensor, out: torch.Tensor, residual: torch.Tensor | None = None,
                       gamma: torch.Tensor | None = None, gain: float = 1.0, eps: float = 1e-6,
                       sum_out: torch.Tensor | None = None) -> torch.Tensor:
        """out = RMSNorm(sum over ranks of x (+ residual)) in one kernel (push all-reduce, fixed-order local reduce);
        ``residual`` is updated in place like vLLM's fused_add_rms_norm."""
        if x_f32.dtype != torch.float32 or x_f32.dim() != 2 or not x_f32.is_contiguous() \
                or x_f32.numel() > self.slot_elems:
            raise ValueError(f"x_f32 must be a contiguous f32 [tokens, hidden] tensor of at most {self.slot_elems} "
                             f"elements, got {x_f32.dtype} {tuple(x_f32.shape)}")
        M, H = x_f32.shape
        _norm_args(out, M, H, residual, gamma)
        if sum_out is not None and (sum_out.dtype != torch.float32 or tuple(sum_out.shape) != (M, H)
                                    or not sum_out.is_contiguous()):
            raise ValueError(f"sum_out must be a contiguous f32 [{M}, {H}] tensor, got {sum_out.dtype} "
                             f"{tuple(sum_out.shape)}")
        rc = L.lib().b200_ep_allreduce_norm(torch.cuda.current_stream().cuda_stream, self._peer_data, self._peer_flags,
                                            self.world, self.rank, x_f32.data_ptr(), M, H, self.slot_elems,
                                            residual.data_ptr() if residual is not None else None,
                                            gamma.data_ptr() if gamma is not None else None, float(gain), float(eps),
                                            out.data_ptr(), sum_out.data_ptr() if sum_out is not None else None,
                                            1 if out.dtype == torch.float16 else 0)
        L.check(rc, "b200_ep_allreduce_norm")
        return out

    # ------------------------------------------------------------------------------ dispatch / combine all-to-all
    def a2a_init(self, m_local: int, hidden: int, top_k: int, experts_per_rank: int, group=None) -> None:
        """Allocate + exchange the static-slot all-to-all buffer for global batches of world*m_local tokens."""
        if m_local < 1 or hidden < 1 or top_k < 1:
            raise ValueError(f"m_local, hidden and top_k must be >= 1, got {m_local}, {hidden}, {top_k}")
        lib = L.lib()
        self.m_local, self.a2a_h, self.a2a_k, self.epr = m_local, hidden, top_k, experts_per_rank
        offs = [C.c_int64() for _ in range(4)]
        total = lib.b200_ep_a2a_layout(self.world * m_local, hidden, top_k, *[C.byref(o) for o in offs])
        self._a2a = C.c_void_p()
        h = (C.c_ubyte * 64)()
        L.check(lib.b200_ep_buffer_create(total, C.byref(self._a2a), h), "ep a2a buffer")
        handles = exchange_handles(bytes(h), group)
        self._peer_a2a = (C.c_void_p * 8)()
        for r, hh in enumerate(handles):
            if r == self.rank:
                self._peer_a2a[r] = self._a2a.value
                continue
            pd = C.c_void_p()
            L.check(lib.b200_ep_buffer_open((C.c_ubyte * 64).from_buffer_copy(hh), C.byref(pd)), "open peer a2a")
            self._peer_a2a[r] = pd.value
        base = self._a2a.value
        self.x_ptr, self.ids_ptr, self.w_ptr, self.y_ptr = (base + o.value for o in offs)
        dist.barrier(group)

    def _ids(self, ids_global: torch.Tensor) -> None:
        if ids_global.dtype != torch.int32 or tuple(ids_global.shape) != (self.m_local, self.a2a_k) \
                or not ids_global.is_contiguous():
            raise ValueError(f"ids_global must be a contiguous int32 [{self.m_local}, {self.a2a_k}] tensor, got "
                             f"{ids_global.dtype} {tuple(ids_global.shape)}")

    def dispatch(self, hidden_local: torch.Tensor, ids_global: torch.Tensor, weights: torch.Tensor) -> None:
        """Push this rank's [m_local, H] rows (+ remapped ids, weights) to the expert owners.  Afterwards run the
        local MoE on (x_ptr, ids_ptr, w_ptr) -> y_ptr with M = world * m_local."""
        if hidden_local.dtype not in (torch.bfloat16, torch.float16) or not hidden_local.is_contiguous() \
                or tuple(hidden_local.shape) != (self.m_local, self.a2a_h):
            raise ValueError(f"hidden_local must be a contiguous bf16 / fp16 [{self.m_local}, {self.a2a_h}] tensor, got "
                             f"{hidden_local.dtype} {tuple(hidden_local.shape)}")
        self._ids(ids_global)
        if weights.dtype != torch.float32 or weights.shape != ids_global.shape or not weights.is_contiguous():
            raise ValueError(f"weights must be a contiguous f32 [{self.m_local}, {self.a2a_k}] tensor, got "
                             f"{weights.dtype} {tuple(weights.shape)}")
        rc = L.lib().b200_ep_dispatch(torch.cuda.current_stream().cuda_stream, self._peer_a2a, self._peer_flags,
                                      self.world, self.rank, hidden_local.data_ptr(), ids_global.data_ptr(),
                                      weights.data_ptr(), self.m_local, self.a2a_k, self.a2a_h, self.epr)
        L.check(rc, "b200_ep_dispatch")

    def combine(self, ids_global: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        """Pull + sum the partial expert outputs of this rank's tokens; out [m_local, H] bf16 / fp16 / f32."""
        self._ids(ids_global)
        if out.dtype not in _OUT or tuple(out.shape) != (self.m_local, self.a2a_h) or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous bf16 / fp16 / f32 [{self.m_local}, {self.a2a_h}] tensor, got "
                             f"{out.dtype} {tuple(out.shape)}")
        od = _OUT[out.dtype]
        rc = L.lib().b200_ep_combine(torch.cuda.current_stream().cuda_stream, self._peer_a2a, self._peer_flags,
                                     self.world, self.rank, ids_global.data_ptr(), self.m_local, self.a2a_k, self.a2a_h,
                                     self.epr, out.data_ptr(), od)
        L.check(rc, "b200_ep_combine")
        return out

    def combine_norm(self, ids_global: torch.Tensor, out: torch.Tensor, residual: torch.Tensor | None = None,
                     gamma: torch.Tensor | None = None, gain: float = 1.0, eps: float = 1e-6) -> torch.Tensor:
        """combine() fused with residual add + RMSNorm (out bf16 / fp16 [m_local, H]; ``residual`` updated in place)."""
        self._ids(ids_global)
        _norm_args(out, self.m_local, self.a2a_h, residual, gamma)
        rc = L.lib().b200_ep_combine_norm(torch.cuda.current_stream().cuda_stream, self._peer_a2a, self._peer_flags,
                                          self.world, self.rank, ids_global.data_ptr(), self.m_local, self.a2a_k, self.a2a_h,
                                          self.epr, residual.data_ptr() if residual is not None else None,
                                          gamma.data_ptr() if gamma is not None else None, float(gain), float(eps),
                                          out.data_ptr(), 1 if out.dtype == torch.float16 else 0)
        L.check(rc, "b200_ep_combine_norm")
        return out
