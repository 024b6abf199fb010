"""torch-tensor front ends of the operator-level C ABI (routing, permutation, decode attention).

Names and argument meaning follow the reference's python op wrappers (vllm/_custom_ops.py ``topk_softmax``,
``grouped_topk``, ``moe_permute`` / ``moe_unpermute``, ``sm100_cutlass_mla_decode``) so that parity tests read
like the reference's own.  All tensors must live on the current CUDA device; there is no CPU path.

The C ABI sees only pointers and sizes, so every op checks the dtype, rank and shape of its tensors here, from metadata
alone (no value is read: that would synchronise and break CUDA-graph capture), and raises ValueError naming the argument
before it checks devices, converts or allocates anything.  Limits the C side checks itself are left to it.
"""
from __future__ import annotations

import torch

from . import _lib as L

_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
_OUT = {torch.bfloat16: 0, torch.float16: 1, torch.float32: 2}
_ACT = (torch.bfloat16, torch.float16)
_INT = (torch.int32, torch.int64)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _device(t: torch.Tensor, name: str) -> torch.Tensor:
    """t itself once it is known to be on a CUDA device: for tensors read or written in place through their strides."""
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (lvllm_b200 has no CPU path)")
    return t


def _cuda(t: torch.Tensor, name: str) -> torch.Tensor:
    return _device(t, name).contiguous()


_SCORING = {"softmax": 0, "sigmoid": 1, "sqrtsoftplus": 2}


def _i32(t: torch.Tensor, name: str) -> torch.Tensor:
    """int32 contiguous CUDA view; converts only when the caller passed another dtype."""
    t = _cuda(t, name)
    return t if t.dtype == torch.int32 else t.to(torch.int32)


def _per_token(T: int, **index_tensors) -> None:
    """Each tensor (positions, slot mappings, request rows, ...) must hold one integer per token; None is an absent one."""
    for name, v in index_tensors.items():
        if v is not None and (v.dtype not in _INT or v.numel() != T):
            raise ValueError(f"{name} needs one int32 / int64 entry per token ({T}), got {v.dtype} {tuple(v.shape)}")


def _int_tensor(t: torch.Tensor, name: str, dim: int | None = None) -> None:
    if t.dtype not in _INT or (dim is not None and t.dim() != dim):
        raise ValueError(f"{name} must be an int32 / int64 tensor{f' of rank {dim}' if dim else ''}, got {t.dtype} "
                         f"{tuple(t.shape)}")


def _cos_sin_cache(cs: torch.Tensor, dtype: torch.dtype = torch.float32) -> None:
    """The RoPE table [max_pos, 64] = cos | sin that the kernels index by position."""
    if cs.dtype != dtype or cs.dim() != 2 or cs.shape[1] != 64 or cs.shape[0] < 1:
        raise ValueError(f"cos_sin_cache must be {dtype} [max_pos, 64], got {cs.dtype} {tuple(cs.shape)}")


def _bias(bias: torch.Tensor | None, E: int) -> None:
    if bias is not None and (not bias.is_floating_point() or bias.numel() != E):
        raise ValueError(f"e_score_correction_bias must hold one float per expert ({E}), got {bias.dtype} "
                         f"{tuple(bias.shape)}")


def _gating(g: torch.Tensor) -> tuple[int, int]:
    if g.dtype not in _DT or g.dim() != 2:
        raise ValueError(f"gating_output must be f32 / bf16 / f16 [tokens, experts], got {g.dtype} {tuple(g.shape)}")
    return g.shape[0], g.shape[1]


def _hash_args(hash_indices_table: torch.Tensor, input_ids: torch.Tensor | None, topk: int, M: int) -> None:
    if input_ids is None:
        raise ValueError("hash routing needs input_ids")
    _int_tensor(hash_indices_table, "hash_indices_table", 2)
    if hash_indices_table.shape[1] != topk:
        raise ValueError(f"hash_indices_table must be [vocab, {topk}], got {tuple(hash_indices_table.shape)}")
    _per_token(M, input_ids=input_ids)


_workspaces: dict = {}


def _persistent_workspace(kind: str, device: torch.device, nbytes: int) -> torch.Tensor:
    """A zero-filled byte buffer of at least nbytes, kept per (kind, device, stream) for kernels whose arrival counters
    must start at zero and that hand them back zeroed.  A larger request replaces the buffer, but the outgrown one stays
    referenced: a CUDA graph captured against it still writes into it on replay."""
    bufs = _workspaces.setdefault((kind, device.index, _stream()), [])
    if not bufs or bufs[-1].numel() < nbytes:
        bufs.append(torch.zeros(nbytes, dtype=torch.uint8, device=device))
    return bufs[-1]


def fused_topk(gating_output: torch.Tensor, topk: int, renormalize: bool, scoring_func: str = "softmax",
               e_score_correction_bias: torch.Tensor | None = None, routed_scaling_factor: float = 1.0,
               return_token_expert_indices: bool = False):
    """reference fused_topk_router.py:81-124 -> _moe_C.topk_softmax / topk_sigmoid, and fused_topk_bias_router.py ->
    topk_softplus_sqrt for ``scoring_func="sqrtsoftplus"`` (DeepSeek-V4: the bias selects, the weights are the
    unbiased scores)."""
    M, E = _gating(gating_output)
    _bias(e_score_correction_bias, E)
    g = _cuda(gating_output, "gating_output")
    w = torch.empty(M, topk, dtype=torch.float32, device=g.device)
    ids = torch.empty(M, topk, dtype=torch.int32, device=g.device)
    tei = torch.empty(M, topk, dtype=torch.int32, device=g.device) if return_token_expert_indices else None
    bias = _cuda(e_score_correction_bias.float(), "bias") if e_score_correction_bias is not None else None
    rc = L.lib().b200_topk_gating(_stream(), g.data_ptr(), _DT[g.dtype], bias.data_ptr() if bias is not None else None,
                                  M, E, topk, _SCORING[scoring_func], int(renormalize),
                                  float(routed_scaling_factor), w.data_ptr(), ids.data_ptr(),
                                  tei.data_ptr() if tei is not None else None)
    L.check(rc, "b200_topk_gating")
    return (w, ids, tei) if return_token_expert_indices else (w, ids)


def grouped_topk(gating_output: torch.Tensor, topk: int, renormalize: bool, num_expert_group: int, topk_group: int,
                 scoring_func: str = "sigmoid", routed_scaling_factor: float = 1.0,
                 e_score_correction_bias: torch.Tensor | None = None):
    """reference grouped_topk_router.py:28-166 (fused kernel semantics: ordered output)."""
    M, E = _gating(gating_output)
    _bias(e_score_correction_bias, E)
    g = _cuda(gating_output, "gating_output")
    if scoring_func == "softmax":  # reference applies the softmax in python first (:58-70)
        g = torch.softmax(g.float(), dim=-1)
        scoring = 0
    else:
        scoring = 1
    w = torch.empty(M, topk, dtype=torch.float32, device=g.device)
    ids = torch.empty(M, topk, dtype=torch.int32, device=g.device)
    bias = _cuda(e_score_correction_bias.float(), "bias") if e_score_correction_bias is not None else None
    rc = L.lib().b200_grouped_topk(_stream(), g.data_ptr(), _DT[g.dtype], bias.data_ptr() if bias is not None else None,
                                   M, E, num_expert_group, topk_group, topk, scoring, int(renormalize),
                                   float(routed_scaling_factor), w.data_ptr(), ids.data_ptr())
    L.check(rc, "b200_grouped_topk")
    return w, ids


def hash_topk(gating_output: torch.Tensor, topk: int, renormalize: bool, input_ids: torch.Tensor,
              hash_indices_table: torch.Tensor, routed_scaling_factor: float = 1.0):
    """DeepSeek-V4 hash routing (reference topk_softplus_sqrt with ``hash_indices_table``): ids = table[input_ids], in
    table order; weights = sqrt(softplus(logits)) of those experts.  table [vocab, topk]; ids or table entries out of
    range give id -1 and weight 0.  Returns (topk_weights f32 [M,k], topk_ids i32 [M,k])."""
    M, E = _gating(gating_output)
    _hash_args(hash_indices_table, input_ids, topk, M)
    g = _cuda(gating_output, "gating_output")
    tab = _i32(hash_indices_table, "hash_indices_table")
    ids_in = _i32(input_ids, "input_ids").reshape(-1)
    w = torch.empty(M, topk, dtype=torch.float32, device=g.device)
    ids = torch.empty(M, topk, dtype=torch.int32, device=g.device)
    rc = L.lib().b200_hash_topk(_stream(), g.data_ptr(), _DT[g.dtype], ids_in.data_ptr(), tab.data_ptr(), tab.shape[0], M,
                                E, topk, int(renormalize), float(routed_scaling_factor), w.data_ptr(), ids.data_ptr())
    L.check(rc, "b200_hash_topk")
    return w, ids


def router_topk(hidden_states: torch.Tensor, gate_weight: torch.Tensor, topk: int, renormalize: bool,
                scoring_func: str = "softmax", e_score_correction_bias: torch.Tensor | None = None,
                routed_scaling_factor: float = 1.0, num_expert_group: int = 0, topk_group: int = 0,
                expert_map: torch.Tensor | None = None, return_logits: bool = False, n_shared: int = 0,
                shared_local_base: int = -1, shared_weight: float = 1.0, input_ids: torch.Tensor | None = None,
                hash_indices_table: torch.Tensor | None = None):
    """Fused router: GateLinear.forward (reference router/gate_linear.py:171-221) + fused_topk / grouped_topk
    (fused_topk_router.py:81-124, grouped_topk_router.py:28-166) + global_to_local_expert_ids in ONE kernel.
    hidden [M,H], gate_weight [E,H] (same 16-bit dtype).  ``num_expert_group > 0`` selects DeepSeek grouped routing.
    ``n_shared`` > 0 appends always-on columns for shared experts held at local ids shared_local_base + s (weight
    ``shared_weight``; reference runner/shared_experts.py) — local_ids are then always returned.
    ``scoring_func="sqrtsoftplus"`` is DeepSeek-V4's top-k; with ``hash_indices_table`` [vocab, k] and ``input_ids``
    it is V4's hash routing (as ``hash_topk``, on the same kernel's logits).
    Returns (topk_weights f32 [M,k'], topk_ids i32 [M,k'] global, local_ids i32 [M,k'] | None[, logits f32 [M,E]]),
    k' = k + n_shared."""
    h, wg = hidden_states, gate_weight
    if h.dtype not in _ACT or h.dim() != 2:
        raise ValueError(f"hidden_states must be bf16 / f16 [tokens, hidden], got {h.dtype} {tuple(h.shape)}")
    M, H = h.shape
    if wg.dtype != h.dtype or wg.dim() != 2 or wg.shape[1] != H:
        raise ValueError(f"gate_weight must be {h.dtype} [experts, {H}], got {wg.dtype} {tuple(wg.shape)}")
    E = wg.shape[0]
    _bias(e_score_correction_bias, E)
    if expert_map is not None:   # the kernel reads expert_map[id] for every id < E
        _int_tensor(expert_map, "expert_map")
        if expert_map.numel() < E:
            raise ValueError(f"expert_map must hold an entry per expert ({E}), got {tuple(expert_map.shape)}")
    if num_expert_group > 0 and scoring_func not in ("sigmoid", "none"):
        raise ValueError(f"grouped routing (num_expert_group > 0) scores by sigmoid or none, got {scoring_func!r}")
    if hash_indices_table is not None:
        _hash_args(hash_indices_table, input_ids, topk, M)
    h, wg = _cuda(h, "hidden_states"), _cuda(wg, "gate_weight")
    dev = h.device
    lib = L.lib()
    # at least 1 MiB: every batch that needs less shares the first buffer
    ws = _persistent_workspace("router", dev, max(int(lib.b200_router_workspace_bytes(M, E, H)), 1 << 20))
    kk = topk + n_shared
    w = torch.empty(M, kk, dtype=torch.float32, device=dev)
    ids = torch.empty(M, kk, dtype=torch.int32, device=dev)
    loc = torch.empty(M, kk, dtype=torch.int32, device=dev) if (expert_map is not None or n_shared) else None
    lg = torch.empty(M, E, dtype=torch.float32, device=dev) if return_logits else None
    bias = _cuda(e_score_correction_bias.float(), "bias") if e_score_correction_bias is not None else None
    em = _cuda(expert_map.to(torch.int32), "expert_map") if expert_map is not None else None
    if num_expert_group > 0:
        mode, scoring = 2, 1 if scoring_func == "sigmoid" else 0
    else:
        mode, scoring = {"softmax": 0, "sigmoid": 1, "sqrtsoftplus": 3}[scoring_func], 0
    args = (_stream(), h.data_ptr(), 1 if h.dtype == torch.float16 else 0, wg.data_ptr(), M, E, H,
            bias.data_ptr() if bias is not None else None, mode, scoring, topk, int(renormalize),
            int(num_expert_group), int(topk_group), float(routed_scaling_factor),
            em.data_ptr() if em is not None else None, int(n_shared), int(shared_local_base),
            float(shared_weight), ws.data_ptr(), ws.numel(), w.data_ptr(),
            ids.data_ptr(), loc.data_ptr() if loc is not None else None,
            lg.data_ptr() if lg is not None else None)
    if hash_indices_table is None:
        L.check(lib.b200_router_topk(*args), "b200_router_topk")
    else:
        tab = _i32(hash_indices_table, "hash_indices_table")
        ids_in = _i32(input_ids, "input_ids").reshape(-1)
        L.check(lib.b200_router_hash_topk(*args, ids_in.data_ptr(), tab.data_ptr(), tab.shape[0]),
                "b200_router_hash_topk")
    return (w, ids, loc, lg) if return_logits else (w, ids, loc)


def global_to_local_expert_ids(topk_ids: torch.Tensor, expert_map: torch.Tensor) -> torch.Tensor:
    """reference routed_experts.py:1332-1342."""
    _int_tensor(topk_ids, "topk_ids")
    _int_tensor(expert_map, "expert_map")
    ids = _cuda(topk_ids.to(torch.int32), "topk_ids")
    em = _cuda(expert_map.to(torch.int32), "expert_map")
    out = torch.empty_like(ids)
    L.check(L.lib().b200_global_to_local_ids(_stream(), ids.data_ptr(), em.data_ptr(), em.numel(), ids.numel(),
                                             out.data_ptr()), "b200_global_to_local_ids")
    return out


def moe_permute(hidden_states: torch.Tensor | None, topk_ids: torch.Tensor, n_local_expert: int):
    """Stable sort by expert (reference moe_permute_unpermute.py:105-231).  Returns
    (permuted_hidden | None, sorted_slot i32 [M*k], expert_first_token_offset i64 [E+1], inv_permuted_idx i32 [M,k])."""
    _int_tensor(topk_ids, "topk_ids", 2)
    M, k = topk_ids.shape
    if hidden_states is not None and (hidden_states.dtype not in _ACT or hidden_states.dim() != 2
                                      or hidden_states.shape[0] != M):
        raise ValueError(f"hidden_states must be bf16 / f16 [{M}, hidden] (a row per token of topk_ids), got "
                         f"{hidden_states.dtype} {tuple(hidden_states.shape)}")
    ids = _cuda(topk_ids.to(torch.int32), "topk_ids")
    dev = ids.device
    sorted_slot = torch.empty(M * k, dtype=torch.int32, device=dev)
    first = torch.empty(n_local_expert + 1, dtype=torch.int64, device=dev)
    inv = torch.empty(M, k, dtype=torch.int32, device=dev)
    perm = None
    hp, H = None, 0
    if hidden_states is not None:
        h = _cuda(hidden_states, "hidden_states")
        H = h.shape[1]
        perm = torch.zeros(M * k, H, dtype=h.dtype, device=dev)
        hp = h.data_ptr()
    rc = L.lib().b200_moe_permute(_stream(), hp, ids.data_ptr(), M, k, n_local_expert, H, sorted_slot.data_ptr(),
                                  first.data_ptr(), inv.data_ptr(), perm.data_ptr() if perm is not None else None)
    L.check(rc, "b200_moe_permute")
    return perm, sorted_slot, first, inv


def moe_unpermute(permuted: torch.Tensor, topk_weights: torch.Tensor, inv_permuted_idx: torch.Tensor,
                  out_dtype: torch.dtype | None = None) -> torch.Tensor:
    """out[t] = sum_j w[t,j] * permuted[inv[t,j]] in fp32 (reference moe_permute_unpermute.py:234-277)."""
    if permuted.dtype not in _ACT or permuted.dim() != 2:
        raise ValueError(f"permuted must be bf16 / f16 [rows, hidden], got {permuted.dtype} {tuple(permuted.shape)}")
    _int_tensor(inv_permuted_idx, "inv_permuted_idx", 2)
    if not topk_weights.is_floating_point() or topk_weights.shape != inv_permuted_idx.shape:
        raise ValueError(f"topk_weights must be float {tuple(inv_permuted_idx.shape)} like inv_permuted_idx, got "
                         f"{topk_weights.dtype} {tuple(topk_weights.shape)}")
    od = out_dtype or permuted.dtype
    if od not in _OUT:
        raise ValueError(f"out_dtype must be bf16, f16 or f32, got {od}")
    p = _cuda(permuted, "permuted")
    w = _cuda(topk_weights.float(), "topk_weights")
    inv = _cuda(inv_permuted_idx.to(torch.int32), "inv_permuted_idx")
    M, k = inv.shape
    H = p.shape[1]
    out = torch.empty(M, H, dtype=od, device=p.device)
    rc = L.lib().b200_moe_unpermute(_stream(), p.data_ptr(), 1 if p.dtype == torch.float16 else 0, w.data_ptr(),
                                    inv.data_ptr(), M, k, H, out.data_ptr(), _OUT[od])
    L.check(rc, "b200_moe_unpermute")
    return out


def rmsnorm_cast(x_f32: torch.Tensor, out: torch.Tensor, gain: float = 1.0, eps: float = 1e-6) -> torch.Tensor:
    """out = cast(x * gain * rsqrt(mean(x^2)+eps)) — the cast Lvllm applies to lk_moe's fp32 output
    (reference routed_experts.py:1855) fused with the RMS normalisation that follows in the layer."""
    if x_f32.dtype != torch.float32 or x_f32.dim() != 2:
        raise ValueError(f"x must be f32 [tokens, hidden], got {x_f32.dtype} {tuple(x_f32.shape)}")
    if out.dtype not in _ACT or out.shape != x_f32.shape or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous bf16 / f16 {tuple(x_f32.shape)} tensor, got {out.dtype} "
                         f"{tuple(out.shape)}")
    x = _cuda(x_f32, "x")
    _device(out, "out")
    M, H = x.shape
    L.check(L.lib().b200_rmsnorm_cast(_stream(), x.data_ptr(), out.data_ptr(), M, H, float(gain), float(eps),
                                      1 if out.dtype == torch.float16 else 0), "b200_rmsnorm_cast")
    return out


def _mla_splits(max_keys: int, rows: int) -> int:
    """Default split count of the MLA-family decode kernel (mla_decode, mla_decode_sparse, dsv4_sparse_decode).  A CTA =
    (grid row, split, value-dim quarter) walks ceil(tiles / splits) of the ceil(max_keys / 128) key tiles with an online
    softmax; rows = grid rows (requests x q-groups, or query tokens).  Enough splits to fill ~2 waves of the 132 SMs, no
    more: each split costs an fp32 partial of the output."""
    return max(1, min(-(-max_keys // 128), 264 // (4 * rows)))


def _mla_queries(q_nope: torch.Tensor, q_pe: torch.Tensor, dtypes: tuple) -> tuple[int, int]:
    """Checks the absorbed MLA query halves q_nope [T, Hq, 512] / q_pe [T, Hq, 64] of one dtype; returns (T, Hq)."""
    if q_nope.dtype not in dtypes or q_nope.dim() != 3 or q_nope.shape[2] != 512:
        raise ValueError(f"q_nope must be {' / '.join(map(str, dtypes))} [tokens, heads, 512], got {q_nope.dtype} "
                         f"{tuple(q_nope.shape)}")
    T, Hq, _ = q_nope.shape
    if q_pe.dtype != q_nope.dtype or tuple(q_pe.shape) != (T, Hq, 64):
        raise ValueError(f"q_pe must be {q_nope.dtype} [{T}, {Hq}, 64], got {q_pe.dtype} {tuple(q_pe.shape)}")
    return T, Hq


def _w_uv(w_uv: torch.Tensor | None, Hq: int) -> None:
    if w_uv is not None and (w_uv.dtype != torch.bfloat16 or tuple(w_uv.shape) != (Hq, 512, 128)):
        raise ValueError(f"w_uv must be bf16 [{Hq}, 512, 128], got {w_uv.dtype} {tuple(w_uv.shape)}")


def mla_decode(q_nope: torch.Tensor, q_pe: torch.Tensor, kv_c_and_k_pe_cache: torch.Tensor, seq_lens: torch.Tensor,
               page_table: torch.Tensor, sm_scale: float, num_kv_splits: int = 0, max_seq_len: int | None = None,
               q_scale: float = 1.0, k_scale: float = 1.0, w_uv: torch.Tensor | None = None, q_len_per_req: int = 1):
    """Paged MLA decode; mirrors ops.sm100_cutlass_mla_decode (reference vllm/_custom_ops.py:3212,
    backends/mla/cutlass_mla.py:176-257).  bf16 q + bf16 cache, or an e4m3 cache (``torch.float8_e4m3fn``, 576 B / token)
    with bf16 or e4m3 queries (the reference's fp8 mode; q_scale / k_scale = per-tensor dequantisation scales).
    ``max_seq_len`` (host-side bound on seq_lens) sizes the split count / workspace instead of the page-table width.
    B = seq_lens.numel(); Q = ``q_len_per_req`` query tokens per request (speculative-decode verification of
    multi-token-prediction drafts, the reference FlashMLA backend's uniform query length with causal=True,
    backends/mla/flashmla.py:120, :284-344): q_nope [B*Q,Hq,512] / q_pe [B*Q,Hq,64] hold request b's Q tokens contiguous in
    draft order, seq_lens[b] counts all its keys including the Q new ones, and token i attends to keys
    [0, seq_lens[b] - Q + i] (a row with no visible key gives out 0 and lse -inf).  Q = 1 (the default) is the
    single-token decode.
    With ``w_uv`` [Hq,512,128] the split merge is fused with the v up-projection and (out_v [B*Q,Hq,128], out, lse) is
    returned.  Returns (out bf16 [B*Q,Hq,512], lse f32 [B*Q,Hq])."""
    f8 = torch.float8_e4m3fn
    kv = kv_c_and_k_pe_cache
    if kv.dtype not in (torch.bfloat16, f8) or kv.dim() != 3 or kv.shape[2] != 576:
        raise ValueError(f"kv_cache must be bf16 or e4m3 [pages, page, 576], got {kv.dtype} {tuple(kv.shape)}")
    T, Hq = _mla_queries(q_nope, q_pe, (torch.bfloat16, f8) if kv.dtype == f8 else (torch.bfloat16,))
    _int_tensor(seq_lens, "seq_lens")
    _int_tensor(page_table, "page_table", 2)
    Q = int(q_len_per_req)
    B = seq_lens.numel()
    if T != B * Q:
        raise ValueError(f"q_nope / q_pe must hold q_len_per_req = {Q} tokens per request: {B * Q} rows for {B} seq_lens, "
                         f"got {T}")
    if page_table.shape[0] < B:   # the kernel reads row b of the table for every request b < B
        raise ValueError(f"page_table must have a row per request ({B}), got {tuple(page_table.shape)}")
    _w_uv(w_uv, Hq)
    qn, qp = _cuda(q_nope, "q_nope"), _cuda(q_pe, "q_pe")
    kv = _cuda(kv, "kv_cache")
    page = kv.shape[1]
    sl = _cuda(seq_lens.reshape(-1).to(torch.int32), "seq_lens")
    pt = _cuda(page_table.to(torch.int32), "page_table")
    max_pages = pt.shape[1]
    if max_seq_len is not None:
        # the kernel only walks pages below the bound: a narrower view of the table keeps the split count (and the
        # B*Q*Hq*splits*514*4-byte workspace) proportional to the real context, not to max_model_len
        max_pages = min(max_pages, -(-int(max_seq_len) // page))
        if max_pages != pt.shape[1]:
            pt = pt[:, :max_pages].contiguous()
    if num_kv_splits <= 0:
        qg = max(1, min(Q, 128 // Hq))   # draft tokens per q-group (the kernel's 128 MMA rows)
        num_kv_splits = _mla_splits(max_pages * page, B * -(-Q // qg))   # grid rows: requests x q-groups
    ws = torch.empty(L.lib().b200_mla_decode_workspace_bytes(T, Hq, num_kv_splits), dtype=torch.uint8, device=qn.device)
    out = torch.empty(T, Hq, 512, dtype=torch.bfloat16, device=qn.device)
    lse = torch.empty(T, Hq, dtype=torch.float32, device=qn.device)
    args = [_stream(), qn.data_ptr(), qp.data_ptr(), int(qn.dtype == f8), kv.data_ptr(), int(kv.dtype == f8), float(q_scale),
            float(k_scale), sl.data_ptr(), pt.data_ptr(), B, Q, Hq, page, max_pages, float(sm_scale), num_kv_splits,
            ws.data_ptr(), out.data_ptr(), lse.data_ptr()]
    if w_uv is not None:
        # split merge fused with the v up-projection (reference _v_up_proj, mla_attention.py:1154-1176)
        wv = _cuda(w_uv, "w_uv")
        out_v = torch.empty(T, Hq, 128, dtype=torch.bfloat16, device=qn.device)
        L.check(L.lib().b200_mla_decode_spec(*args, wv.data_ptr(), out_v.data_ptr()), "b200_mla_decode_vup")
        return out_v, out, lse
    L.check(L.lib().b200_mla_decode_spec(*args, None, None), "b200_mla_decode")
    return out, lse


def mla_decode_sparse(q_nope: torch.Tensor, q_pe: torch.Tensor, kv_cache: torch.Tensor, topk_indices: torch.Tensor,
                      req_id: torch.Tensor, page_table: torch.Tensor, sm_scale: float, num_kv_splits: int = 0,
                      w_uv: torch.Tensor | None = None):
    """Sparse MLA decode of DeepSeek-V3.2 / GLM-5 layers (config.index_topk): query token t attends only to the keys
    topk_indices[t] its lightning indexer picked (request-local positions of request req_id[t]; -1, or a position past the
    page table, is no key).  Replaces the reference's index conversion plus FlashMLA sparse decode
    (sparse_utils.py:120, flashmla_sparse.py:587-611, 763-830) with one kernel.  q_nope [T,Hq,512] / q_pe [T,Hq,64] bf16;
    kv_cache bf16 [pages, page, 576] or the fp8_ds_mla cache, uint8 [pages, page, 656]; topk_indices int32 [T, topk];
    req_id [T]; page_table [R, max_pages].  A token with no valid entry gets out 0 and lse -inf.
    With ``w_uv`` [Hq,512,128] the split merge is fused with the v up-projection and (out_v [T,Hq,128], out, lse) is
    returned.  Returns (out bf16 [T,Hq,512], lse f32 [T,Hq])."""
    if q_nope.dtype != torch.bfloat16 or q_pe.dtype != torch.bfloat16:
        raise ValueError(f"sparse MLA decode takes bf16 queries, got {q_nope.dtype} / {q_pe.dtype}")
    if kv_cache.dim() != 3 or (kv_cache.dtype, kv_cache.shape[-1]) not in ((torch.bfloat16, 576), (torch.uint8, 656)):
        raise ValueError(f"kv_cache must be bf16 [pages, page, 576] or fp8_ds_mla uint8 [pages, page, 656], "
                         f"got {kv_cache.dtype} {tuple(kv_cache.shape)}")
    T, Hq = _mla_queries(q_nope, q_pe, (torch.bfloat16,))
    _int_tensor(topk_indices, "topk_indices", 2)
    if topk_indices.shape[0] != T:
        raise ValueError(f"topk_indices needs one row per query token ({T}), got {tuple(topk_indices.shape)}")
    _per_token(T, req_id=req_id)
    _int_tensor(page_table, "page_table", 2)
    _w_uv(w_uv, Hq)
    qn, qp = _cuda(q_nope, "q_nope"), _cuda(q_pe, "q_pe")
    kv = _cuda(kv_cache, "kv_cache")
    idx = _cuda(topk_indices.to(torch.int32), "topk_indices")
    rid = _cuda(req_id.reshape(-1).to(torch.int32), "req_id")
    pt = _cuda(page_table.to(torch.int32), "page_table")
    topk = idx.shape[1]
    if num_kv_splits <= 0:
        num_kv_splits = _mla_splits(topk, T)
    ws = torch.empty(L.lib().b200_mla_decode_workspace_bytes(T, Hq, num_kv_splits), dtype=torch.uint8, device=qn.device)
    out = torch.empty(T, Hq, 512, dtype=torch.bfloat16, device=qn.device)
    lse = torch.empty(T, Hq, dtype=torch.float32, device=qn.device)
    args = [_stream(), qn.data_ptr(), qp.data_ptr(), kv.data_ptr(), 2 if kv.dtype == torch.uint8 else 0, idx.data_ptr(), topk,
            rid.data_ptr(), pt.data_ptr(), pt.shape[1], T, Hq, kv.shape[1], float(sm_scale), num_kv_splits, ws.data_ptr(),
            out.data_ptr(), lse.data_ptr()]
    if w_uv is not None:
        wv = _cuda(w_uv, "w_uv")
        out_v = torch.empty(T, Hq, 128, dtype=torch.bfloat16, device=qn.device)
        L.check(L.lib().b200_mla_decode_sparse(*args, wv.data_ptr(), out_v.data_ptr()), "b200_mla_decode_sparse")
        return out_v, out, lse
    L.check(L.lib().b200_mla_decode_sparse(*args, None, None), "b200_mla_decode_sparse")
    return out, lse


def _dsv4_cache(c: torch.Tensor, name: str):
    """(block_size, num_blocks, block stride in bytes) of a 584-byte-per-token cache, uint8 [blocks, block_size, 584];
    blocks may be padded (stride(0) > block_size * 584), the bytes of a block are addressed as the per-block layout."""
    if c.dtype != torch.uint8 or c.dim() != 3 or c.shape[2] != 584 or c.stride(2) != 1 or c.stride(1) != 584:
        raise ValueError(f"{name} must be uint8 [blocks, block_size, 584] with rows of 584 contiguous bytes, "
                         f"got {c.dtype} {tuple(c.shape)} strides {c.stride()}")
    return c.shape[1], c.shape[0], c.stride(0)


def dsv4_sparse_decode(q: torch.Tensor, swa_cache: torch.Tensor, swa_indices: torch.Tensor, swa_lens: torch.Tensor,
                       sm_scale: float, attn_sink: torch.Tensor | None = None, extra_cache: torch.Tensor | None = None,
                       extra_indices: torch.Tensor | None = None, extra_lens: torch.Tensor | None = None,
                       num_kv_splits: int = 0) -> torch.Tensor:
    """Sparse attention decode of DeepSeek-V4 layers (the reference's FlashMLA call with indices, extra_k_cache and attn_sink,
    models/deepseek_v4/nvidia/flashmla.py:151-244).  q bf16 [T, Hq, 512] (448 NoPE | 64 RoPE dims); the caches are uint8
    [blocks, block_size, 584] (block layout of flashmla_sparse.py:76-85: block_size x 576 data bytes, then block_size x 8
    ue8m0 scale bytes).  Token t attends to swa_indices[t, :swa_lens[t]] (global slots of swa_cache) followed by
    extra_indices[t, :extra_lens[t]] (global slots of extra_cache, compressed layers only); a slot < 0 or past its cache is
    no key.  One cache row is both key and value.  attn_sink f32 [Hq] adds e^(sink) to each head's softmax denominator.
    A token with no valid key gets out 0.  Returns out bf16 [T, Hq, 512]."""
    if q.dtype != torch.bfloat16 or q.dim() != 3 or q.shape[2] != 512:
        raise ValueError(f"q must be bf16 [tokens, heads, 512], got {q.dtype} {tuple(q.shape)}")
    T, Hq, _ = q.shape
    if not 1 <= Hq <= 128 or not 1 <= T <= 65535:
        raise ValueError(f"dsv4 sparse decode takes 1-128 heads and 1-65535 tokens, got {Hq} heads, {T} tokens")
    sbs, snb, sstride = _dsv4_cache(swa_cache, "swa_cache")

    def _check_lists(idx, lens, name):
        if idx.dtype not in _INT or idx.dim() != 2 or idx.shape[0] != T or idx.shape[1] < 1:
            raise ValueError(f"{name}_indices must be int [{T}, topk >= 1], got {idx.dtype} {tuple(idx.shape)}")
        _per_token(T, **{f"{name}_lens": lens})

    _check_lists(swa_indices, swa_lens, "swa")
    if (extra_cache is None) != (extra_indices is None) or (extra_indices is None) != (extra_lens is None):
        raise ValueError("extra_cache, extra_indices and extra_lens go together")
    if extra_cache is not None:
        ebs, enb, estride = _dsv4_cache(extra_cache, "extra_cache")
        _check_lists(extra_indices, extra_lens, "extra")
    else:
        ebs, enb, estride = 0, 0, 0
    if attn_sink is not None and (not attn_sink.is_floating_point() or attn_sink.numel() != Hq):
        raise ValueError(f"attn_sink must hold one float per head ({Hq}), got {attn_sink.dtype} {tuple(attn_sink.shape)}")
    q = _cuda(q, "q")
    sc = _device(swa_cache, "swa_cache")
    si, sl = _i32(swa_indices, "swa_indices"), _i32(swa_lens.reshape(-1), "swa_lens")
    ec, ei, el = None, None, None
    if extra_cache is not None:
        ec = _device(extra_cache, "extra_cache")
        ei, el = _i32(extra_indices, "extra_indices"), _i32(extra_lens.reshape(-1), "extra_lens")
    sink = _cuda(attn_sink.reshape(-1).to(torch.float32), "attn_sink") if attn_sink is not None else None
    if num_kv_splits <= 0:
        num_kv_splits = _mla_splits(si.shape[1] + (ei.shape[1] if ei is not None else 0), T)
    ws = torch.empty(L.lib().b200_mla_decode_workspace_bytes(T, Hq, num_kv_splits), dtype=torch.uint8, device=q.device)
    out = torch.empty(T, Hq, 512, dtype=torch.bfloat16, device=q.device)
    rc = L.lib().b200_dsv4_sparse_decode(
        _stream(), q.data_ptr(), T, Hq, sc.data_ptr(), sbs, snb, sstride, si.data_ptr(), si.shape[1], sl.data_ptr(),
        ec.data_ptr() if ec is not None else None, ebs, enb, estride, ei.data_ptr() if ei is not None else None,
        ei.shape[1] if ei is not None else 0, el.data_ptr() if el is not None else None,
        sink.data_ptr() if sink is not None else None, float(sm_scale), int(num_kv_splits), ws.data_ptr(), out.data_ptr())
    L.check(rc, "b200_dsv4_sparse_decode")
    return out


def dsv4_qnorm_rope_kv_insert(q: torch.Tensor, kv: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor,
                              slot_mapping: torch.Tensor, swa_cache: torch.Tensor, q_head_padded: int,
                              eps: float) -> torch.Tensor:
    """DeepSeek-V4 q-norm + RoPE + cache insert in one launch (the reference's
    fused_deepseek_v4_qnorm_rope_kv_rope_quant_insert).  q bf16 [T, Hq, 512] gets a per-head RMSNorm without weight and GPT-J
    pair RoPE of its last 64 dims (fp32, rounded to bf16 once); kv bf16 [T, 512] (after kv_norm) gets the RoPE, its 448 NoPE
    dims are quantised per 64 to e4m3 with a ue8m0 scale, and the row goes to slot_mapping[t] of swa_cache (uint8
    [blocks, block_size, 584]; a slot < 0 writes nothing).  positions int64 [T]; cos_sin_cache f32 [max_pos, 64] = cos | sin.
    Returns q_out bf16 [T, q_head_padded, 512], heads past Hq zero."""
    if q.dtype != torch.bfloat16 or q.dim() != 3 or q.shape[2] != 512:
        raise ValueError(f"q must be bf16 [tokens, heads, 512], got {q.dtype} {tuple(q.shape)}")
    T, Hq, _ = q.shape
    if kv.dtype != torch.bfloat16 or tuple(kv.shape) != (T, 512):
        raise ValueError(f"kv must be bf16 [{T}, 512], got {kv.dtype} {tuple(kv.shape)}")
    if int(q_head_padded) < Hq:
        raise ValueError(f"q_head_padded ({q_head_padded}) must be >= the head count ({Hq})")
    _cos_sin_cache(cos_sin_cache)
    _per_token(T, positions=positions, slot_mapping=slot_mapping)
    bs, nb, stride = _dsv4_cache(swa_cache, "swa_cache")
    q, kv = _cuda(q, "q"), _cuda(kv, "kv")
    cs = _cuda(cos_sin_cache, "cos_sin_cache")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    slots = _cuda(slot_mapping.reshape(-1).to(torch.int64), "slot_mapping")
    c = _device(swa_cache, "swa_cache")
    q_out = torch.empty(T, int(q_head_padded), 512, dtype=torch.bfloat16, device=q.device)
    rc = L.lib().b200_dsv4_qnorm_rope_kv_insert(_stream(), q.data_ptr(), kv.data_ptr(), pos.data_ptr(), cs.data_ptr(),
                                                cs.shape[0], slots.data_ptr(), c.data_ptr(), bs, nb, stride, q_out.data_ptr(),
                                                T, Hq, int(q_head_padded), float(eps))
    L.check(rc, "b200_dsv4_qnorm_rope_kv_insert")
    return q_out


def dsv4_compress(kv_score: torch.Tensor, ape: torch.Tensor, positions: torch.Tensor, state_cache: torch.Tensor,
                  slot_mapping: torch.Tensor, token_to_req: torch.Tensor, block_table: torch.Tensor,
                  norm_weight: torch.Tensor, eps: float, cos_sin_cache: torch.Tensor, kv_cache: torch.Tensor,
                  kv_slot_mapping: torch.Tensor, compress_ratio: int) -> None:
    """The DeepSeek-V4 KV compressor (the reference's DeepseekCompressor.forward): the state write, then for every token
    that closes a window of ``compress_ratio`` positions the softmax-pooled compression of the window, RMSNorm, GPT-J RoPE
    of the last 64 dims and the fp8 store.  D = norm_weight.numel(); coff = 2 (overlapping windows) for ratio 4, 1 for 128.
    kv_score f32 [T, 2 coff D] = kv | score (the fused wkv / wgate GEMM output; rows may be strided); ape f32 [ratio, coff D];
    positions [T]; state_cache f32 [blocks, state_block_size, 2 coff D], slot_mapping [T] its slots (< 0: nothing written);
    token_to_req [T] rows of block_table [*, max_blocks] (state block numbers); norm_weight bf16 [D]; cos_sin_cache f32
    [max_pos, 64] = cos | sin.  kv_cache, written at kv_slot_mapping[t] (< 0 or past the cache: nothing written): uint8
    [blocks, block_size, 584] (ops.dsv4_sparse_decode's cache) for D 512 at ratio 4 or 128, uint8 [blocks, block_size, 132]
    (ops.indexer_logits' cache) for D 128 at ratio 4.  Both caches are written in place; returns None."""
    ratio = int(compress_ratio)
    if norm_weight.dtype != torch.bfloat16 or norm_weight.dim() != 1:
        raise ValueError(f"norm_weight must be bf16 [head_dim], got {norm_weight.dtype} {tuple(norm_weight.shape)}")
    D = norm_weight.shape[0]
    row = kv_cache.shape[-1] if kv_cache.dim() == 3 else None
    if (D, ratio, row) not in ((512, 4, 584), (512, 128, 584), (128, 4, 132)):
        raise ValueError(f"dsv4_compress runs head_dim 512 at ratio 4 or 128 into a [blocks, block_size, 584] cache and "
                         f"head_dim 128 at ratio 4 into a [blocks, block_size, 132] cache; got head_dim {D}, ratio {ratio}, "
                         f"kv_cache {tuple(kv_cache.shape)}")
    if kv_cache.dtype != torch.uint8 or kv_cache.stride(2) != 1 or kv_cache.stride(1) != row:
        raise ValueError(f"kv_cache must be uint8 [blocks, block_size, {row}] with rows of {row} contiguous bytes, "
                         f"got {kv_cache.dtype} strides {kv_cache.stride()}")
    half = (2 if ratio == 4 else 1) * D
    T = kv_score.shape[0] if kv_score.dim() == 2 else -1
    if kv_score.dtype != torch.float32 or T < 0 or kv_score.shape[1] != 2 * half or kv_score.stride(1) != 1:
        raise ValueError(f"kv_score must be f32 [tokens, {2 * half}] with contiguous rows, got {kv_score.dtype} "
                         f"{tuple(kv_score.shape)}")
    if ape.dtype != torch.float32 or tuple(ape.shape) != (ratio, half):
        raise ValueError(f"ape must be f32 [{ratio}, {half}], got {ape.dtype} {tuple(ape.shape)}")
    if state_cache.dtype != torch.float32 or state_cache.dim() != 3 or state_cache.shape[2] != 2 * half \
            or state_cache.stride(2) != 1 or state_cache.stride(1) != 2 * half:
        raise ValueError(f"state_cache must be f32 [blocks, block_size, {2 * half}] with contiguous rows, got "
                         f"{state_cache.dtype} {tuple(state_cache.shape)} strides {state_cache.stride()}")
    if block_table.dim() != 2 or block_table.stride(1) != 1 or block_table.dtype not in _INT:
        raise ValueError(f"block_table must be int [requests, max_blocks] with contiguous rows, got {block_table.dtype} "
                         f"{tuple(block_table.shape)}")
    _cos_sin_cache(cos_sin_cache)
    _per_token(T, positions=positions, slot_mapping=slot_mapping, token_to_req=token_to_req,
               kv_slot_mapping=kv_slot_mapping)
    if T == 0:
        return
    # written or read in place, through their strides
    ks, sc, kc = _device(kv_score, "kv_score"), _device(state_cache, "state_cache"), _device(kv_cache, "kv_cache")
    w, cs, ap = _cuda(norm_weight, "norm_weight"), _cuda(cos_sin_cache, "cos_sin_cache"), _cuda(ape, "ape")
    bt = _i32(block_table, "block_table")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    sm = _cuda(slot_mapping.reshape(-1).to(torch.int64), "slot_mapping")
    ksm = _cuda(kv_slot_mapping.reshape(-1).to(torch.int64), "kv_slot_mapping")
    req = _i32(token_to_req.reshape(-1), "token_to_req")
    rc = L.lib().b200_dsv4_compress(
        _stream(), ks.data_ptr(), ks.stride(0) if T > 1 else 2 * half, ap.data_ptr(), pos.data_ptr(), sm.data_ptr(),
        req.data_ptr(), bt.data_ptr(), bt.stride(0), sc.data_ptr(), sc.shape[1], sc.stride(0), w.data_ptr(), float(eps),
        cs.data_ptr(), cs.shape[0], ksm.data_ptr(), kc.data_ptr(), kc.shape[1], kc.shape[0], kc.stride(0), D, ratio, T)
    L.check(rc, "b200_dsv4_compress")


def _mhc_streams(residual: torch.Tensor, name: str = "residual"):
    """bf16 [..., 4, H] -> (leading shape, T, H)."""
    r = residual
    if r.dtype != torch.bfloat16 or r.dim() < 2 or r.shape[-2] != 4:
        raise ValueError(f"{name} must be bf16 [..., 4, hidden] (hc_mult = 4), got {r.dtype} {tuple(r.shape)}")
    return tuple(r.shape[:-2]), r.numel() // (4 * r.shape[-1]) if r.numel() else 0, r.shape[-1]


def _mhc_f32(t: torch.Tensor, numel: int, name: str) -> None:
    if not t.is_floating_point() or t.numel() != numel:
        raise ValueError(f"{name} must hold {numel} float32 values, got {t.dtype} {tuple(t.shape)}")


def _mhc_x(x: torch.Tensor, T: int, H: int) -> None:
    if x.dtype != torch.bfloat16 or x.numel() != T * H:
        raise ValueError(f"x must be bf16 [..., {H}] with the residual's leading shape, got {x.dtype} {tuple(x.shape)}")


def _f32(t: torch.Tensor, name: str) -> torch.Tensor:
    return _cuda(t.to(torch.float32), name)


def _mhc_post_pre(x, residual, post_layer_mix, comb_res_mix, fn, hc_scale, hc_base, rms_eps, hc_pre_eps, hc_sinkhorn_eps,
                  hc_post_mult_value, sinkhorn_repeat, norm_weight, norm_eps):
    lead, T, H = _mhc_streams(residual)
    _mhc_f32(fn, 24 * 4 * H, "fn")
    _mhc_f32(hc_scale, 3, "hc_scale")
    _mhc_f32(hc_base, 24, "hc_base")
    post = x is not None
    if post:
        _mhc_x(x, T, H)
        _mhc_f32(post_layer_mix, T * 4, "post_layer_mix")
        _mhc_f32(comb_res_mix, T * 16, "comb_res_mix")
    if norm_weight is not None and (not norm_weight.is_floating_point() or norm_weight.numel() != H):
        raise ValueError(f"norm_weight must hold {H} values, got {norm_weight.dtype} {tuple(norm_weight.shape)}")
    r = _cuda(residual, "residual")
    fn, sc, base = _f32(fn, "fn"), _f32(hc_scale, "hc_scale"), _f32(hc_base, "hc_base")
    if post:
        x = _cuda(x, "x")
        plm, crm = _f32(post_layer_mix, "post_layer_mix"), _f32(comb_res_mix, "comb_res_mix")
    w = _cuda(norm_weight.to(torch.bfloat16), "norm_weight") if norm_weight is not None else None
    dev = r.device
    r_out = torch.empty_like(r) if post else None
    post_mix = torch.empty(*lead, 4, 1, dtype=torch.float32, device=dev)
    comb_mix = torch.empty(*lead, 4, 4, dtype=torch.float32, device=dev)
    layer_input = torch.empty(*lead, H, dtype=torch.bfloat16, device=dev)
    if T:
        ws = torch.empty(L.lib().b200_mhc_workspace_bytes(T, H), dtype=torch.uint8, device=dev)
        rc = L.lib().b200_mhc_post_pre(
            _stream(), x.data_ptr() if post else None, r.data_ptr(), plm.data_ptr() if post else None,
            crm.data_ptr() if post else None, fn.data_ptr(), sc.data_ptr(), base.data_ptr(),
            w.data_ptr() if w is not None else None, T, H, float(rms_eps), float(hc_pre_eps), float(hc_sinkhorn_eps),
            float(hc_post_mult_value), int(sinkhorn_repeat), float(norm_eps), ws.data_ptr(),
            r_out.data_ptr() if post else None, post_mix.data_ptr(), comb_mix.data_ptr(), layer_input.data_ptr())
        L.check(rc, "b200_mhc_post_pre")
    return r_out, post_mix, comb_mix, layer_input


def mhc_pre(residual: torch.Tensor, fn: torch.Tensor, hc_scale: torch.Tensor, hc_base: torch.Tensor, rms_eps: float,
            hc_pre_eps: float, hc_sinkhorn_eps: float, hc_post_mult_value: float, sinkhorn_repeat: int,
            norm_weight: torch.Tensor | None = None, norm_eps: float = 1e-6):
    """DeepSeek-V4 mHC pre mapping (the reference's mhc_pre_tilelang; kernels/mhc/torch.py:6-91 without the norm).
    residual bf16 [..., 4, H], fn f32 [24, 4H], hc_scale f32 [3], hc_base f32 [24].  The fp32 row's RMS-scaled projection
    gives pre gates, post gates (times hc_post_mult_value) and a 4 x 4 Sinkhorn-normalised mixing matrix; layer_input is the
    pre-gated sum of the streams, RMS-normalised with norm_weight (cast to bf16) when given, as the reference's fused
    kernel does (mean square of the unrounded fp32 row, applied to its bf16 rounding).
    Returns post_mix f32 [..., 4, 1], comb_mix f32 [..., 4, 4], layer_input bf16 [..., H]."""
    _, post_mix, comb_mix, layer_input = _mhc_post_pre(None, residual, None, None, fn, hc_scale, hc_base, rms_eps, hc_pre_eps,
                                                       hc_sinkhorn_eps, hc_post_mult_value, sinkhorn_repeat, norm_weight,
                                                       norm_eps)
    return post_mix, comb_mix, layer_input


def mhc_post(x: torch.Tensor, residual: torch.Tensor, post_layer_mix: torch.Tensor,
             comb_res_mix: torch.Tensor) -> torch.Tensor:
    """DeepSeek-V4 mHC post mapping (the reference's mhc_post_tilelang; torch.py:94-106): x bf16 [..., H], residual bf16
    [..., 4, H], post_layer_mix f32 [..., 4] or [..., 4, 1], comb_res_mix f32 [..., 4, 4];
    out[..., j, :] = bf16(post[j] x + sum_i comb[i, j] residual[i]) in fp32.  Returns bf16 [..., 4, H]."""
    _, T, H = _mhc_streams(residual)
    _mhc_x(x, T, H)
    _mhc_f32(post_layer_mix, T * 4, "post_layer_mix")
    _mhc_f32(comb_res_mix, T * 16, "comb_res_mix")
    r, x = _cuda(residual, "residual"), _cuda(x, "x")
    plm, crm = _f32(post_layer_mix, "post_layer_mix"), _f32(comb_res_mix, "comb_res_mix")
    out = torch.empty_like(r)
    if T:
        rc = L.lib().b200_mhc_post(_stream(), x.data_ptr(), r.data_ptr(), plm.data_ptr(), crm.data_ptr(), T, H, out.data_ptr())
        L.check(rc, "b200_mhc_post")
    return out


def mhc_fused_post_pre(x: torch.Tensor, residual: torch.Tensor, post_layer_mix: torch.Tensor, comb_res_mix: torch.Tensor,
                       fn: torch.Tensor, hc_scale: torch.Tensor, hc_base: torch.Tensor, rms_eps: float, hc_pre_eps: float,
                       hc_sinkhorn_eps: float, hc_post_mult_value: float, sinkhorn_repeat: int,
                       norm_weight: torch.Tensor | None = None, norm_eps: float = 1e-6):
    """mhc_post followed by the next sublayer's mhc_pre in one call (the reference's mhc_fused_post_pre_tilelang).  The mixes
    are computed from the bf16 residual the call returns, so the result is bit-identical to
    mhc_pre(mhc_post(x, residual, post_layer_mix, comb_res_mix), ...).
    Returns residual_cur bf16 [..., 4, H], post_mix f32 [..., 4, 1], comb_mix f32 [..., 4, 4], layer_input bf16 [..., H]."""
    return _mhc_post_pre(x, residual, post_layer_mix, comb_res_mix, fn, hc_scale, hc_base, rms_eps, hc_pre_eps,
                         hc_sinkhorn_eps, hc_post_mult_value, sinkhorn_repeat, norm_weight, norm_eps)


def hc_head(hidden_states: torch.Tensor, hc_fn: torch.Tensor, hc_scale: torch.Tensor, hc_base: torch.Tensor,
            rms_norm_eps: float, hc_eps: float) -> torch.Tensor:
    """DeepSeek-V4 hc_head (the reference's hc_head_fused_kernel_tilelang): collapses the 4 streams before the final norm.
    hidden_states bf16 [T, 4, H], hc_fn f32 [4, 4H], hc_scale f32 [1], hc_base f32 [4];
    out = bf16(sum_i (sigmoid(mix_i * rsqrt(mean(r_flat^2) + rms_norm_eps) * s + base_i) + hc_eps) r_i).  Returns bf16 [T, H]."""
    lead, T, H = _mhc_streams(hidden_states, "hidden_states")
    _mhc_f32(hc_fn, 4 * 4 * H, "hc_fn")
    _mhc_f32(hc_scale, 1, "hc_scale")
    _mhc_f32(hc_base, 4, "hc_base")
    r = _cuda(hidden_states, "hidden_states")
    fn, sc, base = _f32(hc_fn, "hc_fn"), _f32(hc_scale, "hc_scale"), _f32(hc_base, "hc_base")
    out = torch.empty(*lead, H, dtype=torch.bfloat16, device=r.device)
    if T:
        ws = torch.empty(L.lib().b200_mhc_workspace_bytes(T, H), dtype=torch.uint8, device=r.device)
        rc = L.lib().b200_hc_head(_stream(), r.data_ptr(), fn.data_ptr(), sc.data_ptr(), base.data_ptr(), T, H,
                                  float(rms_norm_eps), float(hc_eps), ws.data_ptr(), out.data_ptr())
        L.check(rc, "b200_hc_head")
    return out


def mla_rope_cache_write(q_pe: torch.Tensor, k_pe: torch.Tensor, kv_c: torch.Tensor, positions: torch.Tensor,
                         cos_sin_cache: torch.Tensor, slot_mapping: torch.Tensor, kv_cache: torch.Tensor,
                         is_neox_style: bool = False, kv_scale: float = 1.0) -> None:
    """RoPE of q_pe [T,Hq,64] / k_pe [T,64] IN PLACE (reference RotaryEmbedding.forward_static) fused with
    concat_and_cache_mla: kv_cache [blocks, block_size, 576] (bf16 or e4m3) row slot_mapping[t] <- [kv_c[t] | rope(k_pe[t])].
    A uint8 [blocks, block_size, 656] cache is the fp8_ds_mla layout of concat_and_cache_ds_mla_kernel (per-128-dim fp32
    scales, bf16 rope part; kv_scale is not used)."""
    if q_pe.dtype != torch.bfloat16 or q_pe.dim() != 3 or q_pe.shape[2] != 64 or not q_pe.is_contiguous():
        raise ValueError(f"q_pe must be a contiguous bf16 [tokens, heads, 64] tensor (rotated in place), got {q_pe.dtype} "
                         f"{tuple(q_pe.shape)}")
    T, Hq, _ = q_pe.shape
    if k_pe.dtype != torch.bfloat16 or tuple(k_pe.shape) != (T, 64) or not k_pe.is_contiguous():
        raise ValueError(f"k_pe must be a contiguous bf16 [{T}, 64] tensor (rotated in place), got {k_pe.dtype} "
                         f"{tuple(k_pe.shape)}")
    if kv_c.dtype != torch.bfloat16 or tuple(kv_c.shape) != (T, 512):
        raise ValueError(f"kv_c must be bf16 [{T}, 512], got {kv_c.dtype} {tuple(kv_c.shape)}")
    _cos_sin_cache(cos_sin_cache, torch.bfloat16)
    _per_token(T, positions=positions, slot_mapping=slot_mapping)
    if kv_cache.dim() != 3 or not kv_cache.is_contiguous() or (kv_cache.dtype, kv_cache.shape[2]) not in (
            (torch.bfloat16, 576), (torch.float8_e4m3fn, 576), (torch.uint8, 656)):
        raise ValueError(f"kv_cache must be a contiguous bf16 / e4m3 [blocks, block_size, 576] or uint8 "
                         f"[blocks, block_size, 656] tensor, got {kv_cache.dtype} {tuple(kv_cache.shape)}")
    q_pe, k_pe, kv_cache = _device(q_pe, "q_pe"), _device(k_pe, "k_pe"), _device(kv_cache, "kv_cache")
    kv_c, cs = _cuda(kv_c, "kv_c"), _cuda(cos_sin_cache, "cos_sin_cache")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    sm = _cuda(slot_mapping.reshape(-1).to(torch.int64), "slot_mapping")
    kv_dtype = {torch.bfloat16: 0, torch.float8_e4m3fn: 1, torch.uint8: 2}[kv_cache.dtype]
    rc = L.lib().b200_mla_rope_cache_write(_stream(), q_pe.data_ptr(), k_pe.data_ptr(), kv_c.data_ptr(), pos.data_ptr(),
                                           cs.data_ptr(), int(is_neox_style), sm.data_ptr(), kv_cache.data_ptr(), kv_dtype,
                                           float(kv_scale), T, Hq)
    L.check(rc, "b200_mla_rope_cache_write")


def mla_q_absorb(q_nope: torch.Tensor, w_uk_t: torch.Tensor) -> torch.Tensor:
    """ql_nope [T,Hq,512] = q_nope [T,Hq,128] x W_UK_T [Hq,128,512] (reference mla_attention.py:875-893)."""
    if q_nope.dtype != torch.bfloat16 or q_nope.dim() != 3 or q_nope.shape[2] != 128:
        raise ValueError(f"q_nope must be bf16 [tokens, heads, 128], got {q_nope.dtype} {tuple(q_nope.shape)}")
    T, Hq, _ = q_nope.shape
    if w_uk_t.dtype != torch.bfloat16 or tuple(w_uk_t.shape) != (Hq, 128, 512):
        raise ValueError(f"w_uk_t must be bf16 [{Hq}, 128, 512], got {w_uk_t.dtype} {tuple(w_uk_t.shape)}")
    q, w = _cuda(q_nope, "q_nope"), _cuda(w_uk_t, "w_uk_t")
    out = torch.empty(T, Hq, 512, dtype=torch.bfloat16, device=q.device)
    L.check(L.lib().b200_mla_q_absorb(_stream(), q.data_ptr(), w.data_ptr(), out.data_ptr(), T, Hq), "b200_mla_q_absorb")
    return out


def _kv_cache_strides(k_cache: torch.Tensor, v_cache: torch.Tensor) -> tuple[int, int, int]:
    """(block, page, head) strides in elements of a pair of [blocks, page, Hkv, 128] bf16 cache views, checked against what
    the kernels address: the FlashInfer backend's packed NHD / HND halves (kv_cache.transpose(1, 2).split(128, -1),
    flashinfer.py:2276-2290) or separate contiguous caches.  Never copies: a write through a copy would be lost."""
    for t, n in ((k_cache, "k_cache"), (v_cache, "v_cache")):
        if t.dtype != torch.bfloat16 or t.dim() != 4 or t.shape[-1] != 128:
            raise ValueError(f"{n} must be a bf16 [blocks, page, num_kv_heads, 128] view, got {t.dtype} {tuple(t.shape)}")
    if k_cache.shape != v_cache.shape or k_cache.stride() != v_cache.stride() or k_cache.device != v_cache.device:
        raise ValueError("k_cache and v_cache must be views of the same shape and strides on one device")
    st = k_cache.stride()
    if st[3] != 1 or any(x <= 0 or x % 8 for x in st[:3]) or k_cache.data_ptr() % 16 or v_cache.data_ptr() % 16:
        raise ValueError(f"cache views need a contiguous head dim, strides in positive multiples of 8 elements and "
                         f"16-byte aligned bases (16-byte row loads), got strides {st}")
    return st[0], st[1], st[2]


def gqa_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, seq_lens: torch.Tensor,
               page_table: torch.Tensor, sm_scale: float, num_kv_splits: int = 0, max_seq_len: int | None = None,
               q_len_per_req: int = 1):
    """Paged GQA decode (q [B*Q,Hq,128] bf16; caches [pages,page,Hkv,128] bf16 views).  Returns (out, lse), [B*Q,Hq,128]
    and [B*Q,Hq].  B = seq_lens.numel(); Q = ``q_len_per_req`` query tokens per request (speculative-decode verification,
    the reference decode path's q_len_per_req, flashinfer.py:2183-2188): request b's Q tokens are contiguous in draft
    order, seq_lens[b] counts all its keys including the Q new ones, and token i attends to keys [0, seq_lens[b] - Q + i]
    (a row with no visible key gives out 0 and lse -inf).  Q = 1 (the default) is the single-token decode.
    The caches are read in place through their own strides: separate contiguous caches, or the K / V halves of the
    FlashInfer backend's packed NHD / HND cache exactly as the backend hands them out (kv_cache.transpose(1, 2)
    .split(128, -1)); the head dim must be contiguous and the other strides multiples of 8 elements (ValueError otherwise).
    ``max_seq_len`` (host-side bound on seq_lens, as the reference's attention metadata carries it) sizes the split count
    and the B*Hq*splits*130*4-byte workspace from the real context instead of the page-table width (= max_model_len)."""
    bstride, pstride, hstride = _kv_cache_strides(k_cache, v_cache)
    if q.dtype != torch.bfloat16 or q.dim() != 3 or q.shape[2] != 128:
        raise ValueError(f"q must be bf16 [tokens, heads, 128], got {q.dtype} {tuple(q.shape)}")
    T, Hq, D = q.shape
    Q = int(q_len_per_req)
    page, Hkv = k_cache.shape[1], k_cache.shape[2]
    _int_tensor(seq_lens, "seq_lens")
    _int_tensor(page_table, "page_table", 2)
    B = seq_lens.numel()
    if T != B * Q:
        raise ValueError(f"q must hold q_len_per_req = {Q} tokens per request: {B * Q} rows for {B} seq_lens, got {T}")
    if page_table.shape[0] != B:
        raise ValueError(f"page_table must have one row per request ({B}), got {tuple(page_table.shape)}")
    qq = _cuda(q, "q")
    k_cache, v_cache = _device(k_cache, "k_cache"), _device(v_cache, "v_cache")
    sl = _cuda(seq_lens.reshape(-1).to(torch.int32), "seq_lens")
    pt = _cuda(page_table.to(torch.int32), "page_table")
    if max_seq_len is not None:
        max_pages = max(1, min(pt.shape[1], -(-int(max_seq_len) // page)))
        if max_pages != pt.shape[1]:
            pt = pt[:, :max_pages].contiguous()   # the kernels only walk pages below the bound
    if num_kv_splits <= 0:
        # tensor-core path: one 128-token split per work item, enough splits to cover the page table
        num_kv_splits = max(1, -(-(pt.shape[1] * page) // 128))
        if num_kv_splits > 1024:
            num_kv_splits = max(1, min(32, 592 // max(1, B * Hkv)))
    ws = torch.empty(L.lib().b200_gqa_decode_workspace_bytes(T, Hq, D, num_kv_splits), dtype=torch.uint8, device=qq.device)
    out = torch.empty(T, Hq, D, dtype=torch.bfloat16, device=qq.device)
    lse = torch.empty(T, Hq, dtype=torch.float32, device=qq.device)
    rc = L.lib().b200_gqa_decode_spec(_stream(), qq.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), bstride, pstride,
                                      hstride, sl.data_ptr(), pt.data_ptr(), B, Q, Hq, Hkv, D, page, pt.shape[1],
                                      float(sm_scale), num_kv_splits, ws.data_ptr(), out.data_ptr(), lse.data_ptr())
    L.check(rc, "b200_gqa_decode")
    return out, lse


def gqa_qknorm_rope_cache_write(qkv: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor,
                                slot_mapping: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, num_heads: int,
                                num_kv_heads: int, q_norm_weight: torch.Tensor | None = None,
                                k_norm_weight: torch.Tensor | None = None, eps: float = 1e-6,
                                is_neox_style: bool = True) -> torch.Tensor:
    """One launch for the attention block's work before decode: per-head RMSNorm of q and k (Qwen3, reference
    models/qwen3_moe.py:333-351; skipped where the weight is None), RoPE of q and k (fused_qk_norm_rope,
    vllm/_custom_ops.py:279) and reshape_and_cache_flash of the new k / v (csrc/libtorch_stable/cache_kernels.cu:315-400).
    qkv [T, (Hq + 2 Hkv) * 128] bf16 (the fused QKV projection's rows); positions [T] (clamped to the table's rows);
    cos_sin_cache bf16 [max_position, rotary_dim] = cos | sin; slot_mapping [T] (< 0: padded token, nothing written);
    k_cache / v_cache the views exactly as the reference passes them to reshape_and_cache_flash.
    Returns q_out [T, Hq, 128] bf16, contiguous: the q that gqa_decode takes."""
    x = qkv
    if x.dtype != torch.bfloat16 or x.dim() != 2 or x.shape[1] != (num_heads + 2 * num_kv_heads) * 128:
        raise ValueError(f"qkv must be bf16 [T, (num_heads + 2 * num_kv_heads) * 128], got {x.dtype} {tuple(x.shape)}")
    if cos_sin_cache.dtype != torch.bfloat16 or cos_sin_cache.dim() != 2:
        raise ValueError("cos_sin_cache must be bf16 [max_position, rotary_dim]")
    bstride, pstride, hstride = _kv_cache_strides(k_cache, v_cache)
    if k_cache.shape[2] != num_kv_heads or k_cache.device != x.device:
        raise ValueError("the cache views must hold num_kv_heads heads on qkv's device")
    for w, n in ((q_norm_weight, "q_norm_weight"), (k_norm_weight, "k_norm_weight")):
        if w is not None and (w.dtype != torch.bfloat16 or w.numel() != 128):
            raise ValueError(f"{n} must be bf16 [128]")
    T = x.shape[0]
    _per_token(T, positions=positions, slot_mapping=slot_mapping)
    x = _cuda(x, "qkv")
    cs = _cuda(cos_sin_cache, "cos_sin_cache")
    ws = [_cuda(w, n) if w is not None else None for w, n in ((q_norm_weight, "q_norm_weight"),
                                                               (k_norm_weight, "k_norm_weight"))]
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    sm = _cuda(slot_mapping.reshape(-1).to(torch.int64), "slot_mapping")
    q_out = torch.empty(T, num_heads, 128, dtype=torch.bfloat16, device=x.device)
    rc = L.lib().b200_gqa_qknorm_rope_cache_write(
        _stream(), x.data_ptr(), pos.data_ptr(), cs.data_ptr(), cs.shape[0], cs.shape[1], int(is_neox_style),
        ws[0].data_ptr() if ws[0] is not None else None, ws[1].data_ptr() if ws[1] is not None else None, float(eps),
        sm.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), bstride, pstride, hstride, k_cache.shape[1],
        q_out.data_ptr(), T, num_heads, num_kv_heads, 128)
    L.check(rc, "b200_gqa_qknorm_rope_cache_write")
    return q_out


def _weights_view(weights: torch.Tensor, T: int, H: int) -> None:
    """The indexer weights, bf16 [T, H] read through their row stride (a column slice of the fused projection)."""
    if weights.dtype != torch.bfloat16 or weights.shape != (T, H) or weights.stride(1) != 1 \
            or (T > 1 and weights.stride(0) < H):
        raise ValueError(f"weights must be a bf16 [{T}, {H}] view with contiguous, non-overlapping rows")


def _indexer_cache(k_cache: torch.Tensor) -> None:
    if k_cache.dtype != torch.uint8 or k_cache.dim() != 3 or k_cache.shape[2] != 132 or not k_cache.is_contiguous():
        raise ValueError(f"k_cache must be a contiguous uint8 [num_blocks, block_size, 132], got {k_cache.dtype} "
                         f"{tuple(k_cache.shape)}")


def indexer_qk_rope_quant_cache_write(q: torch.Tensor, weights: torch.Tensor, k: torch.Tensor, positions: torch.Tensor,
                                      cos_sin_cache: torch.Tensor, slot_mapping: torch.Tensor, k_cache: torch.Tensor,
                                      softmax_scale: float, head_scale: float, is_neox_style: bool = True,
                                      use_ue8m0: bool = True):
    """The lightning indexer's q / k preparation in one launch (reference _fused_indexer_q_rope_quant_kernel,
    sparse_attn_indexer.py:127-251; RotaryEmbedding.forward_static of k; indexer_k_quant_and_cache,
    cache_kernels.cu:599-659).  q [T,H,128] bf16 (wq_b output, first 64 dims rotary); weights bf16 [T,H], any row stride
    (a column slice of the fused projection); k [T,128] bf16 after k_norm; cos_sin_cache bf16 [max_position, 64];
    slot_mapping [T] (< 0: nothing written); k_cache uint8 [num_blocks, block_size, 132], written in place.
    Returns (q_fp8 e4m3 [T,H,128], weights_out f32 [T,H] = weight * q_scale * softmax_scale * head_scale)."""
    if q.dtype != torch.bfloat16 or q.dim() != 3 or q.shape[2] != 128:
        raise ValueError(f"q must be bf16 [T, H, 128], got {q.dtype} {tuple(q.shape)}")
    T, H, _ = q.shape
    if k.dtype != torch.bfloat16 or k.shape != (T, 128):
        raise ValueError(f"k must be bf16 [{T}, 128], got {k.dtype} {tuple(k.shape)}")
    _weights_view(weights, T, H)
    _cos_sin_cache(cos_sin_cache, torch.bfloat16)
    _indexer_cache(k_cache)
    _per_token(T, positions=positions, slot_mapping=slot_mapping)
    x, kk = _cuda(q, "q"), _cuda(k, "k")
    weights, k_cache = _device(weights, "weights"), _device(k_cache, "k_cache")
    cs = _cuda(cos_sin_cache, "cos_sin_cache")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    sm = _cuda(slot_mapping.reshape(-1).to(torch.int64), "slot_mapping")
    q_fp8 = torch.empty(T, H, 128, dtype=torch.float8_e4m3fn, device=x.device)
    w_out = torch.empty(T, H, dtype=torch.float32, device=x.device)
    rc = L.lib().b200_indexer_qk_rope_quant_cache_write(
        _stream(), x.data_ptr(), weights.data_ptr(), weights.stride(0) if T > 1 else H, kk.data_ptr(), pos.data_ptr(),
        cs.data_ptr(), cs.shape[0], int(is_neox_style), sm.data_ptr(), k_cache.data_ptr(), k_cache.shape[1],
        int(use_ue8m0), float(softmax_scale), float(head_scale), q_fp8.data_ptr(), w_out.data_ptr(), T, H)
    L.check(rc, "b200_indexer_qk_rope_quant_cache_write")
    return q_fp8, w_out


def _logits_out(logits: torch.Tensor, R: int, width: int) -> None:
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.shape[0] != R or logits.shape[1] < width \
            or logits.stride(1) != 1:
        raise ValueError(f"logits must be f32 [{R}, >= {width}] with contiguous rows")


def indexer_logits(q_fp8: torch.Tensor, weights: torch.Tensor, k_cache: torch.Tensor, seq_lens: torch.Tensor,
                   page_table: torch.Tensor, q_len: int = 1, logits: torch.Tensor | None = None) -> torch.Tensor:
    """Paged MQA logits of the indexer (DeepGEMM fp8_fp4_paged_mqa_logits; fp8_paged_mqa_logits_torch,
    rocm_aiter_mla_sparse.py:264-363): logits[b*Q + i, j] = k_scale[j] * sum_h weights[b*Q + i, h] * relu(q . k_j) for
    j <= seq_lens[b] - Q + i; -inf to the end of the request's last page, the rest untouched.  q_fp8 [B*Q,H,128] e4m3,
    weights f32 [B*Q,H]; H 32 or 64, Q <= 16, page 16 / 32 / 64.  ``logits`` (f32 [B*Q, >= max_pages * page]) is filled
    in place when given.  Returns logits."""
    if q_fp8.dtype != torch.float8_e4m3fn or q_fp8.dim() != 3 or q_fp8.shape[2] != 128:
        raise ValueError(f"q_fp8 must be e4m3 [B*Q, H, 128], got {q_fp8.dtype} {tuple(q_fp8.shape)}")
    R, H, _ = q_fp8.shape
    if weights.dtype != torch.float32 or weights.shape != (R, H):
        raise ValueError(f"weights must be f32 [{R}, {H}]")
    _indexer_cache(k_cache)
    _int_tensor(seq_lens, "seq_lens")
    _int_tensor(page_table, "page_table", 2)
    B, Q = seq_lens.numel(), int(q_len)
    if R != B * Q or page_table.shape[0] < B:
        raise ValueError(f"q_fp8 needs q_len = {Q} rows per request ({B * Q}), page_table a row per request")
    page = k_cache.shape[1]
    width = page_table.shape[1] * page
    if logits is not None:
        _logits_out(logits, R, width)
    q8, w, kc = _cuda(q_fp8, "q_fp8"), _cuda(weights, "weights"), _device(k_cache, "k_cache")
    sl = _cuda(seq_lens.reshape(-1).to(torch.int32), "seq_lens")
    pt = _cuda(page_table.to(torch.int32), "page_table")
    logits = _device(logits, "logits") if logits is not None else torch.empty(R, width, dtype=torch.float32,
                                                                              device=q8.device)
    rc = L.lib().b200_indexer_logits(_stream(), q8.data_ptr(), w.data_ptr(), kc.data_ptr(), kc.shape[0], page,
                                     sl.data_ptr(), pt.data_ptr(), B, Q, H, pt.shape[1], logits.data_ptr(),
                                     logits.stride(0))
    L.check(rc, "b200_indexer_logits")
    return logits


def indexer_topk(logits: torch.Tensor, seq_lens: torch.Tensor, topk: int, q_len: int = 1) -> torch.Tensor:
    """top_k_per_row_decode (sampler.cu:567-614, 661-720): for row b*Q + i, the positions of the topk largest logits of
    [0, min(seq_lens[b] - Q + i + 1, logits.shape[1])) in ascending order, ties at the threshold to the lowest positions,
    -1 padding.  ``logits`` may be a column slice of a wider buffer (rows read through its own row stride).
    Returns int32 [B*Q, topk]."""
    lg = logits
    if lg.dtype != torch.float32 or lg.dim() != 2 or lg.stride(1) != 1 or (lg.shape[0] > 1 and lg.stride(0) < lg.shape[1]):
        raise ValueError("logits must be an f32 [rows, width] tensor with contiguous, non-overlapping rows")
    _int_tensor(seq_lens, "seq_lens")
    B, Q = seq_lens.numel(), int(q_len)
    if lg.shape[0] != B * Q:
        raise ValueError(f"logits needs q_len = {Q} rows per request ({B * Q}), got {lg.shape[0]}")
    lg = _device(lg, "logits")
    sl = _cuda(seq_lens.reshape(-1).to(torch.int32), "seq_lens")
    out = torch.empty(B * Q, int(topk), dtype=torch.int32, device=lg.device)
    row_stride = lg.stride(0) if lg.shape[0] > 1 else lg.shape[1]
    rc = L.lib().b200_indexer_topk(_stream(), lg.data_ptr(), row_stride, lg.shape[1], sl.data_ptr(), B, Q, int(topk),
                                   out.data_ptr())
    L.check(rc, "b200_indexer_topk")
    return out


def indexer_decode(q_fp8: torch.Tensor, weights: torch.Tensor, k_cache: torch.Tensor, seq_lens: torch.Tensor,
                   page_table: torch.Tensor, q_len: int, topk: int) -> torch.Tensor:
    """The indexer's decode step: indexer_logits then indexer_topk.  Returns topk_indices int32 [B*Q, topk], request-local
    positions, the layout mla_decode_sparse takes with req_id = row // q_len and the same page table."""
    logits = indexer_logits(q_fp8, weights, k_cache, seq_lens, page_table, q_len)
    return indexer_topk(logits, seq_lens, topk, q_len)


def dsv4_indexer_q_quant(q: torch.Tensor, weights: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor,
                         softmax_scale: float, head_scale: float):
    """The DeepSeek-V4 indexer's q side (the fp8 path of the reference's fused_indexer_q_rope_quant,
    models/deepseek_v4/common/ops/fused_indexer_q.py:70-176).  q bf16 [T, H, 128] = [64 nope | 64 rope] (wq_b output);
    weights bf16 [T, H], any row stride (a column slice of the fused projection); positions [T]; cos_sin_cache f32
    [max_pos, 64] = cos | sin (the table ops.dsv4_compress takes).  Per (token, head): GPT-J pair RoPE of dims 64-127 in
    fp32, rounded to bf16 once; scale = 2^ceil(log2(max(amax, 1e-4) / 448)); q_fp8 = e4m3(x / scale), saturating.  The model
    passes softmax_scale = 128 ** -0.5 and head_scale = H ** -0.5.  Returns (q_fp8 e4m3 [T, H, 128], weights_out f32
    [T, H] = weights * scale * softmax_scale * head_scale), what ops.dsv4_indexer_decode takes."""
    if q.dtype != torch.bfloat16 or q.dim() != 3 or q.shape[2] != 128 or not 1 <= q.shape[1] <= 128:
        raise ValueError(f"q must be bf16 [T, 1-128 heads, 128], got {q.dtype} {tuple(q.shape)}")
    T, H, _ = q.shape
    _weights_view(weights, T, H)
    _cos_sin_cache(cos_sin_cache)
    _per_token(T, positions=positions)
    weights = _device(weights, "weights")
    x, cs = _cuda(q, "q"), _cuda(cos_sin_cache, "cos_sin_cache")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    q_fp8 = torch.empty(T, H, 128, dtype=torch.float8_e4m3fn, device=x.device)
    w_out = torch.empty(T, H, dtype=torch.float32, device=x.device)
    rc = L.lib().b200_dsv4_indexer_q_quant(_stream(), x.data_ptr(), weights.data_ptr(), weights.stride(0) if T > 1 else H,
                                           pos.data_ptr(), cs.data_ptr(), cs.shape[0], float(softmax_scale),
                                           float(head_scale), q_fp8.data_ptr(), w_out.data_ptr(), T, H)
    L.check(rc, "b200_dsv4_indexer_q_quant")
    return q_fp8, w_out


def dsv4_indexer_decode(q_fp8: torch.Tensor, weights: torch.Tensor, k_cache: torch.Tensor, positions: torch.Tensor,
                        token_to_req: torch.Tensor, block_table: torch.Tensor, compress_ratio: int, topk: int,
                        max_seq_len: int | None = None, logits: torch.Tensor | None = None) -> torch.Tensor:
    """The DeepSeek-V4 C4A indexer's decode step: logits then top-k, one row per token.  q_fp8 e4m3 [T, H, 128] and
    weights f32 [T, H] from ops.dsv4_indexer_q_quant (H 32 or 64); k_cache uint8 [blocks, page, 132] (page 16, 32 or 64),
    the compressed indexer cache ops.dsv4_compress writes; block_table [requests, max_blocks] its block numbers.  Token t
    has (positions[t] + 1) // compress_ratio candidates (at most max_blocks * page) in row token_to_req[t].  ``logits``
    (f32 [T, >= max_blocks * page], contiguous rows) receives the logits when given.  max_seq_len, when given, must be
    > every position: if max_seq_len // compress_ratio <= topk every token selects all of its candidates and no logit is
    computed (the reference's short-context path).  Returns the request-local top-k int32 [T, topk], ascending, -1
    padded; ops.dsv4_global_topk_indices turns it into dsv4_sparse_decode's extra list."""
    if q_fp8.dtype != torch.float8_e4m3fn or q_fp8.dim() != 3 or q_fp8.shape[2] != 128 or q_fp8.shape[1] not in (32, 64):
        raise ValueError(f"q_fp8 must be e4m3 [T, 32 or 64, 128], got {q_fp8.dtype} {tuple(q_fp8.shape)}")
    T, H, _ = q_fp8.shape
    if weights.dtype != torch.float32 or weights.shape != (T, H):
        raise ValueError(f"weights must be f32 [{T}, {H}], got {weights.dtype} {tuple(weights.shape)}")
    _indexer_cache(k_cache)
    if block_table.dim() != 2 or block_table.dtype not in _INT:
        raise ValueError(f"block_table must be int [requests, max_blocks], got {block_table.dtype} "
                         f"{tuple(block_table.shape)}")
    ratio, k = int(compress_ratio), int(topk)
    if ratio not in (4, 128) or not 1 <= k <= 2048:
        raise ValueError(f"compress_ratio must be 4 or 128 and topk 1-2048, got {ratio}, {k}")
    _per_token(T, positions=positions, token_to_req=token_to_req)
    page = k_cache.shape[1]
    width = block_table.shape[1] * page
    if logits is not None:
        _logits_out(logits, T, width)
    if T == 0:
        return torch.empty(T, k, dtype=torch.int32, device=q_fp8.device)
    q8, w, kc = _cuda(q_fp8, "q_fp8"), _cuda(weights, "weights"), _device(k_cache, "k_cache")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    req = _i32(token_to_req.reshape(-1), "token_to_req")
    bt = _i32(block_table, "block_table")
    logits = _device(logits, "logits") if logits is not None else torch.empty(T, width, dtype=torch.float32,
                                                                              device=q8.device)
    out = torch.empty(T, k, dtype=torch.int32, device=q8.device)
    rc = L.lib().b200_dsv4_indexer_decode(
        _stream(), q8.data_ptr(), w.data_ptr(), kc.data_ptr(), kc.shape[0], page, pos.data_ptr(), req.data_ptr(),
        bt.data_ptr(), bt.shape[1], ratio, T, H, int(max_seq_len) if max_seq_len is not None else 0, logits.data_ptr(),
        logits.stride(0) if T > 1 else logits.shape[1], k, out.data_ptr())
    L.check(rc, "b200_dsv4_indexer_decode")
    return out


_DS_IDX_SWA, _DS_IDX_C128A, _DS_IDX_TOPK, _DS_IDX_SLOTMAP = 0, 1, 2, 3


def _dsv4_indices(kind: int, positions, slot_mapping, token_to_req, block_table, block_size: int, param: int,
                  width: int, local_topk=None):
    """One b200_dsv4_indices call; returns (indices int32 [T, width], lens int32 [T]), or the int64 [T] slot mapping."""
    if block_table.dim() != 2 or block_table.dtype not in _INT or block_table.shape[1] < 1:
        raise ValueError(f"block_table must be int [requests, max_blocks >= 1], got {block_table.dtype} "
                         f"{tuple(block_table.shape)}")
    if int(block_size) < 1:
        raise ValueError(f"block_size must be >= 1, got {block_size}")
    T = positions.numel() if local_topk is None else local_topk.shape[0]
    _per_token(T, positions=positions, slot_mapping=slot_mapping, token_to_req=token_to_req)
    dev = block_table.device
    if kind == _DS_IDX_SLOTMAP:
        out, lens = torch.empty(T, dtype=torch.int64, device=dev), None
    else:
        out = torch.empty(T, width, dtype=torch.int32, device=dev)
        lens = torch.empty(T, dtype=torch.int32, device=dev)
    if T == 0:
        return out if lens is None else (out, lens)
    bt = _i32(block_table, "block_table")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions") if positions is not None else None
    sm = _cuda(slot_mapping.reshape(-1).to(torch.int64), "slot_mapping")
    req = _i32(token_to_req.reshape(-1), "token_to_req")
    loc = _i32(local_topk, "topk_indices") if local_topk is not None else None
    rc = L.lib().b200_dsv4_indices(
        _stream(), kind, pos.data_ptr() if pos is not None else None, sm.data_ptr(), req.data_ptr(), bt.data_ptr(), bt.stride(0), bt.shape[1],
        int(block_size), int(param), loc.data_ptr() if loc is not None else None, loc.shape[1] if loc is not None else 0,
        out.data_ptr(), width, width, lens.data_ptr() if lens is not None else None, T)
    L.check(rc, "b200_dsv4_indices")
    return out if lens is None else (out, lens)


def dsv4_swa_indices(positions: torch.Tensor, slot_mapping: torch.Tensor, token_to_req: torch.Tensor,
                     block_table: torch.Tensor, block_size: int, window: int):
    """Sliding-window key list of DeepSeek-V4 decode (the reference's _compute_swa_indices_and_lens_kernel, with p taken
    from positions): token t at position p attends to positions [max(p - window + 1, 0), p] of its request, as global
    slots of the SWA cache: block_table[token_to_req[t]][i // block_size] * block_size + i % block_size (block_table
    [requests, max_blocks]; a block column >= max_blocks is no key, -1).  A token with slot_mapping < 0 gets length 0.
    Returns (swa_indices int32 [T, window], -1 past the length; swa_lens int32 [T]), what ops.dsv4_sparse_decode takes."""
    if int(window) < 1:
        raise ValueError(f"window must be >= 1, got {window}")
    return _dsv4_indices(_DS_IDX_SWA, positions, slot_mapping, token_to_req, block_table, block_size, window, int(window))


def dsv4_c128a_indices(positions: torch.Tensor, slot_mapping: torch.Tensor, token_to_req: torch.Tensor,
                       block_table: torch.Tensor, block_size: int, compress_ratio: int, width: int):
    """Compressed key list of a DeepSeek-V4 C128A layer for decode (the decode branch of the reference's
    _build_c128a_topk_metadata_kernel): every compressed row [0, min((p + 1) // compress_ratio, width)) of the token's
    request, as global slots of the compressed cache (block_table [requests, max_blocks] of the compressed cache, whose
    block size is block_size; a block column >= max_blocks is no key, -1).  A token with slot_mapping < 0 gets length 0.
    Returns (extra_indices int32 [T, width], -1 past the length; extra_lens int32 [T])."""
    if int(compress_ratio) not in (4, 128) or int(width) < 1:
        raise ValueError(f"compress_ratio must be 4 or 128 and width >= 1, got {compress_ratio}, {width}")
    return _dsv4_indices(_DS_IDX_C128A, positions, slot_mapping, token_to_req, block_table, block_size, compress_ratio,
                         int(width))


def dsv4_global_topk_indices(topk_indices: torch.Tensor, slot_mapping: torch.Tensor, token_to_req: torch.Tensor,
                             block_table: torch.Tensor, block_size: int):
    """Request-local C4A top-k (ops.dsv4_indexer_decode's output, int [T, topk]) -> global slots of the compressed
    attention cache (the reference's compute_global_topk_indices_and_lens): entry i >= 0 becomes
    block_table[token_to_req[t]][i // block_size] * block_size + i % block_size (a block column >= max_blocks: -1), -1
    stays -1; the length is the count of entries >= 0, 0 for a token with slot_mapping < 0.
    Returns (extra_indices int32 [T, topk]; extra_lens int32 [T])."""
    if topk_indices.dim() != 2 or topk_indices.dtype not in _INT or topk_indices.shape[1] < 1:
        raise ValueError(f"topk_indices must be int [tokens, topk >= 1], got {topk_indices.dtype} "
                         f"{tuple(topk_indices.shape)}")
    return _dsv4_indices(_DS_IDX_TOPK, None, slot_mapping, token_to_req, block_table, block_size, 0,
                         topk_indices.shape[1], local_topk=topk_indices)


def dsv4_compressed_slot_mapping(positions: torch.Tensor, slot_mapping: torch.Tensor, token_to_req: torch.Tensor,
                                 block_table: torch.Tensor, block_size: int, compress_ratio: int) -> torch.Tensor:
    """The compressor's cache slots (the reference's get_compressed_slot_mapping): a token at position p that closes a
    window ((p + 1) % compress_ratio == 0) writes compressed row p // compress_ratio of its request, global slot
    block_table[token_to_req[t]][row // block_size] * block_size + row % block_size of the compressed cache; every other
    token, a token with slot_mapping < 0 and a block column >= max_blocks get -1.  Returns int64 [T], the kv_slot_mapping
    ops.dsv4_compress takes."""
    if int(compress_ratio) not in (4, 128):
        raise ValueError(f"compress_ratio must be 4 or 128, got {compress_ratio}")
    return _dsv4_indices(_DS_IDX_SLOTMAP, positions, slot_mapping, token_to_req, block_table, block_size, compress_ratio,
                         1)


def _dsv4_o_args(o: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor, n_groups: int):
    """Checks the attention output and rotary arguments of the V4 output projection; returns (T, H, G, token stride)."""
    if o.dtype != torch.bfloat16 or o.dim() != 3 or o.shape[2] != 512 or o.stride(2) != 1 \
            or (o.shape[1] > 1 and o.stride(1) != 512):
        raise ValueError(f"o must be bf16 [T, H, 512] with contiguous heads and dims, got {o.dtype} {tuple(o.shape)} "
                         f"strides {o.stride()}")
    T, H, _ = o.shape
    G = int(n_groups)
    if G < 1 or H % G or not 1 <= H // G <= 16:
        raise ValueError(f"the {H} heads must form n_groups = {n_groups} groups of 1-16 heads")
    if T > 1 << 20:
        raise ValueError(f"at most 2^20 tokens, got {T}")
    stride = o.stride(0) if T > 1 else H * 512
    if stride < H * 512 or stride % 8 or o.data_ptr() % 16:
        raise ValueError(f"o's token stride ({o.stride(0)}) must be >= H * 512 and a multiple of 8, its data 16-byte aligned")
    _cos_sin_cache(cos_sin_cache)
    _per_token(T, positions=positions)
    return T, H, G, stride


def _dsv4_inv_rope_quant(o, positions, cos_sin_cache, n_groups):
    T, H, G, stride = _dsv4_o_args(o, positions, cos_sin_cache, n_groups)
    D = H // G * 512
    o = _device(o, "o")
    pos = _cuda(positions.reshape(-1).to(torch.int64), "positions")
    cs = _cuda(cos_sin_cache, "cos_sin_cache")
    o_fp8 = torch.empty(G, T, D, dtype=torch.float8_e4m3fn, device=o.device)
    o_scale = torch.empty(G, D // 128, T, dtype=torch.float32, device=o.device)
    rc = L.lib().b200_dsv4_inv_rope_quant(_stream(), o.data_ptr(), stride, pos.data_ptr(), cs.data_ptr(), cs.shape[0], T,
                                          H, G, o_fp8.data_ptr(), o_scale.data_ptr())
    L.check(rc, "b200_dsv4_inv_rope_quant")
    return o_fp8, o_scale


def dsv4_inv_rope_quant(o: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor, n_groups: int):
    """Inverse RoPE + block-128 fp8 quantisation of the DeepSeek-V4 attention output (the reference's
    fused_inv_rope_fp8_quant, fp32-scale path, models/deepseek_v4/common/ops/fused_inv_rope_fp8_quant.py).  o bf16
    [T, H, 512] = [448 nope | 64 rope], heads and dims contiguous, any token stride (a head slice of a padded output);
    positions [T]; cos_sin_cache f32 [max_pos, 64] = cos | sin (the table ops.dsv4_qnorm_rope_kv_insert takes).  The H heads
    form n_groups groups of 1-16 heads, D = H / n_groups * 512.  Dims 448-511 of each head get the inverse GPT-J rotation in
    fp32 (not rounded to bf16); every 128 values of a group get scale 2^ceil(log2(max(absmax, 1e-10) / 448)) and e4m3 codes
    x / scale, saturating.  Returns (o_fp8 e4m3 [T, n_groups, D], o_scale f32 [T, n_groups, D / 128]), views of
    group-major storage."""
    o_fp8, o_scale = _dsv4_inv_rope_quant(o, positions, cos_sin_cache, n_groups)
    return o_fp8.transpose(0, 1), o_scale.permute(2, 0, 1)


def dsv4_o_proj(o: torch.Tensor, positions: torch.Tensor, cos_sin_cache: torch.Tensor, wo_a_weight: torch.Tensor,
                wo_a_scale: torch.Tensor, n_groups: int) -> torch.Tensor:
    """The DeepSeek-V4 attention output projection up to wo_b (the reference's deep_gemm_fp8_o_proj without its last
    linear, models/deepseek_v4/nvidia/ops/o_proj.py:28-73): ops.dsv4_inv_rope_quant, then the grouped fp8 GEMM
    z[t, g, :] = wo_a[g] . o_fp8[t, g, :] (DeepGEMM fp8_einsum("bhr,hdr->bhd"), block-128 scales on both sides).
    o, positions, cos_sin_cache and n_groups as ops.dsv4_inv_rope_quant.  wo_a_weight e4m3 [n_groups * R, D] and
    wo_a_scale f32 [n_groups * R / 128, D / 128] are the checkpoint's wo_a, read in place, R = o_lora_rank a multiple of
    128; checkpoints that store the scales as e8m0 (V4-Flash) convert them to f32 once at load, which is exact.  Each
    128-wide k-block is one tensor-core accumulation, added in fp32 times both scales.  A token's result does not depend
    on the other tokens of the call.  Returns z bf16 [T, n_groups * R], the input of wo_b."""
    T, H, G, _ = _dsv4_o_args(o, positions, cos_sin_cache, n_groups)
    hpg = H // G
    D = hpg * 512
    w, ws = wo_a_weight, wo_a_scale
    if w.dtype != torch.float8_e4m3fn or w.dim() != 2 or w.shape[1] != D or w.shape[0] % G \
            or (w.shape[0] // G) % 128 or w.shape[0] == 0:
        raise ValueError(f"wo_a_weight must be e4m3 [n_groups * R, {D}] with R a multiple of 128, got {w.dtype} "
                         f"{tuple(w.shape)}")
    R = w.shape[0] // G
    if not w.is_contiguous() or w.data_ptr() % 16:
        raise ValueError("wo_a_weight must be contiguous and 16-byte aligned (it is read in place)")
    if ws.dtype != torch.float32 or tuple(ws.shape) != (G * R // 128, D // 128):
        raise ValueError(f"wo_a_scale must be f32 [{G * R // 128}, {D // 128}], got {ws.dtype} {tuple(ws.shape)}")
    _device(o, "o")
    w, ws = _device(w, "wo_a_weight"), _cuda(ws, "wo_a_scale")
    z = torch.empty(T, G * R, dtype=torch.bfloat16, device=o.device)
    if T == 0:
        return z
    o_fp8, o_scale = _dsv4_inv_rope_quant(o, positions, cos_sin_cache, G)
    lib = L.lib()
    need = int(lib.b200_dsv4_wo_a_workspace_bytes(T, G, hpg, R))
    buf = _persistent_workspace("dsv4_wo_a", o.device, need) if need else None
    rc = lib.b200_dsv4_wo_a(_stream(), o_fp8.data_ptr(), o_scale.data_ptr(), w.data_ptr(), ws.data_ptr(), T, G, hpg, R,
                            buf.data_ptr() if need else None, buf.numel() if need else 0, z.data_ptr())
    L.check(rc, "b200_dsv4_wo_a")
    return z
