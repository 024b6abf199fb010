"""The router object of a MoE layer (SURVEY.md 8 row a2): the reference's `FusedMoERouter.select_experts` template
(vllm/model_executor/layers/fused_moe/router/fused_moe_router.py:45-81 -> `BaseRouter._select_experts`, base_router.py:259-305:
compute routing -> capture the logical ids -> EPLB map -> index dtype) over this repository's routing kernels.

Two ways in, one way out:
  * `select_experts(hidden_states, router_logits)` — the reference's signature: logits computed by the caller's gate
    (`fused_topk` for plain softmax / sigmoid routing, fused_topk_router.py:81-124; `grouped_topk` for DeepSeek's
    group-limited routing, grouped_topk_router.py:249-330);
  * `select_experts(hidden_states, gate_weight=W_g)` — the fused form: router GEMM + top-k + EP id remap (+ always-on shared
    expert columns) in ONE kernel (`ops.router_topk`), no logits tensor.
DeepSeek-V4 layers use `scoring_func="sqrtsoftplus"` (the bias selects, the weights are the unbiased scores); its first
`num_hash_layers` layers route by `hash_indices_table` [vocab, k] instead, reading `input_ids` in `select_experts`.
Both return `(topk_weights f32 [M, k'], topk_ids [M, k'])` with GLOBAL logical ids, like the reference; the EP-local ids lk_moe
consumes (`RoutedExperts.global_to_local_expert_ids`, routed_experts.py:1332-1342) are kept in `last_local_ids`.
Host-side glue only: every tensor operation is one of the C-ABI kernels behind `lvllm_b200.ops`.
"""
from __future__ import annotations

from typing import Callable

import torch

from . import ops


class Router:
    def __init__(self, top_k: int, global_num_experts: int, renormalize: bool = True, scoring_func: str = "softmax",
                 num_expert_group: int = 0, topk_group: int = 0, routed_scaling_factor: float = 1.0,
                 e_score_correction_bias: torch.Tensor | None = None, expert_map: torch.Tensor | None = None,
                 num_fused_shared_experts: int = 0, shared_local_base: int = -1, shared_weight: float = 1.0,
                 capture_fn: Callable[[torch.Tensor], None] | None = None, eplb_state=None,
                 hash_indices_table: torch.Tensor | None = None):
        if top_k <= 0 or global_num_experts <= 0 or top_k > global_num_experts:
            raise ValueError(f"bad top_k / global_num_experts: {top_k} / {global_num_experts}")
        if (num_expert_group > 0) != (topk_group > 0):
            raise ValueError("num_expert_group and topk_group are set together (grouped routing) or not at all")
        if num_expert_group > 0 and (global_num_experts % num_expert_group or topk_group > num_expert_group):
            raise ValueError("grouped routing: experts must divide into the groups and topk_group <= num_expert_group")
        if scoring_func not in ("softmax", "sigmoid", "sqrtsoftplus"):
            raise ValueError(f"unsupported scoring function {scoring_func!r}")
        if scoring_func == "sqrtsoftplus" and num_expert_group > 0:
            raise ValueError("grouped routing with sqrtsoftplus scores is not supported")
        if hash_indices_table is not None:
            if scoring_func != "sqrtsoftplus":
                raise ValueError("hash routing weights experts by sqrtsoftplus scores: pass scoring_func='sqrtsoftplus'")
            if hash_indices_table.dim() != 2 or hash_indices_table.shape[1] != top_k:
                raise ValueError(f"hash_indices_table must be [vocab, {top_k}], got {tuple(hash_indices_table.shape)}")
        if eplb_state is not None:
            # EPLB (redundant physical experts, vllm/distributed/eplb) is outside the hot-path scope (SURVEY.md 2): refusing
            # is better than silently routing to logical ids
            raise NotImplementedError("EPLB logical -> physical expert mapping is not supported")
        if num_fused_shared_experts and (expert_map is None and shared_local_base < 0):
            raise ValueError("shared experts ride in the routed launch at local ids shared_local_base + s: state the base")
        self.top_k, self.global_num_experts = int(top_k), int(global_num_experts)
        self.renormalize, self.scoring_func = bool(renormalize), scoring_func
        self.num_expert_group, self.topk_group = int(num_expert_group), int(topk_group)
        self.routed_scaling_factor = float(routed_scaling_factor)
        self.e_score_correction_bias = e_score_correction_bias
        self.expert_map = expert_map
        self.num_fused_shared_experts = int(num_fused_shared_experts)
        self.shared_local_base, self.shared_weight = int(shared_local_base), float(shared_weight)
        self.capture_fn = capture_fn
        # int32 once here, so that the per-step call converts nothing
        self.hash_indices_table = hash_indices_table.to(torch.int32).contiguous() if hash_indices_table is not None else None
        self.last_local_ids: torch.Tensor | None = None

    # ---- step 2 of the template: the routing algorithm -----------------------------------------------------------
    def _compute_routing(self, hidden_states: torch.Tensor, router_logits: torch.Tensor | None,
                         gate_weight: torch.Tensor | None, input_ids: torch.Tensor | None):
        hashed = self.hash_indices_table is not None
        if hashed and input_ids is None:
            raise ValueError("this router's layer routes by token-id hash: select_experts needs input_ids")
        if gate_weight is not None:
            if gate_weight.shape[0] != self.global_num_experts:
                raise ValueError(f"gate_weight has {gate_weight.shape[0]} rows, the router {self.global_num_experts} experts")
            if self.num_expert_group > 0 and self.scoring_func != "sigmoid":
                raise ValueError("the fused router serves grouped routing with sigmoid scores (DeepSeek); pass router_logits "
                                 "for grouped softmax routing")
            w, ids, loc = ops.router_topk(hidden_states, gate_weight, self.top_k, self.renormalize, self.scoring_func,
                                          self.e_score_correction_bias, self.routed_scaling_factor, self.num_expert_group,
                                          self.topk_group, self.expert_map, False, self.num_fused_shared_experts,
                                          self.shared_local_base, self.shared_weight,
                                          **(dict(input_ids=input_ids, hash_indices_table=self.hash_indices_table)
                                             if hashed else {}))
            return w, ids, loc
        if router_logits is None:
            raise ValueError("select_experts needs router_logits or gate_weight")
        if router_logits.shape[-1] != self.global_num_experts:
            raise ValueError(f"router_logits has {router_logits.shape[-1]} columns, the router {self.global_num_experts} experts")
        if self.num_fused_shared_experts:
            raise ValueError("shared-expert columns are appended by the fused form (pass gate_weight)")
        if self.num_expert_group > 0:
            w, ids = ops.grouped_topk(router_logits, self.top_k, self.renormalize, self.num_expert_group, self.topk_group,
                                      self.scoring_func, self.routed_scaling_factor, self.e_score_correction_bias)
        elif hashed:
            w, ids = ops.hash_topk(router_logits, self.top_k, self.renormalize, input_ids, self.hash_indices_table,
                                   self.routed_scaling_factor)
        else:
            w, ids = ops.fused_topk(router_logits, self.top_k, self.renormalize, self.scoring_func,
                                    self.e_score_correction_bias, self.routed_scaling_factor)
        loc = ops.global_to_local_expert_ids(ids, self.expert_map) if self.expert_map is not None else None
        return w, ids, loc

    # ---- the template (base_router.py:259-305) ---------------------------------------------------------------------
    def select_experts(self, hidden_states: torch.Tensor, router_logits: torch.Tensor | None = None,
                       topk_indices_dtype: torch.dtype | None = None, *, input_ids: torch.Tensor | None = None,
                       gate_weight: torch.Tensor | None = None):
        """`input_ids` [M] are the token ids; read only by a hash-routed layer (``hash_indices_table`` set), which
        raises ValueError without them."""
        topk_weights, topk_ids, local_ids = self._compute_routing(hidden_states, router_logits, gate_weight, input_ids)
        if self.capture_fn is not None:          # logical ids, before any mapping (base_router.py:291-293)
            self.capture_fn(topk_ids)
        self.last_local_ids = local_ids
        if topk_indices_dtype is not None and topk_ids.dtype != topk_indices_dtype:
            topk_ids = topk_ids.to(dtype=topk_indices_dtype)
        return topk_weights, topk_ids
