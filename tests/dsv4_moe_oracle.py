"""Float32 restatement of DeepSeek-V4's MoE routing and expert activation, as the kernels compute them.

Routing (reference csrc/libtorch_stable/moe/topk_softplus_sqrt_kernels.cu, router/fused_topk_bias_router.py):
  * score s = sqrt(softplus(x)) with softplus(x) = x for x > 20 (F.softplus's threshold), else log1p(exp(x));
    a non-finite score becomes 0;
  * top-k: select by s + bias (one fp32 add), k rounds of arg-max, ties to the lower expert index, output in selection
    order; the weight is the unbiased s (the reference's dsv4_topk and torch paths; its CUDA kernel weights by
    (s + b) - b instead);
  * hash: no bias; ids = table[input_ids[t], j] in table order, weights the s of those experts; an input id outside
    [0, vocab) or a table entry outside [0, E) gives id -1 and weight 0 in that slot;
  * weights: sum sequentially in fp32, scale = rsf / (sum > 0 ? sum : 1) when renormalising (rsf otherwise), w * scale.

Activation type 3 (SiluAndMulWithClamp with alpha 1, beta 0): gate = min(gate, limit), up = clamp(up, -limit, limit),
gate * sigmoid(gate) * up, on the rounded gate and up values the SiLU branch uses.
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch

from oracle import moe_oracle as O

ACT_SILU_CLAMP = 3
F32 = np.float32


def sqrt_softplus(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, F32)
    with np.errstate(over="ignore", invalid="ignore"):
        sp = np.where(x > F32(20.0), x, np.log1p(np.exp(x)).astype(F32)).astype(F32)
        s = np.sqrt(sp).astype(F32)
    return np.where(np.isfinite(s), s, F32(0.0)).astype(F32)


def topk_sqrtsoftplus(logits, k: int, renormalize: bool, bias=None, rsf: float = 1.0, input_ids=None, table=None):
    """(weights f32 [M,k], ids i32 [M,k]) as torch tensors; hash routing when ``table`` [vocab, k] is given."""
    x = torch.as_tensor(logits).detach().to(torch.float32).cpu().numpy()
    M, E = x.shape
    s = sqrt_softplus(x)
    w = np.zeros((M, k), F32)
    ids = np.full((M, k), -1, np.int32)
    rows = np.arange(M)
    if table is not None:
        tab = torch.as_tensor(table).cpu().numpy().astype(np.int64)
        tid = torch.as_tensor(input_ids).cpu().numpy().astype(np.int64).reshape(-1)
        vocab = tab.shape[0]
        for t in range(M):
            if not (0 <= tid[t] < vocab):
                continue
            for j in range(k):
                e = int(tab[tid[t], j])
                if 0 <= e < E:
                    ids[t, j] = e
                    w[t, j] = s[t, e]
    else:
        choice = s.copy()
        if bias is not None:
            b = torch.as_tensor(bias).detach().to(torch.float32).cpu().numpy()
            choice = (choice + b[None, :]).astype(F32)
        for j in range(k):
            idx = choice.argmax(axis=1)   # first occurrence: the lower index wins a tie
            ids[:, j] = idx
            w[:, j] = s[rows, idx]
            choice[rows, idx] = -np.inf
    scale = np.full((M,), F32(rsf), F32)
    if renormalize:
        ssum = np.zeros((M,), F32)
        for j in range(k):
            ssum = (ssum + w[:, j]).astype(F32)
        scale = (scale / np.where(ssum > 0, ssum, F32(1.0))).astype(F32)
    w = (w * scale[:, None]).astype(F32)
    return torch.from_numpy(w), torch.from_numpy(ids)


def silu_clamp(h: torch.Tensor, limit: float) -> torch.Tensor:
    """Activation type 3 on a packed [gate | up] tensor, with the operation order of SiluAndMulWithClamp.forward_native."""
    d = h.shape[-1] // 2
    gate = torch.clamp(h[..., :d], max=limit)
    up = torch.clamp(h[..., d:], min=-limit, max=limit)
    return gate * torch.sigmoid(gate) * up


@contextlib.contextmanager
def clamped_activation(limit: float):
    """Within the block, the expert oracles of oracle.moe_oracle (experts_forward_batched, experts_forward_w8a8_block,
    ...) accept activation_type 3 with this limit; every other type runs as before."""
    base = O.apply_activation

    def apply_activation(h, activation_type, has_gate=True, *args, **kw):
        if activation_type == ACT_SILU_CLAMP and has_gate:
            return silu_clamp(h, limit)
        return base(h, activation_type, has_gate, *args, **kw)

    O.apply_activation = apply_activation
    try:
        yield
    finally:
        O.apply_activation = base
