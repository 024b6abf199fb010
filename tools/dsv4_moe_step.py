"""Time one DeepSeek-V4-Flash MoE layer at decode on the H100, in CUDA graphs.

    python tools/dsv4_moe_step.py [--replays 200] [--warmup 20]

Shapes: 256 routed experts and top-6 (the reference's dsv4_topk serves E 256, k 6); hidden 4096, moe intermediate 2048,
vocab 129280, swiglu_limit 10 and routed_scaling_factor 1.5 are taken from the public DeepSeek-V4-Flash model config,
which is not in the reference tree.  One shared expert is folded into the routed launch as an always-on column (top-7 in
cpu_decode).  Experts are MXFP4 with random weights and scales, generated on the GPU; the gate weight and hidden states
are bf16.  For decode batches M in {1, 16, 64, 256}, for a sqrt-softplus layer (bias ~ 8.08) and a hash layer (table
[vocab, 6]), each captured once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`:
  router        Router.select_experts in the fused form (gate GEMM + routing + shared column, one kernel);
  torch_router  the torch composition of the same routing: bf16 gate matmul, softplus, sqrt, + bias, topk, gather,
                renormalise, scale (hash: table lookup and gather);
  decode_clamp  MOE_MXFP4.cpu_decode with activation_type 3 (swiglu_limit assigned);
  decode_silu   the same weights and routing with plain SiLU, to show what the clamp costs.
Prints one JSON line per (layer, M) in microseconds, with the GPU's name and power limit read in the same run.  Writes
nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import lk_moe  # noqa: E402
from lvllm_b200.router import Router  # noqa: E402

E, K, H, I, VOCAB, LIMIT, RSF = 256, 6, 4096, 2048, 129280, 10.0, 1.5
BATCHES = (1, 16, 64, 256)


def _gpu():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=60)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _graph(fn):
    fn()   # eager warm-up: workspaces are allocated outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    return g


def _time(g, replays, warmup):
    for _ in range(warmup):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / replays


def _layer(clamp, w13, w2, s13, s2):
    c = lk_moe.MOEConfigV2()
    c.expert_num, c.top_k, c.hidden_size, c.intermediate_size = E + 1, K + 1, H, I
    c.max_batch_size, c.max_num_seqs = max(BATCHES), max(BATCHES)
    c.groupN, c.groupK = 1, 32
    if clamp:
        c.swiglu_limit = LIMIT
    return lk_moe.MOE_MXFP4(c, w13.data_ptr(), w2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0,
                            weights_on_device=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = _gpu()
    g = torch.Generator(device=dev).manual_seed(0)
    u8 = dict(dtype=torch.uint8, device=dev, generator=g)
    w13 = torch.randint(0, 256, (E + 1, 2 * I, H // 2), **u8)
    w2 = torch.randint(0, 256, (E + 1, H, I // 2), **u8)
    s13 = torch.randint(118, 122, (E + 1, 2 * I, H // 32), **u8)
    s2 = torch.randint(118, 122, (E + 1, H, I // 32), **u8)
    layers = {"decode_clamp": _layer(True, w13, w2, s13, s2), "decode_silu": _layer(False, w13, w2, s13, s2)}
    del w13, w2, s13, s2
    wg = (torch.randn(E, H, device=dev, generator=g) / 64).bfloat16()
    bias = 8.08 + 1e-3 * torch.randn(E, device=dev, generator=g)
    table = torch.randint(0, E, (VOCAB, K), device=dev, generator=g, dtype=torch.int32)
    routers = {
        "sqrtsoftplus": Router(K, E, True, "sqrtsoftplus", routed_scaling_factor=RSF, e_score_correction_bias=bias,
                               num_fused_shared_experts=1, shared_local_base=E),
        "hash": Router(K, E, True, "sqrtsoftplus", routed_scaling_factor=RSF, num_fused_shared_experts=1,
                       shared_local_base=E, hash_indices_table=table),
    }
    for kind, router in routers.items():
        for M in BATCHES:
            x = (torch.randn(M, H, device=dev, generator=g) / 4).bfloat16()
            input_ids = torch.randint(0, VOCAB, (M,), device=dev, generator=g, dtype=torch.int32)
            out = torch.empty(M, H, dtype=torch.float32, device=dev)
            w, ids = router.select_experts(x, gate_weight=wg, input_ids=input_ids)
            loc = router.last_local_ids

            def route():
                router.select_experts(x, gate_weight=wg, input_ids=input_ids)

            def torch_route():
                logits = (x @ wg.t()).float()
                s = F.softplus(logits).sqrt()
                if kind == "hash":
                    tid = table[input_ids.long()].long()
                else:
                    tid = torch.topk(s + bias, K, dim=-1).indices
                tw = s.gather(1, tid)
                return tw / tw.sum(-1, keepdim=True) * RSF

            res = dict(gpu=name, power_limit=power, layer=kind, M=M, replays=a.replays)
            res["router_us"] = _time(_graph(route), a.replays, a.warmup)
            res["torch_router_us"] = _time(_graph(torch_route), a.replays, a.warmup)
            for key, moe in layers.items():
                def decode(moe=moe):
                    moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, K + 1, x.data_ptr(), loc.data_ptr(),
                                   w.data_ptr(), out.data_ptr())
                res[f"{key}_us"] = _time(_graph(decode), a.replays, a.warmup)
            print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}), flush=True)
    for moe in layers.values():
        moe.close()


if __name__ == "__main__":
    main()
