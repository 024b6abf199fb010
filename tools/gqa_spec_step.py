"""Time multi-token GQA decode (speculative-decode verification) at the two GQA workloads of bench.py (H100, CUDA graphs).

    python tools/gqa_spec_step.py [--replays 1000] [--warmup 50] [--q 1 2 3 4]

Shapes come from bench.WORKLOADS: Mixtral-8x7B (batch 64, KV 2048, page 16, Hq 32 / Hkv 8) and Qwen3-235B-A22B (batch 256,
KV 512, page 16, Hq 64 / Hkv 4), on the FlashInfer backend's packed NHD cache, every request holding KV + Q keys.  For each
Q two variants are captured once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`:
  spec      ops.gqa_decode(q_len_per_req=Q): one call, query token i of request b sees its first S_b - Q + 1 + i keys;
  expanded  the workaround without it: ops.gqa_decode on B*Q single-token requests (page-table rows repeated, seq_len
            S_b - Q + 1 + i), which reads every request's K and V Q times.
Prints one JSON line per (workload, Q): microseconds of each, the algorithmic KV bytes of each (the spec call reads K and V
once per q-group, n_qg = ceil(Q / Qg) with Qg = min(Q, 32 / G) draft tokens per group; the expanded batch Q times), and the
GPU's name and power limit read in the same run.  Writes nothing.
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

from bench import WORKLOADS  # noqa: E402
from lvllm_b200 import ops  # noqa: E402

D = 128


def _gpu():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=60)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _time_graph(fn, replays, warmup):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(warmup):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / replays


def run(name, Q, replays, warmup):
    w = WORKLOADS[name]
    B, S, page, hq, hkv = w["batch"], w["seq"], w["page"], w["Hq"], w["Hkv"]
    G = hq // hkv
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    lens = torch.full((B,), S + Q, dtype=torch.int32, device=dev)
    npg = -(-(S + Q) // page)
    packed = torch.randn(B * npg, page, hkv, 2 * D, generator=gen, device=dev).bfloat16()   # NHD
    kc, vc = packed.permute(0, 2, 1, 3).transpose(1, 2).split(D, dim=-1)
    pt = torch.randperm(B * npg, device=dev).reshape(B, npg).int()
    q = torch.randn(B * Q, hq, D, generator=gen, device=dev).bfloat16()
    i = torch.arange(Q, device=dev, dtype=torch.int32)
    lens_x = (lens[:, None] - Q + 1 + i[None, :]).reshape(-1)
    pt_x = pt.repeat_interleave(Q, dim=0)
    scale = D ** -0.5
    # the same split count in both calls (the default of the spec call's page table)
    splits = -(-(npg * page) // 128)

    def spec():
        return ops.gqa_decode(q, kc, vc, lens, pt, scale, num_kv_splits=splits, q_len_per_req=Q)

    def expanded():
        return ops.gqa_decode(q, kc, vc, lens_x, pt_x, scale, num_kv_splits=splits)

    us = {f.__name__: round(_time_graph(f, replays, warmup), 2) for f in (spec, expanded)}
    qg = min(Q, 32 // G) if G <= 32 else 1
    n_qg = -(-Q // qg) if G <= 32 else Q   # groups of more than 32 heads take the CUDA-core kernel: one pass per token
    kv_bytes = B * (S + Q) * hkv * D * 2 * 2
    return dict(workload=name, batch=B, kv_len=S, q_len=Q, page=page, Hq=hq, Hkv=hkv, num_kv_splits=splits, us=us,
                kv_bytes=dict(spec=kv_bytes * n_qg, expanded=sum(B * (S + 1 + j) * hkv * D * 2 * 2 for j in range(Q))),
                q_groups=n_qg)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--q", type=int, nargs="+", default=[1, 2, 3, 4])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gqa_spec_step.py needs a CUDA device")
    name, power = _gpu()
    for n in ("mixtral-int4", "qwen3-mxfp4"):
        for Q in a.q:
            print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, **run(n, Q, a.replays, a.warmup))),
                  flush=True)


if __name__ == "__main__":
    main()
