"""Time multi-token MLA decode (verification of multi-token-prediction drafts) at DeepSeek-V3 shapes (H100, CUDA graphs).

    python tools/mla_spec_step.py [--replays 1000] [--warmup 50] [--q 1 2 3 4]

Shapes: bench.WORKLOADS["dsv3-fp8"] (Hq 128, batch 1, KV 4096, page 64) and a tensor-parallel shard of it (128 heads / TP8 =
16 heads) at batch 32, KV 4096, each on a bf16 and an e4m3 latent cache, every request holding KV + Q keys.  For each Q two
variants are captured once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`:
  spec      ops.mla_decode(q_len_per_req=Q): one call, query token i of request b sees its first S_b - Q + 1 + i keys;
  expanded  the workaround without it: ops.mla_decode on B*Q single-token requests (page-table rows repeated, seq_len
            S_b - Q + 1 + i), which reads every request's latent cache Q times.
Each variant uses the split count ops.mla_decode picks by default for it.  With Q = 1 the single-token C entry point
b200_mla_decode_ex and b200_mla_decode_spec(q_len = 1) are also timed against each other, alternated twice, on the same
arguments.  Prints one JSON line per (shape, cache, Q): microseconds of each variant, its algorithmic latent-cache bytes (the
spec call reads a request's cache once per q-group, n_qg = ceil(Q / Qg) with Qg = min(Q, 128 / Hq) draft tokens per group;
the expanded batch once per draft token, each over its own prefix), its fp32 partial bytes (B*Q*Hq*splits*514*4), and the GPU's
name and power limit read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import WORKLOADS  # noqa: E402
from lvllm_b200 import _lib as L  # noqa: E402
from lvllm_b200 import ops  # noqa: E402


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
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
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
    return round(a.elapsed_time(b) * 1e3 / replays, 2)


def _n_qg(hq, Q):
    qg = min(Q, 128 // hq)
    return -(-Q // qg)


def _default_splits(B, hq, Q, max_pages, page):
    """The split count ops.mla_decode picks when num_kv_splits is 0."""
    tiles = max(1, -(-(max_pages * page) // 128))
    return max(1, min(tiles, 264 // (4 * B * _n_qg(hq, Q))))


def run(shape, B, S, page, hq, kv_dtype, Q, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    lens = torch.full((B,), S + Q, dtype=torch.int32, device=dev)
    npg = -(-(S + Q) // page)
    cache = torch.randn(B * npg, page, 576, generator=gen, device=dev).to(kv_dtype)
    pt = torch.randperm(B * npg, device=dev).reshape(B, npg).int()
    qn = torch.randn(B * Q, hq, 512, generator=gen, device=dev).bfloat16()
    qp = torch.randn(B * Q, hq, 64, generator=gen, device=dev).bfloat16()
    i = torch.arange(Q, device=dev, dtype=torch.int32)
    lens_x = (lens[:, None] - Q + 1 + i[None, :]).reshape(-1)
    pt_x = pt.repeat_interleave(Q, dim=0)
    scale = 1.0 / math.sqrt(192)
    splits = dict(spec=_default_splits(B, hq, Q, npg, page), expanded=_default_splits(B * Q, hq, 1, npg, page))

    def spec():
        return ops.mla_decode(qn, qp, cache, lens, pt, scale, num_kv_splits=splits["spec"], k_scale=0.5, q_len_per_req=Q)

    def expanded():
        return ops.mla_decode(qn, qp, cache, lens_x, pt_x, scale, num_kv_splits=splits["expanded"], k_scale=0.5)

    us = {f.__name__: _time(_graph(f), replays, warmup) for f in (spec, expanded)}
    esz = 1 if kv_dtype == torch.float8_e4m3fn else 2
    n_qg = _n_qg(hq, Q)
    res = dict(shape=shape, batch=B, kv_len=S, q_len=Q, page=page, Hq=hq,
               cache="e4m3" if esz == 1 else "bf16", q_groups=n_qg, num_kv_splits=splits, us=us,
               cache_bytes=dict(spec=B * (S + Q) * 576 * esz * n_qg,
                                expanded=sum(B * (S + 1 + j) * 576 * esz for j in range(Q))),
               partial_bytes={k: B * Q * hq * v * 514 * 4 for k, v in splits.items()})
    if Q == 1:
        # today's single-token entry point against q_len = 1 of the new one, same arguments, alternated
        lib = L.lib()
        ws = torch.empty(lib.b200_mla_decode_workspace_bytes(B, hq, splits["spec"]), dtype=torch.uint8, device=dev)
        out = torch.empty(B, hq, 512, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(B, hq, dtype=torch.float32, device=dev)
        head = [qn.data_ptr(), qp.data_ptr(), 0, cache.data_ptr(), int(esz == 1), 1.0, 0.5, lens.data_ptr(), pt.data_ptr(), B]
        tail = [hq, page, npg, scale, splits["spec"], ws.data_ptr(), out.data_ptr(), lse.data_ptr()]

        def ex():
            L.check(lib.b200_mla_decode_ex(torch.cuda.current_stream().cuda_stream, *head, *tail), "b200_mla_decode_ex")

        def spec_q1():
            L.check(lib.b200_mla_decode_spec(torch.cuda.current_stream().cuda_stream, *head, 1, *tail, None, None),
                    "b200_mla_decode_spec")

        g_ex, g_sp = _graph(ex), _graph(spec_q1)
        res["single_token_us"] = dict(ex=[], spec_q1=[])
        for _ in range(2):
            res["single_token_us"]["ex"].append(_time(g_ex, replays, warmup))
            res["single_token_us"]["spec_q1"].append(_time(g_sp, replays, warmup))
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--q", type=int, nargs="+", default=[1, 2, 3, 4])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mla_spec_step.py needs a CUDA device")
    name, power = _gpu()
    w = WORKLOADS["dsv3-fp8"]
    shapes = [("dsv3-fp8", w["batch"], w["seq"], w["page"], w["Hq"]),
              ("dsv3-tp8-shard", 32, w["seq"], w["page"], w["Hq"] // 8)]
    for shape, B, S, page, hq in shapes:
        for kv_dtype in (torch.bfloat16, torch.float8_e4m3fn):
            for Q in a.q:
                print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays,
                                      **run(shape, B, S, page, hq, kv_dtype, Q, a.replays, a.warmup))), flush=True)


if __name__ == "__main__":
    main()
