"""Time sparse MLA decode (DeepSeek-V3.2 / GLM-5 layers: attention over each token's top-k keys) on the H100, in CUDA graphs.

    python tools/mla_sparse_step.py [--replays 1000] [--warmup 50]

Shapes (index_topk 2048, context 32K, page 64): Hq 128 at batch 1 (one GPU holding all heads), and a TP8 shard of it
(Hq 16) at batch 32; each on the bf16 cache (576 bf16 per token) and the fp8_ds_mla cache (656 bytes per token).  Every token's
index row holds 2048 distinct random positions of its request's 32K context.  Two variants are captured once in a CUDA
graph and timed with CUDA events over `--replays` replays after `--warmup`, alternated twice:
  sparse  ops.mla_decode_sparse at its default split count;
  dense   ops.mla_decode over 2048 contiguous keys per request on the bf16 cache (the same key count and, on the bf16
          cache, the same key bytes), at its default split count.
Prints one JSON line per (shape, cache): microseconds of each variant, the sparse call's algorithmic bytes
(T * topk_valid * {1152, 656} key bytes + q (T * Hq * 576 * 2) + out (T * Hq * 512 * 2)) and GB/s over its time, and the
GPU's name and power limit read in the same run.  Writes nothing.
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

from lvllm_b200 import ops  # noqa: E402

TOPK, CTX, PAGE = 2048, 32768, 64


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


def run(shape, B, hq, ds_mla, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    npg = CTX // PAGE
    lat = torch.randn(B * npg, PAGE, 576, generator=gen, device=dev).bfloat16()
    if ds_mla:
        x = lat.reshape(-1, 576).float()
        scale = (x[:, :512].reshape(-1, 4, 128).abs().amax(-1) / 448.0).clamp(min=torch.finfo(torch.float32).tiny)
        q8 = (x[:, :512].reshape(-1, 4, 128) / scale[..., None]).to(torch.float8_e4m3fn).reshape(-1, 512)
        cache = torch.cat([q8.view(torch.uint8), scale.contiguous().view(torch.uint8),
                           lat.reshape(-1, 576)[:, 512:].contiguous().view(torch.uint8)], 1).reshape(B * npg, PAGE, 656)
    else:
        cache = lat
    pt = torch.randperm(B * npg, device=dev).reshape(B, npg).int()
    rid = torch.arange(B, dtype=torch.int32, device=dev)
    idx = torch.stack([torch.randperm(CTX, device=dev)[:TOPK] for _ in range(B)]).int()
    qn = torch.randn(B, hq, 512, generator=gen, device=dev).bfloat16()
    qp = torch.randn(B, hq, 64, generator=gen, device=dev).bfloat16()
    lens = torch.full((B,), TOPK, dtype=torch.int32, device=dev)
    pt_dense = pt[:, :TOPK // PAGE].contiguous()
    sm = 1.0 / math.sqrt(192)

    def sparse():
        return ops.mla_decode_sparse(qn, qp, cache, idx, rid, pt, sm)

    def dense():
        return ops.mla_decode(qn, qp, lat, lens, pt_dense, sm)

    gs, gd = _graph(sparse), _graph(dense)
    us = dict(sparse=[], dense=[])
    for _ in range(2):
        us["sparse"].append(_time(gs, replays, warmup))
        us["dense"].append(_time(gd, replays, warmup))
    key_bytes = B * TOPK * (656 if ds_mla else 1152)
    alg = key_bytes + B * hq * 576 * 2 + B * hq * 512 * 2
    return dict(shape=shape, batch=B, Hq=hq, topk=TOPK, context=CTX, page=PAGE, cache="fp8_ds_mla" if ds_mla else "bf16",
                us=us, sparse_bytes=alg, sparse_GBps=round(alg / min(us["sparse"]) / 1e3, 1),
                dense_key_bytes=B * TOPK * 1152)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mla_sparse_step.py needs a CUDA device")
    name, power = _gpu()
    for shape, B, hq in (("dsv32-hq128", 1, 128), ("dsv32-tp8-shard", 32, 16)):
        for ds_mla in (False, True):
            print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, **run(shape, B, hq, ds_mla, a.replays,
                                                                                           a.warmup))), flush=True)


if __name__ == "__main__":
    main()
