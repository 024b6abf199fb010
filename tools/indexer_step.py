"""Time the lightning indexer's decode step (paged fp8 MQA logits, then the per-row top-k) on the H100, in CUDA graphs.

    python tools/indexer_step.py [--replays 1000] [--warmup 50]

Shapes (DeepSeek-V3.2: 64 index heads, index_topk 2048, page 64): batch 1 at 32K and 128K context, batch 32 at 32K context
with one and with two query tokens per request (a multi-token-prediction draft).  The fp8 indexer cache holds random
finite e4m3 values with positive fp32 scales.  Each variant is captured once in a CUDA graph and timed with CUDA events
over `--replays` replays after `--warmup`, alternated twice:
  logits  ops.indexer_logits;
  topk    ops.indexer_topk on those logits;
  torch   the torch composition of the same work on the same card: gather the pages, dequantise, einsum, relu, the
          weighted sum over heads, the causal mask and torch.topk.
Prints one JSON line per shape: microseconds of each variant, the algorithmic bytes of the logits kernel
(sum_b S_b * 132 * n_qg cache bytes, n_qg = the q-groups that each re-read the cache, + q and weights + the logits it
writes) and GB/s over its time, and the GPU's name and power limit read in the same run.  Writes nothing.
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

from lvllm_b200 import ops  # noqa: E402

H, TOPK, PAGE = 64, 2048, 64
SHAPES = (("b1-s32k", 1, 32768, 1), ("b1-s128k", 1, 131072, 1), ("b32-s32k", 32, 32768, 1), ("b32-s32k-q2", 32, 32768, 2))


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


def _e4m3(shape, gen, dev):
    """Random finite e4m3 bytes (no NaN codes 0x7f / 0xff)."""
    mag = torch.randint(0, 0x7F, shape, generator=gen, device=dev, dtype=torch.int32)
    sign = torch.randint(0, 2, shape, generator=gen, device=dev, dtype=torch.int32) * 0x80
    return (mag | sign).to(torch.uint8)


def run(shape, B, S, Q, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    npg = S // PAGE
    nb = B * npg
    cache = torch.empty(nb, PAGE * 132, dtype=torch.uint8, device=dev)
    cache[:, :PAGE * 128] = _e4m3((nb, PAGE * 128), gen, dev)
    cache[:, PAGE * 128:] = (torch.rand(nb, PAGE, generator=gen, device=dev) * 0.01 + 1e-3).view(torch.uint8)
    cache = cache.view(nb, PAGE, 132)
    pt = torch.randperm(nb, device=dev, generator=gen).reshape(B, npg).int()
    q8 = _e4m3((B * Q, H, 128), gen, dev).view(torch.float8_e4m3fn)
    w = torch.randn(B * Q, H, generator=gen, device=dev)
    sl = torch.full((B,), S, dtype=torch.int32, device=dev)
    logits = torch.empty(B * Q, npg * PAGE, dtype=torch.float32, device=dev)
    pos = torch.arange(npg * PAGE, device=dev)
    ends = (sl.repeat_interleave(Q) - Q + torch.arange(B * Q, device=dev) % Q + 1)[:, None]

    def k_logits():
        ops.indexer_logits(q8, w, cache, sl, pt, Q, logits=logits)

    def k_topk():
        return ops.indexer_topk(logits, sl, TOPK, Q)

    def torch_ref():
        blk = cache.view(nb, PAGE * 132)[pt.long()]                                   # [B, npg, page * 132]
        vals = blk[..., :PAGE * 128].contiguous().view(torch.float8_e4m3fn).float().view(B, npg * PAGE, 128)
        sc = blk[..., PAGE * 128:].contiguous().view(torch.float32).view(B, npg * PAGE)
        s = torch.einsum("bqhd,bkd->bqhk", q8.float().view(B, Q, H, 128), vals).relu()
        lg = (s * w.view(B, Q, H, 1)).sum(2) * sc[:, None, :]
        lg = lg.view(B * Q, -1).masked_fill(pos[None, :] >= ends, float("-inf"))
        return torch.topk(lg, TOPK, dim=-1).indices

    graphs = dict(logits=_graph(k_logits), topk=_graph(k_topk), torch=_graph(torch_ref))
    us = {k: [] for k in graphs}
    for _ in range(2):
        for k, g in graphs.items():
            us[k].append(_time(g, replays, warmup))
    qg = min(Q, 128 // H)
    n_qg = -(-Q // qg)
    alg = B * S * 132 * n_qg + B * Q * H * (128 + 4) + B * Q * S * 4
    return dict(shape=shape, batch=B, context=S, q_len=Q, heads=H, page=PAGE, topk=TOPK, us=us, logits_bytes=alg,
                logits_GBps=round(alg / min(us["logits"]) / 1e3, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("indexer_step.py needs a CUDA device")
    name, power = _gpu()
    for shape, B, S, Q in SHAPES:
        print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, **run(shape, B, S, Q, a.replays, a.warmup))),
              flush=True)


if __name__ == "__main__":
    main()
