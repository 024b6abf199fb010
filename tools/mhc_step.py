"""Time DeepSeek-V4's manifold hyper-connection step (post mapping + Sinkhorn pre mapping + fused RMSNorm) on the H100, in
CUDA graphs.

    python tools/mhc_step.py [--replays 1000] [--warmup 50]

hc_mult 4, sinkhorn_repeat 20, hc_post_mult_value 2.0, H in {4096, 7168}, T in {1, 16, 64, 256}.  Three variants, each captured
once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`, alternated twice:
  fused    ops.mhc_fused_post_pre with norm_weight (what every layer runs twice per decode step);
  split    ops.mhc_post, then ops.mhc_pre with norm_weight;
  torch    the same work composed from torch ops on the GPU (fp32 einsum, matmul, sigmoid, Sinkhorn loop, RMSNorm).
Prints one JSON line per shape: microseconds per variant, the largest |fused - torch| of layer_input, the algorithmic bytes
of the fused call T * (20H + 80) + 386H (residual in and out, x, the 4 + 16 mixing inputs and 4 + 16 outputs, layer_input,
fn and the norm weight) and GB/s over its time, and the GPU's name and power limit read in the same run.  Writes nothing.
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

EPS, REPEAT, POST_MULT = 1e-6, 20, 2.0


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
        out = fn()
    return g, out


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


def _torch_step(x, residual, plm, crm, fn, sc, base, w):
    T, _, H = residual.shape
    r = (torch.einsum("tij,tih->tjh", crm, residual.float()) + plm * x.float().unsqueeze(1)).bfloat16()
    rf = r.float().reshape(T, 4 * H)
    mixes = (rf @ fn.t()) * torch.rsqrt(rf.square().sum(-1, keepdim=True) / (4 * H) + EPS)
    pre = torch.sigmoid(mixes[:, :4] * sc[0] + base[:4]) + EPS
    post = torch.sigmoid(mixes[:, 4:8] * sc[1] + base[4:8]) * POST_MULT
    c = torch.softmax((mixes[:, 8:] * sc[2] + base[8:]).view(T, 4, 4), -1) + EPS
    c = c / (c.sum(-2, keepdim=True) + EPS)
    for _ in range(REPEAT - 1):
        c = c / (c.sum(-1, keepdim=True) + EPS)
        c = c / (c.sum(-2, keepdim=True) + EPS)
    o = (pre.unsqueeze(-1) * r.float()).sum(1)
    li = (o.bfloat16().float() * torch.rsqrt(o.square().mean(-1, keepdim=True) + EPS) * w.float()).bfloat16()
    return r, post.unsqueeze(-1), c, li


def run(H, T, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    fn = torch.randn(24, 4 * H, generator=gen, device=dev) * 1e-4
    sc = torch.randn(3, generator=gen, device=dev) * 0.1
    base = torch.randn(24, generator=gen, device=dev) * 0.1
    w = (1 + 0.1 * torch.randn(H, generator=gen, device=dev)).bfloat16()
    residual = torch.randn(T, 4, H, generator=gen, device=dev).bfloat16()
    x = torch.randn(T, H, generator=gen, device=dev).bfloat16()
    plm = torch.rand(T, 4, 1, generator=gen, device=dev) * 2
    crm = torch.softmax(torch.randn(T, 4, 4, generator=gen, device=dev), -2)
    args = (fn, sc, base, EPS, EPS, EPS, POST_MULT, REPEAT)

    def fused():
        return ops.mhc_fused_post_pre(x, residual, plm, crm, *args, norm_weight=w, norm_eps=EPS)

    def split():
        r = ops.mhc_post(x, residual, plm, crm)
        return (r, *ops.mhc_pre(r, *args, norm_weight=w, norm_eps=EPS))

    def composed():
        return _torch_step(x, residual, plm, crm, fn, sc, base, w)

    (gf, of), (gs, _), (gt, ot) = _graph(fused), _graph(split), _graph(composed)
    gf.replay()
    gt.replay()
    torch.cuda.synchronize()
    diff = (of[3].float() - ot[3].float()).abs().max().item()
    us = dict(fused=[], split=[], torch=[])
    for _ in range(2):
        us["fused"].append(_time(gf, replays, warmup))
        us["split"].append(_time(gs, replays, warmup))
        us["torch"].append(_time(gt, replays, warmup))
    alg = T * (20 * H + 80) + 386 * H
    return dict(H=H, T=T, us=us, max_abs_diff_fused_torch=diff, fused_bytes=alg,
                fused_GBps=round(alg / min(us["fused"]) / 1e3, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mhc_step.py needs a CUDA device")
    name, power = _gpu()
    for H in (4096, 7168):
        for T in (1, 16, 64, 256):
            print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, **run(H, T, a.replays, a.warmup))),
                  flush=True)


if __name__ == "__main__":
    main()
