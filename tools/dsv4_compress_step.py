"""Time the DeepSeek-V4 KV compressor (ops.dsv4_compress: state write + softmax-pooled compression, RMSNorm, RoPE and the
fp8 store) on the H100, in CUDA graphs.

    python tools/dsv4_compress_step.py [--replays 1000] [--warmup 50]

V4-Flash decode, one token per request at batch 1, 32 and 256, requests at random context lengths below 8192:
  c4a          a C4A layer: the D 512 call into the 584-byte cache and the D 128 call into the indexer's 132-byte cache
               (both ratio 4, overlapping windows); about a quarter of the tokens close a window;
  c128a        a C128A layer (D 512, ratio 128) in a typical step: at most 2 tokens close a window;
  c128a_worst  the same with every token at a boundary.
Two variants, each captured once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`,
alternated twice:
  kernel  ops.dsv4_compress;
  torch   the same work composed from vectorised torch ops: state write by index_copy_, gather of every boundary token's
          window, softmax, weighted sum, RMSNorm, RoPE, ue8m0 e4m3 quantisation and a scatter into the cache.  It processes
          every token (a graph cannot branch on the boundary count) and masks the non-boundary ones at the scatter.
Prints one JSON line per shape: microseconds per variant, the kernel's algorithmic bytes and GB/s over its time, and the
GPU's name and power limit read in the same run.  Algorithmic bytes: the state write reads and writes T * 2 * coff * D * 4;
a boundary token reads (1 + overlap) * ratio * 2 * D * 4 of state and writes one cache row.  Writes nothing.
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

CTX, SBS, KV_BS, EPS = 8192, 64, 64, 1e-6


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


class Call:
    """One compressor's inputs and caches for B requests, one decode token each at the given positions."""

    def __init__(self, D, ratio, positions, dev, gen):
        B = positions.numel()
        self.D, self.ratio = D, ratio
        self.coff = 2 if ratio == 4 else 1
        half = self.coff * D
        per = CTX // SBS
        self.bt = torch.randperm(B * per, device=dev).reshape(B, per).int()
        self.state = torch.randn(B * per, SBS, 2 * half, device=dev, generator=gen)
        self.kv_score = torch.randn(B, 2 * half, device=dev, generator=gen)
        self.ape = torch.randn(ratio, half, device=dev, generator=gen)
        self.pos = positions.to(dev)
        req = torch.arange(B, device=dev)
        self.req = req.int()
        self.slot = (self.bt[req, self.pos // SBS].long() * SBS + self.pos % SBS)
        kv_rows = B * (CTX // ratio)
        self.kslot = req * (CTX // ratio) + self.pos // ratio
        self.row = 584 if D == 512 else 132
        self.cache = torch.zeros(-(-kv_rows // KV_BS), KV_BS, self.row, dtype=torch.uint8, device=dev)
        self.w = (1 + 0.1 * torch.randn(D, device=dev, generator=gen)).bfloat16()
        inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64, device=dev) / 64))
        f = torch.arange(CTX, dtype=torch.float64, device=dev)[:, None] * inv[None]
        self.cs = torch.cat([f.cos(), f.sin()], 1).float()
        self.n_boundary = int(((self.pos + 1) % ratio == 0).sum())

    def kernel(self):
        ops.dsv4_compress(self.kv_score, self.ape, self.pos, self.state, self.slot, self.req, self.bt, self.w, EPS, self.cs,
                          self.cache, self.kslot, self.ratio)

    def torch(self):
        D, R, half = self.D, self.ratio, self.coff * self.D
        flat = self.state.view(-1, 2 * half)
        sc = self.kv_score[:, half:] + self.ape[self.pos % R]
        flat.index_copy_(0, self.slot, torch.cat([self.kv_score[:, :half], sc], 1))
        W = self.coff * R
        wp = self.pos[:, None] - W + 1 + torch.arange(W, device=self.pos.device)            # [B, W]
        valid = wp >= 0
        wpc = wp.clamp(min=0)
        rows = flat[(self.bt[self.req.long()[:, None], wpc // SBS].long() * SBS + wpc % SBS)]   # [B, W, 2 half]
        if self.coff == 2:
            kv = torch.cat([rows[:, :R, :D], rows[:, R:, D:half]], 1)
            s = torch.cat([rows[:, :R, half:half + D], rows[:, R:, half + D:]], 1)
        else:
            kv, s = rows[..., :D], rows[..., half:]
        s = s.masked_fill(~valid[..., None], float("-inf"))
        c = (torch.softmax(s, 1) * kv).sum(1)
        x = c * torch.rsqrt((c * c).mean(-1, keepdim=True) + EPS) * self.w.float()
        cs = self.cs[(self.pos // R) * R]
        e, o = x[:, D - 64::2], x[:, D - 63::2]
        rot = torch.stack([e * cs[:, :32] - o * cs[:, 32:], o * cs[:, :32] + e * cs[:, 32:]], -1).flatten(1)
        x = torch.cat([x[:, :D - 64], rot], 1).bfloat16().float()
        nb, bs = self.cache.shape[:2]
        cflat = self.cache.view(nb, -1)
        keep = ((self.pos + 1) % R == 0)
        b, p = self.kslot // bs, self.kslot % bs
        if D == 512:
            g = x[:, :448].reshape(-1, 7, 64)
            e8 = torch.ceil(torch.log2(g.abs().amax(-1).clamp(min=1e-4) / 448))
            q8 = (g * torch.exp2(-e8)[..., None]).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).flatten(1)
            data = torch.cat([q8, x[:, 448:].bfloat16().view(torch.uint8)], 1)                # [B, 576]
            rec = torch.cat([(e8 + 127).to(torch.uint8), torch.zeros_like(e8[:, :1], dtype=torch.uint8)], 1)
            doff, roff, dw = p * 576, bs * 576 + p * 8, 576
        else:
            e8 = torch.ceil(torch.log2(x.abs().amax(-1, keepdim=True).clamp(min=1e-4) / 448))
            data = (x * torch.exp2(-e8)).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
            rec = torch.exp2(e8).view(torch.uint8)
            doff, roff, dw = p * 128, bs * 128 + p * 4, 128
        bb = torch.where(keep, b, nb)                                  # non-boundary tokens go to a dropped row
        pad = torch.cat([cflat, cflat[:1]], 0)
        pad[bb[:, None], doff[:, None] + torch.arange(dw, device=b.device)] = data
        pad[bb[:, None], roff[:, None] + torch.arange(rec.shape[1], device=b.device)] = rec
        cflat.copy_(pad[:nb])

    def bytes(self):
        half = self.coff * self.D
        B = self.pos.numel()
        return B * 2 * half * 4 * 2 + self.n_boundary * (self.coff * self.ratio * 2 * self.D * 4 + self.row)


def run(shape, B, replays, warmup, dev):
    gen = torch.Generator(device=dev).manual_seed(0)
    ctx = torch.randint(256, CTX - 1, (B,), device=dev, generator=gen)
    if shape == "c4a":
        calls = [Call(512, 4, ctx, dev, gen), Call(128, 4, ctx, dev, gen)]
    else:
        pos = ctx.clone()
        if shape == "c128a_worst":
            pos = (ctx // 128) * 128 + 127
        else:
            pos = torch.where((pos + 1) % 128 == 0, pos + 1, pos)      # no boundary, then at most 2 of them
            pos[: min(2, B)] = (pos[: min(2, B)] // 128) * 128 + 127
        calls = [Call(512, 128, pos, dev, gen)]
    gk = _graph(lambda: [c.kernel() for c in calls])
    gt = _graph(lambda: [c.torch() for c in calls])
    us = dict(kernel=[], torch=[])
    for _ in range(2):
        us["kernel"].append(_time(gk, replays, warmup))
        us["torch"].append(_time(gt, replays, warmup))
    alg = sum(c.bytes() for c in calls)
    return dict(shape=shape, batch=B, boundary_tokens=[c.n_boundary for c in calls], us=us, bytes=alg,
                GBps=round(alg / min(us["kernel"]) / 1e3, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dsv4_compress_step.py needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = _gpu()
    for shape in ("c4a", "c128a", "c128a_worst"):
        for B in (1, 32, 256):
            print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays,
                                  **run(shape, B, a.replays, a.warmup, dev))), flush=True)


if __name__ == "__main__":
    main()
