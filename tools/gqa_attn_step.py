"""Time the GQA attention step around the decode kernel at the two GQA workloads of bench.py (H100, CUDA graphs).

    python tools/gqa_attn_step.py [--replays 1000] [--warmup 50]

Shapes come from bench.WORKLOADS: Mixtral-8x7B (batch 64, KV 2048, page 16, Hq 32 / Hkv 8, no q/k norm) and
Qwen3-235B-A22B (batch 256, KV 512, page 16, Hq 64 / Hkv 4, per-head q/k norm).  Every variant is captured once in a CUDA
graph and timed with CUDA events over `--replays` replays after `--warmup`:
  write_fused          b200_gqa_qknorm_rope_cache_write alone (q/k norm + RoPE + cache write, one launch);
  write_torch          the unfused torch composition of the same work (per-head RMSNorm, RoPE in bf16 as the reference's
                       forward_static computes it, index_copy_ of k and v into the packed cache views);
  write_decode_packed  the fused write, then GQA decode, on the FlashInfer backend's packed NHD cache;
  decode_packed        GQA decode alone on the packed NHD cache (read through its strides);
  decode_separate      GQA decode on separate contiguous K / V caches (the layout the decode kernel had before strides).
Prints one JSON line: microseconds per variant, the algorithmic bytes of the write and of the decode, and the GPU's name and
power limit read in the same run.  Writes nothing.
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


def _rms(x, w, eps):
    """reference vllm/ir/ops/layernorm.py:10-21 on [T, heads, D]."""
    xf = x.float()
    return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(w.dtype) * w


def _rope(x, cos, sin):
    """NeoX RoPE over the full head in bf16 (reference rotary_embedding/common.py:146-185)."""
    x1, x2 = torch.chunk(x, 2, dim=-1)
    return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1)


def run(name, replays, warmup):
    w = WORKLOADS[name]
    B, S, page, hq, hkv = w["batch"], w["seq"], w["page"], w["Hq"], w["Hkv"]
    norm = name.startswith("qwen3")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    npg = -(-(S + 1) // page)
    blocks = B * npg
    qkv = torch.randn(B, (hq + 2 * hkv) * D, generator=gen, device=dev).bfloat16()
    inv = 1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.float, device=dev) / D))
    fr = torch.einsum("i,j->ij", torch.arange(32768, dtype=torch.float, device=dev), inv)
    table = torch.cat((fr.cos(), fr.sin()), dim=-1).bfloat16()
    qw = kw = None
    if norm:
        qw = (1 + 0.1 * torch.randn(D, generator=gen, device=dev)).bfloat16()
        kw = (1 + 0.1 * torch.randn(D, generator=gen, device=dev)).bfloat16()
    packed = torch.randn(blocks, page, hkv, 2 * D, generator=gen, device=dev).bfloat16()   # NHD
    kc, vc = packed.permute(0, 2, 1, 3).transpose(1, 2).split(D, dim=-1)
    k_sep, v_sep = kc.contiguous(), vc.contiguous()
    pt = torch.randperm(blocks, device=dev).reshape(B, npg).int()
    lens = torch.full((B,), S, dtype=torch.int32, device=dev)
    pos = lens.long()
    slots = pt[torch.arange(B, device=dev), (pos // page)].long() * page + pos % page
    q = torch.randn(B, hq, D, generator=gen, device=dev).bfloat16()
    scale = D ** -0.5
    k_flat, v_flat = kc.reshape(blocks * page, hkv, D), vc.reshape(blocks * page, hkv, D)   # views of `packed`

    def write_fused():
        return ops.gqa_qknorm_rope_cache_write(qkv, pos, table, slots, kc, vc, hq, hkv, qw, kw, 1e-6, True)

    def write_torch():
        qx, kx, vx = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        qx, kx, vx = qx.reshape(B, hq, D), kx.reshape(B, hkv, D), vx.reshape(B, hkv, D)
        if norm:
            qx, kx = _rms(qx, qw, 1e-6), _rms(kx, kw, 1e-6)
        cos, sin = table.index_select(0, pos).unsqueeze(1).chunk(2, dim=-1)
        qx, kx = _rope(qx, cos, sin), _rope(kx, cos, sin)
        k_flat.index_copy_(0, slots, kx)
        v_flat.index_copy_(0, slots, vx)
        return qx

    def write_decode_packed():
        return ops.gqa_decode(write_fused(), kc, vc, lens + 1, pt, scale)

    def decode_packed():
        return ops.gqa_decode(q, kc, vc, lens + 1, pt, scale)

    def decode_separate():
        return ops.gqa_decode(q, k_sep, v_sep, lens + 1, pt, scale)

    us = {f.__name__: round(_time_graph(f, replays, warmup), 2)
          for f in (write_fused, write_torch, write_decode_packed, decode_packed, decode_separate)}
    write_bytes = B * (hq + 2 * hkv) * D * 2 + B * hq * D * 2 + B * 2 * hkv * D * 2   # qkv in, q out, k / v rows out
    decode_bytes = B * (S + 1) * hkv * D * 2 * 2                                       # K and V of every token
    return dict(workload=name, batch=B, kv_len=S, page=page, Hq=hq, Hkv=hkv, qk_norm=norm, us=us,
                write_bytes=write_bytes, decode_bytes=decode_bytes)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gqa_attn_step.py needs a CUDA device")
    name, power = _gpu()
    res = [run(n, a.replays, a.warmup) for n in ("mixtral-int4", "qwen3-mxfp4")]
    print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, shapes=res)))


if __name__ == "__main__":
    main()
