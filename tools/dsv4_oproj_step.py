"""Time DeepSeek-V4's attention output projection up to wo_b on the H100, in CUDA graphs.

    python tools/dsv4_oproj_step.py [--replays 300] [--warmup 20] [--shapes h64-t1,h8-t256,...]

Shapes: 64 / 16 / 8 heads in 8 / 2 / 1 groups of 8 heads (the whole model and tensor-parallel shards of it), o_lora_rank
1024, T = 1, 32 and 256 decode tokens; wo_a is e4m3 [G * 1024, 4096] with f32 block scales.  Each variant is captured
once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`, alternated twice:
  quant   ops.dsv4_inv_rope_quant alone;
  kernels ops.dsv4_o_proj (inverse RoPE + quantisation, then the grouped fp8 GEMM);
  torch   the composition a user without DeepGEMM runs on the same card: inverse RoPE and ue8m0 block quantisation in
          vectorised torch, then an einsum over wo_a dequantised to bf16 once, outside the graph (the reference's ROCm
          path, rocm_inv_rope_einsum).
Prints one JSON line per shape: microseconds per variant (the faster of the two rounds), the algorithmic bytes of the
projection (o in T*H*512*2, the fp8 activations and scales written and read back 2*T*G*D*(1 + 4/128), the weights
G*R*D + G*(R/128)*(D/128)*4, z out T*G*R*2) and GB/s of the kernels, and the GPU's name and power limit read in the same
run.  Writes nothing.
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

R, HPG, MAX_POS = 1024, 8, 4096
SHAPES = [(f"h{H}-t{T}", H, G, T) for H, G in ((64, 8), (16, 2), (8, 1)) for T in (1, 32, 256)]


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
    return a.elapsed_time(b) * 1e3 / replays


def _torch_o_proj(o, positions, cs, w_bf16, G):
    """Inverse RoPE + ue8m0 block quantisation in torch, then the einsum over the bf16 weights."""
    T, H, _ = o.shape
    c, s = cs[positions][:, None, :32], cs[positions][:, None, 32:]
    x = o.float()
    xe, xo = x[..., 448::2], x[..., 449::2]
    rot = torch.stack((xe * c + xo * s, xo * c - xe * s), -1).flatten(-2)
    x = torch.cat((x[..., :448], rot), -1).reshape(T, G, -1, 128)
    scale = torch.exp2(torch.ceil(torch.log2(x.abs().amax(-1, keepdim=True).clamp(min=1e-10) * (1.0 / 448.0))))
    q = (x / scale).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    a = (q.float() * scale).to(torch.bfloat16).reshape(T, G, -1)
    return torch.einsum("tgd,grd->tgr", a, w_bf16).reshape(T, -1)


def run(shape, H, G, T, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    D = HPG * 512
    o = torch.randn(T, H, 512, generator=gen, device=dev).bfloat16()
    pos = torch.randint(0, MAX_POS, (T,), generator=gen, device=dev)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64, device=dev) / 64))
    f = torch.arange(MAX_POS, dtype=torch.float64, device=dev)[:, None] * inv[None]
    cs = torch.cat([f.cos(), f.sin()], dim=1).float()
    w = (torch.randn(G * R, D, generator=gen, device=dev) * 0.05).to(torch.float8_e4m3fn)
    ws = torch.exp2(torch.randint(-10, -4, (G * R // 128, D // 128), generator=gen, device=dev).float())
    w_bf16 = (w.float() * ws.repeat_interleave(128, 0).repeat_interleave(128, 1)).bfloat16().reshape(G, R, D)
    graphs = {
        "quant": _graph(lambda: ops.dsv4_inv_rope_quant(o, pos, cs, G)),
        "kernels": _graph(lambda: ops.dsv4_o_proj(o, pos, cs, w, ws, G)),
        "torch": _graph(lambda: _torch_o_proj(o, pos, cs, w_bf16, G)),
    }
    us = {k: float("inf") for k in graphs}
    for _ in range(2):
        for k, g in graphs.items():
            us[k] = min(us[k], _time(g, replays, warmup))
    nbytes = T * H * 512 * 2 + 2 * T * G * D * (1 + 4 / 128) + G * R * D + G * (R // 128) * (D // 128) * 4 + T * G * R * 2
    return dict(shape=shape, heads=H, groups=G, o_lora_rank=R, tokens=T, us={k: round(v, 2) for k, v in us.items()},
                bytes=int(nbytes), kernels_gbps=round(nbytes / us["kernels"] / 1e3, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--shapes", default="", help="comma-separated subset of " + ",".join(s[0] for s in SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dsv4_oproj_step.py needs a CUDA device")
    want = set(a.shapes.split(",")) if a.shapes else None
    name, power = _gpu()
    for shape, H, G, T in SHAPES:
        if want is None or shape in want:
            print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, **run(shape, H, G, T, a.replays,
                                                                                            a.warmup))), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
