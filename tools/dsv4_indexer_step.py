"""Time DeepSeek-V4's decode key selection on the H100, in CUDA graphs: the C4A indexer (q side, logits, top-k) and the
global key lists.

    python tools/dsv4_indexer_step.py [--replays 300] [--warmup 20] [--shapes b1-s8k,b32-s32k,...]

Shapes: V4-Flash's indexer (64 heads, head dim 128, topk 512, ratio 4, compressed page 64, i.e. 256-token blocks) at batch
1 / 32 / 256 and contexts 8K / 32K / 128K, one decode token per request; every request is at the same position S - 1, so
each token has S / 4 candidates.  The compressed indexer cache holds random finite e4m3 values with positive fp32 scales.
Each variant is captured once in a CUDA graph and timed with CUDA events over `--replays` replays after `--warmup`,
alternated twice:
  q        ops.dsv4_indexer_q_quant;
  decode   ops.dsv4_indexer_decode (logits, then top-k);
  topk     ops.indexer_topk on the same logits with per-token lengths (the same top-k kernel, one row per token);
  lists    ops.dsv4_global_topk_indices + ops.dsv4_swa_indices (window 128) + ops.dsv4_compressed_slot_mapping;
  select   the whole C4A selection: q, decode and lists;
  torch    the torch composition of the same selection on the same card: the q side (RoPE, amax, scale, e4m3 cast), gather
           the pages, dequantise, einsum, relu, the weighted sum over heads, the candidate mask, torch.topk, and the three
           lists by block-table gathers.
The logits' time is decode - topk (derived, not measured alone).  Prints one JSON line per shape: microseconds of each
variant, the logits' algorithmic bytes (B * S / 4 * 132 cache bytes + q and weights + the logits written) and GB/s over
the derived time, and the GPU's name and power limit read in the same run.  Writes nothing.
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

H, TOPK, PAGE, RATIO, WINDOW, SWA_BS = 64, 512, 64, 4, 128, 64
SHAPES = [(f"b{B}-s{S // 1024}k", B, S) for B in (1, 32, 256) for S in (8192, 32768, 131072)]


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


def run(shape, B, S, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    n = S // RATIO                                                   # candidates per token
    npg = n // PAGE
    nb = B * npg
    cache = torch.empty(nb, PAGE * 132, dtype=torch.uint8, device=dev)
    cache[:, :PAGE * 128] = _e4m3((nb, PAGE * 128), gen, dev)
    cache[:, PAGE * 128:] = (torch.rand(nb, PAGE, generator=gen, device=dev) * 0.01 + 1e-3).view(torch.uint8)
    cache = cache.view(nb, PAGE, 132)
    bt = torch.randperm(nb, device=dev, generator=gen).reshape(B, npg).int()
    swa_bt = torch.randperm(B * (S // SWA_BS), device=dev, generator=gen).reshape(B, -1).int()
    q = torch.randn(B, H, 128, generator=gen, device=dev).bfloat16()
    wts = torch.randn(B, H + 8, generator=gen, device=dev).bfloat16()[:, 4:4 + H]
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64, device=dev) / 64))
    f = torch.arange(S, dtype=torch.float64, device=dev)[:, None] * inv[None]
    cs = torch.cat([f.cos(), f.sin()], dim=1).float()
    pos = torch.full((B,), S - 1, dtype=torch.int64, device=dev)
    req = torch.arange(B, dtype=torch.int32, device=dev)
    sm = torch.arange(B, dtype=torch.int64, device=dev)
    lens = torch.full((B,), n, dtype=torch.int32, device=dev)
    logits = torch.empty(B, npg * PAGE, dtype=torch.float32, device=dev)
    q8, w = ops.dsv4_indexer_q_quant(q, wts, pos, cs, 128 ** -0.5, H ** -0.5)
    local = ops.dsv4_indexer_decode(q8, w, cache, pos, req, bt, RATIO, TOPK, logits=logits)

    def k_q():
        ops.dsv4_indexer_q_quant(q, wts, pos, cs, 128 ** -0.5, H ** -0.5)

    def k_decode():
        ops.dsv4_indexer_decode(q8, w, cache, pos, req, bt, RATIO, TOPK, logits=logits)

    def k_topk():
        ops.indexer_topk(logits, lens, TOPK, 1)

    def k_lists():
        ops.dsv4_global_topk_indices(local, sm, req, bt, PAGE)
        ops.dsv4_swa_indices(pos, sm, req, swa_bt, SWA_BS, WINDOW)
        ops.dsv4_compressed_slot_mapping(pos, sm, req, bt, PAGE, RATIO)

    def k_select():
        a8, aw = ops.dsv4_indexer_q_quant(q, wts, pos, cs, 128 ** -0.5, H ** -0.5)
        loc = ops.dsv4_indexer_decode(a8, aw, cache, pos, req, bt, RATIO, TOPK, logits=logits)
        ops.dsv4_global_topk_indices(loc, sm, req, bt, PAGE)
        ops.dsv4_swa_indices(pos, sm, req, swa_bt, SWA_BS, WINDOW)
        ops.dsv4_compressed_slot_mapping(pos, sm, req, bt, PAGE, RATIO)

    keys = torch.arange(npg * PAGE, device=dev)
    win = torch.arange(WINDOW, device=dev)

    def torch_ref():
        x = q.float()
        c, s = cs[pos][:, None, :32], cs[pos][:, None, 32:]
        xe, xo = x[..., 64::2], x[..., 65::2]
        rot = torch.stack(((xe * c - xo * s).bfloat16().float(), (xo * c + xe * s).bfloat16().float()), -1).flatten(-2)
        xr = torch.cat((x[..., :64], rot), -1)
        scale = torch.exp2(torch.ceil(torch.log2(xr.abs().amax(-1).clamp(min=1e-4) / 448.0)))
        qq = (xr / scale[..., None]).to(torch.float8_e4m3fn).float()
        ww = wts.float() * scale * (128 ** -0.5) * (H ** -0.5)
        blk = cache.view(nb, PAGE * 132)[bt[req].long()]                                   # [B, npg, page * 132]
        vals = blk[..., :PAGE * 128].contiguous().view(torch.float8_e4m3fn).float().view(B, npg * PAGE, 128)
        sc = blk[..., PAGE * 128:].contiguous().view(torch.float32).view(B, npg * PAGE)
        lg = (torch.einsum("bhd,bkd->bhk", qq, vals).relu() * ww[..., None]).sum(1) * sc
        ncand = torch.div(pos + 1, RATIO, rounding_mode="floor")
        lg = lg.masked_fill(keys[None] >= ncand[:, None], float("-inf"))
        top = torch.topk(lg, TOPK, dim=-1).indices.sort(-1).values
        g = bt[req.long()].long().gather(1, top // PAGE) * PAGE + top % PAGE
        sp = (pos[:, None] - WINDOW + 1 + win).clamp(min=0)
        sw = swa_bt[req.long()].long().gather(1, sp // SWA_BS) * SWA_BS + sp % SWA_BS
        row = pos // RATIO
        slot = torch.where((pos + 1) % RATIO == 0, bt[req.long(), row // PAGE].long() * PAGE + row % PAGE, -1)
        return g, sw, slot

    graphs = dict(q=_graph(k_q), decode=_graph(k_decode), topk=_graph(k_topk), lists=_graph(k_lists),
                  select=_graph(k_select), torch=_graph(torch_ref))
    us = {k: [] for k in graphs}
    for _ in range(2):
        for k, g in graphs.items():
            us[k].append(_time(g, replays, warmup))
    logits_us = min(us["decode"]) - min(us["topk"])
    alg = B * n * 132 + B * H * (128 + 4) + B * n * 4
    return dict(shape=shape, batch=B, context=S, candidates=n, heads=H, page=PAGE, topk=TOPK, us=us,
                logits_us_derived=round(logits_us, 2), logits_bytes=alg,
                logits_GBps=round(alg / logits_us / 1e3, 1) if logits_us > 0 else None)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--replays", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--shapes", default="", help="comma-separated subset of " + ",".join(s for s, _, _ in SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dsv4_indexer_step.py needs a CUDA device")
    want = set(a.shapes.split(",")) if a.shapes else None
    name, power = _gpu()
    for shape, B, S in SHAPES:
        if want is None or shape in want:
            print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays, **run(shape, B, S, a.replays, a.warmup))),
                  flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
