"""Time DeepSeek-V4 sparse attention decode (sliding-window + compressed top-k keys on the 584-byte fp8 cache, with attention
sinks) on the H100, in CUDA graphs.

    python tools/dsv4_sparse_step.py [--extra-topk 512] [--replays 1000] [--warmup 50]

V4-Flash attention: head dim 512, sliding window 128 (SWA cache block size 64), compressed top-k --extra-topk keys (compressed
cache block size 64; 0 = an SWA-only layer).  Shapes: 64 heads at batch 1, and a TP4 shard (16 heads) at batch 32.  Every
token's lists hold distinct valid slots.  Three variants, each captured once in a CUDA graph and timed with CUDA events over
`--replays` replays after `--warmup`, alternated twice:
  v4      ops.dsv4_sparse_decode at its default split count, with a sink;
  torch   the same work composed from torch ops: gather and dequantise the rows, scores, softmax with the sink, P x rows;
  v32     ops.mla_decode_sparse (DeepSeek-V3.2) on an fp8_ds_mla cache (656 bytes per token) over the same key count.
Prints one JSON line per shape: microseconds per variant, the largest |v4 - torch| of one call, v4's algorithmic bytes
T * valid_keys * 584 + T * Hq * 512 * 2 * 2 (cache rows, q and out) and GB/s over its time, and the GPU's name and power
limit read in the same run.  Writes nothing.
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

WINDOW, SWA_BLOCK, EXTRA_BLOCK, CTX = 128, 64, 64, 32768
SCALE = 512 ** -0.5


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


def _cache(n_tokens, bs, dev, gen):
    """A 584-byte-per-token cache of n_tokens random rows: random e4m3 bytes (finite), ue8m0 scales near 2^-4, bf16 rope."""
    nb = n_tokens // bs
    c = torch.empty(nb, bs * 584, dtype=torch.uint8, device=dev)
    x = torch.randn(nb, bs, 448, generator=gen, device=dev) * 32
    c[:, :bs * 576].view(nb, bs, 576)[..., :448] = x.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    rope = torch.randn(nb, bs, 64, generator=gen, device=dev).bfloat16()
    c[:, :bs * 576].view(nb, bs, 576)[..., 448:] = rope.view(torch.uint8)
    sc = c[:, bs * 576:].view(nb, bs, 8)
    sc[..., :7] = torch.randint(120, 124, (nb, bs, 7), generator=gen, device=dev, dtype=torch.uint8)
    sc[..., 7] = 0
    return c.view(nb, bs, 584)


def _rows(cache, slots):
    """bf16 [B, N, 512] of the given slots (the torch composition's gather + dequantisation)."""
    nb, bs, _ = cache.shape
    flat = cache.view(nb, bs * 584)
    data = flat[:, :bs * 576].reshape(nb, bs, 576)
    sc = flat[:, bs * 576:].reshape(nb, bs, 8)
    b, p = slots.long() // bs, slots.long() % bs
    d = data[b, p]                                                     # [B, N, 576]
    s = torch.exp2(sc[b, p, :7].float() - 127.0).repeat_interleave(64, -1)
    nope = (d[..., :448].contiguous().view(torch.float8_e4m3fn).float() * s).bfloat16()
    return torch.cat([nope, d[..., 448:].contiguous().view(torch.bfloat16)], -1)


def run(shape, B, hq, extra_topk, replays, warmup):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    swa = _cache(B * WINDOW * 2, SWA_BLOCK, dev, gen)
    si = torch.stack([torch.randperm(B * WINDOW * 2, device=dev)[:WINDOW] for _ in range(B)]).int()
    sl = torch.full((B,), WINDOW, dtype=torch.int32, device=dev)
    ext = {}
    if extra_topk:
        ex = _cache(B * CTX // 4, EXTRA_BLOCK, dev, gen)
        ei = torch.stack([torch.randperm(B * CTX // 4, device=dev)[:extra_topk] for _ in range(B)]).int()
        ext = dict(extra_cache=ex, extra_indices=ei, extra_lens=torch.full((B,), extra_topk, dtype=torch.int32, device=dev))
    q = torch.randn(B, hq, 512, generator=gen, device=dev).bfloat16()
    sink = torch.randn(hq, generator=gen, device=dev)
    n_keys = WINDOW + extra_topk

    def v4():
        return ops.dsv4_sparse_decode(q, swa, si, sl, SCALE, attn_sink=sink, **ext)

    def composed():
        kv = _rows(swa, si)
        if extra_topk:
            kv = torch.cat([kv, _rows(ext["extra_cache"], ext["extra_indices"])], 1)
        s = torch.einsum("bhd,bnd->bhn", q.float(), kv.float()) * SCALE
        s = torch.cat([s, sink[None, :, None].expand(B, hq, 1)], -1)
        p = torch.softmax(s, -1)[..., :-1]
        return torch.einsum("bhn,bnd->bhd", p, kv.float()).bfloat16()

    # V3.2 sparse decode over the same key count: one 656-byte fp8_ds_mla row per key, request-local positions
    page = 64
    npg = -(-n_keys // page) * 2
    lat = torch.randn(B * npg * page, 576, generator=gen, device=dev)
    scl = (lat[:, :512].reshape(-1, 4, 128).abs().amax(-1) / 448.0)
    q8 = (lat[:, :512].reshape(-1, 4, 128) / scl[..., None]).to(torch.float8_e4m3fn).reshape(-1, 512)
    ds = torch.cat([q8.view(torch.uint8), scl.contiguous().view(torch.uint8),
                    lat[:, 512:].bfloat16().contiguous().view(torch.uint8)], 1).reshape(B * npg, page, 656)
    pt = torch.randperm(B * npg, device=dev).reshape(B, npg).int()
    rid = torch.arange(B, dtype=torch.int32, device=dev)
    idx32 = torch.stack([torch.randperm(npg * page, device=dev)[:n_keys] for _ in range(B)]).int()
    qn = torch.randn(B, hq, 512, generator=gen, device=dev).bfloat16()
    qp = torch.randn(B, hq, 64, generator=gen, device=dev).bfloat16()

    def v32():
        return ops.mla_decode_sparse(qn, qp, ds, idx32, rid, pt, SCALE)

    (g4, o4), (gt, ot), (g32, _) = _graph(v4), _graph(composed), _graph(v32)
    g4.replay()
    gt.replay()
    torch.cuda.synchronize()
    diff = (o4.float() - ot.float()).abs().max().item()
    us = dict(v4=[], torch=[], v32=[])
    for _ in range(2):
        us["v4"].append(_time(g4, replays, warmup))
        us["torch"].append(_time(gt, replays, warmup))
        us["v32"].append(_time(g32, replays, warmup))
    alg = B * n_keys * 584 + B * hq * 512 * 2 * 2
    return dict(shape=shape, batch=B, Hq=hq, window=WINDOW, extra_topk=extra_topk, us=us, max_abs_diff_v4_torch=diff,
                v4_bytes=alg, v4_GBps=round(alg / min(us["v4"]) / 1e3, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--extra-topk", type=int, default=512)
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dsv4_sparse_step.py needs a CUDA device")
    name, power = _gpu()
    for shape, B, hq in (("v4-flash-hq64", 1, 64), ("v4-flash-tp4-shard", 32, 16)):
        print(json.dumps(dict(gpu=name, power_limit=power, replays=a.replays,
                              **run(shape, B, hq, a.extra_topk, a.replays, a.warmup))), flush=True)


if __name__ == "__main__":
    main()
