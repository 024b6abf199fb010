"""A/B two (or more) builds of libb200moe.so on GQA decode: kernel time and bit-identity of out / lse (H100, CUDA graphs).

    python tools/gqa_decode_ab.py LIB_A LIB_B [--rounds 3] [--replays 500] [--warmup 50]

Each library is loaded in a process of its own (B200MOE_LIB_PATH); the processes alternate, LIB_A, LIB_B, LIB_A, ...,
for `--rounds` rounds, so that drift of the shared machine falls on both sides alike.  Every process builds the same
seeded inputs and times each variant as one CUDA graph over `--replays` replays after `--warmup`:
  {mixtral,qwen3}_{separate,packed}  ops.gqa_decode at the decode shapes of tools/gqa_attn_step.py (bench.WORKLOADS: KV
                                     2048 / 512 + the new token, page 16), on separate contiguous K / V caches and on
                                     the FlashInfer backend's packed NHD cache read through its strides;
  {mixtral,qwen3}_spec_q{Q}          q_len_per_req = Q on the packed cache, the shapes of tools/gqa_spec_step.py
                                     (Mixtral Q = 1-4, Qwen3 Q = 2-4).
The time includes the split merge.  Prints one JSON line: per variant and library the microseconds of every round,
their median and spread (max - min), and whether out and lse of the first round are bit-identical to those of LIB_A
(if not: how many output rows differ and by how much);
the GPU's name and power limit are read in the same run.  Outputs are handed between processes through a temporary
directory; nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 128


def _variants():
    import torch
    from bench import WORKLOADS
    from lvllm_b200 import ops

    dev = torch.device("cuda:0")
    out = {}
    for short, name in (("mixtral", "mixtral-int4"), ("qwen3", "qwen3-mxfp4")):
        w = WORKLOADS[name]
        B, S, page, hq, hkv = w["batch"], w["seq"], w["page"], w["Hq"], w["Hkv"]
        gen = torch.Generator(device=dev).manual_seed(0)
        npg = -(-(S + 1) // page)
        packed = torch.randn(B * npg, page, hkv, 2 * D, generator=gen, device=dev).bfloat16()   # NHD
        kc, vc = packed.permute(0, 2, 1, 3).transpose(1, 2).split(D, dim=-1)
        k_sep, v_sep = kc.contiguous(), vc.contiguous()
        pt = torch.randperm(B * npg, generator=gen, device=dev).reshape(B, npg).int()
        lens = torch.full((B,), S + 1, dtype=torch.int32, device=dev)
        q = torch.randn(B, hq, D, generator=gen, device=dev).bfloat16()
        out[f"{short}_separate"] = lambda q=q, k=k_sep, v=v_sep, lens=lens, pt=pt: ops.gqa_decode(q, k, v, lens, pt, D ** -0.5)
        out[f"{short}_packed"] = lambda q=q, k=kc, v=vc, lens=lens, pt=pt: ops.gqa_decode(q, k, v, lens, pt, D ** -0.5)
        for Q in ((1, 2, 3, 4) if short == "mixtral" else (2, 3, 4)):
            gen = torch.Generator(device=dev).manual_seed(Q)
            npg = -(-(S + Q) // page)
            packed_q = torch.randn(B * npg, page, hkv, 2 * D, generator=gen, device=dev).bfloat16()
            kq, vq = packed_q.permute(0, 2, 1, 3).transpose(1, 2).split(D, dim=-1)
            ptq = torch.randperm(B * npg, generator=gen, device=dev).reshape(B, npg).int()
            lq = torch.full((B,), S + Q, dtype=torch.int32, device=dev)
            qq = torch.randn(B * Q, hq, D, generator=gen, device=dev).bfloat16()
            splits = -(-(npg * page) // 128)
            out[f"{short}_spec_q{Q}"] = (lambda q=qq, k=kq, v=vq, lens=lq, pt=ptq, Q=Q, splits=splits:
                                         ops.gqa_decode(q, k, v, lens, pt, D ** -0.5, num_kv_splits=splits,
                                                        q_len_per_req=Q))
    return out


def child(outputs_path, replays, warmup):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import torch
    from gqa_attn_step import _time_graph

    res, keep = {}, {}
    for name, fn in _variants().items():
        o, lse = fn()
        torch.cuda.synchronize()
        if outputs_path:
            keep[name] = (o.cpu(), lse.cpu())
        res[name] = _time_graph(fn, replays, warmup)
    if outputs_path:
        torch.save(keep, outputs_path)
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--replays", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--outputs", default="", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a.outputs, a.replays, a.warmup)
    if len(a.libs) < 2:
        raise SystemExit("give two or more library paths")
    libs = [os.path.abspath(p) for p in a.libs]
    for p in libs:
        if not os.path.exists(p):
            raise SystemExit(f"{p} does not exist")
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import torch
    from gqa_attn_step import _gpu

    if not torch.cuda.is_available():
        raise SystemExit("gqa_decode_ab.py needs a CUDA device")
    gpu, power = _gpu()
    times = {p: [] for p in libs}
    with tempfile.TemporaryDirectory() as tmp:
        outs = {p: os.path.join(tmp, f"out{i}.pt") for i, p in enumerate(libs)}
        for r in range(a.rounds):
            for p in libs:
                cmd = [sys.executable, os.path.abspath(__file__), "--child", "--replays", str(a.replays), "--warmup",
                       str(a.warmup)] + (["--outputs", outs[p]] if r == 0 else [])
                env = dict(os.environ, B200MOE_LIB_PATH=p)
                cp = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True, check=True)
                times[p].append(json.loads(cp.stdout.strip().splitlines()[-1]))
        base = torch.load(outs[libs[0]])
        other = {p: torch.load(outs[p]) for p in libs[1:]}
    variants = {}
    for v in times[libs[0]][0]:
        row = {}
        for p in libs:
            us = sorted(t[v] for t in times[p])
            row[p] = dict(us=[round(t[v], 2) for t in times[p]], median=round(us[len(us) // 2], 2),
                          spread=round(us[-1] - us[0], 2))
            if p in other:
                (o0, l0), (o1, l1) = base[v], other[p][v]
                row[p]["bit_identical"] = bool(torch.equal(o0, o1) and torch.equal(l0, l1))
                if not row[p]["bit_identical"]:
                    row[p]["out_rows_differing"] = int((o0 != o1).any(-1).sum())
                    row[p]["out_max_abs_diff"] = float((o0.float() - o1.float()).abs().nan_to_num(float("inf")).max())
                    row[p]["lse_max_abs_diff"] = float((l0 - l1).abs().nan_to_num(0.0).max())
        variants[v] = row
    print(json.dumps(dict(gpu=gpu, power_limit=power, rounds=a.rounds, replays=a.replays, libs=libs,
                          variants=variants)))


if __name__ == "__main__":
    main()
