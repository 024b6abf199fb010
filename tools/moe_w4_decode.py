"""Times one 4-bit MoE decode layer (lk_moe cpu_decode -> the fused kernel) in a CUDA graph.

    python tools/moe_w4_decode.py [--replays 1000] [--dump DIR]

The library is the one lvllm_b200 loads (B200MOE_LIB_PATH selects another build of it, for A/B runs).  Per case it
prints one JSON line: microseconds per layer, distinct active experts, 64-row chunks, algorithmic bytes (the weights of
the distinct active experts) over time, and the card's name and power limit.  --dump DIR writes each case's fp32 output
as .npy, so that two builds can be compared on the same seeded inputs."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def expert_bytes(fmt, H, I):
    nib = 3 * H * I // 2                      # gate + up + down, two weights per byte
    return nib + {"int4": 3 * H * I // 32 * 2, "mxfp4": 3 * H * I // 32, "nvfp4": 3 * H * I // 16}[fmt]


def make_layer(fmt, E, k, H, I, max_seqs, dev, g):
    import lk_moe
    cfg = lk_moe.MOEConfigV2()
    cfg.expert_num, cfg.top_k, cfg.hidden_size, cfg.intermediate_size = E, k, H, I
    cfg.max_batch_size, cfg.max_num_seqs = max(max_seqs, 16), max(max_seqs, 16)
    cfg.gpu_id = 0
    p13 = torch.randint(0, 256, (E, 2 * I, H // 2), device=dev, dtype=torch.uint8, generator=g)
    p2 = torch.randint(0, 256, (E, H, I // 2), device=dev, dtype=torch.uint8, generator=g)
    if fmt == "int4":
        cfg.groupN, cfg.groupK = 1, 32
        s13 = (torch.rand(E, 2 * I, H // 32, device=dev, generator=g) * 0.01 + 0.002).bfloat16()
        s2 = (torch.rand(E, H, I // 32, device=dev, generator=g) * 0.01 + 0.002).bfloat16()
        return lk_moe.MOE_WNA16(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0,
                                weights_on_device=True)
    if fmt == "mxfp4":
        cfg.groupN, cfg.groupK = 1, 32
        s13 = torch.randint(117, 122, (E, 2 * I, H // 32), device=dev, dtype=torch.uint8, generator=g)
        s2 = torch.randint(117, 122, (E, H, I // 32), device=dev, dtype=torch.uint8, generator=g)
        return lk_moe.MOE_MXFP4(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0,
                                weights_on_device=True)
    cfg.groupN, cfg.groupK = 1, 16
    s13 = (torch.rand(E, 2 * I, H // 16, device=dev, generator=g) * 2 + 0.5).to(torch.float8_e4m3fn)
    s2 = (torch.rand(E, H, I // 16, device=dev, generator=g) * 2 + 0.5).to(torch.float8_e4m3fn)
    g13 = torch.full((E, 2), 0.004, device=dev)
    g2 = torch.full((E,), 0.004, device=dev)
    return lk_moe.MOE_NVFP4(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), g13.data_ptr(),
                            g2.data_ptr(), weights_on_device=True)


def random_ids(M, E, k, g, local=None):
    ids = torch.stack([torch.randperm(E if local is None else local[0], generator=g)[:k] for _ in range(M)]).int()
    if local is not None:   # an EP shard: only ids in [0, E_local) are this rank's, the rest -1
        ids = torch.where(ids < local[1], ids, torch.full_like(ids, -1))
    return ids


def bench_like_ids(dev):
    """ids of layer 0 from one eager step of the benchmark's Mixtral INT4 model (its router on a seeded batch)."""
    import bench
    w = dict(bench.WORKLOADS["mixtral-int4"])
    w["layers"] = 1
    model = bench.HotPathModel(w, 0, 1, dev)
    g = torch.Generator(device=dev).manual_seed(1)
    model.hidden_in.copy_(torch.randn(model.hidden_in.shape, device=dev, generator=g).bfloat16())
    model.step(record_ids=True)
    torch.cuda.synchronize()
    ids = model.last_ids[0].cpu().int()
    for L in model.layers:
        L["moe"].close()
    del model
    torch.cuda.empty_cache()
    return ids


def run_case(name, fmt, E, k, H, I, ids, dev, replays, dump, chunk_rows=64):
    g = torch.Generator(device=dev).manual_seed(7)
    M = ids.shape[0]
    moe = make_layer(fmt, E, k, H, I, M, dev, g)
    hidden = (torch.randn(M, H, device=dev, generator=g) / 10).bfloat16()
    tw = torch.softmax(torch.randn(M, k, device=dev, generator=g), -1).float().contiguous()
    idd = ids.to(dev).contiguous()
    out = torch.zeros(M, H, dtype=torch.float32, device=dev)
    st = torch.cuda.Stream()

    def launch():
        moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, k, hidden.data_ptr(), idd.data_ptr(), tw.data_ptr(),
                       out.data_ptr())

    with torch.cuda.stream(st):
        for _ in range(3):
            launch()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(graph, stream=st):
            launch()
        for _ in range(20):
            graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(replays):
            graph.replay()
        e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / replays
    cnt = torch.bincount(ids[ids >= 0].long(), minlength=E)
    distinct = int((cnt > 0).sum())
    chunks = int(((cnt + chunk_rows - 1) // chunk_rows).sum())
    gbs = distinct * expert_bytes(fmt, H, I) / (us * 1e-6) / 1e9
    if dump:
        os.makedirs(dump, exist_ok=True)
        np.save(os.path.join(dump, f"{name}.npy"), out.cpu().numpy())
    moe.close()
    return {"case": name, "us": round(us, 2), "distinct_experts": distinct, "chunks_64": chunks,
            "algo_GBps": round(gbs, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=1000)
    ap.add_argument("--dump", default=None, metavar="DIR")
    ap.add_argument("--only", default=None, help="comma-separated case names")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    name, pl = card()
    g = torch.Generator().manual_seed(0)
    mix = dict(fmt="int4", E=8, k=2, H=4096, I=14336)
    uni = torch.stack([torch.arange(64) * 2 % 8, (torch.arange(64) * 2 + 1) % 8], 1).int()   # 16 rows per expert
    # the benchmark's routing in closed form: every token picks expert 0, and expert 1 or (one token in 8) expert 2 ->
    # chunks of 64, 56 and 8 rows, run by the 64-column instantiation
    conc = torch.stack([torch.zeros(64, dtype=torch.long), torch.where(torch.arange(64) % 8 == 0, 2, 1)], 1).int()
    cases = [
        ("mixtral_int4_m64_bench_routing", mix, lambda: bench_like_ids(dev)),
        ("mixtral_int4_m64_uniform", mix, lambda: uni),
        ("mixtral_int4_m64_concentrated", mix, lambda: conc),
        ("mixtral_mxfp4_m64_concentrated", dict(mix, fmt="mxfp4"), lambda: conc),
        ("mixtral_nvfp4_m64_concentrated", dict(mix, fmt="nvfp4"), lambda: conc),
        ("mixtral_int4_m1", mix, lambda: random_ids(1, 8, 2, g)),
        ("mixtral_int4_m16", mix, lambda: random_ids(16, 8, 2, g)),
        ("mixtral_int4_m256", mix, lambda: random_ids(256, 8, 2, g)),
        ("qwen3_mxfp4_m256", dict(fmt="mxfp4", E=128, k=8, H=4096, I=1536), lambda: random_ids(256, 128, 8, g)),
        # DeepSeek-V3 NVFP4 under EP8: 32 local experts of 256, one token, top-8 -> the ids outside the shard are -1
        ("dsv3_nvfp4_ep8_shard_m1", dict(fmt="nvfp4", E=32, k=8, H=7168, I=2048),
         lambda: torch.tensor([[3, 17, -1, -1, -1, -1, -1, -1]], dtype=torch.int32)),
    ]
    only = set(args.only.split(",")) if args.only else None
    for cname, c, mk in cases:
        if only and cname not in only:
            continue
        ids = mk()
        r = run_case(cname, c["fmt"], c["E"], c["k"], c["H"], c["I"], ids, dev, args.replays, args.dump)
        r.update({"card": name, "power_limit": pl, "lib": os.environ.get("B200MOE_LIB_PATH", "in-tree")})
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
