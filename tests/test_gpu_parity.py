"""GPU parity tests (-m gpu): CUDA path through the C ABI vs the CPU oracle on the same seeded inputs, the
committed golden fixtures, and size-independent properties at BASELINE sizes."""
import math
import os

import pytest
import torch

from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _ulp_tie_ok(logits_row, ids_a, ids_b, scores_fn):
    """ids may differ only where the competing scores are within a few ulp (fp32 expf / tanhf differ
    by <= 2 ulp between libm and CUDA)."""
    sa, sb = set(ids_a.tolist()), set(ids_b.tolist())
    if sa == sb:
        return True
    sc = scores_fn(logits_row)
    diff = list(sa ^ sb)
    vals = sc[diff]
    return float(vals.max() - vals.min()) <= 8 * torch.finfo(torch.float32).eps * float(vals.abs().max())


# ------------------------------------------------------------------------------------------ routing
@pytest.mark.parametrize("M,E,k,scoring,use_bias,renorm", [
    (1, 8, 2, "softmax", False, True), (64, 8, 2, "softmax", False, True), (256, 128, 8, "softmax", False, True),
    (33, 64, 6, "sigmoid", False, False), (57, 256, 8, "sigmoid", True, True), (7, 192, 4, "softmax", True, False),
    (300, 512, 10, "softmax", False, True), (5, 1000, 8, "sigmoid", True, True),
])
def test_topk_gating_vs_oracle(dev, M, E, k, scoring, use_bias, renorm):
    from lvllm_b200 import ops
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(M, E, generator=g)
    bias = torch.randn(E, generator=g) if use_bias else None
    w_ref, i_ref = O.topk_gating(logits, k, renorm, scoring, bias, 2.5 if use_bias else 1.0)
    w, ids, tei = ops.fused_topk(logits.to(dev), k, renorm, scoring, bias.to(dev) if use_bias else None,
                                 2.5 if use_bias else 1.0, return_token_expert_indices=True)
    w, ids = w.cpu(), ids.cpu()
    assert torch.equal(tei.cpu(), (torch.arange(k).view(1, k) * M + torch.arange(M).view(M, 1)).int())
    if not torch.equal(ids, i_ref):
        bad = (ids != i_ref).any(dim=1).nonzero().flatten()
        for t in bad.tolist():
            fn = (lambda r: torch.softmax(r, -1)) if scoring == "softmax" else torch.sigmoid
            sc = lambda r: fn(r) + (bias if use_bias else 0)
            assert _ulp_tie_ok(logits[t], ids[t], i_ref[t], sc), f"row {t}: {ids[t]} vs {i_ref[t]}"
        good = (ids == i_ref).all(dim=1)
        w, w_ref = w[good], w_ref[good]
    torch.testing.assert_close(w, w_ref, atol=2e-6, rtol=2e-5)


def test_topk_gating_exact_ties_and_nan(dev):
    from lvllm_b200 import ops
    logits = torch.zeros(4, 16)
    logits[1, 5] = logits[1, 9] = 3.0           # exact tie -> lower index first
    logits[2, :] = float("nan")                # NaN row -> scores 0 -> ids 0..k-1 (reference :466-471)
    logits[3, 7] = float("inf")
    w, ids = ops.fused_topk(logits.to(dev), 4, True)
    w_ref, i_ref = O.topk_gating(logits, 4, True)
    assert torch.equal(ids.cpu(), i_ref)
    assert ids[0].tolist() == [0, 1, 2, 3] and ids[1, :2].tolist() == [5, 9] and ids[2].tolist() == [0, 1, 2, 3]
    torch.testing.assert_close(w.cpu(), w_ref, atol=1e-6, rtol=1e-5, equal_nan=True)


def test_topk_golden(dev, golden):
    from lvllm_b200 import ops
    for c in golden["fused_topk"]:
        w, ids = ops.fused_topk(c["logits"].to(dev), c["k"], c["renorm"], c["scoring"],
                                c["bias"].to(dev) if c["bias"] is not None else None)
        assert torch.equal(ids.cpu().long(), c["ids"].long())
        torch.testing.assert_close(w.cpu(), c["weights"], atol=2e-6, rtol=2e-5)


@pytest.mark.parametrize("M,E,ng,tg,k,use_bias,scoring", [
    (1, 256, 8, 4, 8, True, "sigmoid"), (64, 256, 8, 4, 8, True, "sigmoid"), (19, 64, 4, 2, 6, False, "softmax"),
    (8, 128, 8, 3, 4, True, "sigmoid"), (3, 384, 1, 1, 8, True, "sigmoid"),
])
def test_grouped_topk_vs_oracle(dev, M, E, ng, tg, k, use_bias, scoring):
    from lvllm_b200 import ops
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(M, E, generator=g)
    bias = torch.randn(E, generator=g) if use_bias else None
    w_ref, i_ref = O.grouped_topk(logits, bias, ng, tg, k, True, 2.5, scoring)
    w, ids = ops.grouped_topk(logits.to(dev), k, True, ng, tg, scoring, 2.5, bias.to(dev) if use_bias else None)
    w, ids = w.cpu(), ids.cpu()
    same = (ids == i_ref).all(dim=1)
    # rows may differ only on genuine near-ties (fp32 sigmoid differs by <= 2 ulp between libm and CUDA, SURVEY 8a4):
    # either two experts, or two groups (score = sum of the group's top-2), compete within a few ulp
    eps = 8 * torch.finfo(torch.float32).eps
    sc_all = (torch.sigmoid(logits) if scoring == "sigmoid" else torch.softmax(logits, -1)) + (bias if use_bias else 0)
    for t in (~same).nonzero().flatten().tolist():
        sa, sb = set(ids[t].tolist()), set(i_ref[t].tolist())
        if sa == sb:
            continue   # same experts, order differs: only possible on an exact tie of the (unbiased) weights
        gsz = E // ng
        ga, gb = {i // gsz for i in sa}, {i // gsz for i in sb}
        if ga != gb:
            gs = sc_all[t].view(ng, gsz).topk(2, dim=-1).values.sum(-1)
            vals = gs[list(ga ^ gb)]
        else:
            vals = sc_all[t][list(sa ^ sb)]
        assert float(vals.max() - vals.min()) <= eps * float(vals.abs().max()), f"row {t}: {ids[t]} vs {i_ref[t]}"
    torch.testing.assert_close(w[same], w_ref[same], atol=2e-5, rtol=1e-4)


def test_grouped_topk_golden_and_degenerate(dev, golden):
    from lvllm_b200 import ops
    for c in golden["grouped_topk_native"]:
        w, ids = ops.grouped_topk(c["logits"].to(dev), c["k"], c["renorm"], c["n_group"], c["topk_group"],
                                  c["scoring"], c["rsf"], c["bias"].to(dev) if c["bias"] is not None else None)
        o1 = torch.argsort(ids.cpu().long(), 1)
        o2 = torch.argsort(c["ids"].long(), 1)
        assert torch.equal(torch.gather(ids.cpu().long(), 1, o1), torch.gather(c["ids"].long(), 1, o2))
        torch.testing.assert_close(torch.gather(w.cpu(), 1, o1), torch.gather(c["weights"], 1, o2), atol=2e-5, rtol=1e-4)
    # all groups -inf -> ids 0..k-1, w = 1/k (reference grouped_topk_kernels.cu:603-618)
    logits = torch.full((2, 64), float("-inf"))
    w, ids = ops.grouped_topk(logits.to(dev), 4, True, 4, 2, "none" if False else "sigmoid", 1.0, torch.zeros(64).to(dev))
    # sigmoid(-inf)=0 -> finite group scores: selection proceeds; just require valid distinct ids
    assert all(len(set(r.tolist())) == 4 for r in ids.cpu())


def test_global_to_local_ids(dev):
    from lvllm_b200 import ops
    local, emap = O.determine_expert_map(8, 3, 256)
    ids = torch.randint(-1, 256, (37, 8), dtype=torch.int32)
    out = ops.global_to_local_expert_ids(ids.to(dev), emap.to(dev)).cpu()
    assert torch.equal(out, O.global_to_local_expert_ids(ids, emap))


# ------------------------------------------------------------------------------------------ permute
@pytest.mark.parametrize("M,k,E", [(1, 8, 32), (64, 2, 8), (256, 8, 128), (1000, 8, 256), (3, 4, 600)])
def test_permute_unpermute_bit_exact(dev, M, k, E):
    from lvllm_b200 import ops
    g = torch.Generator().manual_seed(M)
    H = 256
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(M)]).int()
    ids[torch.rand(M, k, generator=g) < 0.1] = -1           # skipped / non-local slots
    hidden = torch.randn(M, H, generator=g).bfloat16()
    srt_ref, off_ref, inv_ref = O.moe_permute(ids, E)
    perm, srt, off, inv = ops.moe_permute(hidden.to(dev), ids.to(dev), E)
    nv = int(off_ref[-1])
    assert torch.equal(off.cpu(), off_ref)
    assert torch.equal(srt.cpu()[:nv], srt_ref[:nv])
    assert torch.equal(inv.cpu().flatten(), inv_ref)
    assert torch.equal(perm.cpu()[:nv], hidden[(srt_ref[:nv] // k).long()])
    # sortedness + permutation property
    keys = ids.flatten()[srt.cpu()[:nv].long()]
    assert bool((keys[1:] >= keys[:-1]).all())
    # unpermute: fp32 weighted reduce, fixed k order -> compare against the same fp32 formula
    w = torch.rand(M, k, generator=g)
    out = ops.moe_unpermute(perm, w.to(dev), inv, torch.float32).cpu()
    ref = torch.zeros(M, H)
    pc = perm.cpu().float()
    for j in range(k):
        r = inv_ref.view(M, k)[:, j].long()
        ok = r >= 0
        ref[ok] = torch.addcmul(ref[ok], w[ok, j:j + 1], pc[r[ok]])
    torch.testing.assert_close(out, ref, atol=1e-5, rtol=1e-5)


# ------------------------------------------------------------------------------------------ experts
def _route(M, E, k, g, frac_skip=0.0):
    score = torch.randn(M, E, generator=g)
    w, ids = torch.topk(torch.softmax(score, -1), k)
    w = (w / w.sum(-1, keepdim=True)).float()
    ids = ids.int()
    if frac_skip:
        ids[torch.rand(M, k, generator=g) < frac_skip] = -1
    return w.contiguous(), ids.contiguous()


def _cfg(E, k, H, I, max_seqs=64, gN=0, gK=0, gated=True, act=0):
    import lk_moe
    c = lk_moe.MOEConfigV2()
    c.expert_num, c.top_k, c.hidden_size, c.intermediate_size = E, k, H, I
    c.max_batch_size, c.max_num_seqs = 4096, max_seqs
    c.groupN, c.groupK = gN, gK
    c.has_gate_proj = gated
    c.activation_type = act
    c.gpu_id = 0
    return c


def _run_all_entry_points(moe, hidden, ids, w, dev):
    """cpu_prefill (host ptrs), cpu_decode under CUDA-graph capture, gpu_prefill (device ptrs)."""
    M, H = hidden.shape
    k = ids.shape[1]
    outs = {}
    out_host = torch.empty(M, H, dtype=torch.float32)
    moe.cpu_prefill(M, k, ids.data_ptr(), w.data_ptr(), hidden.data_ptr(), out_host.data_ptr())
    outs["cpu_prefill"] = out_host
    hd, idd, wd = hidden.to(dev), ids.to(dev), w.to(dev)
    out_dev = torch.zeros(M, H, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            assert torch.cuda.is_current_stream_capturing()
            moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, k, hd.data_ptr(), idd.data_ptr(),
                           wd.data_ptr(), out_dev.data_ptr())
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    outs["cpu_decode(graph)"] = out_dev.cpu()
    out2 = torch.empty(M, H, dtype=hidden.dtype, device=dev)
    moe.gpu_prefill(hd.data_ptr(), out2.data_ptr(), idd.data_ptr(), wd.data_ptr(), M, k,
                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    outs["gpu_prefill"] = out2.float().cpu()
    return outs


@pytest.mark.parametrize("M", [1, 3, 16, 33, 64])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_moe_16bit_vs_oracle(dev, M, dtype):
    import lk_moe
    E, k, H, I = 8, 2, 512, 256
    g = torch.Generator().manual_seed(100 + M)
    hidden = (torch.randn(M, H, generator=g) / 10).to(dtype)
    w13 = (torch.randn(E, 2 * I, H, generator=g) / 10).to(dtype)
    w2 = (torch.randn(E, H, I, generator=g) / 10).to(dtype)
    w, ids = _route(M, E, k, g, 0.1)
    ref = O.experts_forward_batched(hidden, O.DequantExperts(w13.float(), w2.float()), ids, w, act_dtype=dtype)
    cls = lk_moe.MOE_BF16 if dtype == torch.bfloat16 else lk_moe.MOE_FP16
    moe = cls(_cfg(E, k, H, I), w13.data_ptr(), w2.data_ptr(), 0, 0, 0, 0)
    outs = _run_all_entry_points(moe, hidden, ids, w, dev)
    for name, o in outs.items():
        tol = 2e-2 if name == "gpu_prefill" else 3e-3   # reference bf16 tolerance tests/kernels/moe/test_moe.py:233
        torch.testing.assert_close(o, ref, atol=tol, rtol=2e-2, msg=lambda m: f"{name}: {m}")
    # the three entry points run the same kernels: fp32 outputs must agree bit for bit
    assert torch.equal(outs["cpu_prefill"], outs["cpu_decode(graph)"])
    moe.close()


def test_moe_bf16_golden(dev, golden):
    import lk_moe
    c = golden["experts_bf16"]
    a, w1, w2 = c["a"], c["w1"].contiguous(), c["w2"].contiguous()
    E, N1, H = w1.shape
    moe = lk_moe.MOE_BF16(_cfg(E, c["topk_ids"].shape[1], H, N1 // 2), w1.data_ptr(), w2.data_ptr(), 0, 0, 0, 0)
    M = a.shape[0]
    out = torch.empty(M, H, dtype=torch.float32)
    ids, tw = c["topk_ids"].int().contiguous(), c["topk_weight"].float().contiguous()
    moe.cpu_prefill(M, ids.shape[1], ids.data_ptr(), tw.data_ptr(), a.contiguous().data_ptr(), out.data_ptr())
    torch.testing.assert_close(out, c["out"].float(), atol=2e-2, rtol=0)   # reference tolerance test_moe.py:233


@pytest.mark.parametrize("M", [1, 5, 16, 40, 64, 150])
def test_moe_fp8_block_vs_oracle(dev, M):
    import lk_moe
    E, k, H, I = 8, 4, 1024, 512
    g = torch.Generator().manual_seed(200 + M)
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16()
    w13q, w13s = O.quant_fp8_block(torch.randn(E, 2 * I, H, generator=g) / 10)
    w2q, w2s = O.quant_fp8_block(torch.randn(E, H, I, generator=g) / 10)
    w, ids = _route(M, E, k, g, 0.05)
    ref = O.experts_forward_w8a8_block(hidden, w13q, w13s, w2q, w2s, ids, w)
    moe = lk_moe.MOE_FP8(_cfg(E, k, H, I, gN=128, gK=128), w13q.data_ptr(), w2q.data_ptr(), w13s.data_ptr(),
                         w2s.data_ptr(), 0, 0)
    outs = _run_all_entry_points(moe, hidden, ids, w, dev)
    scale = ref.abs().mean()
    for name, o in outs.items():
        err = (o - ref).abs().mean() / scale
        # reference block-fp8 tolerance is 0.035 relative (tests/kernels/moe/test_block_fp8.py:207-210)
        assert err < 0.01, f"{name}: rel err {err}"
    assert torch.equal(outs["cpu_prefill"], outs["cpu_decode(graph)"])
    moe.close()


def test_moe_fp8_golden(dev, golden):
    import lk_moe
    c = golden["experts_fp8_block"]
    a = c["a"].contiguous()
    w1q, w2q = c["w1q"].contiguous(), c["w2q"].contiguous()
    w1s, w2s = c["w1s"].contiguous(), c["w2s"].contiguous()
    E, N1, H = w1q.shape
    ids, tw = c["topk_ids"].int().contiguous(), c["topk_weight"].float().contiguous()
    moe = lk_moe.MOE_FP8(_cfg(E, ids.shape[1], H, N1 // 2, gN=128, gK=128), w1q.data_ptr(), w2q.data_ptr(),
                         w1s.data_ptr(), w2s.data_ptr(), 0, 0)
    M = a.shape[0]
    out = torch.empty(M, H, dtype=torch.float32)
    moe.cpu_prefill(M, ids.shape[1], ids.data_ptr(), tw.data_ptr(), a.data_ptr(), out.data_ptr())
    ref = c["out"].float()
    assert ((out - ref).abs().mean() / ref.abs().mean()) < 0.035


def test_moe_properties_at_baseline_width(dev):
    """DeepSeek-V3 widths (H=7168, I=2048) with few experts: linearity in the routing weights, skipped
    slots contribute zero, batch-invariance of a token's result (same kernels for M=1 and M=8)."""
    import lk_moe
    E, k, H, I = 4, 2, 7168, 2048
    g = torch.Generator().manual_seed(7)
    w13q, w13s = O.quant_fp8_block(torch.randn(E, 2 * I, H, generator=g) / 10)
    w2q, w2s = O.quant_fp8_block(torch.randn(E, H, I, generator=g) / 10)
    moe = lk_moe.MOE_FP8(_cfg(E, k, H, I, gN=128, gK=128), w13q.data_ptr(), w2q.data_ptr(), w13s.data_ptr(),
                         w2s.data_ptr(), 0, 0)
    M = 8
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16()
    w, ids = _route(M, E, k, g)

    def run(hh, ii, ww):
        out = torch.empty(hh.shape[0], H, dtype=torch.float32)
        moe.cpu_prefill(hh.shape[0], k, ii.data_ptr(), ww.data_ptr(), hh.data_ptr(), out.data_ptr())
        return out

    base = run(hidden, ids, w)
    assert torch.isfinite(base).all() and base.abs().mean() > 0
    torch.testing.assert_close(run(hidden, ids, (w * 2).contiguous()), base * 2, atol=1e-6, rtol=1e-5)
    ids2 = ids.clone()
    ids2[:, 1] = -1
    w0 = w.clone()
    w0[:, 1] = 0
    assert torch.equal(run(hidden, ids2, w), run(hidden, ids, w0.contiguous()))
    one = run(hidden[3:4].contiguous(), ids[3:4].contiguous(), w[3:4].contiguous())
    # stream-K split points depend on the number of tiles, so M=1 and M=8 differ in fp32 summation order only
    torch.testing.assert_close(one[0], base[3], rtol=1e-4, atol=1e-5)
    assert torch.equal(run(hidden, ids, w), base)   # and a given batch is bit-reproducible
    # spot-check one token against the oracle at full width
    ref = O.experts_forward_w8a8_block(hidden[:1], w13q, w13s, w2q, w2s, ids[:1], w[:1])
    assert ((base[:1] - ref).abs().mean() / ref.abs().mean()) < 0.01


def _w4_case(fmt, M, E, k, H, I, seed):
    import lk_moe
    g = torch.Generator().manual_seed(seed)
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16()
    w13f = torch.randn(E, 2 * I, H, generator=g) / 10
    w2f = torch.randn(E, H, I, generator=g) / 10
    w, ids = _route(M, E, k, g, 0.05)
    if fmt == "int4":
        p13, s13 = O.quant_int4_group(w13f, 32)
        p2, s2 = O.quant_int4_group(w2f, 32)
        dq = O.DequantExperts(O.dequant_int4_group(p13, s13, 32), O.dequant_int4_group(p2, s2, 32))
        moe = lk_moe.MOE_WNA16(_cfg(E, k, H, I, gN=1, gK=32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0)
    elif fmt == "nvfp4":
        p13, s13, _ = O.quant_nvfp4(w13f.reshape(E * 2, I, H))   # separate global scale for the gate / up halves
        g13 = _.reshape(E, 2).contiguous()
        p13, s13 = p13.reshape(E, 2 * I, H // 2), s13.reshape(E, 2 * I, H // 16)
        p2, s2, g2 = O.quant_nvfp4(w2f)
        d13 = O.dequant_nvfp4(p13.reshape(E * 2, I, H // 2), s13.reshape(E * 2, I, H // 16), g13.reshape(E * 2)).reshape(E, 2 * I, H)
        dq = O.DequantExperts(d13, O.dequant_nvfp4(p2, s2, g2))
        g2 = g2.contiguous()
        moe = lk_moe.MOE_NVFP4(_cfg(E, k, H, I, gN=1, gK=16), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(),
                               g13.data_ptr(), g2.data_ptr())
    else:
        p13, s13 = O.quant_mxfp4(w13f)
        p2, s2 = O.quant_mxfp4(w2f)
        dq = O.DequantExperts(O.dequant_mxfp4(p13, s13), O.dequant_mxfp4(p2, s2))
        moe = lk_moe.MOE_MXFP4(_cfg(E, k, H, I, gN=1, gK=32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0)
    ref = O.experts_forward_batched(hidden, dq, ids, w, act_dtype=torch.float16)
    return moe, hidden, ids, w, ref


@pytest.mark.parametrize("M", [1, 16, 100])
def test_moe_mxfp4_dequant_path_vs_oracle(dev, M, monkeypatch):
    """MXFP4 through the W4A16 dequant kernel (the path INT4 / NVFP4 take too)."""
    moe, hidden, ids, w, ref = _w4_case("mxfp4", M, 8, 2, 512, 256, 300 + M)
    assert moe.query(0) == 0
    outs = _run_all_entry_points(moe, hidden, ids, w, dev)
    for name, o in outs.items():
        assert (o - ref).abs().mean() / ref.abs().mean() < 0.02, f"{name}"
    moe.close()


@pytest.mark.parametrize("fmt", ["int4", "nvfp4", "mxfp4"])
@pytest.mark.parametrize("M", [1, 7, 16, 40, 100])
def test_moe_w4a16_vs_oracle(dev, fmt, M):
    """W4A16 formats (weight-only dequant oracle; reference tolerances 4e-2 .. 1e-1, tests/kernels/moe/test_moe.py:1026-1182,
    test_nvfp4_moe.py:110-160)"""
    moe, hidden, ids, w, ref = _w4_case(fmt, M, 8, 2, 512, 256, 300 + M)
    outs = _run_all_entry_points(moe, hidden, ids, w, dev)
    scale = ref.abs().mean()
    for name, o in outs.items():
        err = (o - ref).abs().mean() / scale
        assert err < 0.02, f"{fmt} {name}: rel err {err}"
        assert (o - ref).abs().max() < 4e-2 * max(1.0, float(ref.abs().max()))
    moe.close()


def test_ctor_rejects_bad_input(dev):
    import lk_moe
    from lvllm_b200._lib import B200Error
    w = torch.zeros(2, 256, 200, dtype=torch.bfloat16)
    with pytest.raises(B200Error):
        lk_moe.MOE_BF16(_cfg(2, 2, 200, 128), w.data_ptr(), w.data_ptr(), 0, 0, 0, 0)   # H % 128 != 0
    with pytest.raises(B200Error):
        lk_moe.MOE_FP8(_cfg(2, 2, 256, 128, gN=128, gK=128), w.data_ptr(), w.data_ptr(), 0, 0, 0, 0)  # no scales


# ------------------------------------------------------------------------------------------ attention
def _cos_diff(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return 1 - 2 * (a * b).sum() / max((a * a + b * b).sum(), 1e-12)


@pytest.mark.parametrize("B,S,page,Hq", [(1, 4096, 64, 128), (3, 300, 16, 16), (2, 1, 128, 128), (4, 1000, 32, 32)])
def test_mla_decode_vs_oracle(dev, B, S, page, Hq):
    from lvllm_b200 import ops
    g = torch.Generator().manual_seed(42)
    lens = torch.tensor([max(1, S - 37 * b) for b in range(B)], dtype=torch.int32)
    npg = -(-S // page)
    cache = torch.randn(B * npg + 3, page, 576, generator=g).bfloat16()
    pt = torch.randperm(B * npg + 3, generator=g)[:B * npg].reshape(B, npg).int()   # shuffled pages
    qn = torch.randn(B, Hq, 512, generator=g).bfloat16()
    qp = torch.randn(B, Hq, 64, generator=g).bfloat16()
    scale = 1.0 / math.sqrt(576)
    ref, lse_ref = O.mla_decode(qn, qp, cache, lens, pt, scale)
    out, lse = ops.mla_decode(qn.to(dev), qp.to(dev), cache.to(dev), lens.to(dev), pt.to(dev), scale)
    # metric + thresholds of reference tests/kernels/attention/test_cutlass_mla_decode.py:15-32
    assert _cos_diff(out.cpu().float(), ref) < 1e-5
    torch.testing.assert_close(lse.cpu(), lse_ref, atol=1e-3, rtol=1e-3)
    from lvllm_b200._lib import B200Error
    with pytest.raises(B200Error, match="num_heads <= 128"):   # one head more than the kernel serves
        ops.mla_decode(torch.zeros(B, 129, 512, dtype=torch.bfloat16, device=dev),
                       torch.zeros(B, 129, 64, dtype=torch.bfloat16, device=dev), cache.to(dev), lens.to(dev), pt.to(dev),
                       scale)


@pytest.mark.parametrize("splits", [0, 3])   # 0: tensor-core path (128-token splits); 3: CUDA-core split-KV path
@pytest.mark.parametrize("B,S,page,Hq,Hkv", [(64, 2048, 16, 32, 8), (3, 77, 16, 64, 4), (2, 5, 32, 8, 8), (5, 513, 64, 32, 2),
                                             (7, 1300, 16, 64, 4),
                                             # groups of 32 and 24 query heads (the wider instantiation), several work items
                                             # per CTA (512 and 480 items over the SMs)
                                             (64, 1024, 16, 32, 1), (40, 700, 16, 48, 2)])
def test_gqa_decode_vs_oracle(dev, B, S, page, Hq, Hkv, splits):
    from lvllm_b200 import ops
    g = torch.Generator().manual_seed(1)
    D = 128
    lens = torch.tensor([max(1, S - 11 * (b % 7)) for b in range(B)], dtype=torch.int32)
    npg = -(-S // page)
    kc = torch.randn(B * npg, page, Hkv, D, generator=g).bfloat16()
    vc = torch.randn(B * npg, page, Hkv, D, generator=g).bfloat16()
    pt = torch.randperm(B * npg, generator=g).reshape(B, npg).int()
    q = torch.randn(B, Hq, D, generator=g).bfloat16()
    scale = D ** -0.5
    # oracle on a subset of requests keeps the CPU side in seconds: the first and the last ones (a CTA's later work items)
    sel = torch.tensor(sorted(set(range(min(B, 3))) | set(range(max(0, B - 3), B))))
    ref, lse_ref = O.gqa_decode(q[sel], kc, vc, lens[sel], pt[sel], scale)
    out, lse = ops.gqa_decode(q.to(dev), kc.to(dev), vc.to(dev), lens.to(dev), pt.to(dev), scale, num_kv_splits=splits)
    assert _cos_diff(out.cpu().float()[sel], ref) < 1e-5
    torch.testing.assert_close(lse.cpu()[sel], lse_ref, atol=1e-3, rtol=1e-3)
    assert torch.isfinite(out.float()).all()


def test_gqa_golden(dev, golden):
    from lvllm_b200 import ops
    c = golden["gqa_decode"]
    D = c["q"].shape[-1]
    assert D == 128
    out, _ = ops.gqa_decode(c["q"].bfloat16().to(dev), c["k_cache"].bfloat16().to(dev), c["v_cache"].bfloat16().to(dev),
                            torch.tensor(c["kv_lens"], dtype=torch.int32).to(dev), c["block_tables"].to(dev), c["scale"])
    # fixture is fp32 (reference ref_paged_attn); bf16 inputs/outputs -> cos_diff threshold of the reference MLA test
    assert _cos_diff(out.cpu().float(), c["out"].float()) < 5e-5
