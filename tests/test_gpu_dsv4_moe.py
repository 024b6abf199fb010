"""DeepSeek-V4 MoE on the GPU: sqrt-softplus top-k and token-id hash routing in the stand-alone routing kernel and the
fused router, the clamped SwiGLU (activation_type 3) in every expert format's decode and in gpu_prefill, and one
V4-Flash-shaped layer (router -> MXFP4 cpu_decode with a folded shared expert) under CUDA-graph replay.  References:
tests/dsv4_moe_oracle.py and the expert oracles of oracle/moe_oracle.py."""
import pytest
import torch

import dsv4_moe_oracle as D
from oracle import moe_oracle as O
from test_gpu_parity import _ulp_tie_ok

pytestmark = pytest.mark.gpu

LIMIT = 10.0   # V4-Flash's swiglu_limit
RSF = 1.5


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _bias(kind, E, g):
    if kind == "normal":
        return torch.randn(E, generator=g)
    return 8.08 + 1e-3 * torch.randn(E, generator=g)   # V4-Flash's correction biases are all about 8.08


def _biased_scores(bias):
    return lambda row: torch.from_numpy(D.sqrt_softplus(row.float().numpy())) + bias.float()


def _check_routing(w, ids, w_ref, i_ref, logits, bias, rtol=2e-6):
    w, ids = w.cpu(), ids.cpu()
    for t in range(ids.shape[0]):
        if not torch.equal(ids[t], i_ref[t]):
            assert _ulp_tie_ok(logits[t], ids[t], i_ref[t], _biased_scores(bias)), (t, ids[t], i_ref[t])
            continue
        torch.testing.assert_close(w[t], w_ref[t], rtol=rtol, atol=0)


# ------------------------------------------------------------------------------------------ stand-alone routing
@pytest.mark.parametrize("renorm", [True, False])
@pytest.mark.parametrize("bias_kind", ["normal", "v4flash"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,E,k", [(1, 256, 6), (37, 384, 8), (1000, 256, 8), (200, 384, 6)])
def test_topk_gating_sqrtsoftplus_vs_oracle(dev, M, E, k, dtype, bias_kind, renorm):
    from lvllm_b200 import ops
    g = torch.Generator().manual_seed(M * 7 + E + k)
    logits = (torch.randn(M, E, generator=g) * 2).to(dtype)
    bias = _bias(bias_kind, E, g)
    w_ref, i_ref = D.topk_sqrtsoftplus(logits, k, renorm, bias, RSF)
    w, ids = ops.fused_topk(logits.to(dev), k, renorm, "sqrtsoftplus", bias.to(dev), RSF)
    torch.cuda.synchronize()
    _check_routing(w, ids, w_ref, i_ref, logits, bias)


@pytest.mark.parametrize("M", [1, 64, 513])
def test_hash_topk_vs_oracle(dev, M):
    from lvllm_b200 import ops
    E, k, vocab = 256, 6, 129280
    g = torch.Generator().manual_seed(M)
    logits = torch.randn(M, E, generator=g) * 2
    table = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(64)]).repeat(vocab // 64 + 1, 1)[:vocab]
    input_ids = torch.randint(0, vocab, (M,), generator=g)
    for renorm in (True, False):
        w_ref, i_ref = D.topk_sqrtsoftplus(logits, k, renorm, None, RSF, input_ids, table)
        # int64 ids and table here: converted in the op
        w, ids = ops.hash_topk(logits.to(dev), k, renorm, input_ids.to(dev), table.to(dev), RSF)
        torch.cuda.synchronize()
        assert torch.equal(ids.cpu(), table[input_ids].int())
        torch.testing.assert_close(w.cpu(), w_ref, rtol=2e-6, atol=0)


def test_hash_topk_out_of_range(dev):
    from lvllm_b200 import ops
    E, k, vocab, M = 256, 6, 64, 8
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(M, E, generator=g).bfloat16()
    table = torch.randint(0, E, (vocab, k), generator=g, dtype=torch.int32)
    table[5, 2], table[5, 4] = E, -7
    input_ids = torch.tensor([0, -1, vocab, 5, 63, 2**31 - 1, 5, 1], dtype=torch.int32)
    w_ref, i_ref = D.topk_sqrtsoftplus(logits, k, True, None, RSF, input_ids, table)
    w, ids = ops.hash_topk(logits.to(dev), k, True, input_ids.to(dev), table.to(dev), RSF)
    torch.cuda.synchronize()
    w, ids = w.cpu(), ids.cpu()
    assert torch.equal(ids, i_ref)
    assert (ids[[1, 2, 5]] == -1).all() and (w[[1, 2, 5]] == 0).all()
    assert ids[3, 2] == -1 and ids[3, 4] == -1 and w[3, 2] == 0 and w[3, 4] == 0
    torch.testing.assert_close(w, w_ref, rtol=2e-6, atol=0)


# ------------------------------------------------------------------------------------------ fused router
@pytest.mark.parametrize("hashed", [False, True])
@pytest.mark.parametrize("M", [1, 64, 300])
def test_fused_router_matches_standalone_bitwise(dev, M, hashed):
    """The fused router's ids and weights are the stand-alone kernel's on the fused router's own logits_out, bit for bit,
    with an EP expert map and one shared column."""
    from lvllm_b200 import ops
    E, k, H, vocab = 256, 6, 4096, 1000
    g = torch.Generator().manual_seed(300 + M + hashed)
    hidden = torch.randn(M, H, generator=g).bfloat16().to(dev)
    wg = (torch.randn(E, H, generator=g) / 32).bfloat16().to(dev)
    bias = _bias("v4flash", E, g).to(dev)
    emap = torch.full((E,), -1, dtype=torch.int32)
    emap[64:128] = torch.arange(64, dtype=torch.int32)
    emap = emap.to(dev)
    table = torch.randint(0, E, (vocab, k), generator=g, dtype=torch.int32).to(dev)
    input_ids = torch.randint(0, vocab, (M,), generator=g, dtype=torch.int32).to(dev)
    kw = dict(input_ids=input_ids, hash_indices_table=table) if hashed else {}
    w, ids, loc, lg = ops.router_topk(hidden, wg, k, True, "sqrtsoftplus", bias, RSF, expert_map=emap, return_logits=True,
                                      n_shared=1, shared_local_base=64, shared_weight=1.0, **kw)
    if hashed:
        w_s, ids_s = ops.hash_topk(lg, k, True, input_ids, table, RSF)
    else:
        w_s, ids_s = ops.fused_topk(lg, k, True, "sqrtsoftplus", bias, RSF)
    torch.cuda.synchronize()
    assert torch.equal(ids[:, :k], ids_s) and torch.equal(w[:, :k], w_s)
    assert (ids[:, k] == E).all() and (w[:, k] == 1.0).all() and (loc[:, k] == 64).all()
    assert torch.equal(loc[:, :k], ops.global_to_local_expert_ids(ids_s, emap))
    ref = hidden.float() @ wg.float().t()
    torch.testing.assert_close(lg, ref, rtol=1e-4, atol=1e-3)


# ------------------------------------------------------------------------------------------ clamped experts
def _moe_cfg(E, k, H, I, gN=0, gK=0, max_seqs=256):
    import lk_moe
    c = lk_moe.MOEConfigV2()
    c.expert_num, c.top_k, c.hidden_size, c.intermediate_size = E, k, H, I
    c.max_batch_size, c.max_num_seqs = 4096, max_seqs
    c.groupN, c.groupK = gN, gK
    c.gpu_id = 0
    c.swiglu_limit = LIMIT   # assigned: activation_type 0 goes to the library as 3
    return c


def _clamped_layer(fmt, E, k, H, I, g, w13_scale):
    """(layer, oracle(hidden, ids, w, act_type), tolerance, fp32 w13 before quantisation, keep-alive)"""
    import lk_moe
    w13f = torch.randn(E, 2 * I, H, generator=g) * w13_scale
    w2f = torch.randn(E, H, I, generator=g) / 10
    if fmt == "bf16":
        w13, w2 = w13f.bfloat16(), w2f.bfloat16()
        moe = lk_moe.MOE_BF16(_moe_cfg(E, k, H, I), w13.data_ptr(), w2.data_ptr(), 0, 0, 0, 0)
        dq = O.DequantExperts(w13.float(), w2.float())
        ref = lambda x, ids, w, act: O.experts_forward_batched(x, dq, ids, w, activation_type=act, act_dtype=torch.bfloat16)
        return moe, ref, 5e-3, w13f, (w13, w2)
    if fmt == "fp8":
        w13q, w13s = O.quant_fp8_block(w13f)
        w2q, w2s = O.quant_fp8_block(w2f)
        moe = lk_moe.MOE_FP8(_moe_cfg(E, k, H, I, 128, 128), w13q.data_ptr(), w2q.data_ptr(), w13s.data_ptr(),
                             w2s.data_ptr(), 0, 0)
        ref = lambda x, ids, w, act: O.experts_forward_w8a8_block(x, w13q, w13s, w2q, w2s, ids, w, activation_type=act)
        return moe, ref, 1e-2, w13f, (w13q, w13s, w2q, w2s)
    if fmt == "int4":
        p13, s13 = O.quant_int4_group(w13f, 32)
        p2, s2 = O.quant_int4_group(w2f, 32)
        dq = O.DequantExperts(O.dequant_int4_group(p13, s13, 32), O.dequant_int4_group(p2, s2, 32))
        moe = lk_moe.MOE_WNA16(_moe_cfg(E, k, H, I, 1, 32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(),
                               0, 0)
        keep = (p13, p2, s13, s2)
    elif fmt == "nvfp4":
        p13, s13, g13 = O.quant_nvfp4(w13f.reshape(E * 2, I, H))
        g13 = g13.reshape(E, 2).contiguous()
        p13, s13 = p13.reshape(E, 2 * I, H // 2), s13.reshape(E, 2 * I, H // 16)
        p2, s2, g2 = O.quant_nvfp4(w2f)
        d13 = O.dequant_nvfp4(p13.reshape(E * 2, I, H // 2), s13.reshape(E * 2, I, H // 16), g13.reshape(E * 2))
        dq = O.DequantExperts(d13.reshape(E, 2 * I, H), O.dequant_nvfp4(p2, s2, g2))
        g2 = g2.contiguous()
        moe = lk_moe.MOE_NVFP4(_moe_cfg(E, k, H, I, 1, 16), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(),
                               g13.data_ptr(), g2.data_ptr())
        keep = (p13, p2, s13, s2, g13, g2)
    else:
        p13, s13 = O.quant_mxfp4(w13f)
        p2, s2 = O.quant_mxfp4(w2f)
        dq = O.DequantExperts(O.dequant_mxfp4(p13, s13), O.dequant_mxfp4(p2, s2))
        moe = lk_moe.MOE_MXFP4(_moe_cfg(E, k, H, I, 1, 32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(),
                               0, 0)
        keep = (p13, p2, s13, s2)
    ref = lambda x, ids, w, act: O.experts_forward_batched(x, dq, ids, w, activation_type=act, act_dtype=torch.float16)
    return moe, ref, 2e-2, w13f, keep


FORMATS = ["bf16", "fp8", "int4", "nvfp4", "mxfp4"]


def _run_clamped(dev, fmt, M, prefill):
    E, k, H, I = 8, 2, 512, 256
    g = torch.Generator().manual_seed(900 + M + len(fmt))
    # hidden ~ 0.1, H = 512: w13 ~ 5.5 puts the gate / up pre-activations at ~1.25 x the limit
    moe, ref_fn, tol, w13f, keep = _clamped_layer(fmt, E, k, H, I, g, 5.5)
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16()
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(M)]).int()
    w = torch.softmax(torch.randn(M, k, generator=g), -1).float().contiguous()
    pre = hidden.float() @ w13f[0].t()
    assert (pre[:, :I] > LIMIT).float().mean() > 0.1 and (pre[:, I:].abs() > LIMIT).float().mean() > 0.1
    with D.clamped_activation(LIMIT):
        ref = ref_fn(hidden, ids, w, D.ACT_SILU_CLAMP)
    ref_plain = ref_fn(hidden, ids, w, O.ACT_SILU)
    scale = float(ref.abs().mean())
    assert float((ref_plain - ref).abs().mean()) / scale > 20 * tol   # the clamp is visible far above the tolerance
    hd, idd, wd = hidden.to(dev), ids.to(dev), w.to(dev)
    if prefill:
        out = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        moe.gpu_prefill(hd.data_ptr(), out.data_ptr(), idd.data_ptr(), wd.data_ptr(), M, k,
                        torch.cuda.current_stream().cuda_stream)
    else:
        out = torch.zeros(M, H, dtype=torch.float32, device=dev)
        moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, k, hd.data_ptr(), idd.data_ptr(), wd.data_ptr(),
                       out.data_ptr())
    torch.cuda.synchronize()
    moe.close()
    o = out.float().cpu()
    err = float((o - ref).abs().mean()) / scale
    assert err < (2 * tol if prefill else tol), f"{fmt} M={M}: rel err {err}"


@pytest.mark.parametrize("M", [1, 7, 64, 256])
@pytest.mark.parametrize("fmt", FORMATS)
def test_clamped_experts_decode(dev, fmt, M):
    _run_clamped(dev, fmt, M, prefill=False)


@pytest.mark.parametrize("fmt", FORMATS)
def test_clamped_experts_gpu_prefill(dev, fmt):
    _run_clamped(dev, fmt, 1100, prefill=True)


# ------------------------------------------------------------------------------------------ one V4-Flash-shaped layer
@pytest.mark.parametrize("hashed", [False, True])
def test_v4flash_layer_graph(dev, hashed):
    """Router (sqrt-softplus + bias, or hash) in the fused form -> MOE_MXFP4.cpu_decode over 256 routed experts + 1 shared
    expert folded in as an always-on column, top-6; captured in a CUDA graph and replayed twice with identical bits.
    H and I are cut to 512 / 256 to keep the host-side quantisation and oracle small."""
    import lk_moe
    from lvllm_b200.router import Router
    E, k, H, I, M, vocab = 256, 6, 512, 256, 16, 129280
    g = torch.Generator().manual_seed(77 + hashed)
    w13f = torch.randn(E + 1, 2 * I, H, generator=g) * 5.5
    w2f = torch.randn(E + 1, H, I, generator=g) / 10
    p13, s13 = O.quant_mxfp4(w13f)
    p2, s2 = O.quant_mxfp4(w2f)
    dq = O.DequantExperts(O.dequant_mxfp4(p13, s13), O.dequant_mxfp4(p2, s2))
    cfg = _moe_cfg(E + 1, k + 1, H, I, 1, 32, max_seqs=M)
    moe = lk_moe.MOE_MXFP4(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0)
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16().to(dev)
    wg = (torch.randn(E, H, generator=g) / 8).bfloat16().to(dev)
    bias = _bias("v4flash", E, g).to(dev)
    table = torch.randint(0, E, (vocab, k), generator=g)
    input_ids = torch.randint(0, vocab, (M,), generator=g, dtype=torch.int32).to(dev)
    router = Router(k, E, True, "sqrtsoftplus", routed_scaling_factor=RSF, e_score_correction_bias=bias,
                    num_fused_shared_experts=1, shared_local_base=E, shared_weight=1.0,
                    hash_indices_table=table.to(dev) if hashed else None)
    outs = [torch.zeros(M, H, dtype=torch.float32, device=dev) for _ in range(2)]
    box = {}

    def step(out):
        w, ids = router.select_experts(hidden, gate_weight=wg, input_ids=input_ids)
        loc = router.last_local_ids
        box.update(w=w, ids=ids, loc=loc)
        moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, k + 1, hidden.data_ptr(), loc.data_ptr(), w.data_ptr(),
                       out.data_ptr())

    step(outs[0])   # eager warm-up: allocates the router workspace outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            step(outs[1])
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    first = outs[1].clone()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(first, outs[1]), "two replays differ"
    assert torch.equal(first, outs[0]), "eager and graph replay differ"

    # oracle chain: routing from fp32 logits, experts from the kernel's own routing
    w, ids, loc = box["w"].cpu(), box["ids"].cpu(), box["loc"].cpu()
    logits = hidden.float().cpu() @ wg.float().cpu().t()
    if hashed:
        w_ref, i_ref = D.topk_sqrtsoftplus(logits, k, True, None, RSF, input_ids.cpu(), table)
        assert torch.equal(ids[:, :k], i_ref)
        torch.testing.assert_close(w[:, :k], w_ref, rtol=1e-4, atol=0)
    else:
        w_ref, i_ref = D.topk_sqrtsoftplus(logits, k, True, bias.cpu(), RSF)
        for t in range(M):
            if torch.equal(ids[t, :k], i_ref[t]):
                torch.testing.assert_close(w[t, :k], w_ref[t], rtol=1e-4, atol=0)
            else:   # the GEMM's summation order moves the logits by ~1e-6: only a near-tie may swap an expert
                sc = _biased_scores(bias.cpu())(logits[t])
                diff = list(set(ids[t, :k].tolist()) ^ set(i_ref[t].tolist()))
                assert float(sc[diff].max() - sc[diff].min()) < 1e-4 * float(sc[diff].abs().max()), t
    assert (ids[:, k] == E).all() and (loc[:, k] == E).all() and (w[:, k] == 1.0).all()
    with D.clamped_activation(LIMIT):
        ref = O.experts_forward_batched(hidden.cpu(), dq, loc, w, activation_type=D.ACT_SILU_CLAMP,
                                        act_dtype=torch.float16)
    moe.close()
    err = float((first.cpu() - ref).abs().mean() / ref.abs().mean())
    assert err < 2e-2, f"rel err {err}"
