"""4-bit fused decode (W4A16: int4, nvfp4, mxfp4) at routings that exercise the 64-row chunks: experts of 33-64 rows read
once per launch, experts of more than 64 rows split into several chunks, and chunks of every instruction width
16 / 32 / 48 / 64.  Each case is checked against the weight-only dequant oracle, for bit-reproducibility between two
launches, and for bit-identity between an eager launch and a CUDA-graph replay."""
import pytest
import torch

from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cfg(E, k, H, I, max_seqs, gK):
    import lk_moe
    c = lk_moe.MOEConfigV2()
    c.expert_num, c.top_k, c.hidden_size, c.intermediate_size = E, k, H, I
    c.max_batch_size, c.max_num_seqs = 4096, max_seqs
    c.groupN, c.groupK = 1, gK
    c.gpu_id = 0
    return c


def _ids_with_counts(counts, M, k):
    """ids [M, k] in which expert e gets counts[e] rows; slot p = (token p % M, column p // M), so a run of <= M
    consecutive slots never gives a token the same expert twice."""
    assert sum(counts) == M * k and max(counts) <= M
    flat = torch.cat([torch.full((c,), e, dtype=torch.int32) for e, c in enumerate(counts)])
    return flat.reshape(k, M).t().contiguous()


def _layer(fmt, E, H, I, max_seqs, g):
    import lk_moe
    w13f = torch.randn(E, 2 * I, H, generator=g) / 10
    w2f = torch.randn(E, H, I, generator=g) / 10
    if fmt == "int4":
        p13, s13 = O.quant_int4_group(w13f, 32)
        p2, s2 = O.quant_int4_group(w2f, 32)
        dq = O.DequantExperts(O.dequant_int4_group(p13, s13, 32), O.dequant_int4_group(p2, s2, 32))
        moe = lk_moe.MOE_WNA16(_cfg(E, 2, H, I, max_seqs, 32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(),
                               s2.data_ptr(), 0, 0)
        keep = (p13, p2, s13, s2)
    elif fmt == "nvfp4":
        p13, s13, g13 = O.quant_nvfp4(w13f.reshape(E * 2, I, H))   # separate global scales for gate and up
        g13 = g13.reshape(E, 2).contiguous()
        p13, s13 = p13.reshape(E, 2 * I, H // 2), s13.reshape(E, 2 * I, H // 16)
        p2, s2, g2 = O.quant_nvfp4(w2f)
        d13 = O.dequant_nvfp4(p13.reshape(E * 2, I, H // 2), s13.reshape(E * 2, I, H // 16), g13.reshape(E * 2))
        dq = O.DequantExperts(d13.reshape(E, 2 * I, H), O.dequant_nvfp4(p2, s2, g2))
        g2 = g2.contiguous()
        moe = lk_moe.MOE_NVFP4(_cfg(E, 2, H, I, max_seqs, 16), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(),
                               s2.data_ptr(), g13.data_ptr(), g2.data_ptr())
        keep = (p13, p2, s13, s2, g13, g2)
    else:
        p13, s13 = O.quant_mxfp4(w13f)
        p2, s2 = O.quant_mxfp4(w2f)
        dq = O.DequantExperts(O.dequant_mxfp4(p13, s13), O.dequant_mxfp4(p2, s2))
        moe = lk_moe.MOE_MXFP4(_cfg(E, 2, H, I, max_seqs, 32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(),
                               s2.data_ptr(), 0, 0)
        keep = (p13, p2, s13, s2)
    return moe, dq, keep


CASES = {
    # M = 64, top-2 over 8 experts, concentrated: chunks of 64 / 48 / 32 / 16 padded rows, two experts of 33-64 rows
    "widths_m64": (64, [50, 34, 20, 12, 6, 3, 2, 1]),
    # every active expert between 33 and 64 rows (the shape of a concentrated Mixtral batch)
    "mixtral_like_m64": (64, [64, 40, 24, 0, 0, 0, 0, 0]),
    # experts of more than 64 rows: several 64-row chunks per expert, plus a remainder chunk
    "split_m200": (200, [150, 100, 70, 40, 20, 10, 5, 5]),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("fmt", ["int4", "nvfp4", "mxfp4"])
def test_w4_decode_chunks(dev, fmt, case):
    M, counts = CASES[case]
    E, k, H, I = 8, 2, 512, 256
    g = torch.Generator().manual_seed(4000 + M + len(fmt))
    moe, dq, keep = _layer(fmt, E, H, I, max(M, 64), g)
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16()
    ids = _ids_with_counts(counts, M, k)
    w = torch.softmax(torch.randn(M, k, generator=g), -1).float().contiguous()
    ref = O.experts_forward_batched(hidden, dq, ids, w, act_dtype=torch.float16)

    hd, idd, wd = hidden.to(dev), ids.to(dev), w.to(dev)
    outs = [torch.zeros(M, H, dtype=torch.float32, device=dev) for _ in range(3)]
    st = torch.cuda.current_stream()

    def launch(o):
        moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, k, hd.data_ptr(), idd.data_ptr(), wd.data_ptr(),
                       o.data_ptr())

    launch(outs[0])
    launch(outs[1])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(st)
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            launch(outs[2])
    st.wait_stream(side)
    outs[2].zero_()
    graph.replay()
    torch.cuda.synchronize()
    moe.close()

    o = outs[0].cpu()
    err = float((o - ref).abs().mean() / ref.abs().mean())
    assert err < 2e-2, f"{fmt} {case}: rel err {err}"
    assert float((o - ref).abs().max()) < 4e-2 * max(1.0, float(ref.abs().max()))
    assert torch.equal(outs[0], outs[1]), "two launches differ"
    assert torch.equal(outs[0], outs[2]), "eager and CUDA-graph replay differ"
