"""4-bit tiles are stored in the fused decode kernel's wgmma fragment order (lvllm_b200/csrc/w4_layout.cuh).  These layers
make a misplaced nibble or scale show up far above tolerance: every weight code is a function of (expert, row, column)
that differs between rows 8, 16, 64 and 128 apart, and the scales change with the row of the tile and with the group.  H = 768 and I = 384 give 3 gate/up tiles
and 3 w2 tile pairs per expert.  Each layer runs as a decode batch (eagerly and as a CUDA-graph replay, which must agree
bit for bit) and through the prefill path, which expands the same tiles to fp16; both are checked against the W4A16
oracle."""
import pytest
import torch

from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu

E, K_TOP, H, I = 4, 2, 768, 384
COUNTS = [64, 40, 16, 8]   # M = 64, top-2: chunks of 64, 48 and 16 padded rows


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _codes(n_rows, k):
    """[E, n_rows, k] 4-bit codes that depend on expert, row and column."""
    e = torch.arange(E).view(E, 1, 1)
    r = torch.arange(n_rows).view(1, n_rows, 1)
    c = torch.arange(k).view(1, 1, k)
    return ((r * 5 + c * 3 + (c // 16) * 7 + e * 11 + (r // 8) * 2 + (r // 64) * 3) % 16).to(torch.int32)


def _pack(codes):
    return (codes[..., 0::2] | (codes[..., 1::2] << 4)).to(torch.uint8).contiguous()


def _row_group(n_rows, n_groups):
    """(row of the tile, group) of every scale position [E, n_rows, n_groups]"""
    r = torch.arange(n_rows).view(1, n_rows, 1).expand(E, n_rows, n_groups)
    g = torch.arange(n_groups).view(1, 1, n_groups).expand(E, n_rows, n_groups)
    return r % 128, g


def _mix(r, g, n):
    """one of n scale codes; rows 1, 8, 16, 32 and 64 apart and neighbouring groups of a tile get different codes"""
    return (r + (r // 16) * 3 + (r // 64) * 5 + g * 7) % n


def _layer(fmt):
    import lk_moe
    c13, c2 = _codes(2 * I, H), _codes(H, I)
    p13, p2 = _pack(c13), _pack(c2)
    cfg = lk_moe.MOEConfigV2()
    cfg.expert_num, cfg.top_k, cfg.hidden_size, cfg.intermediate_size = E, K_TOP, H, I
    cfg.max_batch_size, cfg.max_num_seqs, cfg.groupN = 4096, 64, 1
    cfg.gpu_id = 0
    if fmt == "int4":
        def scales(n_rows, k):   # bf16 scales, distinct for every (row, group) of a tile and exact in fp16
            r, g = _row_group(n_rows, k // 32)
            idx = r * 2 + g % 2
            return (2.0 ** -8 * (1 + (idx % 128) / 128) * 2.0 ** (idx // 128)).bfloat16().contiguous()
        s13, s2 = scales(2 * I, H), scales(H, I)
        dq = O.DequantExperts(O.dequant_int4_group(p13, s13, 32), O.dequant_int4_group(p2, s2, 32))
        cfg.groupK = 32
        moe = lk_moe.MOE_WNA16(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0)
        return moe, dq, (p13, p2, s13, s2)
    if fmt == "nvfp4":
        def scales(n_rows, k):   # e4m3 block scales 0.25 .. 60: too few values for 512 distinct ones per tile
            r, g = _row_group(n_rows, k // 16)
            return (0x28 + _mix(r, g % 4, 64)).to(torch.uint8).view(torch.float8_e4m3fn).contiguous()
        s13, s2 = scales(2 * I, H), scales(H, I)
        g13 = torch.tensor([[0.004, 0.003]] * E, dtype=torch.float32)
        g2 = torch.full((E,), 0.002, dtype=torch.float32)
        d13 = torch.cat([O.dequant_nvfp4(p13[:, :I], s13[:, :I], g13[:, 0]), O.dequant_nvfp4(p13[:, I:], s13[:, I:], g13[:, 1])], 1)
        dq = O.DequantExperts(d13, O.dequant_nvfp4(p2, s2, g2))
        cfg.groupK = 16
        moe = lk_moe.MOE_NVFP4(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), g13.data_ptr(),
                               g2.data_ptr())
        return moe, dq, (p13, p2, s13, s2, g13, g2)

    def scales(n_rows, k):   # e8m0 scales 2^-14 .. 2^1 (the fused kernel flushes smaller ones to zero)
        r, g = _row_group(n_rows, k // 32)
        return (113 + _mix(r, g % 2, 16)).to(torch.uint8).contiguous()
    s13, s2 = scales(2 * I, H), scales(H, I)
    dq = O.DequantExperts(O.dequant_mxfp4(p13, s13), O.dequant_mxfp4(p2, s2))
    cfg.groupK = 32
    moe = lk_moe.MOE_MXFP4(cfg, p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(), 0, 0)
    return moe, dq, (p13, p2, s13, s2)


def _inputs(seed):
    M = sum(COUNTS) // K_TOP
    g = torch.Generator().manual_seed(seed)
    hidden = (torch.randn(M, H, generator=g) / 10).bfloat16()
    flat = torch.cat([torch.full((c,), e, dtype=torch.int32) for e, c in enumerate(COUNTS)])
    ids = flat.reshape(K_TOP, M).t().contiguous()   # a token never gets the same expert twice
    w = torch.softmax(torch.randn(M, K_TOP, generator=g), -1).float().contiguous()
    return hidden, ids, w


def _check(out, ref, what):
    err = float((out - ref).abs().mean() / ref.abs().mean())
    assert err < 2e-2, f"{what}: rel err {err}"
    assert float((out - ref).abs().max()) < 4e-2 * max(1.0, float(ref.abs().max())), what


@pytest.mark.parametrize("fmt", ["int4", "nvfp4", "mxfp4"])
def test_w4_fragment_layout_decode(dev, fmt):
    moe, dq, keep = _layer(fmt)
    hidden, ids, w = _inputs(11)
    M = hidden.shape[0]
    ref = O.experts_forward_batched(hidden, dq, ids, w, act_dtype=torch.float16)
    hd, idd, wd = hidden.to(dev), ids.to(dev), w.to(dev)
    outs = [torch.zeros(M, H, dtype=torch.float32, device=dev) for _ in range(2)]

    def launch(o):
        moe.cpu_decode(torch.cuda.current_stream().cuda_stream, M, K_TOP, hd.data_ptr(), idd.data_ptr(), wd.data_ptr(),
                       o.data_ptr())

    launch(outs[0])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            launch(outs[1])
    torch.cuda.current_stream().wait_stream(side)
    outs[1].zero_()
    graph.replay()
    torch.cuda.synchronize()
    moe.close()
    _check(outs[0].cpu(), ref, f"{fmt} decode")
    assert torch.equal(outs[0], outs[1]), "eager and CUDA-graph replay differ"


@pytest.mark.parametrize("fmt", ["int4", "nvfp4", "mxfp4"])
def test_w4_fragment_layout_prefill(dev, fmt, monkeypatch):
    monkeypatch.setenv("B200MOE_W4_PREFILL_MIN", "1")   # expand the tiles to fp16 even at this batch
    moe, dq, keep = _layer(fmt)
    hidden, ids, w = _inputs(12)
    M = hidden.shape[0]
    ref = O.experts_forward_batched(hidden, dq, ids, w, act_dtype=torch.float16)
    out = torch.empty(M, H, dtype=torch.float32)
    moe.cpu_prefill(M, K_TOP, ids.data_ptr(), w.data_ptr(), hidden.data_ptr(), out.data_ptr())
    moe.close()
    _check(out, ref, f"{fmt} prefill")
