"""GPU (-m gpu): the DeepSeek-V4 attention output projection (ops.dsv4_inv_rope_quant, ops.dsv4_o_proj).

Against the oracle (tests/dsv4_oproj_oracle.py): the inverse RoPE + quantisation bit for bit, also on a head slice of a
padded output; z against the float64 GEMM on the kernel's own fp8 operands within one bf16 ulp plus 2^-12 of the summed
magnitudes (the fp8 tensor core's accumulation inside a k-block); at the reference test's shape, calc_diff < 1e-2 to the
unquantised bf16 composition (its threshold).  A token's z is the same bits alone and in a batch, in repeated calls and in
a CUDA-graph replay; T = 0 writes nothing; sparse decode followed by the projection matches the oracle composition."""
import pytest
import torch

import dsv4_oproj_oracle as O
import dsv4_sparse_oracle as V4
from lvllm_b200 import _lib as L
from lvllm_b200 import ops

pytestmark = pytest.mark.gpu

MAX_POS = 4096
ACC_TOL = 2 ** -12
SHAPES = [(64, 8), (16, 2), (8, 1)]   # (heads, groups): V4-Flash-style 64 heads in 8 groups and tensor-parallel shards


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_sin(n=MAX_POS):
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(n, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


def _o(gen, T, H):
    """bf16 [T, H, 512] with per-head magnitudes over four decades, so that scales differ between blocks."""
    mag = torch.logspace(-2, 2, H)[None, :, None]
    return (torch.randn(T, H, 512, generator=gen) * mag).bfloat16()


def _positions(gen, T):
    p = torch.randint(0, MAX_POS, (T,), generator=gen)
    if T > 2:
        p[0], p[1] = -3, MAX_POS + 5   # clamped to the table
    return p


def _weights(gen, G, R, D):
    w = torch.randn(G * R, D, generator=gen) * torch.logspace(-1, 1, G * R // 128).repeat_interleave(128)[:, None]
    return O.quant_weight(w)


def _bytes(t):
    return t.contiguous().view(torch.uint8)


def _ulp_bf16(x):
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126)))
    return torch.exp2(e - 7)


def _check_z(z, o8, s8, w, ws):
    ref, bound = O.wo_a(o8, s8, w, ws)
    err = (z.double().to(ref.device) - ref).abs()
    tol = _ulp_bf16(ref) + ACC_TOL * bound
    bad = err > tol
    assert not bad.any(), f"{int(bad.sum())} outputs off, worst excess {(err - tol).max().item():.3e}"


@pytest.mark.parametrize("T", [1, 7, 64, 256])
@pytest.mark.parametrize("H,G", SHAPES)
def test_quant_bit_exact(dev, H, G, T):
    gen = torch.Generator().manual_seed(1000 * H + T)
    o, pos, cs = _o(gen, T, H), _positions(gen, T), _cos_sin()
    q, s = ops.dsv4_inv_rope_quant(o.to(dev), pos.to(dev), cs.to(dev), G)
    rq, rs = O.inv_rope_quant(o, pos, cs, G)
    D = H // G * 512
    assert q.shape == (T, G, D) and s.shape == (T, G, D // 128)
    assert torch.equal(_bytes(q.cpu()), _bytes(rq))
    assert torch.equal(s.cpu(), rs)


def test_quant_strided_input(dev):
    gen = torch.Generator().manual_seed(7)
    T, H, G = 33, 64, 8
    padded = _o(gen, T, 128).to(dev)
    o = padded[:, :H]
    pos, cs = _positions(gen, T).to(dev), _cos_sin().to(dev)
    q1, s1 = ops.dsv4_inv_rope_quant(o, pos, cs, G)
    q2, s2 = ops.dsv4_inv_rope_quant(o.contiguous(), pos, cs, G)
    assert torch.equal(_bytes(q1), _bytes(q2)) and torch.equal(s1, s2)
    rq, rs = O.inv_rope_quant(o.cpu(), pos.cpu(), cs.cpu(), G)
    assert torch.equal(_bytes(q1.cpu()), _bytes(rq)) and torch.equal(s1.cpu(), rs)


@pytest.mark.parametrize("T", [1, 7, 64, 100, 256])
@pytest.mark.parametrize("H,G,R", [(64, 8, 1024), (16, 2, 1024), (8, 1, 1024), (16, 1, 512), (3, 3, 128), (4, 1, 256)])
def test_z_against_float64(dev, H, G, R, T):
    gen = torch.Generator().manual_seed(H * 7 + G * 131 + R + T)
    D = H // G * 512
    o, pos, cs = _o(gen, T, H), _positions(gen, T), _cos_sin()
    w, ws = _weights(gen, G, R, D)
    od, pd, cd, wd, wsd = o.to(dev), pos.to(dev), cs.to(dev), w.to(dev), ws.to(dev)
    z = ops.dsv4_o_proj(od, pd, cd, wd, wsd, G)
    assert z.shape == (T, G * R) and z.dtype == torch.bfloat16
    q, s = ops.dsv4_inv_rope_quant(od, pd, cd, G)
    _check_z(z, q, s, wd, wsd)


@pytest.mark.parametrize("T", [1, 7, 32, 256])
def test_reference_shape_calc_diff(dev, T):
    """The reference test's shape (test_einsum_end_to_end): 64 heads in 8 groups, o_lora_rank 1024, randn inputs, against
    the unquantised composition (inverse RoPE rounded to bf16, einsum over wo_a dequantised to bf16)."""
    gen = torch.Generator().manual_seed(T)
    H, G, R = 64, 8, 1024
    D = H // G * 512
    o = torch.randn(T, H, 512, generator=gen).bfloat16()
    pos, cs = torch.randint(0, MAX_POS, (T,), generator=gen), _cos_sin()
    w, ws = O.quant_weight(torch.randn(G * R, D, generator=gen))
    z = ops.dsv4_o_proj(o.to(dev), pos.to(dev), cs.to(dev), w.to(dev), ws.to(dev), G).cpu()
    o_ref = O.inv_rope(o, pos, cs).bfloat16().reshape(T, G, D)
    w_bf = (w.float() * ws.repeat_interleave(128, 0).repeat_interleave(128, 1)).bfloat16().reshape(G, R, D)
    z_ref = torch.einsum("tgd,grd->tgr", o_ref.float(), w_bf.float()).reshape(T, G * R)
    assert O.calc_diff(z, z_ref) < 1e-2


@pytest.mark.parametrize("H,G", [(64, 8), (8, 1)])
def test_batch_invariance_determinism_graph(dev, H, G):
    gen = torch.Generator().manual_seed(H)
    T, R = 64, 1024
    D = H // G * 512
    o, pos, cs = _o(gen, T, H).to(dev), _positions(gen, T).to(dev), _cos_sin().to(dev)
    w, ws = (x.to(dev) for x in _weights(gen, G, R, D))
    z = ops.dsv4_o_proj(o, pos, cs, w, ws, G)
    assert torch.equal(z, ops.dsv4_o_proj(o, pos, cs, w, ws, G))
    for t in (0, 1, 17, 63):
        assert torch.equal(ops.dsv4_o_proj(o[t:t + 1], pos[t:t + 1], cs, w, ws, G)[0], z[t]), t
    # graph capture and replay (warm-up on a side stream first, as torch.cuda.graphs requires)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.dsv4_o_proj(o, pos, cs, w, ws, G)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        zg = ops.dsv4_o_proj(o, pos, cs, w, ws, G)
    for _ in range(3):
        zg.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(zg, z)


def test_zero_tokens_write_nothing(dev):
    H, G, R = 16, 2, 256
    D = H // G * 512
    lib = L.lib()
    stream = torch.cuda.current_stream().cuda_stream
    o = torch.zeros(1, H, 512, dtype=torch.bfloat16, device=dev)
    pos = torch.zeros(1, dtype=torch.int64, device=dev)
    cs = _cos_sin().to(dev)
    q = torch.full((G * D,), 0x5A, dtype=torch.uint8, device=dev)
    s = torch.full((G * D // 128,), 3.0, device=dev)
    L.check(lib.b200_dsv4_inv_rope_quant(stream, o.data_ptr(), H * 512, pos.data_ptr(), cs.data_ptr(), MAX_POS, 0, H, G,
                                         q.data_ptr(), s.data_ptr()), "inv_rope_quant T=0")
    w = torch.zeros(G * R, D, dtype=torch.uint8, device=dev)
    ws = torch.ones(G * R // 128, D // 128, device=dev)
    z = torch.full((G * R,), 7.0, dtype=torch.bfloat16, device=dev)
    L.check(lib.b200_dsv4_wo_a(stream, q.data_ptr(), s.data_ptr(), w.data_ptr(), ws.data_ptr(), 0, G, H // G, R, None, 0,
                               z.data_ptr()), "wo_a T=0")
    torch.cuda.synchronize()
    assert (q == 0x5A).all() and (s == 3.0).all() and (z == 7.0).all()
    assert lib.b200_dsv4_wo_a_workspace_bytes(0, G, H // G, R) == 0
    e = ops.dsv4_o_proj(o[:0], pos[:0], cs, w.view(torch.float8_e4m3fn), ws, G)
    assert e.shape == (0, G * R)


def test_chain_after_sparse_decode(dev):
    """ops.dsv4_sparse_decode's output, head-sliced from a padded q like the reference's o_padded[:, :n_local_heads], into
    ops.dsv4_o_proj, against the oracle composition."""
    gen = torch.Generator().manual_seed(5)
    T, H, G, R, bs, blocks, topk = 6, 16, 2, 512, 64, 4, 96
    D = H // G * 512
    q = (torch.randn(T, 64, 512, generator=gen)).bfloat16()
    cache = V4.pack((torch.randn(blocks * bs, 512, generator=gen) * 0.5).bfloat16(), bs, num_blocks=blocks)
    idx = torch.randint(0, blocks * bs, (T, topk), generator=gen, dtype=torch.int32)
    lens = torch.randint(1, topk + 1, (T,), generator=gen, dtype=torch.int32)
    scale = 512 ** -0.5
    out = ops.dsv4_sparse_decode(q.to(dev), cache.to(dev), idx.to(dev), lens.to(dev), scale)
    o = out[:, :H]
    pos, cs = _positions(gen, T), _cos_sin()
    w, ws = _weights(gen, G, R, D)
    z = ops.dsv4_o_proj(o, pos.to(dev), cs.to(dev), w.to(dev), ws.to(dev), G).cpu()
    # the projection on the kernel's attention output: the float64 GEMM bound
    q8, s8 = O.inv_rope_quant(o.cpu(), pos, cs, G)
    _check_z(z, q8, s8, w, ws)
    # the whole chain against the float64 attention oracle
    o64 = V4.decode(q, cache, idx, lens, scale)[:, :H]
    q64, s64 = O.inv_rope_quant(o64.bfloat16(), pos, cs, G)
    z64, _ = O.wo_a(q64, s64, w, ws)
    assert O.calc_diff(z, z64) < 1e-3
