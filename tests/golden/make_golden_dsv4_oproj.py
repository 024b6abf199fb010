"""Golden fixture for the DeepSeek-V4 attention output projection (tests/dsv4_oproj_oracle.py; ops.dsv4_inv_rope_quant,
ops.dsv4_o_proj).

Everything stored is computed by the reference's own code, read from its files with `ast` and run on the CPU:
  interp  _fused_inv_rope_fp8_quant_per_head (vllm/models/deepseek_v4/common/ops/fused_inv_rope_fp8_quant.py), the SM90
          path (TMA_ALIGNED_SCALES=False, USE_GDC=False), run by Triton's interpreter (TRITON_INTERPRET=1).  The
          interpreter's fp32 -> e4m3 cast is not the hardware's (make_golden_dsv4_sparse.py explains how), so its bytes
          are kept as `q_interp` / `s_interp` and the hardware's bytes come from the next item.
  q, s    the reference test's reference_inv_rope_fp8_quant with rotate_gptj and _ref_ue8m0_quant_block
          (tests/kernels/test_fused_inv_rope_fp8_quant.py:115-248): the kernel's statements in torch, with torch's e4m3
          cast.  The script checks that the interpreter's scales equal these everywhere and reports where its bytes agree.
  z       for the GEMM case: the reference test's reference_inv_rope (bf16 output), the weights expanded by
          _expand_2d_block_scales and _decode_e8m0_scales and dequantised to bf16 once, and the einsum "tgd,grd->tgr"
          of rocm_inv_rope_einsum (vllm/v1/attention/ops/rocm_aiter_mla_sparse.py:939-999): the unquantised z.

Needs the reference tree; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_dsv4_oproj.py [out.pt]

Cases (T 5, positions spread over a 4096-position f32 table):
  quant   G 2, 8 heads per group (D 4096).  Block 0 of head 0 has absmax 3.5, so absmax * (1 / 448) is exactly 2^-7;
          block 1 of head 0 has absmax 3.515625, the next bf16 above it (scale 2^-6); head 1 is all zero (the 1e-10
          clamp, scale 2^-42); head 2 of token 1 holds values around 1e37 and one of 448 * 2^118 (1.49e38, code 448,
          the e4m3 maximum) in its NoPE dims and values around 2^100 in its RoPE dims (no overflow in the rotation); the other heads are randn over four decades of magnitude.
  gemm    G 2, 2 heads per group (D 1024), o_lora_rank 256: o, e4m3 weights [512, 1024] with power-of-two block scales
          [4, 8], the quantised operands and the unquantised z.
Goes to tests/golden/golden_dsv4_oproj.pt.  Nothing here is imported by the product.
"""
import ast
import math
import os
import sys

os.environ["TRITON_INTERPRET"] = "1"   # before triton is imported: its kernels then run on CPU tensors

import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_dsv4_oproj.pt")
KERNEL_FILE = os.path.join("vllm", "models", "deepseek_v4", "common", "ops", "fused_inv_rope_fp8_quant.py")
TEST_FILE = os.path.join("tests", "kernels", "test_fused_inv_rope_fp8_quant.py")
ROCM_FILE = os.path.join("vllm", "v1", "attention", "ops", "rocm_aiter_mla_sparse.py")
MAX_POS = 4096
TEST_CONSTANTS = {"HEAD_DIM", "NOPE_DIM", "ROPE_DIM", "QUANT_GROUP_SIZE", "FP8_MAX", "FP8_DTYPE", "EPS"}


def _functions(rel, names, ns, constants=()):
    path = next((os.path.join(p, rel) for p in sys.path if p and os.path.isfile(os.path.join(p, rel))), None)
    if path is None:
        raise SystemExit(f"{rel} not found on PYTHONPATH: put the reference tree there")
    tree = ast.parse(open(path).read(), filename=path)
    consts = [n for n in tree.body if isinstance(n, ast.Assign) and any(getattr(t, "id", None) in constants
                                                                       for t in n.targets)]
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(fns) == len(names), (rel, names)
    exec(compile(ast.Module(body=consts + fns, type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in names]


def _reference():
    import triton
    import triton.language as tl
    ns = dict(torch=torch, triton=triton, tl=tl, math=math)
    (kernel,) = _functions(KERNEL_FILE, ["_fused_inv_rope_fp8_quant_per_head"], ns)
    tns = dict(torch=torch)
    _, _, quant, inv_rope = _functions(TEST_FILE, ["rotate_gptj", "_ref_ue8m0_quant_block", "reference_inv_rope_fp8_quant",
                                                  "reference_inv_rope"], tns, TEST_CONSTANTS)
    rns = dict(torch=torch, math=math)
    _, expand = _functions(ROCM_FILE, ["_decode_e8m0_scales", "_expand_2d_block_scales"], rns)
    return kernel, quant, inv_rope, expand


def _cos_sin():
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(MAX_POS, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


def _interp(kernel, o, pos, cs, G, hpg):
    """The Triton kernel under the interpreter, launched as _fused_inv_rope_fp8_quant_kernel_impl launches it on SM90."""
    T, H, _ = o.shape
    d, S = hpg * 512, hpg * 4
    Ta = (T + 3) // 4 * 4                    # get_tma_aligned_size(T, 4) for f32 scales
    fp8 = torch.zeros(G, T, d, dtype=torch.float8_e4m3fn)
    sc = torch.zeros(G * S * Ta, dtype=torch.float32).as_strided((G, T, S), (S * Ta, 1, Ta))
    kernel[(Ta, H)](o, pos, cs, fp8, sc, T, heads_per_group=hpg, o_stride_token=o.stride(0), o_stride_head=o.stride(1),
                    cache_stride_pos=cs.stride(0), fp8_stride_group=fp8.stride(0), fp8_stride_token=fp8.stride(1),
                    scale_stride_group=sc.stride(0), scale_stride_k=sc.stride(2), fp8_max=448.0, eps=1e-10,
                    QUANT_GROUP_SIZE=128, CHUNKS_PER_HEAD=4, ROPE_START=64, HALF_ROPE=32, TMA_ALIGNED_SCALES=False,
                    USE_GDC=False, launch_pdl=False)
    return fp8.transpose(0, 1), sc.transpose(0, 1)


def _quant_case(ref, gen, G, hpg, special):
    kernel, quant, _, _ = ref
    T, H = 5, G * hpg
    o = torch.randn(T, H, 512, generator=gen) * torch.logspace(-2, 2, H)[None, :, None]
    if special:
        o[0, 0, :128] = torch.rand(128, generator=gen) * 3.0
        o[0, 0, 3] = 3.5                              # block 0: absmax * (1 / 448) = 2^-7 exactly
        o[0, 0, 128:256] = torch.rand(128, generator=gen) * 3.0
        o[0, 0, 130] = -3.515625                      # block 1: the next bf16 above 3.5
        o[:, 1] = 0.0                                 # all-zero head
        o[1, 2, :448] = torch.randn(448, generator=gen) * 1e37
        o[1, 2, 7] = 448.0 * 2.0 ** 118                # 1.49e38: code 448, the e4m3 maximum
        o[1, 2, 448:] = torch.randn(64, generator=gen) * 2.0 ** 100
    o = o.bfloat16()
    pos = torch.tensor([0, 1, 517, 2048, MAX_POS - 1])
    cs = _cos_sin()
    q, s = quant(o, pos, cs, G, hpg)
    qi, si = _interp(kernel, o, pos, cs, G, hpg)
    assert torch.equal(si, s), "the interpreter's scales differ from the reference statement"
    same = (qi.contiguous().view(torch.uint8) == q.contiguous().view(torch.uint8))
    print(f"G {G} hpg {hpg}: interpreter bytes equal to the reference statement on {int(same.sum())} of {same.numel()}")
    if special:
        assert float(s[0, 0, 0]) == 2.0 ** -7 and float(s[0, 0, 1]) == 2.0 ** -6 and float(s[0, 0, 4]) == 2.0 ** -42
        assert float(q[1, 0, 2 * 512 + 7].float()) == 448.0
    return dict(o=o, positions=pos, n_groups=G, q=q.contiguous().view(torch.uint8), s=s.contiguous(),
                q_interp=qi.contiguous().view(torch.uint8), s_interp=si.contiguous())


def _gemm_case(ref, gen):
    _, _, inv_rope, expand = ref
    G, hpg, R = 2, 2, 256
    case = _quant_case(ref, gen, G, hpg, special=False)
    T, D = case["o"].shape[0], hpg * 512
    w = (torch.randn(G * R, D, generator=gen) * 30).clamp(-448, 448).to(torch.float8_e4m3fn)
    ws = torch.exp2(torch.randint(-12, -4, (G * R // 128, D // 128), generator=gen).float())
    o_ref = inv_rope(case["o"], case["positions"], _cos_sin()).view(T, G, D)
    cached = (w.float().view(G, R, D) * expand(ws.view(G, R // 128, D // 128), R, D)).to(torch.bfloat16)
    z = torch.einsum("tgd,grd->tgr", o_ref, cached)
    case.update(R=R, w=w.view(torch.uint8), w_scale=ws, z=z.reshape(T, G * R))
    return case


def main(out_path: str = OUT):
    ref = _reference()
    gen = torch.Generator().manual_seed(0)
    torch.save(dict(cos_sin_positions=MAX_POS, quant=_quant_case(ref, gen, 2, 8, special=True),
                    gemm=_gemm_case(ref, gen)), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
