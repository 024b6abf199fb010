"""Golden fixture for the DeepSeek-V4 C4A indexer's q side and V4's decode key lists (tests/dsv4_indexer_oracle.py;
ops.dsv4_indexer_q_quant, dsv4_indexer_decode, dsv4_swa_indices, dsv4_c128a_indices, dsv4_global_topk_indices,
dsv4_compressed_slot_mapping).

Everything stored is computed by the reference's own Triton kernels, read from its files with `ast` and run on the CPU by
Triton's interpreter (TRITON_INTERPRET=1):
  q       _fused_indexer_q_rope_quant_kernel with _get_cos_sin (vllm/models/deepseek_v4/common/ops/fused_indexer_q.py:14-27,
          70-176), fp8 path.  The interpreter's casts are not the hardware's: fp32 -> bf16 truncates where the hardware
          rounds to nearest even, which moves rotated values and sometimes a head's amax and scale, and fp32 -> e4m3
          differs as make_golden_dsv4_sparse.py explains.  So the e4m3 bytes and weights_out of every head are re-encoded
          from the kernel's own statements evaluated by torch (the same fp32 products and sums, a round-to-nearest-even
          bf16 cast, tl.div_rn as an exact quotient, exp2(ceil(log2(.))) and torch's e4m3 cast); weights_out as the kernel
          computes it is kept as `w_interp`, and the script checks that it equals the re-encoded value on every head
          whose scale the truncation did not move.
  short   _fill_short_context_topk_indices (models/deepseek_v4/attention.py:72-86);
  swa     _compute_swa_indices_and_lens_kernel (v1/attention/backends/mla/sparse_swa.py:744-800);
  c128a   _build_c128a_topk_metadata_kernel, decode tokens only (models/deepseek_v4/sparse_mla.py:353-408);
  global  _compute_global_topk_indices_and_lens_kernel (models/deepseek_v4/common/ops/cache_utils.py:477-525);
  slots   _compressed_slot_mapping_kernel (v1/attention/backends/mla/compressor_utils.py:8-50), output filled with -1
          first as get_compressed_slot_mapping does.
The lists of tokens with is_valid = 0 are the reference's to leave: the SWA kernel writes only their length, the others
fill their rows; the tests compare lengths for those tokens and rows for the others.  No case reaches past a block
table's width (the reference would read the next row there).

Needs the reference tree; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_dsv4_indexer.py [out.pt]

Cases:
  q       T 5, H 64, weights a column slice of a wider matrix, positions 0..300 of a 320-position f32 table;
          head (0, 0) has amax exactly 3.5 = 448 * 2^-7 (the scale where max(amax, 1e-4) / 448 and the V3.2 kernel's
          amax * (1 / 448) part), head (1, 1) is all zero (the 1e-4 clamp), head (2, 2) has values up to 2^20.
  lists   4 requests as (seq_len, query_len): (3, 1), (9, 1), (26, 3), (40, 2) -> 7 tokens, one padded token (request 0,
          is_valid 0) appended; block tables of width 12 over 48 shuffled blocks; SWA window 8 on block size 4 (windows
          crossing blocks, p < W); ratio 4 on compressed block size 2 for C128A (width 6, below some tokens' counts) and
          the slot mapping (positions before, at and after a boundary); the global top-k over local lists with -1 padding.
  short   the same positions, ratio 4, top-k 8.
Goes to tests/golden/golden_dsv4_indexer.pt.  Nothing here is imported by the product.
"""
import ast
import math
import os
import sys

os.environ["TRITON_INTERPRET"] = "1"   # before triton is imported: its kernels then run on CPU tensors

import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_dsv4_indexer.pt")
Q_FILE = os.path.join("vllm", "models", "deepseek_v4", "common", "ops", "fused_indexer_q.py")
ATTN_FILE = os.path.join("vllm", "models", "deepseek_v4", "attention.py")
SWA_FILE = os.path.join("vllm", "v1", "attention", "backends", "mla", "sparse_swa.py")
C128_FILE = os.path.join("vllm", "models", "deepseek_v4", "sparse_mla.py")
GLOBAL_FILE = os.path.join("vllm", "models", "deepseek_v4", "common", "ops", "cache_utils.py")
SLOT_FILE = os.path.join("vllm", "v1", "attention", "backends", "mla", "compressor_utils.py")
MAX_POS = 320


def _functions(rel, names, ns):
    path = next((os.path.join(p, rel) for p in sys.path if p and os.path.isfile(os.path.join(p, rel))), None)
    if path is None:
        raise SystemExit(f"{rel} not found on PYTHONPATH: put the reference tree there")
    tree = ast.parse(open(path).read(), filename=path)
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(fns) == len(names), (rel, names)
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in names]


def _reference():
    import triton
    import triton.language as tl
    ns = dict(torch=torch, triton=triton, tl=tl, math=math)
    _, qk = _functions(Q_FILE, ["_get_cos_sin", "_fused_indexer_q_rope_quant_kernel"], ns)
    (short,) = _functions(ATTN_FILE, ["_fill_short_context_topk_indices"], ns)
    (swa,) = _functions(SWA_FILE, ["_compute_swa_indices_and_lens_kernel"], ns)
    (c128,) = _functions(C128_FILE, ["_build_c128a_topk_metadata_kernel"], ns)
    (glob,) = _functions(GLOBAL_FILE, ["_compute_global_topk_indices_and_lens_kernel"], ns)
    (slots,) = _functions(SLOT_FILE, ["_compressed_slot_mapping_kernel"], ns)
    return triton, qk, short, swa, c128, glob, slots


def _cos_sin():
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(MAX_POS, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


def _q_statement(q, w, pos, cs, softmax_scale, head_scale):
    """The kernel's statements in torch, with the hardware's casts."""
    c, s = cs[pos][:, None, :32], cs[pos][:, None, 32:]
    x = q.float()
    xe, xo = x[..., 64::2], x[..., 65::2]
    re = (xe * c - xo * s).bfloat16().float()
    ro = (xo * c + xe * s).bfloat16().float()
    amax = torch.maximum(torch.maximum(re.abs().amax(-1), ro.abs().amax(-1)), x[..., :64].abs().amax(-1))
    scale = torch.exp2(torch.ceil(torch.log2(torch.clamp(amax, min=1e-4) / 448.0)))
    xr = torch.cat((x[..., :64], torch.stack((re, ro), -1).flatten(-2)), -1)
    q8 = (xr / scale[..., None]).to(torch.float8_e4m3fn)
    wo = w.float() * scale
    wo = wo * softmax_scale
    wo = wo * head_scale
    return q8, wo, scale


def _q_case(ref, gen):
    triton, qk = ref[0], ref[1]
    T, H = 5, 64
    q = (torch.randn(T, H, 128, generator=gen) * torch.logspace(-2, 1, H)[None, :, None]).bfloat16()
    q[0, 0] = (torch.rand(128, generator=gen) * 3.0).bfloat16()
    q[0, 0, 70] = 0.0
    q[0, 0, 3] = 3.5
    q[1, 1] = 0.0
    q[2, 2, :64] = (torch.randn(64, generator=gen) * 2 ** 18).bfloat16()
    q[2, 2, 5] = 2.0 ** 20
    fused = torch.randn(T, H + 24, generator=gen).bfloat16()
    w = fused[:, 16:16 + H]
    pos = torch.tensor([0, 1, 37, 255, 300])
    cs = _cos_sin()
    ss, hs = 128 ** -0.5, H ** -0.5
    q8 = torch.zeros(T, H, 128, dtype=torch.float8_e4m3fn)
    wo = torch.zeros(T, H)
    qk[(T, H)](pos, q, q.stride(0), q.stride(1), cs, cs.stride(0), INDEX_Q_HALF_ROT_DIM=32, index_q_fp8_ptr=q8,
               index_q_fp8_stride0=q8.stride(0), index_q_fp8_stride1=q8.stride(1), INDEX_Q_HEAD_DIM=128,
               index_weights_ptr=w, index_weights_stride=w.stride(0), index_weights_softmax_scale=ss,
               index_weights_head_scale=hs, index_weights_out_ptr=wo, index_weights_out_stride=wo.stride(0))
    tq8, two, tscale = _q_statement(q, w, pos, cs, ss, hs)
    # the interpreter's scale per head, from its weights_out (exact: a power of two times w)
    same = wo == two
    print(f"q: weights_out of the interpreter equal to the torch statement on {int(same.sum())} of {T * H} heads")
    moved = ~same
    assert bool(moved.sum() <= T * H // 4), "the truncation moved too many scales: re-check the inputs"
    assert float(tscale[0, 0]) == 2.0 ** -7 and float(tscale[1, 1]) == 2.0 ** -22
    return dict(q=q, weights=fused, weights_cols=(16, 16 + H), positions=pos, softmax_scale=ss, head_scale=hs,
                q_fp8=tq8.view(torch.uint8), weights_out=two, w_interp=wo)


def _lists_case(ref, gen):
    triton, _, short, swa, c128, glob, slots = ref
    reqs = [(3, 1), (9, 1), (26, 3), (40, 2)]
    W, SWA_BS, RATIO, CBS, WIDTH, MAXB, TOPK = 8, 4, 4, 2, 6, 12, 8
    R = len(reqs)
    qsl = [0]
    for _, ql in reqs:
        qsl.append(qsl[-1] + ql)
    T = qsl[-1] + 1                                              # + one padded token
    query_start_loc = torch.tensor(qsl, dtype=torch.int32)
    seq_lens = torch.tensor([s for s, _ in reqs], dtype=torch.int32)
    token_to_req = torch.tensor([r for r, (_, ql) in enumerate(reqs) for _ in range(ql)] + [0], dtype=torch.int32)
    positions = torch.tensor([s - ql + i for s, ql in reqs for i in range(ql)] + [0], dtype=torch.int64)
    is_valid = torch.ones(T, dtype=torch.bool)
    is_valid[-1] = False
    slot_map = torch.where(is_valid, torch.arange(T), torch.full((T,), -1)).long()
    bt = torch.randperm(48, generator=gen)[:R * MAXB].reshape(R, MAXB).int()
    # SWA (decode tokens; the padded token's row is not written)
    swa_idx = torch.full((T, W), -7, dtype=torch.int32)
    swa_len = torch.full((T,), -7, dtype=torch.int32)
    swa[(T,)](swa_idx, swa_idx.stride(0), swa_len, W, query_start_loc, seq_lens, token_to_req, is_valid.int(), bt,
              bt.stride(0), SWA_BS, 0, TRITON_BLOCK_SIZE=8)
    # C128A at ratio 4 on compressed blocks of 2, width 6
    c_idx = torch.full((T, WIDTH), -7, dtype=torch.int32)
    c_len = torch.full((T,), -7, dtype=torch.int32)
    pre = torch.zeros(1, WIDTH, dtype=torch.int32)
    c128[(T,)](c_idx, c_idx.stride(0), c_len, pre, pre.stride(0), positions, RATIO, WIDTH, T, token_to_req, bt,
               bt.stride(0), CBS, slot_map, BLOCK_SIZE=8)
    # global top-k over local lists (ascending, -1 padded) of the tokens' candidates
    n = torch.div(positions + 1, RATIO, rounding_mode="floor")
    local = torch.full((T, TOPK), -1, dtype=torch.int32)
    for t in range(T):
        k = min(int(n[t]), TOPK)
        if k:
            local[t, :k] = torch.randperm(int(n[t]), generator=gen)[:k].sort().values.int()
    g_idx = torch.full((T, TOPK), -7, dtype=torch.int32)
    g_len = torch.full((T,), -7, dtype=torch.int32)
    glob[(T,)](g_idx, g_idx.stride(0), g_len, local, local.stride(0), TOPK, token_to_req, bt, bt.stride(0), CBS,
               is_valid.int(), TRITON_BLOCK_SIZE=8)
    # compressor slot mapping, per request
    sm = torch.full((T,), -1, dtype=torch.int64)
    slots[(R,)](sm, query_start_loc, seq_lens, bt, bt.stride(0), CBS, COMPRESS_RATIO=RATIO, PAD_ID=-1,
                TRITON_BLOCK_SIZE=8)
    # short context
    sc = torch.full((T, TOPK), -7, dtype=torch.int32)
    short[(T,)](sc, positions, TOP_K=TOPK, COMPRESS_RATIO=RATIO, PADDED_TOP_K=TOPK)
    return dict(positions=positions, token_to_req=token_to_req, slot_mapping=slot_map, block_table=bt, window=W,
                swa_block_size=SWA_BS, ratio=RATIO, c_block_size=CBS, width=WIDTH, topk=TOPK, swa_indices=swa_idx,
                swa_lens=swa_len, c128a_indices=c_idx, c128a_lens=c_len, local_topk=local, global_indices=g_idx,
                global_lens=g_len, kv_slot_mapping=sm, short_topk=sc)


def main(out_path: str = OUT):
    ref = _reference()
    gen = torch.Generator().manual_seed(0)
    torch.save(dict(cos_sin=_cos_sin(), q=_q_case(ref, gen), lists=_lists_case(ref, gen)), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
