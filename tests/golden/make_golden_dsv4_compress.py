"""Golden fixture for the DeepSeek-V4 KV compressor (tests/dsv4_compress_oracle.py, ops.dsv4_compress).

Everything stored is computed by the reference's own code, read from its files with `ast` and executed here:
  state     _save_partial_states_kernel (vllm/models/deepseek_v4/common/ops/save_partial_states.py:48-101);
  compress  _fused_kv_compress_norm_rope_insert_sparse_attn (D 512) and _fused_kv_compress_norm_rope_insert_indexer_attn
            (D 128) (common/ops/fused_compress_quant_cache.py:113-297, 657-828), all three Triton kernels run on the CPU
            by Triton's interpreter (TRITON_INTERPRET=1).  The interpreter's casts are not the hardware's: fp32 -> bf16
            truncates (the hardware rounds to nearest even, which moves a block's amax and so its scale) and fp32 -> e4m3
            differs as make_golden_dsv4_sparse.py explains.  So the compress kernels decide which rows are written, where,
            and the pad bytes; the values of every written row (e4m3 bytes, scales, rope bytes) are re-encoded from the
            reference test's torch statement by its own _ue8m0_reference (tests/kernels/test_compressor_kv_cache.py:55-78,
            exact quotient, per 64 NoPE dims for D 512, one block for D 128);
  rows      _reference_kv_compress_norm_rope (same file :502-580), its bf16 rows (return_full_cache).

Needs the reference tree; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_dsv4_compress.py [out.pt]

One case per shape (D, ratio): (512, 4), (512, 128), (128, 4), each with two requests whose state blocks are shuffled over
a shared pool, eps 1e-6 and a 160-position cos | sin cache.  To keep the file small, kv_score and ape values are numbers
of a narrow format, stored in it and run as fp32: bf16 at ratio 4, e4m3 at ratio 128 (whose two windows alone are 256
rows of 1024 values); the state cache starts with random bf16-valued rows (earlier calls) where a window reaches back.
  ratio 4    request 0 at positions 0..11 (the window of position 3 starts at -4), request 1 at 20..27 (its window of 23
             reads rows 16..19 written before the call); one padded token (state and cache slot -1) at a boundary
             position; one boundary token with cache slot -1; D 512: request 1's kv columns 64..127 scaled by 1e-6, so
             that its rows' second quant block falls under the 1e-4 amax clamp.
  ratio 128  request 0 at positions 0..127, request 1 at 128..255, one boundary each, and a padded token.
Stored per case: the inputs, the score half of some of the state rows the call wrote (the boundary tokens' rows and six
others), the cache after the call (zeros before) and the torch rows.
Goes to tests/golden/golden_dsv4_compress.pt.  Nothing here is imported by the product.
"""
import ast
import math
import os
import sys

os.environ["TRITON_INTERPRET"] = "1"   # before triton is imported: its kernels then run on CPU tensors

import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_dsv4_compress.pt")
STATE_FILE = os.path.join("vllm", "models", "deepseek_v4", "common", "ops", "save_partial_states.py")
COMP_FILE = os.path.join("vllm", "models", "deepseek_v4", "common", "ops", "fused_compress_quant_cache.py")
TEST_FILE = os.path.join("tests", "kernels", "test_compressor_kv_cache.py")
EPS, MAX_POS = 1e-6, 160


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
    (save,) = _functions(STATE_FILE, ["_save_partial_states_kernel"], ns)
    k512, k128 = _functions(COMP_FILE, ["_fused_kv_compress_norm_rope_insert_sparse_attn",
                                        "_fused_kv_compress_norm_rope_insert_indexer_attn"], ns)
    rows, ue8m0 = _functions(TEST_FILE, ["_reference_kv_compress_norm_rope", "_ue8m0_reference"], ns)
    return triton, save, k512, k128, rows, ue8m0


def _cos_sin():
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(MAX_POS, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


def _case(ref, gen, D, ratio):
    triton, save, k512, k128, ref_rows, ue8m0 = ref
    ovl = int(ratio == 4)
    half = (1 + ovl) * D
    sbs = 8 if ratio == 4 else 32
    if ratio == 4:
        req_pos = [(0, list(range(0, 12))), (1, list(range(20, 28)))]
        early = [(1, p) for p in range(16, 20)]                # rows written by an earlier call
    else:
        req_pos = [(0, list(range(0, 128))), (1, list(range(128, 256)))]
        early = []
    blocks_per_req = -(-max(p for _, ps in req_pos for p in ps) // sbs) + 1
    nblk = 2 * blocks_per_req + 2
    perm = torch.randperm(nblk, generator=gen).int()
    block_table = torch.stack([perm[:blocks_per_req], perm[blocks_per_req:2 * blocks_per_req]])
    # tokens of the call: both requests interleaved in position order, then a padded token
    toks = sorted([(p, r) for r, ps in req_pos for p in ps])
    req = torch.tensor([r for _, r in toks] + [0], dtype=torch.int32)
    pos = torch.tensor([p for p, _ in toks] + [ratio - 1], dtype=torch.int64)
    T = pos.numel()
    slot = torch.tensor([int(block_table[r, p // sbs]) * sbs + p % sbs for p, r in toks] + [-1], dtype=torch.int64)
    kv_score = torch.randn(T, 2 * half, generator=gen).to(torch.bfloat16 if ratio == 4 else torch.float8_e4m3fn)
    if D == 512 and ratio == 4:
        for c0 in (64, D + 64):                                  # request 1's kv columns 64..127 of both halves
            kv_score[req == 1, c0:c0 + 64] = (kv_score[req == 1, c0:c0 + 64].float() * 1e-6).bfloat16()
    ape = torch.randn(ratio, half, generator=gen).to(torch.bfloat16 if ratio == 4 else torch.float8_e4m3fn)
    state = torch.zeros(nblk, sbs, 2 * half)
    for r, p in early:
        x = torch.randn(2 * half, generator=gen)
        if D == 512:
            x[64:128] *= 1e-6
            x[D + 64:D + 128] *= 1e-6
        state[int(block_table[r, p // sbs]), p % sbs] = x.bfloat16().float()   # bf16 numbers: stored as bf16
    state_before = state.clone()
    ks = kv_score.float()
    save[(T,)](ks[:, :half], ks.stride(0), ks[:, half:], ks.stride(0), ape.float(), ape.stride(0), pos, state,
               state.stride(0), state.stride(1), slot, sbs, HEAD_SIZE=half,
               TRITON_BLOCK_SIZE=triton.next_power_of_2(half), STATE_WIDTH=half, COMPRESS_RATIO=ratio)
    # cache slots: boundary tokens get distinct shuffled rows; one boundary token gets -1
    bound = [t for t in range(T) if (int(pos[t]) + 1) % ratio == 0 and slot[t] >= 0]
    kvb, kvnb = 4, 4
    kslot = torch.full((T,), -1, dtype=torch.int64)
    kslot[bound] = torch.randperm(kvb * kvnb, generator=gen)[:len(bound)]
    if ratio == 4:
        kslot[bound[1]] = -1
    kslot[T - 1] = 5                                             # the padded token names a row: still nothing written
    w = (1.0 + 0.25 * torch.randn(D, generator=gen)).bfloat16()
    cs = _cos_sin()
    row = 584 if D == 512 else 132
    cache = torch.zeros(kvnb, kvb, row, dtype=torch.uint8)
    flat = cache.view(kvnb, -1)
    kern = k512 if D == 512 else k128
    ts, sd, qb = (576, 8, 64) if D == 512 else (128, 4, 128)
    kern[(T,)](state, state.stride(0), state.stride(1), req, pos, slot, block_table, block_table.stride(0), sbs, w, EPS,
               cs, cs.stride(0), flat, kslot, kvb, HEAD_SIZE=D, TRITON_BLOCK_SIZE=D, STATE_WIDTH=half,
               COMPRESS_RATIO=ratio, OVERLAP=ovl, ROPE_HEAD_DIM=64, FP8_MAX=448.0, QUANT_BLOCK=qb, TOKEN_STRIDE=ts,
               SCALE_DIM=sd, KV_BLOCK_STRIDE=flat.stride(0))
    # the torch statement, per request (it reads block_table[0])
    torch_rows = {}
    for r in (0, 1):
        ps = [int(pos[t]) for t in bound if int(req[t]) == r]
        out = ref_rows(state, block_table[r:r + 1], torch.tensor(ps), w, cs, ratio, ovl, rms_eps=EPS,
                       return_full_cache=True)
        for p, x in zip(ps, out):
            torch_rows[(r, p)] = x
    rows = torch.stack([torch_rows[(int(req[t]), int(pos[t]))] for t in bound])          # bf16 [n, D]
    # re-encode the values of every row the kernel wrote (see the module docstring)
    for i, t in enumerate(bound):
        s = int(kslot[t])
        if s < 0:
            continue
        blk, p = flat[s // kvb], s % kvb
        x = rows[i]
        if D == 512:
            assert blk[p * 576:p * 576 + 576].any() and int(blk[kvb * 576 + p * 8 + 7]) == 0
            q8, sc = ue8m0(x[:448].float(), 64, 448.0)
            blk[p * 576:p * 576 + 448] = q8.view(torch.uint8)
            blk[p * 576 + 448:p * 576 + 576] = x[448:].contiguous().view(torch.uint8)
            blk[kvb * 576 + p * 8:][:7] = (torch.log2(sc) + 127).to(torch.uint8)
        else:
            assert blk[p * 128:p * 128 + 128].any()
            q8, sc = ue8m0(x.float(), 128, 448.0)
            blk[p * 128:p * 128 + 128] = q8.view(torch.uint8)
            blk[kvb * 128 + p * 4:][:4] = sc.contiguous().view(torch.uint8)
    assert int((flat != 0).any(1).sum()) >= 1
    written = sorted({int(slot[t]) for t in range(T) if slot[t] >= 0})
    keep = {int(slot[t]) for t in bound} | {written[i] for i in torch.randperm(len(written), generator=gen)[:6].tolist()}
    written = sorted(keep)
    st = state.view(nblk * sbs, 2 * half)
    return dict(head_dim=D, ratio=ratio, kv_score=kv_score, ape=ape, positions=pos, slot_mapping=slot, token_to_req=req,
                block_table=block_table, state_blocks=nblk, state_block_size=sbs,
                early_slots=torch.tensor([int(block_table[r, p // sbs]) * sbs + p % sbs for r, p in early],
                                         dtype=torch.int64),
                early_rows=state_before.view(nblk * sbs, 2 * half)[[int(block_table[r, p // sbs]) * sbs + p % sbs
                                                                    for r, p in early]].bfloat16(),
                written_slots=torch.tensor(written, dtype=torch.int64), state_score=st[written, half:].clone(),
                norm_weight=w, kv_slot_mapping=kslot, cache=cache, boundary_tokens=torch.tensor(bound),
                torch_rows=rows)


def main(out_path: str = OUT):
    ref = _reference()
    gen = torch.Generator().manual_seed(0)
    cases = [_case(ref, gen, D, r) for D, r in ((512, 4), (512, 128), (128, 4))]
    torch.save(dict(eps=EPS, cos_sin=_cos_sin(), cases=cases), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
