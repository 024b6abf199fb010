"""Golden fixture for DeepSeek-V4 sparse decode and its cache insert (tests/dsv4_sparse_oracle.py, ops.dsv4_sparse_decode,
ops.dsv4_qnorm_rope_kv_insert).

Everything stored is computed by the reference's own code, read from its files with `ast` and executed here:
  packer   quantize_and_insert_k_kernel (vllm/models/deepseek_v4/common/ops/cache_utils.py:37-160), the Triton kernel the
           reference test's _pack_fp8_ds_mla_cache calls, run on the CPU by Triton's interpreter (TRITON_INTERPRET=1); its
           e4m3 bytes are re-encoded with torch's round-to-nearest-even cast (see packer: the interpreter's cast differs from
           the hardware's);
  reader   _read_fp8_ds_mla_cache (tests/kernels/attention/test_rocm_triton_attn_dsv4.py:125-147);
  decode   _ref_sparse_decode_ragged (same file :150-190), with and without attn_sink, and _ref_sparse_prefill_ragged (:61-88)
           for a token without keys (the decode reference cannot stack an empty key list);
  insert   make_cos_sin_cache, apply_rope_gptj_last_k, rmsnorm_no_weight, _ue8m0_per_block_scales
           (tests/kernels/test_fused_deepseek_v4_qnorm_rope_kv_insert.py:51-124, 285-296), and the packer on the roped kv, as
           that test's KV-path comparison does.

Needs the reference tree; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_dsv4_sparse.py [out.pt]

Cases (all seeded):
  pack     40 tokens, one block group scaled below the 1e-4 clamp and one near the e4m3 limit, into slots of a 3-block
           cache of block size 16 (four tokens with slot -1); the packed bytes and the reader's row of every written slot.
  decode   a main cache (block size 16, 64 tokens) and an extra cache (block size 16, 128 tokens), packed by the reference;
           index rows with -1 and out-of-range entries anywhere, lengths shorter than the rows.  The reference reader takes one
           block size for both caches, so both use 16.  (Hq, T, extra, sink):
             (20, 4, no, no)    a head count that does not divide 128; token 1 has a single valid key, token 3 none;
             (16, 2, yes, yes)  SWA + compressed with a sink;
             (64, 2, yes, no)   the V4-Flash head count; token 1 has no valid key.
  insert   3 tokens, 5 heads, positions 0, 1000 and 4095 of a 4096-position cos|sin cache (only those rows stored),
           eps 1e-6, slots [5, -1, 2] of a 2-block cache of block size 4.
Goes to tests/golden/golden_dsv4_sparse.pt.  Nothing here is imported by the product.
"""
import ast
import os
import sys

os.environ["TRITON_INTERPRET"] = "1"   # before triton is imported: its kernels then run on CPU tensors

import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_dsv4_sparse.pt")
PACK_FILE = os.path.join("vllm", "models", "deepseek_v4", "common", "ops", "cache_utils.py")
DEC_FILE = os.path.join("tests", "kernels", "attention", "test_rocm_triton_attn_dsv4.py")
INS_FILE = os.path.join("tests", "kernels", "test_fused_deepseek_v4_qnorm_rope_kv_insert.py")
SCALE = 512 ** -0.5
DEC_CASES = ((20, 4, False, False), (16, 2, True, True), (64, 2, True, False))


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
    ns = dict(torch=torch, triton=triton, tl=tl, NOPE_HEAD_DIM=448, ROPE_HEAD_DIM=64, HEAD_DIM=512, NOPE_DIM=448,
              ROPE_DIM=64, FP8_MAX=448.0)
    (kern,) = _functions(PACK_FILE, ["quantize_and_insert_k_kernel"], ns)

    def packer(kv, cache, slots, block_size):   # quantize_and_insert_k_cache's launch (cache_utils.py:162-226), OCP e4m3
        flat = cache.view(cache.shape[0], -1)
        kern[(slots.numel(),)](kv, slots.long(), flat, slots.numel(), input_dim=512, fp8_dim=448, bf16_dim=64, scale_dim=8,
                               quant_block=64, cache_block_size=block_size, token_data_size=576,
                               block_stride=flat.stride(0), fp8_max=448.0, n_quant_blocks=8, use_fnuz=False)
        # The interpreter's fp32 -> e4m3 cast is not the hardware's: it rounds ties away from zero and loses the carry of a
        # mantissa that rounds up into the next exponent (-31.625 -> -16).  The kernel's bytes are
        # x_clamped.to(tl.float8e4nv), a round-to-nearest-even cast, so the NoPE bytes are re-encoded from the kernel's own
        # scale bytes with torch's cast; addressing, scale bytes, pad byte and rope bytes are the interpreter's.
        for i, s in enumerate(slots.tolist()):
            if s < 0:
                continue
            blk, pos = flat[s // block_size], s % block_size
            e = blk[block_size * 576 + pos * 8:][:7].float()
            x = kv[i, :448].float() / torch.pow(2.0, e - 127.0).repeat_interleave(64)
            blk[pos * 576:pos * 576 + 448] = x.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)
        return cache

    read, dec, pre = _functions(DEC_FILE, ["_read_fp8_ds_mla_cache", "_ref_sparse_decode_ragged",
                                           "_ref_sparse_prefill_ragged"], ns)
    ins = _functions(INS_FILE, ["make_cos_sin_cache", "apply_rope_gptj_last_k", "rmsnorm_no_weight",
                                "_ue8m0_per_block_scales"], ns)
    return packer, read, dec, pre, ins


def _index_row(gen, width, n_valid, n_slots):
    """width entries: n_valid distinct slots, the rest -1 or out of range (>= n_slots), all in random order."""
    row = torch.full((width,), -1, dtype=torch.int32)
    row[torch.randperm(width, generator=gen)[:width // 4]] = n_slots + 7
    row[torch.randperm(width, generator=gen)[:n_valid]] = torch.randperm(n_slots, generator=gen)[:n_valid].int()
    return row


def _lists(row, n, n_slots):
    return [int(s) for s in row[:n] if 0 <= int(s) < n_slots]


def main(out_path: str = OUT):
    packer, read, dec, pre, (make_cs, rope, rmsnorm, ue8m0_scales) = _reference()
    gen = torch.Generator().manual_seed(0)

    # ---- pack / read
    kv = torch.randn(40, 512, generator=gen).bfloat16()
    kv[3, 64:128] *= 1e-6          # below the 1e-4 clamp
    kv[7, :64] *= 100.0            # large values
    slots = torch.randperm(48, generator=gen)[:40]
    slots[[2, 11, 25, 38]] = -1
    pcache = packer(kv, torch.zeros(3, 16, 584, dtype=torch.uint8), slots, 16)
    ok = slots[slots >= 0]
    prows = torch.stack([read(pcache, int(s), 16, False) for s in ok])
    pack = dict(kv=kv, slots=slots.int(), block_size=16, cache=pcache, read_slots=ok.int(), read_rows=prows)

    # ---- decode
    main_kv = torch.randn(64, 512, generator=gen).bfloat16()
    extra_kv = torch.randn(128, 512, generator=gen).bfloat16()
    mc = packer(main_kv, torch.zeros(4, 16, 584, dtype=torch.uint8), torch.arange(64), 16)
    ec = packer(extra_kv, torch.zeros(8, 16, 584, dtype=torch.uint8), torch.arange(128), 16)
    decode = []
    for hq, T, extra, with_sink in DEC_CASES:
        q = torch.randn(T, hq, 512, generator=gen).bfloat16()
        sink = (torch.randn(hq, generator=gen) * 2).float() if with_sink else None
        si = torch.stack([_index_row(gen, 96, 40, 64) for _ in range(T)])
        sl = torch.randint(48, 97, (T,), generator=gen, dtype=torch.int32)
        ei = torch.stack([_index_row(gen, 160, 90, 128) for _ in range(T)]) if extra else None
        el = torch.randint(100, 161, (T,), generator=gen, dtype=torch.int32) if extra else None
        if hq == 20:               # token 1: one valid key; token 3: none
            si[1] = -1
            si[1, 5] = 17
            sl[3] = 0
        if hq == 64:               # token 1: no valid key in either list
            si[1], ei[1] = -1, 64 + 128
        out = torch.zeros(T, hq, 512, dtype=torch.bfloat16)
        for t in range(T):
            mrows = _lists(si[t], int(sl[t]), 64)
            erows = _lists(ei[t], int(el[t]), 128) if extra else []
            if mrows or erows:
                out[t] = dec(q[t:t + 1], mc, [mrows], SCALE, sink, 16, ec if extra else None, [erows] if extra else None)[0]
            else:
                out[t] = pre(q[t:t + 1], torch.zeros(1, 512), [[]], SCALE, sink)[0]
        decode.append(dict(num_heads=hq, q=q, attn_sink=sink, swa_indices=si, swa_lens=sl, extra_indices=ei, extra_lens=el,
                           out=out))

    # ---- insert
    T, hq, eps = 3, 5, 1e-6
    positions = torch.tensor([0, 1000, 4095])
    cs = make_cs(4096, 64, torch.float32, "cpu")[positions]
    pos_local = torch.arange(T)
    q = torch.randn(T, hq, 512, generator=gen).bfloat16()
    ikv = torch.randn(T, 512, generator=gen).bfloat16()
    q_ref = rope(rmsnorm(q, eps), pos_local, cs)
    kv_ref = rope(ikv, pos_local, cs)
    islots = torch.tensor([5, -1, 2])
    icache = packer(kv_ref, torch.zeros(2, 4, 584, dtype=torch.uint8), islots, 4)
    insert = dict(q=q, kv=ikv, positions=positions, cos_sin_rows=cs, eps=eps, slots=islots, block_size=4, q_ref=q_ref,
                  kv_ref=kv_ref, cache=icache, scales=ue8m0_scales(kv_ref[:, :448].float(), 64))

    torch.save(dict(scale=SCALE, pack=pack, main_cache=mc, extra_cache=ec, decode=decode, insert=insert), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
