"""Golden fixture for sparse MLA decode (tests/mla_sparse_oracle.py, ops.mla_decode_sparse).

Two parts, both computed from the reference at generation time:
  conversion  the reference test's own _triton_convert_reference_impl (tests/v1/attention/test_sparse_mla_backends.py:557-605,
              the Python statement of triton_convert_req_index_to_global_index), read from the reference file with `ast` and
              executed here; nothing of it is stored.  Inputs follow the reference's decode-only test (:614-661): random
              request ids and block table, indices with -1 runs and runs one page past the table.
  attention   the reference test's sparse SDPA (:386-412): per query token, gather the keys its valid indices name, then
              torch.nn.functional.scaled_dot_product_attention over all heads, fp32 on the CPU, and the v up-projection
              einsum("qnl,lnv->qnv", out, W_UV).  SDPA has no page table: indices are positions in the request's key list.

Needs the reference tree on PYTHONPATH; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_mla_sparse.py [out.pt]

Inputs are seeded uniform [0, 1) bf16 values like the reference test's torch.rand (stored as bf16, computed in fp32).  One
key pool [320, 576] is shared by the attention cases (the request's keys are its first rows) and the queries of every case
are the first rows of one pool of 576-dim query vectors.  W_UV is mla_sparse_oracle.golden_w_uv(Hq), a fixed pattern, so the
file stays under 1 MB; for the same reason the latent output keeps every fourth value dim (out_dims = 0, 4, ..., 508), and
out_v = latent x W_UV is stored in full.  Attention cases (Hq, S keys, index rows):
  128, 300, 1 token, topk 2048   the DeepSeek-V3.2 shape: 200 distinct keys in random order with interior -1 runs, the rest -1;
  16, 300, 3 tokens, topk 256    a TP8 shard, three tokens of one request (draft tokens), each with its own key set;
  20, 160, 2 tokens, topk 128    a head count that does not divide 128; one token has a single valid entry.
Conversion cases (page, topk): (16, 128), (64, 256), (64, 2048).  Goes to tests/golden/golden_mla_sparse.pt.
Nothing here is imported by the product.
"""
import ast
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import mla_sparse_oracle as SP  # noqa: E402

OUT = os.path.join(HERE, "golden_mla_sparse.pt")
REF_FILE = os.path.join("tests", "v1", "attention", "test_sparse_mla_backends.py")
POOL_KEYS = 320
OUT_DIMS = torch.arange(0, 512, 4)
# (Hq, S, T, topk, valid entries per token)
ATTN_CASES = ((128, 300, 1, 2048, [200]), (16, 300, 3, 256, [180, 97, 256]), (20, 160, 2, 128, [1, 90]))
CONV_CASES = ((16, 128), (64, 256), (64, 2048))


def _reference_convert():
    path = next((os.path.join(p, REF_FILE) for p in sys.path if p and os.path.isfile(os.path.join(p, REF_FILE))), None)
    if path is None:
        raise SystemExit(f"{REF_FILE} not found on PYTHONPATH: put the reference tree there")
    tree = ast.parse(open(path).read(), filename=path)
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "_triton_convert_reference_impl")
    ns = dict(torch=torch)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    return ns["_triton_convert_reference_impl"]


def _index_row(gen, S, topk, n_valid):
    """n_valid distinct key positions < S in random order, scattered over the row with -1 between them; -1 after."""
    keys = torch.randperm(S, generator=gen)[:n_valid].int()
    row = torch.full((topk,), -1, dtype=torch.int32)
    span = min(topk, n_valid + n_valid // 4 + (1 if n_valid < topk else 0))
    pos = torch.randperm(span, generator=gen)[:n_valid].sort().values
    row[pos] = keys
    return row


def main(out_path: str = OUT):
    gen = torch.Generator().manual_seed(0)
    convert = _reference_convert()
    conv = []
    for page, topk in CONV_CASES:
        T, R, max_blocks = 8, 4, 10
        req_id = torch.randint(0, R, (T,), generator=gen, dtype=torch.int32)
        bt = torch.randint(0, 100, (R, max_blocks), generator=gen, dtype=torch.int32)
        idx = torch.randint(0, page * max_blocks, (T, topk), generator=gen, dtype=torch.int32)
        idx[0, :10] = -1
        idx[3, 50:60] = -1
        idx[2, 100:110] = max_blocks * page           # one page past the table
        idx[6, topk - 20:] = max_blocks * page + 5
        idx[5, topk // 2:] = -1                       # trailing -1
        conv.append(dict(page=page, req_id=req_id, block_table=bt, indices=idx,
                         slots=convert(req_id, bt, idx, page, topk)))

    keys = torch.rand(POOL_KEYS, 576, generator=gen).bfloat16()
    q_pool = torch.rand(max(hq * T for hq, _, T, _, _ in ATTN_CASES), 576, generator=gen).bfloat16()
    scale = 1.0 / math.sqrt(576)
    attn = []
    for hq, S, T, topk, n_valid in ATTN_CASES:
        w_uv = SP.golden_w_uv(hq).float()
        q = q_pool[:T * hq].reshape(T, hq, 576).float()
        k_mqa = keys[:S].float()
        v_mqa = k_mqa[:, :512]
        rows = torch.stack([_index_row(gen, S, topk, n) for n in n_valid])
        out = torch.empty(T, hq, 512)
        out_v = torch.empty(T, hq, 128)
        for t in range(T):
            valid = rows[t][rows[t] >= 0].long()
            k_sparse = k_mqa[valid].unsqueeze(1).expand(-1, hq, -1)
            v_sparse = v_mqa[valid].unsqueeze(1).expand(-1, hq, -1)
            o = torch.nn.functional.scaled_dot_product_attention(
                q[t:t + 1].unsqueeze(0).transpose(1, 2), k_sparse.unsqueeze(0).transpose(1, 2),
                v_sparse.unsqueeze(0).transpose(1, 2), scale=scale).transpose(1, 2).squeeze(0)   # [1, hq, 512]
            out[t] = o[0]
            out_v[t] = torch.einsum("qnl,lnv->qnv", o, w_uv.transpose(0, 1))[0]   # the reference's W_UV is [512, Hq, 128]
        attn.append(dict(num_heads=hq, kv_len=S, topk_indices=rows, q_rows=T * hq,
                         out=out[..., OUT_DIMS].contiguous(), out_v=out_v))
    torch.save(dict(scale=scale, keys=keys, q_pool=q_pool, out_dims=OUT_DIMS, attention=attn, conversion=conv), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
