"""Golden fixture for the lightning indexer (tests/indexer_oracle.py, ops.indexer_*).

Every expected value is computed at generation time by the reference's own pure-torch functions, read from the reference
files with `ast` and executed here; nothing of their code is stored:
  fp8_paged_mqa_logits_torch    vllm/v1/attention/ops/rocm_aiter_mla_sparse.py:264-363, both branches: next_n == 1 (the
                                block cache layout) and next_n > 1;
  kv_cache_cast_to_fp8,         tests/kernels/attention/test_deepgemm_attention.py:21-50: the block-layout fp8 cache
  per_custom_dims_cast_to_fp8   (scale = amax / 448, no ue8m0) and the per-row ue8m0 cast;
  torch.topk                    the reference top-k tests' comparison.
Stand-ins: `current_platform` is an object whose fp8_dtype() returns torch.float8_e4m3fn; `cdiv` and `_ceil_to_ue8m0`
(vllm/utils/math_utils.py, vllm/utils/deep_gemm.py:644-645) are given to the functions as ceil division and
pow(2, ceil(log2(|x|))); the `from vllm.utils.math_utils import cdiv` statement inside fp8_paged_mqa_logits_torch is
dropped for that.  The functions use their inputs' device, so no "cuda" -> "cpu" rewrite is needed.
The next_n > 1 branch slices each row as [128 value bytes | 4 scale bytes] (kv_cache[..., :dim], kv_cache[..., dim:]), not
the block layout: its input is the same cache with each row's scale moved beside its values, a byte rearrangement done
here.  Inputs follow the reference test (torch.randn q, kv and fp32 weights; q cast straight to e4m3).

Cases (batch, next_n, heads, page, seq_lens):
  logits_q1   4, 1, 64, 16, [0, 1, 37, 100]  (an empty request, one key, lengths not a multiple of the page)
  logits_q2   2, 2, 32, 64, [70, 130]
  logits_q3   2, 3, 32, 16, [2, 45]         (a request shorter than next_n)
  topk        torch.topk(k = 8) over [0, row_end) of every row of the three logits cases
  kquant      64 rows of bf16 k: kv_cache_cast_to_fp8 (no ue8m0) and per_custom_dims_cast_to_fp8(ue8m0 = True)

Needs the reference tree on PYTHONPATH; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_indexer.py [out.pt]
Goes to tests/golden/golden_indexer.pt.  Nothing here is imported by the product.
"""
import ast
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_indexer.pt")
LOGITS_FILE = os.path.join("vllm", "v1", "attention", "ops", "rocm_aiter_mla_sparse.py")
TEST_FILE = os.path.join("tests", "kernels", "attention", "test_deepgemm_attention.py")
CASES = (("logits_q1", 4, 1, 64, 16, [0, 1, 37, 100]), ("logits_q2", 2, 2, 32, 64, [70, 130]),
         ("logits_q3", 2, 3, 32, 16, [2, 45]))
TOPK = 8


class _Platform:
    @staticmethod
    def fp8_dtype():
        return torch.float8_e4m3fn


def _cdiv(a, b):
    return -(a // -b)


def _ceil_to_ue8m0(x):
    return torch.pow(2.0, torch.ceil(torch.log2(x.abs())))


class _DropImports(ast.NodeTransformer):
    def visit_ImportFrom(self, node):
        return None


def _load(rel, names):
    path = next((os.path.join(p, rel) for p in sys.path if p and os.path.isfile(os.path.join(p, rel))), None)
    if path is None:
        raise SystemExit(f"{rel} not found on PYTHONPATH: put the reference tree there")
    tree = ast.parse(open(path).read(), filename=path)
    fns = [_DropImports().visit(n) for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    ns = dict(torch=torch, F=torch.nn.functional, current_platform=_Platform(), cdiv=_cdiv, _ceil_to_ue8m0=_ceil_to_ue8m0)
    exec(compile(ast.fix_missing_locations(ast.Module(body=fns, type_ignores=[])), path, "exec"), ns)
    return [ns[n] for n in names]


def _per_row_layout(cache_block):
    """[nb, bs, 1, 132] block layout (bs x 128 values, then bs scales) -> [nb, bs, 1, 132] rows of [128 values | scale]."""
    nb, bs = cache_block.shape[:2]
    flat = cache_block.reshape(nb, bs * 132)
    vals = flat[:, :bs * 128].reshape(nb, bs, 128)
    sc = flat[:, bs * 128:].reshape(nb, bs, 4)
    return torch.cat([vals, sc], dim=-1).reshape(nb, bs, 1, 132).contiguous()


def main(out_path: str = OUT):
    (logits_ref,) = _load(LOGITS_FILE, ["fp8_paged_mqa_logits_torch"])
    kv_cast, row_cast = _load(TEST_FILE, ["kv_cache_cast_to_fp8", "per_custom_dims_cast_to_fp8"])
    gen = torch.Generator().manual_seed(0)
    res = {}
    for name, B, Q, H, page, lens in CASES:
        npg = max(1, -(-max(lens) // page))
        nb = B * npg + 3
        q = torch.randn(B, Q, H, 128, generator=gen).bfloat16()
        kv = torch.randn(nb, page, 1, 128, generator=gen).bfloat16()
        w = torch.randn(B * Q, H, generator=gen)
        bt = torch.randperm(nb, generator=gen)[:B * npg].reshape(B, npg).int()
        sl = torch.tensor(lens, dtype=torch.int32)
        q8 = q.to(torch.float8_e4m3fn)
        cache = kv_cast(kv)                                           # uint8 [nb, page, 1, 132], block layout
        width = npg * page
        if Q == 1:
            lg = logits_ref(q8, cache, w, sl, bt, width)
        else:
            lg = logits_ref(q8, _per_row_layout(cache), w, sl, bt, width)
        res[name] = dict(q_fp8=q8.reshape(B * Q, H, 128).contiguous().view(torch.uint8), weights=w,
                         k_cache=cache.reshape(nb, page, 132).contiguous(), seq_lens=sl, page_table=bt, q_len=Q,
                         logits=lg)
    tk = {}
    for name, B, Q, _, _, lens in CASES:
        lg = res[name]["logits"]
        rows = []
        for r in range(B * Q):
            end = max(0, lens[r // Q] - Q + r % Q + 1)
            k = min(TOPK, end)
            rows.append(torch.topk(lg[r, :end], k).indices.int() if k else torch.zeros(0, dtype=torch.int32))
        tk[name] = rows
    k = (torch.randn(64, 128, generator=gen) * torch.logspace(-3, 2, 64)[:, None]).bfloat16()
    k[5] = 0
    cache1 = kv_cast(k.reshape(1, 64, 1, 128))
    v8, sf = row_cast(k, (0,), True)
    res["topk"] = dict(k=TOPK, indices=tk)
    res["kquant"] = dict(k=k, plain_cache=cache1.reshape(1, 64, 132),
                         ue8m0_values=v8.view(torch.uint8), ue8m0_scales=sf.float())
    torch.save(res, out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
