"""Golden fixture for multi-token MLA decode (tests/mla_spec_oracle.py, ops.mla_decode(q_len_per_req=Q)): the reference's
OWN causal attention, scaled_dot_product_attention(..., is_causal=True) of tests/kernels/attention/test_flashmla.py:138-155
(mask tril(diagonal = s_k - s_q): query token i of a request with s_k keys and s_q = Q queries sees keys [0, s_k - Q + i]),
on the CPU in fp32.

That function is nested inside the reference's test, so it is not importable: it is read from the reference file with `ast`
at generation time and executed with h_q / h_kv bound; nothing of it is stored here.  It hard-codes the softmax scale
1 / sqrt(576) (the query's last dim), so the fixture uses that scale.

Needs the reference tree on PYTHONPATH; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_mla_spec.py [out.pt]

Inputs are seeded bf16 values (stored as bf16, computed in fp32); the reference output is fp32.  One paged latent cache
[9 pages, 16, 576] is shared by the cases (each request walks its pages in its own order), and the queries of every case
are the first rows of one pool of 576-dim query vectors (q_nope | q_pe), which keeps the file under 1 MB.  For the same
reason the stored output keeps every fourth value dim (out_dims = 0, 4, ..., 508: all four 128-dim quarters and all eight
64-dim blocks of V); lse is stored in full.  Cases (Hq, Q, kv_lens):
  128, Q 2, [37]        the bench head count: one draft token per q-group of the kernel;
  16, Q 4, [4, 129]     a TP8 shard (8 draft tokens fit one pass): kv_len == Q, and kv_len 129, where the draft
                        (positions 125-128) crosses a 128-token tile and a page boundary;
  16, Q 8, [50]         an exactly full q-group;
  64, Q 3, [45]         two q-groups (2 + 1 draft tokens);
  20, Q 3, [23]         a head count that does not divide 128.
No row has kv_len - Q + 1 + i <= 0 (the reference gives NaN there).  Goes to tests/golden/golden_mla_spec.pt.
Nothing here is imported by the product.
"""
import ast
import math
import os
import sys

import torch

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_mla_spec.pt")
REF_FILE = os.path.join("tests", "kernels", "attention", "test_flashmla.py")
PAGE = 16
POOL_PAGES = 9
OUT_DIMS = torch.arange(0, 512, 4)
# (Hq, Q, kv_lens)
CASES = (
    (128, 2, [37]),
    (16, 4, [4, 129]),
    (16, 8, [50]),
    (64, 3, [45]),
    (20, 3, [23]),
)


def _reference_sdpa(h_q: int, h_kv: int):
    """The reference's nested scaled_dot_product_attention, with h_q / h_kv bound."""
    path = next((os.path.join(p, REF_FILE) for p in sys.path if p and os.path.isfile(os.path.join(p, REF_FILE))), None)
    if path is None:
        raise SystemExit(f"{REF_FILE} not found on PYTHONPATH: put the reference tree there")
    tree = ast.parse(open(path).read(), filename=path)
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "scaled_dot_product_attention")
    ns = dict(torch=torch, math=math, h_q=h_q, h_kv=h_kv)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    return ns["scaled_dot_product_attention"]


def main(out_path: str = OUT):
    gen = torch.Generator().manual_seed(0)
    kv_cache = torch.randn(POOL_PAGES, PAGE, 576, generator=gen).bfloat16()
    q_pool = torch.randn(max(hq * q * len(lens) for hq, q, lens in CASES), 576, generator=gen).bfloat16()
    scale = 1.0 / math.sqrt(576)
    cases = []
    for hq, Q, kv_lens in CASES:
        B = len(kv_lens)
        assert all(Q <= s <= POOL_PAGES * PAGE for s in kv_lens)
        sdpa = _reference_sdpa(hq, 1)
        q = q_pool[:B * Q * hq].reshape(B * Q, hq, 576)
        bt = torch.stack([torch.randperm(POOL_PAGES, generator=gen) for _ in range(B)]).int()
        out = torch.empty(B * Q, hq, 512)
        lse = torch.empty(B * Q, hq)
        for b, S in enumerate(kv_lens):
            kv = kv_cache[bt[b].long()].reshape(-1, 576)[:S].float()
            # reference layout: query [h_q, s_q, d], key [h_kv, s_k, d], value [h_kv, s_k, dv]
            o, l = sdpa(q[b * Q:(b + 1) * Q].float().transpose(0, 1), kv[None], kv[None, :, :512], is_causal=True)
            out[b * Q:(b + 1) * Q] = o.transpose(0, 1)
            lse[b * Q:(b + 1) * Q] = l.transpose(0, 1)
        cases.append(dict(num_heads=hq, q_len=Q, kv_lens=kv_lens, block_tables=bt, q_rows=B * Q * hq,
                          out=out[..., OUT_DIMS].contiguous(), lse=lse))
    torch.save(dict(page_size=PAGE, scale=scale, kv_cache=kv_cache, q_pool=q_pool, out_dims=OUT_DIMS, cases=cases),
               out_path)
    print("wrote", out_path, len(cases), "cases")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
