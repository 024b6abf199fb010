"""Golden fixture for multi-token GQA decode (tests/gqa_spec_oracle.py, ops.gqa_decode(q_len_per_req=Q)): the reference's
OWN ref_paged_attn (tests/kernels/attention/test_flashinfer.py:29-80) with query_lens = [Q] * B, on the CPU in fp32.

Needs the reference tree on PYTHONPATH; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_gqa_spec.py [out.pt]

Inputs are seeded bf16 values (stored as bf16, computed in fp32); the reference output is fp32.  One paged K / V pool per kv
head count is shared by the cases (page 16).  Cases (Hq / Hkv, Q, kv_lens):
  32 / 8, Q 2 and 4     Mixtral's group of 4 (Q <= 4: one q-group of 16 columns);
  64 / 4, Q 3           Qwen3's group of 16: two q-groups (2 + 1 draft tokens);
  8 / 8, Q 5            group 1, kv_len == Q and a longer request;
  48 / 1, Q 2           group 48: the CUDA-core kernel;
  4 / 1, Q 4            kv_len 129: query token 0 sees nothing of the second 128-token split, and the draft (positions
                        125-128) crosses a page boundary.
No row has kv_len - Q + 1 + i <= 0 (ref_paged_attn would give NaN there).  Goes to tests/golden/golden_gqa_spec.pt.
Nothing here is imported by the product.
"""
import os
import sys

import torch

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_gqa_spec.pt")
D = 128
PAGE = 16
POOL_PAGES = {8: 1, 4: 1, 1: 9}   # pages of the shared pool per kv head count
# (Hq, Hkv, Q, kv_lens)
CASES = (
    (32, 8, 2, [11]),
    (32, 8, 4, [16]),
    (64, 4, 3, [13]),
    (8, 8, 5, [5, 16]),
    (48, 1, 2, [30]),
    (4, 1, 4, [129]),
)


def main(out_path: str = OUT):
    from tests.kernels.attention.test_flashinfer import ref_paged_attn  # :29-80
    gen = torch.Generator().manual_seed(0)
    pools = {}
    for hkv, npg in POOL_PAGES.items():
        pools[hkv] = dict(k_cache=torch.randn(npg, PAGE, hkv, D, generator=gen).bfloat16(),
                          v_cache=torch.randn(npg, PAGE, hkv, D, generator=gen).bfloat16())
    scale = D ** -0.5
    cases = []
    for hq, hkv, Q, kv_lens in CASES:
        B = len(kv_lens)
        npg = POOL_PAGES[hkv]
        assert all(Q <= s <= npg * PAGE for s in kv_lens)
        q = torch.randn(B * Q, hq, D, generator=gen).bfloat16()
        # each request walks the pool's pages in its own order (requests may share pages: the cache is only read)
        bt = torch.stack([torch.randperm(npg, generator=gen) for _ in range(B)]).int()
        p = pools[hkv]
        out = ref_paged_attn(q.float().clone(), p["k_cache"].float(), p["v_cache"].float(), [Q] * B, kv_lens, bt, scale)
        cases.append(dict(num_heads=hq, num_kv_heads=hkv, q_len=Q, kv_lens=kv_lens, block_tables=bt, q=q, out=out))
    torch.save(dict(head_dim=D, page_size=PAGE, scale=scale, pools=pools, cases=cases), out_path)
    print("wrote", out_path, len(cases), "cases")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
