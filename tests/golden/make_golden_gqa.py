"""Golden fixture for the GQA q/k-norm + RoPE oracle (tests/gqa_oracle.py): the reference's OWN native ops.

Needs the reference tree on PYTHONPATH; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_gqa.py [out.pt]

The reference's RMSNorm.forward_native (layers/layernorm.py) and RotaryEmbedding.forward_native (rotary_embedding/base.py:
203-220 -> forward_static :161-201) are composed exactly as tests/kernels/core/test_fused_qk_norm_rope.py:21-47 composes
them, on seeded bf16 qkv rows of head_dim 128: Qwen3-like heads (16 q / 4 kv, per-head norm) and Mixtral-like heads
(32 / 8), NeoX and GPT-J pairing, rotary_dim 128 / 64 / 32, eps 1e-6 / 1e-5, with and without the norm, positions up to
tens of thousands.  Only the cos | sin rows of the positions used are stored (the full table is 10 MB); inputs and the
rotated q / k go to tests/golden/golden_gqa.pt.  Nothing here is imported by the product.
"""
import os
import sys

import torch

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_gqa.pt")
D = 128
MAX_POS = 40960          # Qwen3's max_position_embeddings
BASE = 1e6               # rope_theta of Qwen3 and Mixtral
HEADS = ((16, 4), (32, 8))
# (heads index, tokens, neox, rotary_dim, norm, eps)
CASES = (
    (0, 2, True, 128, True, 1e-6), (0, 2, True, 64, True, 1e-5), (0, 2, True, 32, True, 1e-6),
    (0, 2, False, 128, True, 1e-5), (0, 2, False, 64, True, 1e-6), (0, 2, False, 32, True, 1e-5),
    (0, 2, False, 32, False, 1e-6),
    (1, 1, True, 128, False, 1e-6), (1, 1, False, 64, False, 1e-6), (1, 1, True, 32, False, 1e-6),
    (1, 1, False, 128, True, 1e-5),
)


def main(out_path: str = OUT):
    from vllm.config import DeviceConfig, VllmConfig, set_current_vllm_config
    from vllm.model_executor.layers.layernorm import RMSNorm
    from vllm.model_executor.layers.rotary_embedding import RotaryEmbedding
    gen = torch.Generator().manual_seed(0)
    qkv = [(torch.randn(2, (hq + 2 * hkv) * D, generator=gen) * 2).bfloat16() for hq, hkv in HEADS]
    cases = []
    with set_current_vllm_config(VllmConfig(device_config=DeviceConfig(device="cpu"))), torch.inference_mode():
        for hi, T, neox, rot, norm, eps in CASES:
            hq, hkv = HEADS[hi]
            x = qkv[hi][:T]
            pos = torch.cat([torch.randint(0, 64, (1,), generator=gen),
                             torch.randint(20000, MAX_POS, (T - 1,), generator=gen)])[-T:] if T > 1 else \
                torch.randint(20000, MAX_POS, (1,), generator=gen)
            rope = RotaryEmbedding(head_size=D, rotary_dim=rot, max_position_embeddings=MAX_POS, base=BASE,
                                   is_neox_style=neox, dtype=torch.bfloat16)
            q, k, _ = x.split([hq * D, hkv * D, hkv * D], dim=-1)
            qw = kw = None
            if norm:   # test_fused_qk_norm_rope.py:21-47 (weights ~ N(1, 0.1) as there)
                q_norm, k_norm = RMSNorm(D, eps=eps).to(torch.bfloat16), RMSNorm(D, eps=eps).to(torch.bfloat16)
                qw = (1 + 0.1 * torch.randn(D, generator=gen)).bfloat16()
                kw = (1 + 0.1 * torch.randn(D, generator=gen)).bfloat16()
                q_norm.weight.data.copy_(qw)
                k_norm.weight.data.copy_(kw)
                q = q_norm.forward_native(q.reshape(T, hq, D)).reshape(T, hq * D)
                k = k_norm.forward_native(k.reshape(T, hkv, D)).reshape(T, hkv * D)
            qo, ko = rope.forward_native(pos, q.clone(), k.clone())
            cs = rope._match_cos_sin_cache_dtype(x)
            cases.append(dict(heads=hi, num_heads=hq, num_kv_heads=hkv, tokens=T, is_neox=neox, rotary_dim=rot, norm=norm,
                              eps=eps, q_weight=qw, k_weight=kw, positions=pos, cos_sin_rows=cs[pos].clone(),
                              q_out=qo.reshape(T, hq, D).clone(), k_out=ko.reshape(T, hkv, D).clone()))
    torch.save(dict(head_dim=D, max_position=MAX_POS, qkv=qkv, cases=cases), out_path)
    print("wrote", out_path, len(cases), "cases")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
