"""Golden fixture for DeepSeek-V4's manifold hyper-connections (tests/mhc_oracle.py, ops.mhc_pre / mhc_post /
mhc_fused_post_pre / hc_head).

Everything stored is computed by the reference's own code, read from its files with `ast` and executed here on the CPU:
  vllm/model_executor/kernels/mhc/torch.py    mhc_pre_torch, mhc_post_torch (the native forward of the mHC ops);
  tests/kernels/test_mhc_kernels.py           sinkhorn_normalize_ref, mhc_pre_ref, mhc_post_ref, hc_head_ref;
  vllm/ir/ops/layernorm.py                    rms_norm (decorators dropped), applied to mhc_pre_torch's layer_input: the
                                              unfused composition that the fused norm replaces.

Needs the reference tree; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_mhc.py [out.pt]

H = 1280 (the reference's smallest mHC size), hc_mult 4, eps 1e-6, sinkhorn_repeat 20, hc_post_mult_value 2.0 (what the
model passes).  One fn [24, 4H] and one hc_head fn [4, 4H], drawn as the reference test draws them (fn ~ 1e-4 with a
per-stream factor, scale and base ~ 0.1).  Cases (all seeded):
  t1       T = 1, the reference test's distribution;
  t5_pad   T = 5, token 3 an all-zero padding row (residual and x);
  t2_big   T = 2, hc_scale = (30, 30, 500), so the comb logits span several units and Sinkhorn has real work to do.
Per case: the inputs, mhc_post_torch / mhc_post_ref, mhc_pre_torch on the residual and on the post output (the fused op's
order), mhc_pre_ref, rms_norm of mhc_pre_torch's layer_input, hc_head_ref, and sinkhorn_normalize_ref of stored logits.
Goes to tests/golden/golden_mhc.pt.  Nothing here is imported by the product.
"""
import ast
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_mhc.pt")
TORCH_FILE = os.path.join("vllm", "model_executor", "kernels", "mhc", "torch.py")
TEST_FILE = os.path.join("tests", "kernels", "test_mhc_kernels.py")
NORM_FILE = os.path.join("vllm", "ir", "ops", "layernorm.py")
H, HC, EPS, REPEAT, POST_MULT, NORM_EPS = 1280, 4, 1e-6, 20, 2.0, 1e-6


def _functions(rel, names, ns):
    path = next((os.path.join(p, rel) for p in sys.path if p and os.path.isfile(os.path.join(p, rel))), None)
    if path is None:
        raise SystemExit(f"{rel} not found on PYTHONPATH: put the reference tree there")
    tree = ast.parse(open(path).read(), filename=path)
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(fns) == len(names), (rel, names)
    for f in fns:
        f.decorator_list = []
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in names]


def main(out_path: str = OUT):
    ns = dict(torch=torch, Tensor=torch.Tensor)
    pre_torch, post_torch = _functions(TORCH_FILE, ["mhc_pre_torch", "mhc_post_torch"], ns)
    sink_ref, pre_ref, post_ref, head_ref = _functions(
        TEST_FILE, ["sinkhorn_normalize_ref", "mhc_pre_ref", "mhc_post_ref", "hc_head_ref"], ns)
    (rms_norm,) = _functions(NORM_FILE, ["rms_norm"], ns)
    gen = torch.Generator().manual_seed(0)
    n3 = 2 * HC + HC * HC
    fn = (torch.randn(n3, HC, H, generator=gen) * 1e-4 * (1 + torch.arange(HC).mul(0.01).view(1, -1, 1))).flatten(1, 2)
    head_fn = torch.randn(HC, HC * H, generator=gen) * 1e-4
    head_scale = torch.randn(1, generator=gen) * 0.1
    head_base = torch.randn(HC, generator=gen) * 0.1
    norm_weight = (1 + 0.1 * torch.randn(H, generator=gen)).bfloat16()

    cases = []
    for name, T in (("t1", 1), ("t5_pad", 5), ("t2_big", 2)):
        residual = torch.randn(T, HC, H, generator=gen).bfloat16()
        x = torch.randn(T, H, generator=gen).bfloat16()
        plm = torch.rand(T, HC, 1, generator=gen) * 2
        crm = torch.rand(T, HC, HC, generator=gen)
        crm = crm / crm.sum(-2, keepdim=True)
        hc_scale = torch.randn(3, generator=gen) * 0.1
        hc_base = torch.randn(n3, generator=gen) * 0.1
        if name == "t5_pad":
            residual[3] = 0
            x[3] = 0
        if name == "t2_big":
            hc_scale = torch.tensor([30.0, 30.0, 500.0])
        args = (fn, hc_scale, hc_base, EPS, EPS, EPS, POST_MULT, REPEAT)
        r_post = post_torch(x, residual, plm, crm)
        pre_res = pre_torch(residual, *args)
        pre_post = pre_torch(r_post, *args)
        logits = torch.randn(T, HC, HC, generator=gen) * 3
        cases.append(dict(
            name=name, residual=residual, x=x, post_layer_mix=plm, comb_res_mix=crm, hc_scale=hc_scale, hc_base=hc_base,
            post_torch=r_post, post_ref=post_ref(x, residual, plm, crm),
            pre_torch=pre_res, pre_torch_on_post=pre_post, pre_ref=pre_ref(residual, *args),
            pre_torch_normed=rms_norm(pre_res[2], norm_weight, NORM_EPS),
            hc_head=head_ref(residual, head_fn, head_scale, head_base, EPS, EPS),
            sinkhorn_logits=logits, sinkhorn=sink_ref(logits, REPEAT, EPS)))
    torch.save(dict(H=H, eps=EPS, repeat=REPEAT, post_mult=POST_MULT, norm_eps=NORM_EPS, fn=fn, norm_weight=norm_weight,
                    head_fn=head_fn, head_scale=head_scale, head_base=head_base, cases=cases), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
