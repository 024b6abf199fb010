"""Golden fixture for DeepSeek-V4's MoE routing and clamped SwiGLU (tests/dsv4_moe_oracle.py, ops.fused_topk /
ops.hash_topk with scoring "sqrtsoftplus", activation_type 3).

Everything stored is computed by the reference's own code, read from its files with `ast` and executed here on the CPU:
  tests/kernels/moe/test_topk_softplus_sqrt.py                     _torch_topk_softplus_sqrt;
  vllm/model_executor/layers/fused_moe/router/fused_topk_bias_router.py   _topk_softplus_sqrt_torch;
  vllm/model_executor/layers/fused_moe/utils.py                    _swiglu_limit_torch (torch.compile decorator dropped);
  vllm/model_executor/layers/activation.py                         SiluAndMulWithClamp.forward_native (alpha 1, beta 0).

Needs the reference tree; run from outside both trees:
    PYTHONPATH=<reference tree> python <repository>/tests/golden/make_golden_dsv4_moe.py [out.pt]

Routing cases (all seeded, M = 40 tokens, k = 6, rsf 1.5, logits N(0, 2^2) with a few entries above softplus's threshold
of 20): E 256 and 384, each with bias N(0, 1) and with V4-Flash-like bias 8.08 + N(0, 1e-3^2), renormalised; one E 256
case without renormalisation; rows 3 and 17 all NaN in the biased cases.  Hash cases: a table [64, 6] over E 256 and
input ids drawn from the 64 token ids, renormalised and not.  Activation: x [32, 2 * 96] uniform over +-3 * limit,
limit 10.  Goes to tests/golden/golden_dsv4_moe.pt.  Nothing here is imported by the product.
"""
import ast
import os
import sys
import types

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_dsv4_moe.pt")
TEST_FILE = os.path.join("tests", "kernels", "moe", "test_topk_softplus_sqrt.py")
ROUTER_FILE = os.path.join("vllm", "model_executor", "layers", "fused_moe", "router", "fused_topk_bias_router.py")
UTILS_FILE = os.path.join("vllm", "model_executor", "layers", "fused_moe", "utils.py")
ACT_FILE = os.path.join("vllm", "model_executor", "layers", "activation.py")
M, K, RSF, VOCAB, LIMIT = 40, 6, 1.5, 64, 10.0
NAN_ROWS = (3, 17)


def _path(rel):
    path = next((os.path.join(p, rel) for p in sys.path if p and os.path.isfile(os.path.join(p, rel))), None)
    if path is None:
        raise SystemExit(f"{rel} not found on PYTHONPATH: put the reference tree there")
    return path


def _functions(rel, names, ns):
    path = _path(rel)
    tree = ast.parse(open(path).read(), filename=path)
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(fns) == len(names), (rel, names)
    for f in fns:
        f.decorator_list = []
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in names]


def _method(rel, cls, name, ns):
    path = _path(rel)
    tree = ast.parse(open(path).read(), filename=path)
    c = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls)
    f = next(n for n in c.body if isinstance(n, ast.FunctionDef) and n.name == name)
    f.decorator_list = []
    exec(compile(ast.Module(body=[f], type_ignores=[]), path, "exec"), ns)
    return ns[name]


def _logits(gen, E):
    x = torch.randn(M, E, generator=gen) * 2
    x[torch.rand(M, E, generator=gen) < 0.01] = 25.0   # softplus(x) = x above 20
    return x


def _route(test_ref, torch_ref, logits, renorm, bias=None, input_ids=None, table=None):
    a_w, a_ids = test_ref(logits, K, renorm, RSF, bias, input_ids, table)
    b_w = torch.empty(M, K, dtype=torch.float32)
    b_ids = torch.empty(M, K, dtype=torch.int32)
    torch_ref(b_w, b_ids, torch.empty(M, K, dtype=torch.int32), logits, renorm, bias, input_ids, table, RSF)
    return dict(test_w=a_w, test_ids=a_ids, torch_w=b_w, torch_ids=b_ids)


def main(out_path: str = OUT):
    ns = dict(torch=torch, F=F, Tensor=torch.Tensor)
    (test_ref,) = _functions(TEST_FILE, ["_torch_topk_softplus_sqrt"], ns)
    (torch_ref,) = _functions(ROUTER_FILE, ["_topk_softplus_sqrt_torch"], ns)
    (swiglu_limit,) = _functions(UTILS_FILE, ["_swiglu_limit_torch"], ns)
    forward_native = _method(ACT_FILE, "SiluAndMulWithClamp", "forward_native", ns)
    gen = torch.Generator().manual_seed(0)

    topk = []
    for E in (256, 384):
        for bias_kind in ("normal", "v4flash"):
            logits = _logits(gen, E)
            logits[list(NAN_ROWS)] = float("nan")
            if bias_kind == "normal":
                bias = torch.randn(E, generator=gen)
            else:
                bias = 8.08 + 1e-3 * torch.randn(E, generator=gen)
            topk.append(dict(E=E, bias_kind=bias_kind, renorm=True, logits=logits, bias=bias,
                             **_route(test_ref, torch_ref, logits, True, bias)))
    logits = _logits(gen, 256)
    bias = torch.randn(256, generator=gen)
    topk.append(dict(E=256, bias_kind="normal", renorm=False, logits=logits, bias=bias,
                     **_route(test_ref, torch_ref, logits, False, bias)))

    table = torch.stack([torch.randperm(256, generator=gen)[:K] for _ in range(VOCAB)]).to(torch.int32)
    hashed = []
    for renorm in (True, False):
        logits = _logits(gen, 256)
        input_ids = torch.randint(0, VOCAB, (M,), generator=gen, dtype=torch.int32)
        hashed.append(dict(E=256, renorm=renorm, logits=logits, input_ids=input_ids,
                           **_route(test_ref, torch_ref, logits, renorm, None, input_ids, table)))

    x = (torch.rand(32, 2 * 96, generator=gen) * 2 - 1) * 3 * LIMIT
    out_limit = torch.empty(32, 96)
    swiglu_limit(out_limit, x, LIMIT)
    act = dict(x=x, limit=LIMIT, forward_native=forward_native(types.SimpleNamespace(swiglu_limit=LIMIT, alpha=1.0,
                                                                                     beta=0.0), x),
               swiglu_limit_torch=out_limit)

    torch.save(dict(M=M, k=K, rsf=RSF, vocab=VOCAB, nan_rows=list(NAN_ROWS), topk=topk, hash_table=table, hash=hashed,
                    act=act), out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
