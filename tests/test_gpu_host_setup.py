"""GPU (-m gpu): the host side of kernel launches.

- Launch set-up is per device (api.cu kernel_smem / device_sms): a kernel's raised dynamic shared-memory limit belongs to
  the device's context, so a process that drives two devices must launch on the second exactly as on the first.  Every
  path run here reduces in a fixed order, so the outputs are bit-identical across two devices of the same SM count.
- The 4-bit prefill expansion runs in several passes with a short last pass, which stays on the fp16 shadow's grouped
  GEMM."""
import pytest
import torch

from oracle import moe_oracle as O
from test_gpu_shapes import _cfg, _decode, _ids, _rel

pytestmark = pytest.mark.gpu


def _run_every_set_up_path(d):
    """On cuda:d, every launch site with per-device set-up: the fused 4-bit decode, a 16-bit layer at M > 256 (grouped
    GEMM; the single-CTA routing sort and the multi-CTA one), the fused router, GQA and MLA decode (all four tensor-core
    instantiations of each).  Inputs come from one seed, so two devices get the same bytes."""
    import lk_moe
    from lvllm_b200 import ops
    dev = torch.device("cuda", d)
    g = torch.Generator().manual_seed(2024)
    outs = {}
    with torch.cuda.device(d):
        E, H, I = 16, 512, 256
        p13, s13 = O.quant_mxfp4(torch.randn(E, 2 * I, H, generator=g) / 10)
        p2, s2 = O.quant_mxfp4(torch.randn(E, H, I, generator=g) / 10)
        moe = lk_moe.MOE_MXFP4(_cfg(E, 2, H, I, gN=1, gK=32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(),
                               s2.data_ptr(), 0, 0)
        hid = (torch.randn(64, H, generator=g) / 10).bfloat16()
        ids, w = _ids(64, E, 2, g)
        outs["fused_w4"] = _decode(moe, hid, ids, w, dev)
        moe.close()

        w13 = (torch.randn(E, 2 * I, H, generator=g) / 10).bfloat16()
        w2 = (torch.randn(E, H, I, generator=g) / 10).bfloat16()
        moe = lk_moe.MOE_BF16(_cfg(E, 8, H, I), w13.data_ptr(), w2.data_ptr(), 0, 0, 0, 0)
        for M in (300, 1100):   # 2400 and 8800 routed slots: below and above the multi-CTA sort's 8192
            hid = (torch.randn(M, H, generator=g) / 10).bfloat16()
            ids, w = _ids(M, E, 8, g)
            out = torch.empty(M, H, dtype=torch.float32)
            moe.cpu_prefill(M, 8, ids.data_ptr(), w.data_ptr(), hid.data_ptr(), out.data_ptr())
            outs[f"grouped_{M}"] = out
        moe.close()

        hid = (torch.randn(64, 1024, generator=g) / 4).bfloat16()
        wg = (torch.randn(128, 1024, generator=g) * 0.05).bfloat16()
        outs["router"] = [t.cpu() for t in ops.router_topk(hid.to(dev), wg.to(dev), 8, True, "softmax")[:2]]

        B, S, page = 4, 300, 16
        npg = -(-S // page)
        for hq, hkv in ((32, 8), (64, 2)):   # G = 4: N = 16; G = 32: N = 32
            kc = torch.randn(B * npg, page, hkv, 128, generator=g).bfloat16().to(dev)
            vc = torch.randn(B * npg, page, hkv, 128, generator=g).bfloat16().to(dev)
            pt = torch.randperm(B * npg, generator=g).reshape(B, npg).int().to(dev)
            lens = torch.tensor([S, S - 13, 129, 40], dtype=torch.int32).to(dev)
            for Q in (1, 2):
                q = torch.randn(B * Q, hq, 128, generator=g).bfloat16().to(dev)
                outs[f"gqa_{hq}_{Q}"] = [t.cpu() for t in ops.gqa_decode(q, kc, vc, lens, pt, 128 ** -0.5, q_len_per_req=Q)]

        B, page = 2, 64
        npg = -(-S // page)
        pt = torch.arange(B * npg, dtype=torch.int32).reshape(B, npg).to(dev)
        lens = torch.tensor([S, 129], dtype=torch.int32).to(dev)
        for kv_dtype in (torch.bfloat16, torch.float8_e4m3fn):
            cache = torch.randn(B * npg, page, 576, generator=g).to(kv_dtype).to(dev)
            for Q in (1, 2):
                qn = torch.randn(B * Q, 16, 512, generator=g).bfloat16().to(dev)
                qp = torch.randn(B * Q, 16, 64, generator=g).bfloat16().to(dev)
                outs[f"mla_{kv_dtype}_{Q}"] = [t.cpu() for t in ops.mla_decode(qn, qp, cache, lens, pt, 0.07,
                                                                              q_len_per_req=Q)]
        torch.cuda.synchronize()
    return outs


def test_two_devices_in_one_process():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    props = [torch.cuda.get_device_properties(d) for d in (0, 1)]
    if props[0].multi_processor_count != props[1].multi_processor_count:
        pytest.skip("the two GPUs differ in SM count, so the persistent kernels' reduction orders differ")
    first, second = _run_every_set_up_path(0), _run_every_set_up_path(1)
    assert first.keys() == second.keys()
    for name in first:
        a, b = first[name], second[name]
        for x, y in zip(a, b) if isinstance(a, list) else [(a, b)]:
            assert torch.equal(x, y), f"{name}: cuda:0 and cuda:1 differ"


@pytest.mark.parametrize("act", ["bf16", "fp16"])
def test_moe_w4_prefill_expansion_passes(act):
    """max_batch_size = 256 cuts a 1100-token 4-bit prefill into four expansion passes of 256 tokens and a last pass of
    76.  That pass is small enough for the fused decode kernel, but it stays on the fp16 shadow's grouped GEMM: the fused
    kernel does not convert bf16 rows to fp16, and with fp16 activations a kernel switch would change bits.  So 1100
    tokens take one grouped-GEMM pass of launches more than 1024 (routing sort, gather, two GEMMs, combine).
    Tolerances of test_moe_w4_prefill_expansion."""
    import lk_moe
    from lvllm_b200 import _lib as L
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    dev = torch.device("cuda:0")
    E, k, H, I, M = 8, 2, 512, 256, 1100
    dt = torch.bfloat16 if act == "bf16" else torch.float16
    g = torch.Generator().manual_seed(1100)
    hid = (torch.randn(M, H, generator=g) / 10).to(dt)
    p13, s13 = O.quant_mxfp4(torch.randn(E, 2 * I, H, generator=g) / 10)
    p2, s2 = O.quant_mxfp4(torch.randn(E, H, I, generator=g) / 10)
    ids, w = _ids(M, E, k, g, 0.05)
    ref = O.experts_forward_batched(hid, O.DequantExperts(O.dequant_mxfp4(p13, s13), O.dequant_mxfp4(p2, s2)), ids, w,
                                    act_dtype=torch.float16)
    cls = lk_moe.MOE_MXFP4 if act == "bf16" else lk_moe.MOE_MXFP4_FP16
    moe = cls(_cfg(E, k, H, I, max_batch=256, gN=1, gK=32), p13.data_ptr(), p2.data_ptr(), s13.data_ptr(), s2.data_ptr(),
              0, 0)
    lib = L.lib()
    launches = {}
    for m in (1024, M):   # the first m rows of the row-major inputs
        out = torch.empty(m, H, dtype=torch.float32)
        n0 = lib.b200moe_launch_count()
        moe.cpu_prefill(m, k, ids.data_ptr(), w.data_ptr(), hid.data_ptr(), out.data_ptr())
        launches[m] = lib.b200moe_launch_count() - n0
    assert launches[M] - launches[1024] == 5, launches
    assert _rel(out, ref) < 0.01, f"cpu_prefill {act}: {_rel(out, ref)}"
    hd, idd, wd = hid.to(dev), ids.to(dev), w.to(dev)
    od = torch.empty(M, H, dtype=dt, device=dev)
    moe.gpu_prefill(hd.data_ptr(), od.data_ptr(), idd.data_ptr(), wd.data_ptr(), M, k, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    moe.close()
    assert _rel(od.float().cpu(), ref) < 0.015, f"gpu_prefill {act}: {_rel(od.float().cpu(), ref)}"
