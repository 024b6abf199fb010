"""CPU: the DeepSeek-V4 output projection oracle (tests/dsv4_oproj_oracle.py) against the reference's own code stored in
tests/golden/golden_dsv4_oproj.pt (the inverse RoPE + quantisation bytes and scales, the unquantised z), the C ABI and
Python refusals of dsv4_inv_rope_quant and dsv4_o_proj, and the SASS of the wo_a GEMM kernel."""
import os
import shutil
import subprocess
import sys

import pytest
import torch

import dsv4_oproj_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "golden_dsv4_oproj.pt")


def _load():
    return torch.load(GOLDEN, weights_only=True)


def _cos_sin(n):
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    f = torch.arange(n, dtype=torch.float64)[:, None] * inv[None]
    return torch.cat([f.cos(), f.sin()], dim=1).float()


@pytest.mark.parametrize("case", ["quant", "gemm"])
def test_quant_matches_reference(case):
    g = _load()
    c = g[case]
    q, s = O.inv_rope_quant(c["o"], c["positions"], _cos_sin(g["cos_sin_positions"]), c["n_groups"])
    assert torch.equal(q.view(torch.uint8), c["q"])
    assert torch.equal(s, c["s"])
    # the interpreter's scales are the same; its e4m3 cast is not the hardware's, so most but not all of its bytes agree
    assert torch.equal(s, c["s_interp"])
    assert float((q.view(torch.uint8) == c["q_interp"]).float().mean()) > 0.9


def test_quant_edge_blocks():
    c = _load()["quant"]
    s, q = c["s"], c["q"].view(torch.float8_e4m3fn)
    assert float(s[0, 0, 0]) == 2.0 ** -7          # absmax * (1 / 448) exactly a power of two keeps it
    assert float(s[0, 0, 1]) == 2.0 ** -6          # the next bf16 above goes up one
    assert float(s[0, 0, 4]) == 2.0 ** -42         # all-zero head: the 1e-10 clamp
    assert int(c["q"][0, 0, 512:1024].sum()) == 0
    assert float(q[1, 0, 2 * 512 + 7].float()) == 448.0   # the e4m3 maximum


def test_z_matches_reference():
    c = _load()["gemm"]
    w = c["w"].view(torch.float8_e4m3fn)
    z, bound = O.wo_a(c["q"].view(torch.float8_e4m3fn), c["s"], w, c["w_scale"])
    assert z.shape == c["z"].shape == (5, c["n_groups"] * c["R"])
    assert O.calc_diff(z, c["z"].float()) < 1e-2
    assert bool((z.abs() <= bound).all())


def test_ue8m0_ceil_is_exact():
    x = torch.tensor([2.0 ** -7, 2.0 ** -7 * (1 + 2 ** -23), 1.0, 3.0, 2.0 ** -140 * 2 ** 20], dtype=torch.float32)
    assert O.ue8m0_ceil(x).tolist() == [2.0 ** -7, 2.0 ** -6, 1.0, 4.0, 2.0 ** -120]


def _args(T=3, H=16, G=2, R=256):
    o = torch.zeros(T, H, 512, dtype=torch.bfloat16)
    D = H // G * 512
    w = torch.zeros(G * R, D, dtype=torch.float8_e4m3fn)
    ws = torch.ones(G * R // 128, D // 128)
    return o, torch.zeros(T, dtype=torch.int64), _cos_sin(64), w, ws, G


def test_python_refusals():
    from lvllm_b200 import ops
    o, pos, cs, w, ws, G = _args()
    bad_o = [
        (o.float(), G), (o[:, :, :256], G), (o.transpose(0, 1), G),
        (torch.zeros(3, 16, 1024, dtype=torch.bfloat16)[:, :, ::2], G),                       # strided dims
        (torch.zeros(3, 16, 516, dtype=torch.bfloat16)[:, :, :512], G),                       # head stride 516
        (torch.zeros(3 * (16 * 512 + 4), dtype=torch.bfloat16).as_strided((3, 16, 512), (16 * 512 + 4, 512, 1)), G),
        (o, 3), (o, 0), (o, -2), (torch.zeros(3, 34, 512, dtype=torch.bfloat16), 2),          # 17 heads per group
    ]
    for ob, g in bad_o:
        with pytest.raises(ValueError):
            ops.dsv4_inv_rope_quant(ob, pos, cs, g)
        with pytest.raises(ValueError):
            ops.dsv4_o_proj(ob, pos, cs, w, ws, g)
    for pb, cb in [(pos[:2], cs), (pos, cs.double()), (pos, cs[:, :32])]:
        with pytest.raises(ValueError):
            ops.dsv4_inv_rope_quant(o, pb, cb, G)
        with pytest.raises(ValueError):
            ops.dsv4_o_proj(o, pb, cb, w, ws, G)
    bad_w = [
        (w.view(torch.uint8), ws), (w.to(torch.bfloat16), ws), (w[:, :1024], ws), (w[:384], ws),
        (torch.zeros(2 * 192, 4096, dtype=torch.float8_e4m3fn), ws), (w.t().contiguous().t(), ws),
        (w, ws.double()), (w, ws[:, :16]), (w, ws[:2]),
    ]
    for wb, wsb in bad_w:
        with pytest.raises(ValueError):
            ops.dsv4_o_proj(o, pos, cs, wb, wsb, G)
    # valid shapes on the CPU: there is no CPU path
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_inv_rope_quant(o, pos, cs, G)
    with pytest.raises(ValueError, match="CUDA"):
        ops.dsv4_o_proj(o, pos, cs, w, ws, G)


P = 1 << 20   # a 16-byte aligned stand-in address: refusals happen before anything is dereferenced


def _ir_abi(lib, **kw):
    a = dict(o=P, ostride=16 * 512, pos=P, cs=P, maxpos=64, T=2, H=16, G=2, q=P, s=P)
    a.update(kw)
    return lib.b200_dsv4_inv_rope_quant(None, *a.values())


def _wa_abi(lib, **kw):
    a = dict(q=P, s=P, w=P, ws=P, T=2, G=2, hpg=8, R=256, work=P, work_bytes=1 << 40, z=P)
    a.update(kw)
    return lib.b200_dsv4_wo_a(None, *a.values())


def test_c_abi_refuses_bad_arguments():
    from lvllm_b200 import _lib as L
    lib = L.lib()
    assert _ir_abi(lib, T=0) == 0 and _wa_abi(lib, T=0) == 0
    assert _ir_abi(lib, H=16, G=1, T=0) == 0 and _ir_abi(lib, H=3, G=3, ostride=3 * 512, T=0) == 0
    for bad in (dict(o=None), dict(o=P + 8), dict(ostride=16 * 512 - 8), dict(ostride=16 * 512 + 4), dict(pos=None),
                dict(pos=P + 4), dict(cs=None), dict(cs=P + 2), dict(maxpos=0), dict(T=-1), dict(T=(1 << 20) + 1),
                dict(H=0), dict(G=0), dict(G=3), dict(H=34, G=2, ostride=34 * 512), dict(q=None), dict(q=P + 8),
                dict(s=None), dict(s=P + 2)):
        assert _ir_abi(lib, **bad) == -1, bad
    for bad in (dict(q=None), dict(q=P + 8), dict(s=None), dict(s=P + 2), dict(w=None), dict(w=P + 8), dict(ws=None),
                dict(ws=P + 2), dict(z=None), dict(z=P + 1), dict(T=-1), dict(T=(1 << 20) + 1), dict(G=0), dict(hpg=0),
                dict(hpg=17), dict(R=0), dict(R=192), dict(R=64), dict(G=1 << 12, R=1 << 20)):
        assert _wa_abi(lib, **bad) == -1, bad
    for G, hpg, R in ((0, 8, 256), (2, 0, 256), (2, 17, 256), (2, 8, 192), (1 << 12, 8, 1 << 20)):
        assert lib.b200_dsv4_wo_a_workspace_bytes(2, G, hpg, R) == 0
    assert lib.b200_dsv4_wo_a_workspace_bytes(0, 2, 8, 256) == 0


def test_wo_a_kernel_sass():
    """The grouped GEMM runs on the Hopper data path: warpgroup fp8 MMAs (QGMMA) fed by tensor-map loads (UTMALDG), no
    warp-level MMA, in every token-tile width."""
    if not (shutil.which("cuobjdump") or os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("cuobjdump not available")
    from lvllm_b200 import build
    build.build_lib()
    env = dict(os.environ, PATH=os.environ.get("PATH", "") + ":/usr/local/cuda/bin")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_evidence.py")], stdout=subprocess.PIPE, text=True,
                         check=True, env=env).stdout
    rows = [ln for ln in out.splitlines() if ln.startswith("dsv4_wo_a_kernel")]
    assert len(rows) == 4, out
    for ln in rows:
        counts = eval("{" + ln.split("{", 1)[1])   # noqa: S307 — our own tool's dict repr
        assert counts.get("QGMMA", 0) >= 4 and counts.get("UTMALDG", 0) >= 2, ln
        assert counts.get("HMMA", 0) + counts.get("IMMA", 0) + counts.get("QMMA", 0) == 0, ln
