"""In-tree build of libb200moe.so (nvcc, sm_90a) and of the C oracle.  No torch dependency."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libb200moe.so")
SOURCES = ["api.cu", "moe_prep.cu", "moe_gemm.cu", "moe_fused.cu", "repack.cu", "routing.cu", "router.cu", "attention.cu", "attention_mla.cu", "mla_aux.cu", "attention_gqa.cu", "gqa_aux.cu", "indexer.cu", "ep.cu", "mhc.cu", "dsv4_compress.cu", "dsv4_indices.cu", "dsv4_oproj.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_lib(force: bool = False, verbose: bool = False) -> str:
    """nvcc every csrc/*.cu for sm_90a and link libb200moe.so in-tree.  Objects are rebuilt when a source / header is
    newer; B200MOE_FORCE_BUILD=1 (or force=True) recompiles everything.  What was done is recorded in
    lvllm_b200/build/build_record.json (sources compiled this call, nvcc version, flags) so that a run can prove which
    binary it used."""
    force = force or os.environ.get("B200MOE_FORCE_BUILD") == "1"
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(ROOT, "include", "b200moe.h"))
    objdir = os.path.join(PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            cmd = [nvcc] + [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")] + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{out}")
    linked = False
    if force or procs or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs  # cudart is linked statically (nvcc default)
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}")
        linked = True
    try:
        import hashlib
        import json
        import time
        ver = subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[-1]
        rec = {"time": time.strftime("%Y-%m-%dT%H:%M:%S"), "forced": bool(force), "compiled": [s for s, _ in procs],
               "linked": linked, "nvcc": ver, "flags": NVCC_FLAGS, "lib": os.path.relpath(LIB, ROOT),
               "lib_sha256_16": hashlib.sha256(open(LIB, "rb").read()).hexdigest()[:16]}
        with open(os.path.join(objdir, "build_record.json"), "w") as f:
            json.dump(rec, f, indent=1)
    except Exception:
        pass
    return LIB


def build_oracle_c(force: bool = False) -> str | None:
    """Compile the plain-C restatement of the expert path (test infrastructure / CPU baseline)."""
    src = os.path.join(ROOT, "oracle", "moe_ref.c")
    if not os.path.exists(src):
        return None
    outdir = os.path.join(ROOT, "oracle", "_build")
    os.makedirs(outdir, exist_ok=True)
    out = os.path.join(outdir, "libmoe_ref.so")
    if force or _stale(out, [src]):
        cmd = ["gcc", "-O3", "-march=native", "-fopenmp", "-fPIC", "-shared", "-o", out, src, "-lm"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"gcc failed for oracle:\n{r.stdout}")
    return out


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose=True))
    print(build_oracle_c(force="--force" in sys.argv))
