"""Count the SASS mnemonics that prove the Hopper data path per kernel of lvllm_b200/libb200moe.so (cuobjdump -sass):
warpgroup MMAs (HGMMA 16-bit / QGMMA fp8), tensor-map TMA (UTMALDG), bulk async copies (UBLKCP), cp.async (LDGSTS), and the
warp-level HMMA / IMMA / QMMA that must NOT appear.  WGDEPBAR1 counts `WARPGROUP.DEPBAR.LE gsb0, 0x1`: a wait that leaves one
wgmma group in flight, i.e. MMAs that ptxas did not serialise.  usage: python tools/sass_evidence.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lvllm_b200", "libb200moe.so")
PAT = re.compile(r"\b(HGMMA|QGMMA|UTMALDG|UTMASTG|UBLKCP|LDGSTS|HMMA|IMMA|QMMA|F2FP)\b")
DEPBAR1 = re.compile(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b")


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    per = collections.OrderedDict()
    cur = None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            per[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = PAT.search(ln)
        if m:
            per[cur][m.group(1)] += 1
        if DEPBAR1.search(ln):
            per[cur]["WGDEPBAR1"] += 1
    try:
        names = subprocess.run(["c++filt"], input="\n".join(per), stdout=subprocess.PIPE, text=True).stdout.splitlines()
    except OSError:
        names = list(per)
    tot = collections.Counter()
    print(f"# SASS evidence: cuobjdump -sass {os.path.relpath(LIB, ROOT)} ({len(per)} kernels); counts of instruction SITES per kernel")
    for (mangled, c), nm in zip(per.items(), names):
        tot.update(c)
        short = re.sub(r"\(.*", "", nm).replace("void b200::", "")
        print(f"{short:90s} {dict(c)}")
    print("# totals:", dict(tot))
    print("# legacy mma.sync sites (HMMA / IMMA / QMMA), must be 0:", tot["HMMA"] + tot["IMMA"] + tot["QMMA"])


if __name__ == "__main__":
    sys.exit(main())
