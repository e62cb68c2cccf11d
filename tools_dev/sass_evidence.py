"""Tensor-core / TMA / mbarrier mnemonic counts per kernel of the built library.

  python tools_dev/sass_evidence.py                 # table on stdout
  python tools_dev/sass_evidence.py --check         # CI gate: the kernels that must use wgmma / TMA do
  cuobjdump -sass lib.so | python tools_dev/sass_evidence.py -     # read a listing from stdin
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "hugectr_b200", "lib", "libhctr_cuda.so")
PAT = re.compile(r'\b(HGMMA|QGMMA|WARPGROUP|UTMALDG|UTMASTG|UBLKCP|SYNCS|UTMAPF)[A-Z0-9_.]*')
# kernel-name pattern (re.search on the mangled name) -> mnemonics it must contain
REQUIRED = {
    "gemm_tc_kernel": ("HGMMA", "UTMALDG", "SYNCS"),
    # instantiations with the TMA epilogue (last template argument, TMA_EPI, true) store their output by TMA
    r"gemm_tc_kernelI.*ELb1EE": ("UTMASTG",),
    "gemm_mxfp8_kernel": ("QGMMA", "UTMALDG", "UBLKCP"),
    "interaction": ("HGMMA",),
}


def counts(lines):
    cur, cnt = None, collections.defaultdict(collections.Counter)
    for l in lines:
        m = re.search(r'Function : (\S+)', l)
        if m:
            cur = m.group(1)
            continue
        if cur:
            for x in PAT.findall(l):
                cnt[cur][x] += 1
    return cnt


def main(argv):
    if "-" in argv:
        lines = sys.stdin
    else:
        lines = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout.splitlines()
    cnt = counts(lines)
    if "--check" in argv:
        bad = []
        for frag, need in REQUIRED.items():
            ks = [k for k in cnt if re.search(frag, k)]
            if not ks:
                bad.append(f"no kernel named *{frag}* in the library")
            for k in ks:
                missing = [m for m in need if not cnt[k].get(m)]
                if missing:
                    bad.append(f"{k[:100]}: missing {missing}")
        print("\n".join(bad) if bad else f"ok: {sum(1 for k in cnt if cnt[k])} kernels carry wgmma / TMA / bulk-copy SASS")
        return 1 if bad else 0
    print("cuobjdump -sass hugectr_b200/lib/libhctr_cuda.so : tensor-core / TMA / bulk-copy mnemonic counts per kernel")
    print("HGMMA / QGMMA = wgmma.mma_async bf16 / fp8   WARPGROUP = wgmma fence / wait   UTMALDG / UTMASTG = TMA tensor load / store")
    print("UBLKCP = cp.async.bulk (1-D)   SYNCS = mbarrier ops\n")
    for k, v in sorted(cnt.items()):
        if v:
            print(k[:150])
            print("    " + ", ".join(f"{a}:{b}" for a, b in sorted(v.items())))
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
