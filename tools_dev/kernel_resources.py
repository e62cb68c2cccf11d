"""Static resource usage of every kernel in libhctr_cuda.so (cuobjdump -res-usage): registers, static shared
memory, stack (spills show up as stack).  `--max-stack N` makes it a CI gate for the hot kernels."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "hugectr_b200", "lib", "libhctr_cuda.so")
HOT = ("gemm_tc_kernel", "gemm_mxfp8_kernel", "emb_fwd_kernel", "emb_dispatch_kernel")


def main(argv):
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    rows = collections.defaultdict(list)
    name = None
    for l in out.splitlines():
        m = re.search(r"Function (\S+):", l)
        if m:
            raw = m.group(1)
            d = subprocess.run(["c++filt", raw], capture_output=True, text=True).stdout.strip() or raw
            name = re.sub(r"\(.*", "", re.sub(r"<.*", "", d)).replace("void ", "")
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", l)
        if m and name:
            rows[name].append(tuple(int(x) for x in m.groups()))
            name = None
    print("# kernel x instantiations   regs min-max   static smem max   stack min-max (bytes; > 0 in a hot loop = spills)")
    worst = 0
    for k in sorted(rows):
        r = rows[k]
        regs, stack, sm = [x[0] for x in r], [x[1] for x in r], [x[2] for x in r]
        print(f"{k[:48]:48s} x{len(r):3d}  regs {min(regs):3d}-{max(regs):3d}  smem {max(sm):6d}  stack {min(stack)}-{max(stack)}")
        if any(h in k for h in HOT):
            worst = max(worst, max(stack))
    if "--max-stack" in argv:
        lim = int(argv[argv.index("--max-stack") + 1])
        if worst > lim:
            print(f"FAIL: a hot kernel uses {worst} B of stack (> {lim})")
            return 1
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
