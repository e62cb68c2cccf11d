"""Static resource usage of every kernel in libhctr_cuda.so (cuobjdump -res-usage): registers, static shared
memory, stack (spills show up as stack).  `--max-stack N` makes it a CI gate for the hot kernels, and for the
sparse-update kernels at no more than their stack of today (UPDATE_MAX_STACK)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "hugectr_b200", "lib", "libhctr_cuda.so")
HOT = ("gemm_tc_kernel", "gemm_mxfp8_kernel", "emb_fwd_kernel", "emb_dispatch_kernel")
# fused sparse-update kernels: today's worst stack per kernel (the G = 8, ev <= 128, reduce-update
# instantiations of stateful optimizers spill under their 80-register launch bound; FTRL / Nesterov heavy
# rows and one accumulate-path instantiation spill a little); the gate keeps every one of them from growing
UPDATE_MAX_STACK = {"emb_bwd_reduce_update_kernel": 64, "emb_bwd_heavy_kernel": 24, "emb_update_kernel": 16}


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
    worst_update = {}
    for k in sorted(rows):
        r = rows[k]
        regs, stack, sm = [x[0] for x in r], [x[1] for x in r], [x[2] for x in r]
        print(f"{k[:48]:48s} x{len(r):3d}  regs {min(regs):3d}-{max(regs):3d}  smem {max(sm):6d}  stack {min(stack)}-{max(stack)}")
        if any(h in k for h in HOT):
            worst = max(worst, max(stack))
        for u in UPDATE_MAX_STACK:
            if k.endswith(u):
                worst_update[u] = max(stack)
    if "--max-stack" in argv:
        lim = int(argv[argv.index("--max-stack") + 1])
        if worst > lim:
            print(f"FAIL: a hot kernel uses {worst} B of stack (> {lim})")
            return 1
        for u, cap in UPDATE_MAX_STACK.items():
            if worst_update.get(u, 0) > min(lim, cap):
                print(f"FAIL: {u} uses {worst_update[u]} B of stack (> {min(lim, cap)})")
                return 1
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
