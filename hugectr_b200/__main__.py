"""``python -m hugectr_b200``: installation report (version, native libraries, device, kernel inventory)."""
import os
import sys

import torch

import hugectr_b200 as h
from hugectr_b200 import _native


def main():
    print(f"hugectr_b200 {h.__version__}  (python {sys.version.split()[0]}, torch {torch.__version__})")
    for name, path in (("sm_90a kernels", _native.CUDA_SO), ("host runtime", _native.HOST_SO)):
        st = f"{os.path.getsize(path) / 1e6:.1f} MB" if os.path.exists(path) else "NOT BUILT (python __graft_entry__.py)"
        print(f"  {name:16s} {path}  {st}")
    if torch.cuda.is_available():
        p = torch.cuda.get_device_properties(0)
        print(f"  device 0         {p.name}, sm_{p.major}{p.minor}, {p.multi_processor_count} SMs, "
              f"{p.total_memory / 2**30:.0f} GiB, {torch.cuda.device_count()} visible")
        if (p.major, p.minor) != (9, 0):
            print("  WARNING: the kernels are compiled for sm_90a only")
    else:
        print("  device           none (CPU reference paths and gloo collectives only)")
    try:
        from hugectr_b200.utils.diagnose import kernel_summary
        ks = kernel_summary()
        fam = {}
        for k in ks:
            base = k.split("(")[0].split("<")[0].split("::")[-1].replace("void ", "")
            fam[base] = fam.get(base, 0) + 1
        print(f"  kernels          {len(ks)} instantiations of {len(fam)} kernels: " +
              ", ".join(f"{k} x{v}" for k, v in sorted(fam.items(), key=lambda x: -x[1])[:8]) + ", ...")
    except Exception as e:  # cuobjdump not installed
        print(f"  kernels          (cuobjdump unavailable: {e})")
    from hugectr_b200.layers import LAYER_REGISTRY
    print(f"  layers           {len(LAYER_REGISTRY)} Layer_t types; model zoo: " +
          ", ".join(n[6:] for n in dir(__import__("hugectr_b200.models.zoo", fromlist=["x"])) if n.startswith("build_")))


if __name__ == "__main__":
    main()
