"""Device time of the embedding lookup + fused backward with every input weighted, and with every input
position-weighted, against the same collection unweighted, at the DLRM-DCNv2 embedding shapes.

  python tools_dev/bench_emb_weighted.py [--steps 30] [--warmup 5] [--rounds 3] [--ev 128] [--cap-rows 2500000]
      [--arms unweighted,weighted,position_weighted]

The 26 Criteo-TB tables, batch 6912, the DCNv2 multi-hot sizes (214 keys per sample), power-law keys (alpha
1.1), AdaGrad, fp32 weights and activations, one GPU.  Tables are capped at --cap-rows rows: the collections of all
arms (fp32 weights and AdaGrad state, about 16.6 GB each at 2.5M rows) live on the card at once, so that the arms can
alternate in one process; bench.py's 10M-row cap holds one of them only.  All collections start from the same tables.
The position-weighted arm's step adds the fill of the weights from P, the weight-gradient dot products of every
looked-up row and their column sums into P's gradient (P stays at 1: the step does not run the dense optimizer).  Each round times
--steps steps of each arm (forward + backward between CUDA events, median), the arms alternating; the result
is the median over rounds, printed as one JSON line with the card name and its power limit, the keys per step
and the extra bytes the weights add per step (one fp32 weight read per key by the lookup and by the backward
index).  ``--profile`` adds, from one more step of each arm under torch.profiler, the device time per kernel
name (summed over launches) of every arm.  Without a CUDA device it exits and measures nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BATCH = 6912


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl or "unknown"


def collection(sizes, hot, ev, arm, dev):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    tabs = [EmbeddingTableConfig(str(i), v, ev) for i, v in enumerate(sizes)]
    names = [f"s{i}" for i in range(len(hot))]
    cfg.embedding_lookup(tabs, names, "emb", ["sum"] * len(hot))
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.0, epsilon=1e-8)
    e = EmbeddingCollection(cfg, BATCH, dict(zip(names, hot)), dev, torch.float32, Comm.single(dev), opt, seed=1,
                            weighted=names if arm == "weighted" else (),
                            position_weighted=names if arm == "position_weighted" else ())
    if arm == "position_weighted":
        e.bind_position_weights({n: (torch.ones(1, h, device=dev), torch.zeros(1, h, device=dev))
                                 for n, h in zip(names, hot)})
    return e


def batches(sizes, hot, n, dev):
    from hugectr_b200.data.batch import power_law_keys
    gen = torch.Generator().manual_seed(0)
    out = []
    for _ in range(n):
        keys = torch.cat([power_law_keys(BATCH * h, v, 1.1, gen, torch.int32) for v, h in zip(sizes, hot)])
        out.append((keys.to(dev), (torch.rand(keys.numel(), generator=gen) + 0.5).to(dev)))
    return out


def run(e, data, steps, warmup):
    dev = data[0][0].device
    lr, st = torch.tensor([0.01], device=dev), torch.tensor([1], dtype=torch.int32, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for it in range(warmup + steps):
        keys, w = data[it % len(data)]
        e.set_keys(keys)
        if e.has_data_weights:
            e.set_weights(w)
        ev[0].record()
        e.forward()
        e.top_grad["emb"].fill_(1e-3)
        e.backward(lr, st)
        ev[1].record()
        torch.cuda.synchronize()
        if it >= warmup:
            ts.append(ev[0].elapsed_time(ev[1]))
    return sorted(ts)[len(ts) // 2]


def kernel_times(e, data):
    """{kernel name: device microseconds} of one step of ``e`` under torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    run(e, data, 1, 1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(e, data, 1, 0)
    res = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            res[ev.key[:90]] = round(t, 1)
    return res


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ev", type=int, default=128)
    ap.add_argument("--cap-rows", type=int, default=2_500_000)
    ap.add_argument("--arms", default="unweighted,weighted,position_weighted")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_emb_weighted: no CUDA device; nothing measured")
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    hot = list(CRITEO_TB_MULTI_HOT)
    sizes = [min(t, a.cap_rows) for t in CRITEO_TB_TABLE_SIZES]
    dev = torch.device("cuda")
    name, plim = card()
    data = batches(sizes, hot, 8, dev)
    arms = {k: collection(sizes, hot, a.ev, k, dev) for k in a.arms.split(",")}
    first = next(iter(arms.values()))
    for e in arms.values():
        for g, g0 in zip(e.groups, first.groups):
            g.table.copy_(g0.table)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, e in arms.items():
            times[k].append(run(e, data, a.steps, a.warmup))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    n_keys = BATCH * sum(hot)
    print(json.dumps({"tables": len(hot), "batch": BATCH, "keys_per_step": n_keys, "ev": a.ev, "cap_rows": a.cap_rows,
                      "optimizer": "AdaGrad", **{f"{k}_ms": round(v, 4) for k, v in med.items()},
                      **{f"{k}_over_unweighted": round(v / med["unweighted"], 4) for k, v in med.items()
                         if k != "unweighted" and "unweighted" in med},
                      "rounds_ms": {k: [round(x, 4) for x in v] for k, v in times.items()},
                      "weight_bytes_per_step": 2 * n_keys * 4, "row_bytes_per_step_fwd": n_keys * a.ev * 4,
                      # the weight gradient reads every looked-up row once more
                      "pw_grad_row_bytes_per_step": n_keys * a.ev * 4,
                      "card": name, "power_limit": plim}), flush=True)
    if a.profile:
        kt = {k: kernel_times(e, data) for k, e in arms.items()}
        names = sorted(set().union(*kt.values()), key=lambda n: -max(t.get(n, 0) for t in kt.values()))
        print(json.dumps({"arms": list(kt), "kernel_us": [[n] + [t.get(n, 0) for t in kt.values()] for n in names[:25]]}),
              flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
