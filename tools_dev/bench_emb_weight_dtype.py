"""fp32 vs bf16 embedding weights: device time of the model-parallel lookup (forward) and of the fused
backward (bwd_index + bwd_reduce_update, AdaGrad with fp32 state) at DLRM-DCNv2 shapes.

  python tools_dev/bench_emb_weight_dtype.py [--iters 20] [--rounds 5] [--max-rows 4000000]

One arena of the 26 Criteo-TB tables (rows capped at --max-rows, far larger than the 50 MB L2), ev 128,
batch 6912, the DCNv2 multi-hot sizes, power-law keys (alpha 1.1), bf16 activations and gradients.  Both
arenas live in one process and the two weight types are timed alternately, with CUDA events after a
warm-up.  Prints the card name and power limit read in the same run, the nominal bytes per step
computed from the shapes, and one JSON line per (weight type, phase) with the median over rounds.
Needs a CUDA device: without one it exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hugectr_b200.data.batch import power_law_keys  # noqa: E402
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.enums import Optimizer_t  # noqa: E402
from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES  # noqa: E402

BATCH, EV = 6912, 128


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl or "unknown"


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        print("bench_emb_weight_dtype: needs a CUDA device (an H100); nothing was measured", file=sys.stderr)
        return 1
    dev = torch.device("cuda")
    name, plim = card()
    print(f"# device: {name}, power limit {plim}", flush=True)
    rows = [min(s, a.max_rows) for s in CRITEO_TB_TABLE_SIZES]
    hot = list(CRITEO_TB_MULTI_HOT)
    n = len(rows)
    gen = torch.Generator().manual_seed(0)
    lookups, roff, koff, keys = [], 0, 0, []
    width = n * EV
    for i in range(n):
        lookups.append(E.LookupDesc(table_row_off=roff, key_off=koff, out_off=i * EV, grad_off=i * EV,
                                    hotness=hot[i], key_stride=hot[i], num_shards=1, shard_idx=0,
                                    out_stride=width, grad_stride=width, combiner=0, ev_size=EV, rows=rows[i]))
        keys.append(power_law_keys(BATCH * hot[i], rows[i], 1.1, gen, torch.int32))
        roff += rows[i]
        koff += BATCH * hot[i]
    po = 0
    for lk in lookups:
        lk.pair_off = po
        po += BATCH * lk.hotness
    pairs, total_rows = po, roff
    keys_h = torch.cat(keys)
    uniq = sum(int(torch.unique(k).numel()) for k in keys)
    key_d = keys_h.to(dev)
    ld = E.lookups_to_device(lookups, dev)
    out = torch.zeros(BATCH * width, dtype=torch.bfloat16, device=dev)
    grad = (torch.randn(BATCH * width, device=dev) * 1e-3).to(torch.bfloat16)
    state = torch.zeros(total_rows * EV, device=dev)
    tables = {"fp32": torch.empty(total_rows * EV, device=dev).uniform_(-0.01, 0.01)}
    tables["bf16"] = tables["fp32"].to(torch.bfloat16)
    ws = E.UniqueWorkspace(pairs, EV, dev, indexed=True)
    lr_t = torch.full((1,), 1e-3, device=dev)
    st_t = torch.ones(1, dtype=torch.int32, device=dev)
    hp = {"epsilon": 1e-8, "sr_seed": 1}

    def fwd(t):
        E.forward(lookups, ld, t, EV, [key_d], [out], BATCH)

    def bwd(t):
        E.bwd_index(lookups, ld, t, EV, [key_d], BATCH, ws)
        E.bwd_reduce_update(Optimizer_t.AdaGrad, lookups, ld, t, state, None, EV, [key_d], [grad], BATCH, ws,
                            hp, lr_t, st_t)

    def timed(fn, t):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            fn(t)
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / a.iters

    for t in tables.values():
        for _ in range(a.warmup):
            fwd(t)
            bwd(t)
    torch.cuda.synchronize()
    res = {(w, ph): [] for w in tables for ph in ("forward", "backward")}
    for _ in range(a.rounds):
        for w, t in tables.items():                    # alternate fp32 / bf16 within every round
            res[(w, "forward")].append(timed(fwd, t))
            res[(w, "backward")].append(timed(bwd, t))
    E.check_workspace_overflow(ws, "benchmark")
    print(f"# {n} tables, {total_rows} rows x {EV}, batch {BATCH}, {pairs} keys per step, {uniq} distinct rows",
          flush=True)
    for w, t in tables.items():
        wb = t.element_size()
        nbytes = {"forward": pairs * EV * wb + pairs * 4 + BATCH * width * 2,
                  # weight read + write and AdaGrad state read + write per distinct row, gradient rows per key
                  "backward": uniq * EV * (2 * wb + 8) + pairs * (EV * 2 + 4)}
        for ph in ("forward", "backward"):
            ts = sorted(res[(w, ph)])
            ms = ts[len(ts) // 2]
            print(json.dumps({"weights": w, "phase": ph, "ms": round(ms, 4), "min_ms": round(ts[0], 4),
                              "max_ms": round(ts[-1], 4), "nominal_MB": round(nbytes[ph] / 1e6, 1),
                              "nominal_GBps": round(nbytes[ph] / ms / 1e6, 1), "device": name,
                              "power_limit": plim}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
