"""Row-wise AdaGrad against element-wise AdaGrad: device time of the fused embedding backward
(bwd_index + bwd_reduce_update) at DLRM-DCNv2 shapes, and (--full-model) the uncapped DLRM-DCNv2
Criteo-TB tables with bf16 weights and row-wise AdaGrad on one GPU.

  python tools_dev/bench_emb_rowwise_adagrad.py [--iters 20] [--rounds 5] [--max-rows 4000000]
  python tools_dev/bench_emb_rowwise_adagrad.py --full-model [--steps 20] [--warmup 3]

Kernel mode: one arena of the 26 Criteo-TB tables (rows capped at --max-rows, far larger than the
50 MB L2), ev 128, batch 6912, the DCNv2 multi-hot sizes, power-law keys (alpha 1.1), bf16 gradients.
Six arms -- {AdaGrad fp32 state, AdaGrad bf16 state, RowWiseAdaGrad} x {fp32, bf16 weights} -- live in
one process and are timed alternately with CUDA events after a warm-up; one JSON line per arm with the
median over rounds and the nominal bytes of the update computed from the shapes.

Full-model mode: build_dlrm_dcnv2(num_gpus=1, batchsize=6912, embedding_optimizer="rowwise_adagrad",
weight_dtype="bf16") with the full table sizes, CUDA-graph training steps timed with CUDA events; prints
the table + state bytes, torch.cuda.max_memory_allocated, the step time and the final loss.

Both modes print the card name and power limit read in the same run.  Without a CUDA device the tool
exits with an error and measures nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def kernels(a, name, plim):
    dev = torch.device("cuda")
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
    uniq = sum(int(torch.unique(k).numel()) for k in keys)
    key_d = torch.cat(keys).to(dev)
    ld = E.lookups_to_device(lookups, dev)
    grad = (torch.randn(BATCH * width, device=dev) * 1e-3).to(torch.bfloat16)
    w32 = torch.empty(total_rows * EV, device=dev).uniform_(-0.01, 0.01)
    tables = {"fp32": w32, "bf16": w32.to(torch.bfloat16)}
    states = {"adagrad_fp32_state": (Optimizer_t.AdaGrad, torch.zeros(total_rows * EV, device=dev), 8),
              "adagrad_bf16_state": (Optimizer_t.AdaGrad,
                                     torch.zeros(total_rows * EV, dtype=torch.bfloat16, device=dev), 4),
              "rowwise_adagrad": (Optimizer_t.RowWiseAdaGrad, torch.zeros(total_rows, device=dev), None)}
    ws = E.UniqueWorkspace(pairs, EV, dev, indexed=True)
    lr_t = torch.full((1,), 1e-3, device=dev)
    st_t = torch.ones(1, dtype=torch.int32, device=dev)
    hp = {"epsilon": 1e-8, "sr_seed": 1}
    arms = [(o, w) for o in states for w in tables]

    def bwd(arm):
        o, w = arm
        opt, st, _ = states[o]
        t = tables[w]
        E.bwd_index(lookups, ld, t, EV, [key_d], BATCH, ws)
        E.bwd_reduce_update(opt, lookups, ld, t, st, None, EV, [key_d], [grad], BATCH, ws, hp, lr_t, st_t)

    def timed(arm):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            bwd(arm)
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / a.iters

    for arm in arms:
        for _ in range(a.warmup):
            bwd(arm)
    torch.cuda.synchronize()
    res = {arm: [] for arm in arms}
    for _ in range(a.rounds):
        for arm in arms:                     # every arm once per round
            res[arm].append(timed(arm))
    E.check_workspace_overflow(ws, "benchmark")
    print(f"# {n} tables, {total_rows} rows x {EV}, batch {BATCH}, {pairs} keys per step, {uniq} distinct rows",
          flush=True)
    for o, w in arms:
        wb = tables[w].element_size()
        sb = states[o][2]
        # weight read + write and state read + write per distinct row, one bf16 gradient row + locator per key
        row_bytes = EV * 2 * wb + (EV * sb if sb is not None else 8)
        nbytes = uniq * row_bytes + pairs * (EV * 2 + 4)
        ts = sorted(res[(o, w)])
        ms = ts[len(ts) // 2]
        print(json.dumps({"optimizer": o, "weights": w, "phase": "fused backward", "ms": round(ms, 4),
                          "min_ms": round(ts[0], 4), "max_ms": round(ts[-1], 4),
                          "update_bytes_per_row": row_bytes, "nominal_MB": round(nbytes / 1e6, 1),
                          "nominal_GBps": round(nbytes / ms / 1e6, 1), "device": name, "power_limit": plim}),
              flush=True)
    return 0


def full_model(a, name, plim):
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    torch.cuda.set_device(0)
    t0 = time.time()
    m = build_dlrm_dcnv2(batchsize=BATCH, num_gpus=1, embedding_optimizer="rowwise_adagrad", weight_dtype="bf16",
                         use_cuda_graph=True)
    m.compile()
    e = m.ebcs_train[0]
    tb = sum(g.table.numel() * g.table.element_size() for g in e.groups)
    sb = sum(g.s0.numel() * g.s0.element_size() for g in e.groups if g.s0 is not None)
    print(f"# built in {time.time() - t0:.0f} s: {sum(CRITEO_TB_TABLE_SIZES)} rows, tables {tb / 1e9:.2f} GB, "
          f"row-wise state {sb / 1e9:.2f} GB", flush=True)
    for _ in range(a.warmup):
        m.train()
    torch.cuda.synchronize()
    s, ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(a.steps):
        m.train()
    ev.record()
    ev.synchronize()
    ms = s.elapsed_time(ev) / a.steps
    loss = m.get_current_loss()
    print(json.dumps({"mode": "full-model", "table_GB": round(tb / 1e9, 2), "state_GB": round(sb / 1e9, 3),
                      "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                      "step_ms": round(ms, 3), "steps": a.steps, "final_loss": loss, "batch": BATCH,
                      "device": name, "power_limit": plim}), flush=True)
    return 0 if loss == loss else 1


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-rows", type=int, default=4_000_000)
    ap.add_argument("--full-model", action="store_true")
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        print("bench_emb_rowwise_adagrad: needs a CUDA device (an H100); nothing was measured", file=sys.stderr)
        return 1
    name, plim = card()
    print(f"# device: {name}, power limit {plim}", flush=True)
    return full_model(a, name, plim) if a.full_model else kernels(a, name, plim)


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
