"""Device time of the model-parallel embedding lookup (forward) and of the fused sparse update (bwd_index +
bwd_reduce_update) at DLRM-DCNv2 shapes, per optimizer, optimizer-state dtype and weight dtype; and
(--full-model) the DLRM-DCNv2 Criteo-TB tables with bf16 weights and row-wise AdaGrad (or partial row-wise
Adam) on one GPU.

  python tools_dev/bench_emb_update.py [--opts adagrad,rowwise_adagrad] [--ev 128] [--iters 20] [--rounds 5]
                                       [--max-rows N] [--tree DIR]
  python tools_dev/bench_emb_update.py --check-bits TREE [--keys uniform] [--opts all] [--ev 128] [--steps 3]
  python tools_dev/bench_emb_update.py --full-model [--opts rowwise_adagrad] [--max-rows N] [--steps 20]
                                       [--warmup 3]

Kernel mode: one arena of the 26 Criteo-TB tables, ev 128 by default (the DLRM-DCNv2 width, which runs the
G = 8 update kernels; --ev 256 runs the G = 32 ones), batch 6912, the DCNv2 multi-hot sizes, power-law keys
(alpha 1.1), bf16 activations and gradients.  Rows are capped at --max-rows (default 4 M x 128 / ev, so the
arena keeps its size, far larger than the 50 MB L2).  --opts takes a comma-separated list of
sgd, adagrad, adam, ftrl, momentum, nesterov, rmsprop, rowwise_adagrad, partial_rowwise_adam, or `all`.
Every optimizer with per-element state runs with fp32 and with bf16 state (partial row-wise Adam: its first
moment; the second is one fp32 value per row); each of these arms runs with fp32 and bf16 weights.
The default is the six arms {AdaGrad fp32 state, AdaGrad bf16 state, RowWiseAdaGrad} x {fp32, bf16 weights}.
All arms live in one process and are timed alternately with CUDA events after a warm-up; the arms share
their state buffers, which are zeroed before every timed block.  One JSON line per (weight dtype, forward)
and per arm, with the median over rounds and the nominal bytes computed from the shapes.

--tree DIR imports hugectr_b200 from another checkout (built in place), so that two builds can be timed
alternately, one process per run, in one session.

--check-bits TREE times nothing: it runs --steps seeded fused-backward steps of every selected arm, each from
the same initial weights and zero state, under this tree, under TREE and under TREE a second time (one process
each), and compares 64-bit checksums of the arena and of both state arrays (computed on the device, position
weighted).  Rows are capped at 500 k unless --max-rows says otherwise.  The gradients are multiples of 2^-12, so
every row's fp32 sum is exact and the result does not depend on the order in which the counting sort lists a row's
buckets or the heavy rows' atomics land: every arm must agree bit for bit, and TREE against TREE is the control
(an arm that differs there is reported and not counted).  --keys uniform draws uniform keys and keeps only the
tables whose rows then occur 16 times on average at most (and stops if a row has more than 64 occurrences), so
that only the light- and medium-row code runs; the default power-law keys add the heavy rows.

Full-model mode: build_dlrm_dcnv2(num_gpus=1, batchsize=6912, embedding_optimizer=--opts (rowwise_adagrad
unless one of rowwise_adagrad / partial_rowwise_adam is given), weight_dtype="bf16") with the full table
sizes, or each capped at --max-rows (the uncapped tables do not fit one 80 GB card under partial row-wise
Adam), CUDA-graph training steps timed with CUDA events; prints the row cap, the table + state bytes,
torch.cuda.max_memory_allocated, the step time and the final loss.

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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH = 6912
OPTS = ("sgd", "adagrad", "adam", "ftrl", "momentum", "nesterov", "rmsprop", "rowwise_adagrad",
        "partial_rowwise_adam")
# per-element state vectors of each optimizer; ROW_STATE: the index of its state that is one fp32 value per
# row instead (row-wise AdaGrad's accumulator, partial row-wise Adam's second moment)
STATES = {"sgd": 0, "adagrad": 1, "adam": 2, "ftrl": 2, "momentum": 1, "nesterov": 1, "rmsprop": 1,
          "rowwise_adagrad": 0, "partial_rowwise_adam": 1}
ROW_STATE = {"rowwise_adagrad": 0, "partial_rowwise_adam": 1}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl or "unknown"


def parse_opts(s):
    opts = list(OPTS) if s == "all" else [o.strip() for o in s.split(",") if o.strip()]
    bad = [o for o in opts if o not in OPTS]
    if bad or not opts:
        raise SystemExit(f"bench_emb_update: unknown optimizer(s) {bad}; choose from {', '.join(OPTS)} or all")
    return opts


def checksum(t):
    """Position-weighted 64-bit sum of a tensor's 32-bit words (wraps), computed on the device in chunks."""
    w = t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)
    tot = torch.zeros((), dtype=torch.int64, device=t.device)
    for o in range(0, w.numel(), 1 << 26):
        c = w[o:o + (1 << 26)].to(torch.int64)
        tot += (c * (torch.arange(o, o + c.numel(), device=t.device) * 2 + 1)).sum()
    return format(int(tot.item()) & 0xFFFFFFFFFFFFFFFF, "016x")


def kernels(a, name, plim):
    from hugectr_b200.data.batch import power_law_keys
    from hugectr_b200.embedding import ops as E
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    names = {"sgd": "SGD", "adagrad": "AdaGrad", "adam": "Adam", "ftrl": "Ftrl", "momentum": "MomentumSGD",
             "nesterov": "Nesterov", "rmsprop": "RMSProp", "rowwise_adagrad": "RowWiseAdaGrad",
             "partial_rowwise_adam": "PartialRowWiseAdam"}
    # (an older tree, timed or compared with --tree, may lack an optimizer: its arms are left out)
    opt_t = {k: getattr(Optimizer_t, v) for k, v in names.items() if hasattr(Optimizer_t, v)}
    dev = torch.device("cuda")
    EV = a.ev
    max_rows = a.max_rows or (500_000 if a.digests else 4_000_000 * 128 // EV)
    rows = [min(s, max_rows) for s in CRITEO_TB_TABLE_SIZES]
    hot = list(CRITEO_TB_MULTI_HOT)
    if a.keys == "uniform":      # no heavy rows: tables whose rows occur 16 times on average at most
        keep = [i for i in range(len(rows)) if BATCH * hot[i] <= 16 * rows[i]]
        rows, hot = [rows[i] for i in keep], [hot[i] for i in keep]
    n = len(rows)
    gen = torch.Generator().manual_seed(0)
    lookups, roff, koff, keys = [], 0, 0, []
    width = n * EV
    for i in range(n):
        lookups.append(E.LookupDesc(table_row_off=roff, key_off=koff, out_off=i * EV, grad_off=i * EV,
                                    hotness=hot[i], key_stride=hot[i], num_shards=1, shard_idx=0,
                                    out_stride=width, grad_stride=width, combiner=0, ev_size=EV, rows=rows[i]))
        if a.keys == "uniform":
            keys.append(torch.randint(0, rows[i], (BATCH * hot[i],), generator=gen, dtype=torch.int32))
            most = int(torch.unique(keys[-1], return_counts=True)[1].max())
            if most > 64:
                raise SystemExit(f"bench_emb_update: a row of table {i} occurs {most} times: it would be heavy")
        else:
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
    out = torch.zeros(BATCH * width, dtype=torch.bfloat16, device=dev)
    torch.manual_seed(0)
    if a.digests:     # multiples of 2^-12: a row's sum is exact, whatever order the index lists its buckets in
        grad = (torch.randint(-64, 65, (BATCH * width,), device=dev) / 4096).to(torch.bfloat16)
    else:
        grad = (torch.randn(BATCH * width, device=dev) * 1e-3).to(torch.bfloat16)
    w32 = torch.empty(total_rows * EV, device=dev).uniform_(-0.01, 0.01)
    tables = {"fp32": w32, "bf16": w32.to(torch.bfloat16)}
    opts = [o for o in parse_opts(a.opts) if o in opt_t]
    # arms: (optimizer, state dtype or None); state buffers per dtype, shared by the arms
    arms = []
    for o in opts:
        arms += [(o, sd) for sd in ("fp32", "bf16")] if STATES[o] else [(o, None)]
    need = max([STATES[o] for o, sd in arms] + [0])
    sdt = {"fp32": torch.float32, "bf16": torch.bfloat16}
    bufs = {sd: [torch.zeros(total_rows * EV, dtype=sdt[sd], device=dev) for _ in range(need)]
            for sd in {sd for _, sd in arms if sd}}
    if any(o in ROW_STATE for o in opts):
        bufs["row"] = [torch.zeros(total_rows, device=dev)]
    ws = E.UniqueWorkspace(pairs, EV, dev, indexed=True)
    lr_t = torch.full((1,), 1e-3, device=dev)
    st_t = torch.ones(1, dtype=torch.int32, device=dev)
    hp = {"epsilon": 1e-8, "sr_seed": 1, "beta1": 0.9, "beta2": 0.999}

    def arm_name(o, sd):
        return f"{o}_{sd}_state" if sd else o

    def states(o, sd):
        s = bufs.get(sd, [])[:STATES[o]]
        if o in ROW_STATE:
            s.insert(ROW_STATE[o], bufs["row"][0])
        return s + [None] * (2 - len(s))

    def fwd(w):
        E.forward(lookups, ld, tables[w], EV, [key_d], [out], BATCH)

    def bwd(arm, w):
        o, sd = arm
        s0, s1 = states(o, sd)
        E.bwd_index(lookups, ld, tables[w], EV, [key_d], BATCH, ws)
        E.bwd_reduce_update(opt_t[o], lookups, ld, tables[w], s0, s1, EV, [key_d], [grad], BATCH, ws, hp,
                            lr_t, st_t)

    if a.digests:       # every arm from the same weights and zero state; one JSON object on the last line
        res = {}
        for w in tables:
            first = tables[w].clone()
            for arm in arms:
                tables[w].copy_(first)
                for s in states(*arm):
                    if s is not None:
                        s.zero_()
                for _ in range(a.steps):
                    bwd(arm, w)
                torch.cuda.synchronize()
                res[f"{arm_name(*arm)}/{w}"] = {k: checksum(t) for k, t in
                                                zip(("table", "s0", "s1"), [tables[w]] + states(*arm)) if t is not None}
        E.check_workspace_overflow(ws, "benchmark")
        print(json.dumps(res))
        return 0

    def timed(fn, *args):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            fn(*args)
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / a.iters

    def reset(arm):
        for s in states(*arm):
            if s is not None:
                s.zero_()

    for w in tables:
        for _ in range(a.warmup):
            fwd(w)
        for arm in arms:
            reset(arm)
            for _ in range(a.warmup):
                bwd(arm, w)
    torch.cuda.synchronize()
    res = {k: [] for k in [(w, "forward") for w in tables] + [(w, arm) for w in tables for arm in arms]}
    for _ in range(a.rounds):
        for w in tables:                     # every arm once per round
            res[(w, "forward")].append(timed(fwd, w))
            for arm in arms:
                reset(arm)
                res[(w, arm)].append(timed(bwd, arm, w))
    E.check_workspace_overflow(ws, "benchmark")
    print(f"# {n} tables, {total_rows} rows x {EV}, batch {BATCH}, {pairs} keys per step, {uniq} distinct rows",
          flush=True)

    def line(rec, ts, nbytes):
        ts = sorted(ts)
        ms = ts[len(ts) // 2]
        rec.update({"ev": EV, "ms": round(ms, 4), "min_ms": round(ts[0], 4), "max_ms": round(ts[-1], 4),
                    "nominal_MB": round(nbytes / 1e6, 1), "nominal_GBps": round(nbytes / ms / 1e6, 1),
                    "device": name, "power_limit": plim})
        print(json.dumps(rec), flush=True)

    for w, t in tables.items():
        wb = t.element_size()
        line({"weights": w, "phase": "forward"}, res[(w, "forward")],
             pairs * EV * wb + pairs * 4 + BATCH * width * 2)
        for o, sd in arms:
            # weight read + write and state read + write per distinct row, one bf16 gradient row + locator per key
            srow = EV * 2 * STATES[o] * (sdt[sd].itemsize if sd else 0) + (8 if o in ROW_STATE else 0)
            row_bytes = EV * 2 * wb + srow
            line({"optimizer": arm_name(o, sd), "weights": w, "phase": "fused backward",
                  "update_bytes_per_row": row_bytes}, res[(w, (o, sd))], uniq * row_bytes + pairs * (EV * 2 + 4))
    return 0


def check_bits(a):
    """Digests of every arm under this tree and (twice) under a.check_bits, one process each, compared."""
    runs = []
    for tree in (a.tree, a.check_bits, a.check_bits):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--tree", tree, "--digests", "--opts", a.opts,
                            "--ev", str(a.ev), "--steps", str(a.steps), "--max-rows", str(a.max_rows),
                            "--keys", a.keys], capture_output=True, text=True)
        if r.returncode != 0:
            print(r.stdout[-2000:] + r.stderr[-4000:], file=sys.stderr)
            return 1
        runs.append(json.loads(r.stdout.strip().splitlines()[-1]))
    mine, other, again = runs
    bad = 0
    for arm in sorted(set(mine) - set(other)):     # optimizers TREE does not have
        print(json.dumps({"arm": arm, "new": True}), flush=True)
    for arm in other:
        same = {k: mine.get(arm, {}).get(k) == v for k, v in other[arm].items()}
        stable = {k: again[arm][k] == v for k, v in other[arm].items()}
        fail = any(stable[k] and not same[k] for k in same)
        bad += fail
        print(json.dumps({"arm": arm, "equal": same, "other_tree_equals_itself": stable, "fail": fail}), flush=True)
    print(json.dumps({"check_bits": os.path.abspath(a.check_bits), "keys": a.keys, "ev": a.ev, "steps": a.steps,
                      "arms": len(other), "failed": bad}), flush=True)
    return 1 if bad or not set(other) <= set(mine) else 0


def full_model(a, name, plim):
    from hugectr_b200.models.dlrm import CRITEO_TB_TABLE_SIZES, build_dlrm_dcnv2
    torch.cuda.set_device(0)
    t0 = time.time()
    opt = "partial_rowwise_adam" if "partial_rowwise_adam" in parse_opts(a.opts) else "rowwise_adagrad"
    sizes = [min(s, a.max_rows) if a.max_rows else s for s in CRITEO_TB_TABLE_SIZES]
    m = build_dlrm_dcnv2(batchsize=BATCH, num_gpus=1, table_sizes=sizes, embedding_optimizer=opt,
                         weight_dtype="bf16", use_cuda_graph=True)
    m.compile()
    e = m.ebcs_train[0]
    tb = sum(g.table.numel() * g.table.element_size() for g in e.groups)
    sb = sum(s.numel() * s.element_size() for g in e.groups for s in (g.s0, g.s1) if s is not None)
    print(f"# built in {time.time() - t0:.0f} s: {opt}, {sum(sizes)} rows (cap {a.max_rows or 'none'}), tables "
          f"{tb / 1e9:.2f} GB, state {sb / 1e9:.2f} GB", flush=True)
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
    print(json.dumps({"mode": "full-model", "optimizer": opt, "row_cap": a.max_rows or None, "rows": sum(sizes),
                      "table_GB": round(tb / 1e9, 2), "state_GB": round(sb / 1e9, 3),
                      "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                      "step_ms": round(ms, 3), "steps": a.steps, "final_loss": loss, "batch": BATCH,
                      "device": name, "power_limit": plim}), flush=True)
    return 0 if loss == loss else 1


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--opts", default="adagrad,rowwise_adagrad")
    ap.add_argument("--ev", type=int, default=128, choices=(128, 256))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-rows", type=int, default=0)
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--full-model", action="store_true")
    ap.add_argument("--steps", type=int, default=0, help="full model: 20 training steps; --check-bits: 3 updates")
    ap.add_argument("--check-bits", default="", metavar="TREE",
                    help="compare the updated weights and states of every arm with TREE's, bit for bit")
    ap.add_argument("--keys", default="power-law", choices=("power-law", "uniform"))
    ap.add_argument("--digests", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args(argv)
    a.steps = a.steps or (3 if a.check_bits or a.digests else 20)
    parse_opts(a.opts)
    if a.check_bits and not os.path.isdir(os.path.join(a.check_bits, "hugectr_b200")):
        raise SystemExit(f"bench_emb_update: {a.check_bits} holds no hugectr_b200 package")
    if not os.path.isdir(os.path.join(a.tree, "hugectr_b200")):
        raise SystemExit(f"bench_emb_update: {a.tree} holds no hugectr_b200 package")
    if not torch.cuda.is_available():
        print("bench_emb_update: needs a CUDA device (an H100); nothing was measured", file=sys.stderr)
        return 1
    if a.check_bits:
        return check_bits(a)
    sys.path.insert(0, os.path.abspath(a.tree))
    name, plim = card()
    print(f"# device: {name}, power limit {plim}, tree {os.path.abspath(a.tree)}", flush=True)
    return full_model(a, name, plim) if a.full_model else kernels(a, name, plim)


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
