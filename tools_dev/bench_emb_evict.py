"""Device time of the evicting dynamic-table translate (touch + insert-or-evict + re-initialisation) against the
growing dynamic table's translate on the same keys, and of the lookup + fused backward behind each, with and
without admission (admit_threshold).

  python tools_dev/bench_emb_evict.py [--steps 20] [--warmup 5] [--pool 1000000] [--capacity 393216]
                                      [--ev 128] [--strategy lru|lfu[,...]] [--admit-threshold 1[,2,4]]
                                      [--admit-decay-steps 0] [--batches 8]

Shapes of tools_dev/bench_emb_update.py: the 26 DLRM-DCNv2 tables, batch 6912, the DCNv2 multi-hot sizes,
power-law keys (alpha 1.1), here drawn from a pool of --pool keys per table and scrambled into 64-bit ids, in
--batches pre-drawn batches that the steps cycle through (every key of a batch recurs --batches steps later; a
value of at least --warmup + --steps gives a stream that does not repeat).
Every table is dynamic: the evicting collection holds --capacity rows per table (below the distinct keys of
the pool, so eviction is in steady state after the warm-up), the growing one enough rows for the whole pool
(it never overflows).  Both run AdaGrad with fp32 weights and activations.  Phases are timed with CUDA events
around the translate (forward_begin) and around the lookup + backward, median over --steps steps.  Prints one
JSON line per collection with the card name and its power limit, and the admitted / evicted / dropped counters of
the evicting one.  Every strategy of --strategy and the growing table run once per threshold of
--admit-threshold; each line also carries the rejected positions, the rows in use at the end, and the fraction of
the timed steps' key occurrences whose key had a row before the step (read with the read-only get, outside the
timed windows).  Without a CUDA device it exits and measures nothing.
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


def batches(hot, pool, n_batches, dev):
    """n_batches feature-major key slabs: power-law indices into the pool, scrambled into 64-bit ids"""
    from hugectr_b200.data.batch import power_law_keys
    gen = torch.Generator().manual_seed(0)
    out = []
    for _ in range(n_batches):
        ks = []
        for i, h in enumerate(hot):
            idx = power_law_keys(BATCH * h, pool, 1.1, gen, torch.int64)
            ks.append((idx * 0x5851F42D4C957F2D + ((i * 0x632BE59BD9B4E019) & ((1 << 62) - 1))) & ((1 << 62) - 1))
        out.append(torch.cat(ks).to(dev))
    return out


def collection(hot, ev, capacity, strategy, dev, admit_threshold=1, admit_decay_steps=0):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    kw = dict(max_capacity=capacity, evict_strategy=strategy) if strategy else dict(init_capacity=capacity)
    if admit_threshold > 1:
        kw.update(admit_threshold=admit_threshold, admit_decay_steps=admit_decay_steps)
    tabs = [EmbeddingTableConfig(str(i), -1, ev, **kw) for i in range(len(hot))]
    cfg.embedding_lookup(tabs, [f"s{i}" for i in range(len(hot))], "emb", ["sum"] * len(hot))
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.0, epsilon=1e-8)
    return EmbeddingCollection(cfg, BATCH, {f"s{i}": h for i, h in enumerate(hot)}, dev, torch.float32,
                               Comm.single(dev), opt, key_dtype=torch.int64, seed=1)


def present(e, keys):
    """(key occurrences of the batch whose key has a row, occurrences), by the tables' read-only get"""
    from hugectr_b200.embedding.hashtable import SetAssocTable
    hit = torch.zeros((), dtype=torch.int64, device=keys.device)
    for gl in e.glookups:
        k = keys[gl["key_off"]:gl["key_off"] + e.b * gl["hotness"]].view(1, -1).clone()
        ht = e._dyn_tables[(gl["table"], 0, 0)]
        if isinstance(ht, SetAssocTable):
            ht.get(k, 0, k.shape[1])
            rows = k
        else:
            rows = ht.get(k.view(-1))
        hit += (rows >= 0).sum()
    return int(hit), int(e.user_key_elems)


def run(e, keys, steps, warmup):
    dev = keys[0].device
    lr, st = torch.tensor([0.01], device=dev), torch.tensor([1], dtype=torch.int32, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tr, lb = [], []
    hit = tot = 0
    for it in range(warmup + steps):
        if it >= warmup:
            h, n = present(e, keys[it % len(keys)])
            hit, tot = hit + h, tot + n
        e.set_keys(keys[it % len(keys)])
        ev[0].record()
        e.forward_begin()
        ev[1].record()
        e.forward_compute()
        e.forward_end()
        e.top_grad["emb"].fill_(1e-3)
        e.backward(lr, st)
        ev[2].record()
        torch.cuda.synchronize()
        if it >= warmup:
            tr.append(ev[0].elapsed_time(ev[1]))
            lb.append(ev[1].elapsed_time(ev[2]))
    med = lambda x: sorted(x)[len(x) // 2]
    return med(tr), med(lb), hit / max(tot, 1)


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pool", type=int, default=1_000_000)
    ap.add_argument("--capacity", type=int, default=393_216)
    ap.add_argument("--ev", type=int, default=128)
    ap.add_argument("--strategy", default="lru", help="comma-separated evicting strategies (lru, lfu)")
    ap.add_argument("--admit-threshold", default="1", help="comma-separated admit_threshold values")
    ap.add_argument("--admit-decay-steps", type=int, default=0)
    ap.add_argument("--batches", type=int, default=8, help="pre-drawn batches the steps cycle through")
    a = ap.parse_args(argv)
    strategies = a.strategy.split(",")
    if any(x not in ("lru", "lfu") for x in strategies):
        raise SystemExit(f"--strategy: lru and / or lfu, not {a.strategy!r}")
    thresholds = [int(x) for x in a.admit_threshold.split(",")]
    if not torch.cuda.is_available():
        raise SystemExit("bench_emb_evict: no CUDA device; nothing measured")
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT
    hot = list(CRITEO_TB_MULTI_HOT)
    dev = torch.device("cuda")
    name, plim = card()
    keys = batches(hot, a.pool, a.batches, dev)
    n_keys = sum(BATCH * h for h in hot)
    runs = [("evicting", s_, a.capacity) for s_ in strategies] + [("growing", None, a.pool + a.pool // 4)]
    for thr in thresholds:
        for label, strategy, cap in runs:
            e = collection(hot, a.ev, cap, strategy, dev, thr, a.admit_decay_steps if thr > 1 else 0)
            t_tr, t_lb, had_row = run(e, keys, a.steps, a.warmup)
            res = {"collection": label, "strategy": strategy, "rows_per_table": cap, "tables": len(hot),
                   "batch": BATCH, "keys_per_step": n_keys, "key_pool_per_table": a.pool, "batches": a.batches,
                   "ev": a.ev,
                   "admit_threshold": thr, "admit_decay_steps": a.admit_decay_steps if thr > 1 else 0,
                   "translate_ms": round(t_tr, 4), "lookup_backward_ms": round(t_lb, 4),
                   "had_row_fraction": round(had_row, 4), "card": name, "power_limit": plim}
            if strategy:
                tot = {"live": 0, "admitted": 0, "evicted": 0, "dropped": 0}
                for v in e.eviction_stats().values():
                    for k in tot:
                        tot[k] += v[k]
                res.update(tot)
                res["set_bytes_per_step"] = n_keys * 256
            else:
                # a growing table admits by handing out rows, and never evicts; it drops nothing below its rows
                rows = sum(ht.size() for ht in e._dyn_tables.values())
                res.update(live=rows, admitted=rows, evicted=0, dropped=0)
            res["rejected"] = sum(v["rejected"] for v in e.admission_stats().values())
            print(json.dumps(res), flush=True)
            del e
            torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
