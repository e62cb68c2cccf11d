"""Sharding planner: greedy cost model -> (shard_matrix, shard_strategy).

Capabilities of the reference planner (samples/dlrm/sharding/planner.py:22-327,
generate_plan.py:23-131): data-parallel threshold for tiny tables, hot-table split (row-wise over
several GPUs) when one table's lookup cost exceeds the balanced share, memory-cap split, then
greedy longest-processing-time placement by cost = hotness * (1 + comm/mem ratio).
H100 SXM data-sheet rates: HBM3 3.35 TB/s, NVLink 450 GB/s per direction -> ratio ~7.4 (not measured here).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple


def generate_plan(table_sizes: Sequence[int], multi_hot: Sequence[int], num_gpus: int,
                  ev_size: int = 128, plan: str = "auto", dp_threshold_rows: int = 4096,
                  mem_comm_bw_ratio: float = 3.35e12 / 450e9, mem_cap_gb: float = 70.0,
                  bytes_per_elem: int = 8, num_nodes: int = 1) -> Tuple[List[List[int]], list]:
    """``num_nodes`` > 1 (hier-auto of the reference planner): the shards of a row-split table are
    kept inside ONE node (the least loaded) so that the hierarchical exchange reduces their partial
    sums before anything crosses the node boundary."""
    n = len(table_sizes)
    names = [str(i) for i in range(n)]
    if num_gpus == 1:
        return [[1] * n], [("mp", names)]
    if plan == "round_robin":
        sm = [[1 if (t % num_gpus) == g else 0 for t in range(n)] for g in range(num_gpus)]
        return sm, [("mp", names)]
    if plan == "uniform":      # every table row-sharded over every GPU
        return [[1] * n for _ in range(num_gpus)], [("mp", names)]
    dp = [t for t in range(n) if table_sizes[t] <= dp_threshold_rows]
    mp = [t for t in range(n) if t not in dp]
    # cost of a table = rows gathered per sample (HBM) + pooled vector sent per shard (NVLink)
    def cost(t, k):
        return multi_hot[t] / k + mem_comm_bw_ratio * 0.5
    total = sum(cost(t, 1) for t in mp)
    share = total / num_gpus
    shards = {}
    for t in mp:
        k = 1
        mem_gb = table_sizes[t] * ev_size * bytes_per_elem / 1e9
        while k < num_gpus and (cost(t, k) > 1.25 * share or mem_gb / k > mem_cap_gb):
            k *= 2
        shards[t] = min(k, num_gpus)
    load = [0.0] * num_gpus
    mem = [0.0] * num_gpus
    sm = [[0] * n for _ in range(num_gpus)]
    gpn = num_gpus // max(1, num_nodes)
    for t in sorted(mp, key=lambda t: -cost(t, shards[t]) * shards[t]):
        k = shards[t]
        cand = range(num_gpus)
        if num_nodes > 1 and 1 < k <= gpn:
            node_load = [sum(load[nd * gpn:(nd + 1) * gpn]) for nd in range(num_nodes)]
            nd = min(range(num_nodes), key=lambda i: node_load[i])
            cand = range(nd * gpn, (nd + 1) * gpn)
        order = sorted(cand, key=lambda g: (load[g], mem[g]))
        for g in order[:k]:
            sm[g][t] = 1
            load[g] += cost(t, k)
            mem[g] += table_sizes[t] * ev_size * bytes_per_elem / 1e9 / k
    for t in dp:
        for g in range(num_gpus):
            sm[g][t] = 1
    strategy = []
    if mp:
        strategy.append(("mp", [names[t] for t in mp]))
    if dp:
        strategy.append(("dp", [names[t] for t in dp]))
    return sm, strategy


# ------------------------------------------------------------------------------------------------
# heterogeneous planner: per-table widths / combiners, row- AND column-wise splits, time-based costs
class HardwareModel:
    """Per-GPU rates the cost model divides by (defaults: H100 SXM data-sheet bandwidths, not measured here):
    random 512-byte row gathers are assumed to run at ~0.8 of the 3.35 TB/s HBM3 bandwidth, the read-modify-write
    sparse update at ~0.55, one NVLink direction carries 450 GB/s, inter-node links 50 GB/s per GPU; 70 of the
    80 GB are given to embedding tables."""

    def __init__(self, hbm_gbps: float = 3350.0, gather_eff: float = 0.8, update_eff: float = 0.55,
                 nvlink_gbps: float = 450.0, internode_gbps: float = 50.0, hbm_capacity_gb: float = 70.0):
        self.hbm, self.gather_eff, self.update_eff = hbm_gbps * 1e9, gather_eff, update_eff
        self.nvlink, self.internode, self.capacity = nvlink_gbps * 1e9, internode_gbps * 1e9, hbm_capacity_gb * 1e9


def plan_tables(table_sizes: Sequence[int], hotness: Sequence[int], ev_sizes, num_gpus: int,
                global_batch: int = 65536, combiners: Sequence[str] = None, num_nodes: int = 1,
                hw: HardwareModel = None, weight_bytes: int = 4, state_bytes: int = 4,
                act_bytes: int = 2, dp_threshold_bytes: float = 4e6, min_rows_per_shard: int = 1024,
                min_cols_per_shard: int = 32, balance_tol: float = 1.10, per_key_bytes: float = 96.0,
                state_row_bytes: int = 0):
    """Plan for tables of different widths and combiners (the role of the reference's larger planner,
    benchmarks/embedding_collection/hugectr/sharding/planner.py:38-620: cost model with per-table
    ev sizes, hot-shard / out-of-memory splits that may be column-wise, hierarchical mode).

    Costs are seconds per training step on the owning GPU:
      lookup   = keys hitting the shard * row bytes / (HBM * gather_eff)            (forward gather)
      update   = 2 * unique-ish rows * (weight+state) bytes / (HBM * update_eff)    (backward RMW)
      per key  = per_key_bytes of index-build / sort / key traffic for every key the shard sees
                 (independent of the row width: NOT reduced by a column split)
      exchange = pooled (or per-key for ``concat``) vectors of the WHOLE global batch leaving the shard
                 and their gradients coming back, over NVLink (intra-node) or the NIC share
    A row split by k divides lookup / update by k but every shard still sends a full-width partial
    vector (exchange unchanged per shard -> total x k); a column split by c divides all three by c.
    Tables whose replicated gradient all-reduce is cheaper than the exchange and that fit
    ``dp_threshold_bytes`` become data-parallel.  The most expensive shard is split until the critical
    GPU is within ``balance_tol`` of the mean or nothing can be split; shards are then placed
    longest-first on the least-loaded GPU that does not hold the table yet (same node for the shards
    of one table when ``num_nodes`` > 1) and that has memory left.

    ``state_bytes`` is optimizer state per weight, ``state_row_bytes`` per row and column slice (row-wise
    AdaGrad: 4, with ``state_bytes=0``; partial row-wise Adam: 4, with ``state_bytes`` 4 or 2 for its fp32 or bf16
    first moment); both enter the memory and update terms.

    Returns (shard_matrix, shard_strategy, report); strategy entries are ``name`` or
    ``(name, column_wise_factor)``."""
    hw = hw or HardwareModel()
    n = len(table_sizes)
    evs = [int(ev_sizes)] * n if isinstance(ev_sizes, int) else [int(e) for e in ev_sizes]
    comb = list(combiners) if combiners else ["sum"] * n
    names = [str(i) for i in range(n)]
    gpn = max(1, num_gpus // max(1, num_nodes))
    link = hw.nvlink if num_nodes == 1 else (hw.nvlink * (gpn - 1) + hw.internode * (num_gpus - gpn)) / max(1, num_gpus - 1)

    def mem(t, k=1, c=1):
        return table_sizes[t] * (evs[t] * (weight_bytes + state_bytes) / c + state_row_bytes) / k

    def vec_per_sample(t):
        return hotness[t] if comb[t] == "concat" else 1

    def shard_cost(t, k, c):
        keys = global_batch * hotness[t] / k
        row = evs[t] / c
        lookup = keys * row * weight_bytes / (hw.hbm * hw.gather_eff)
        update = 2.0 * min(keys, table_sizes[t] / k) * (row * (weight_bytes + state_bytes) + state_row_bytes) \
            / (hw.hbm * hw.update_eff) \
            + keys * row * act_bytes / hw.hbm
        exch = 2.0 * global_batch * vec_per_sample(t) * row * act_bytes * (num_gpus - 1) / num_gpus / link
        return lookup + update + exch + keys * per_key_bytes / hw.hbm

    def dp_cost(t):
        keys = global_batch / num_gpus * hotness[t]
        lookup = keys * evs[t] * weight_bytes / (hw.hbm * hw.gather_eff)
        allreduce = 2.0 * table_sizes[t] * evs[t] * 4 / link
        dense_update = 3.0 * table_sizes[t] * (evs[t] * (weight_bytes + state_bytes) + state_row_bytes) / hw.hbm
        return lookup + allreduce + dense_update + keys * per_key_bytes / hw.hbm

    if num_gpus == 1:
        return [[1] * n], [("mp", names)], {"step_cost_us": [sum(shard_cost(t, 1, 1) for t in range(n)) * 1e6],
                                            "memory_gb": [sum(mem(t) for t in range(n)) / 1e9],
                                            "imbalance": 1.0, "splits": {}, "dp": []}
    dp = [t for t in range(n) if mem(t) <= dp_threshold_bytes and dp_cost(t) * num_gpus <= shard_cost(t, 1, 1) * 2
          and comb[t] != "concat"]
    mp = [t for t in range(n) if t not in dp]
    split = {t: [1, 1] for t in mp}                      # table -> [row shards k, column parts c]
    dp_load = sum(dp_cost(t) for t in dp)

    def can_row(t):
        k, c = split[t]
        return k * c * 2 <= num_gpus and table_sizes[t] / (k * 2) >= min_rows_per_shard

    def can_col(t):
        k, c = split[t]
        return k * c * 2 <= num_gpus and evs[t] % (c * 2) == 0 and evs[t] / (c * 2) >= min_cols_per_shard \
            and comb[t] != "concat"

    def split_once(t):
        """prefer the split with the lower resulting per-shard cost (rows when the table is big and
        lookup-bound, columns when the exchange dominates or the table has few rows)"""
        k, c = split[t]
        opts = []
        if can_row(t):
            opts.append((shard_cost(t, k * 2, c), 0))
        if can_col(t):
            opts.append((shard_cost(t, k, c * 2), 1))
        if not opts:
            return False
        split[t][min(opts)[1]] *= 2
        return True

    cap = hw.capacity
    for t in mp:                                          # out-of-memory splits first
        while mem(t, *split[t]) > cap and split_once(t):
            pass
    for _ in range(8 * max(1, len(mp))):
        costs = {t: shard_cost(t, *split[t]) for t in mp}
        total = sum(costs[t] * split[t][0] * split[t][1] for t in mp)
        share = total / num_gpus
        worst = max(mp, key=lambda t: costs[t]) if mp else None
        if worst is None or costs[worst] <= balance_tol * share or not split_once(worst):
            break
    # placement: longest shard first
    load = [dp_load] * num_gpus
    used = [sum(mem(t) for t in dp)] * num_gpus
    sm = [[0] * n for _ in range(num_gpus)]
    order = sorted(mp, key=lambda t: -shard_cost(t, *split[t]))
    for t in order:
        k, c = split[t]
        cnt, cst, mb = k * c, shard_cost(t, k, c), mem(t, k, c)
        cand = list(range(num_gpus))
        if num_nodes > 1 and 1 < cnt <= gpn:
            nd = min(range(num_nodes), key=lambda i: sum(load[i * gpn:(i + 1) * gpn]))
            cand = list(range(nd * gpn, (nd + 1) * gpn))
        fit = [g for g in cand if used[g] + mb <= cap] or cand
        for g in sorted(fit, key=lambda g: (load[g], used[g]))[:cnt]:
            sm[g][t] = 1
            load[g] += cst
            used[g] += mb
        if sum(sm[g][t] for g in range(num_gpus)) < cnt:           # not enough GPUs with memory left
            for g in sorted(cand, key=lambda g: (sm[g][t], load[g]))[:cnt - sum(sm[g][t] for g in range(num_gpus))]:
                sm[g][t] = 1
                load[g] += cst
                used[g] += mb
    for t in dp:
        for g in range(num_gpus):
            sm[g][t] = 1
    strategy = []
    if mp:
        strategy.append(("mp", [names[t] if split[t][1] == 1 else (names[t], split[t][1]) for t in mp]))
    if dp:
        strategy.append(("dp", [names[t] for t in dp]))
    report = {"step_cost_us": [x * 1e6 for x in load], "memory_gb": [x / 1e9 for x in used],
              "imbalance": max(load) / (sum(load) / num_gpus) if sum(load) else 1.0,
              "splits": {names[t]: tuple(split[t]) for t in mp if split[t] != [1, 1]}, "dp": [names[t] for t in dp]}
    return sm, strategy, report


def plan_report(table_sizes: Sequence[int], multi_hot: Sequence[int], shard_matrix, ev_size: int = 128,
                bytes_per_elem: int = 8) -> dict:
    """per-GPU lookup load (rows gathered per sample) and table memory (GB) of a plan"""
    g = len(shard_matrix)
    n = len(table_sizes)
    k = [sum(shard_matrix[r][t] for r in range(g)) for t in range(n)]
    load = [sum(multi_hot[t] / k[t] for t in range(n) if shard_matrix[r][t]) for r in range(g)]
    mem = [sum(table_sizes[t] * ev_size * bytes_per_elem / 1e9 / k[t] for t in range(n)
               if shard_matrix[r][t]) for r in range(g)]
    return {"shards_per_table": k, "lookups_per_sample": load, "memory_gb": mem,
            "imbalance": max(load) / (sum(load) / g) if sum(load) else 1.0}


def save_plan(path: str, shard_matrix, shard_strategy, column_wise=None):
    import json
    with open(path, "w") as f:
        json.dump({"shard_matrix": shard_matrix, "shard_strategy": [[k, list(v)] for k, v in shard_strategy],
                   "shard_column_wise": column_wise or []}, f, indent=1)


def load_plan(path: str):
    import json
    with open(path) as f:
        d = json.load(f)
    return d["shard_matrix"], [(k, v) for k, v in d["shard_strategy"]], d.get("shard_column_wise", [])


def main(argv=None):
    """python -m hugectr_b200.tools.planner --num-gpus 8 [--num-nodes 1] [--plan auto] --out plan.json
    (Criteo-TB DLRM-DCNv2 tables by default; --slot-sizes / --multi-hot override)"""
    import argparse
    from ..models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    ap = argparse.ArgumentParser()
    ap.add_argument("--num-gpus", type=int, required=True)
    ap.add_argument("--num-nodes", type=int, default=1)
    ap.add_argument("--plan", default="auto", choices=["auto", "round_robin", "uniform"])
    ap.add_argument("--slot-sizes", default="")
    ap.add_argument("--multi-hot", default="")
    ap.add_argument("--ev-size", type=int, default=128)
    ap.add_argument("--ev-sizes", default="", help="per-table widths: selects the heterogeneous planner")
    ap.add_argument("--combiners", default="", help="per-table sum|mean|concat (heterogeneous planner)")
    ap.add_argument("--global-batch", type=int, default=65536)
    ap.add_argument("--out", default="")
    a = ap.parse_args(argv)
    sizes = [int(x) for x in a.slot_sizes.split(",")] if a.slot_sizes else CRITEO_TB_TABLE_SIZES
    hot = [int(x) for x in a.multi_hot.split(",")] if a.multi_hot else CRITEO_TB_MULTI_HOT
    if a.ev_sizes or a.combiners:
        evs = [int(x) for x in a.ev_sizes.split(",")] if a.ev_sizes else a.ev_size
        sm, st, rep = plan_tables(sizes, hot, evs, a.num_gpus, a.global_batch,
                                  a.combiners.split(",") if a.combiners else None, a.num_nodes)
        print("step cost per GPU (us):", [round(x, 1) for x in rep["step_cost_us"]])
        print("table memory per GPU (GB):", [round(x, 2) for x in rep["memory_gb"]])
        print("imbalance (max/mean): %.3f" % rep["imbalance"], " splits (rows, cols):", rep["splits"], " dp:", rep["dp"])
        if a.out:
            save_plan(a.out, sm, [(k, [list(x) if isinstance(x, tuple) else x for x in v]) for k, v in st])
        return sm, st
    sm, st = generate_plan(sizes, hot, a.num_gpus, ev_size=a.ev_size, plan=a.plan, num_nodes=a.num_nodes)
    rep = plan_report(sizes, hot, sm, a.ev_size)
    print("lookups/sample per GPU:", [round(x, 1) for x in rep["lookups_per_sample"]])
    print("table memory per GPU (GB):", [round(x, 1) for x in rep["memory_gb"]])
    print("imbalance (max/mean): %.3f" % rep["imbalance"])
    if a.out:
        save_plan(a.out, sm, st)
    return sm, st


if __name__ == "__main__":
    main()
