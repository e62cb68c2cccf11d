"""Device time of the serving lookup over fp32, bf16 and fp8 (e4m3 + one power-of-two scale per row) tables, at the
DLRM-DCNv2 embedding shapes.

  python tools_dev/bench_emb_fp8.py [--steps 20] [--warmup 5] [--rounds 5] [--ev 128] [--cap-rows 4000000]
                                    [--act bf16] [--full-size]

The 26 Criteo-TB tables, batch 6912, the DCNv2 multi-hot sizes (214 keys per sample), power-law keys (alpha 1.1),
one GPU, lookup only (serving collections: no optimizer state, no gradients).  The three arms are built from the
same fp32 values (bf16 rounds them to nearest, fp8 quantizes them) and live on the card at once, so tables are
capped at --cap-rows rows; each arm still holds several GB, far beyond the 50 MB L2.  Each round times --steps
lookups of each arm between CUDA events, the arms alternating; the result is the median over rounds, printed as
one JSON line with the card name and its power limit, each arm's memory_bytes, the bytes a lookup asks for (computed
from the shapes: one row read per key, the exponent byte per key of fp8, the keys and the pooled outputs) and that
count over the lookup time.  Power-law keys repeat, and the repeated rows come from L2, so this logical rate can
exceed the HBM bandwidth: it is not a share of peak.  ``--full-size`` builds only the fp8 arm at the uncapped
Criteo-TB sizes (204M rows) and reports its memory_bytes and lookup time.  Without a CUDA device it exits and
measures nothing.
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


def collection(sizes, hot, ev, storage, act, dev):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import OptParamsPy
    cfg = EmbeddingCollectionConfig()
    wd = "bf16" if storage == "bf16" else "fp32"
    tabs = [EmbeddingTableConfig(str(i), v, ev, weight_dtype=wd) for i, v in enumerate(sizes)]
    names = [f"s{i}" for i in range(len(hot))]
    cfg.embedding_lookup(tabs, names, "emb", ["sum"] * len(hot))
    return EmbeddingCollection(cfg, BATCH, dict(zip(names, hot)), dev, act, Comm.single(dev), OptParamsPy(),
                               seed=1, is_train=False, fp8_quant=storage == "fp8")


def copy_values(src, dst):
    """dst's tables take src's fp32 values: rounded to nearest (bf16) or quantized (fp8), a chunk of rows at a time"""
    from hugectr_b200.embedding.collection import FP8_STORE_CHUNK_ROWS
    for gs, gd in zip(src.groups, dst.groups):
        if gd.exps is None:
            gd.table.copy_(gs.table)
            continue
        for sl in gd.table_slices:
            lo, n = sl["row_off"], sl["rows"]
            for c in range(lo, lo + n, FP8_STORE_CHUNK_ROWS):
                m = min(FP8_STORE_CHUNK_ROWS, lo + n - c)
                dst._store_rows(gd, sl["table"], torch.arange(c, c + m, device=gd.table.device),
                                gs.table.view(-1, gs.pitch)[c:c + m])
    dst.check_quantized()


def batches(sizes, hot, n, dev):
    from hugectr_b200.data.batch import power_law_keys
    gen = torch.Generator().manual_seed(0)
    return [torch.cat([power_law_keys(BATCH * h, v, 1.1, gen, torch.int32) for v, h in zip(sizes, hot)]).to(dev)
            for _ in range(n)]


def run(e, data, steps, warmup):
    """ms per lookup over ``steps`` lookups between two CUDA events (after ``warmup`` lookups)"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(warmup):
        e.set_keys(data[it % len(data)])
        e.forward(False)
    torch.cuda.synchronize()
    ev[0].record()
    for it in range(steps):
        e.set_keys(data[it % len(data)])
        e.forward(False)
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def lookup_bytes(n_keys, n_out, ev, storage, act_bytes):
    """bytes one lookup moves: a row per key (+ its exponent byte for fp8), the int32 keys, the pooled outputs"""
    row = {"fp32": 4 * ev, "bf16": 2 * ev, "fp8": ev + 1}[storage]
    return n_keys * row + n_keys * 4 + n_out * act_bytes


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ev", type=int, default=128)
    ap.add_argument("--cap-rows", type=int, default=4_000_000)
    ap.add_argument("--act", choices=("fp32", "bf16"), default="bf16")
    ap.add_argument("--full-size", action="store_true")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_emb_fp8: no CUDA device; nothing measured")
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    hot = list(CRITEO_TB_MULTI_HOT)
    sizes = list(CRITEO_TB_TABLE_SIZES) if a.full_size else [min(t, a.cap_rows) for t in CRITEO_TB_TABLE_SIZES]
    dev = torch.device("cuda")
    act = torch.bfloat16 if a.act == "bf16" else torch.float32
    name, plim = card()
    data = batches(sizes, hot, 8, dev)
    n_keys, n_out = BATCH * sum(hot), BATCH * len(hot) * a.ev
    if a.full_size:
        arms = {"fp8": collection(sizes, hot, a.ev, "fp8", act, dev)}
    else:
        arms = {"fp32": collection(sizes, hot, a.ev, "fp32", act, dev)}
        for s in ("bf16", "fp8"):
            arms[s] = collection(sizes, hot, a.ev, s, act, dev)
            copy_values(arms["fp32"], arms[s])
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, e in arms.items():
            times[k].append(run(e, data, a.steps, a.warmup))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    nb = {k: lookup_bytes(n_keys, n_out, a.ev, k, act.itemsize) for k in arms}
    res = {"tables": len(hot), "rows": sum(sizes), "batch": BATCH, "keys_per_lookup": n_keys, "ev": a.ev,
           "cap_rows": None if a.full_size else a.cap_rows, "act": a.act,
           "ms": {k: round(v, 4) for k, v in med.items()},
           "rounds_ms": {k: [round(x, 4) for x in v] for k, v in times.items()},
           "bytes_per_lookup": nb, "logical_GBps": {k: round(nb[k] / med[k] / 1e6, 1) for k in arms},
           "memory_bytes": {k: e.memory_bytes() for k, e in arms.items()},
           "card": name, "power_limit": plim}
    print(json.dumps(res), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
