"""NVLink byte accounting of the fused embedding paths for the benchmark's sharding plan (no GPU needed: the routes
are pure metadata).  Per rank and step: key-dispatch stores, pooled-vector stores (owner -> requester), gradient
push stores; max over ranks.  python tools_dev/nvlink_accounting.py > nvlink_bytes.txt"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,  # noqa: E402
                                               EmbeddingTableConfig, resolve_placement)
from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES  # noqa: E402
from hugectr_b200.tools.planner import generate_plan  # noqa: E402

B, EV, LINK = 6912, 128, 900e9      # per-GPU batch, vector width, NVLink 5 bytes/s per direction


def collection(world, rank):
    n = len(CRITEO_TB_TABLE_SIZES)
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig(str(i), CRITEO_TB_TABLE_SIZES[i], EV) for i in range(n)],
                         [f"d{i}" for i in range(n)], "emb", ["sum"] * n)
    plan = generate_plan(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, world)
    cfg.shard(plan[0], plan[1])
    e = EmbeddingCollection.__new__(EmbeddingCollection)
    e.cfg, e.b, e.world, e.rank, e.device = cfg, B, world, rank, torch.device("cpu")
    e.tables = cfg.tables()
    e.tmap = {t.name: t for t in e.tables}
    e.placement = resolve_placement(cfg, world)
    e.shard_split, e._kb, e._abf = world > 1, 4, True
    e._build_layout({f"d{i}": CRITEO_TB_MULTI_HOT[i] for i in range(n)})
    e._build_key_routes()
    e._build_grad_routes()
    return e


print("NVLink bytes per step of the fused embedding exchange, DLRM-DCNv2 benchmark plan, b = 6912 / GPU, bf16 vectors")
print("(stores leaving a GPU; max over ranks; time at 900 GB/s per direction = the NVLink roofline of the phase)\n")
print(f"{'GPUs':>4} {'key dispatch':>14} {'pooled vectors':>15} {'gradient push':>14} {'fwd us @link':>13} {'bwd us @link':>13}")
for W in (2, 4, 8):
    kmax = omax = gmax = 0
    for r in range(W):
        e = collection(W, r)
        kmax = max(kmax, e.dispatch_key_bytes)
        gmax = max(gmax, e.push_grad_bytes)
        out = 0
        for gl in e.glookups:                     # vectors this rank (as owner) stores into the other requesters
            owners = {o[0] for o in e._mp_owners(gl)}
            if r in owners:
                out += (W - 1) * B * gl["ev"] * 2
        omax = max(omax, out)
    print(f"{W:>4} {kmax / 1e6:>11.1f} MB {omax / 1e6:>12.1f} MB {gmax / 1e6:>11.1f} MB "
          f"{(kmax + omax) / LINK * 1e6:>13.1f} {gmax / LINK * 1e6:>13.1f}")
