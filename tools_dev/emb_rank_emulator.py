"""Emulate ONE rank of an N-GPU job on a single GPU to tune the owner-side embedding kernels cheaply.

The embedding collection is built for (world=N, rank=r) in fused mode over a stub communicator whose
"symmetric heap" is local memory: every source rank's row of the key inbox is filled by the real key
dispatch of that rank's routes, so the kernels run with N source-rank key / gradient buffers exactly as
on the real machine (same lookup descriptors, same requester-side split of row-sharded tables, same
index / reduce+update work) -- only the buffers are local instead of peer mapped.  The sharding plan is
the benchmark's for the full table sizes; ``--cap-rows`` only shrinks the tables.  Usage:

    python tools_dev/emb_rank_emulator.py --world 8 --rank 0 [--cap-rows 4000000] [--batch 6912]
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hugectr_b200.data.batch import power_law_keys  # noqa: E402
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,  # noqa: E402
                                               EmbeddingTableConfig)
from hugectr_b200.enums import Optimizer_t  # noqa: E402
from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES  # noqa: E402
from hugectr_b200.solver import CreateOptimizer  # noqa: E402
from hugectr_b200.tools.planner import generate_plan  # noqa: E402


class EmuComm:
    """rank r of N without peers: collectives are no-ops (the buffers are pre-filled by the tool), the
    symmetric heap is local memory and every rank's "peer" buffer is the local one"""

    def __init__(self, rank, world, device):
        self.rank, self.world_size, self.device = rank, world, device
        self.p2p_available = True
        self.emulated = True
        self.num_nodes = 1

    def symm_alloc(self, numel, dtype): return torch.zeros(max(int(numel), 1), dtype=dtype, device=self.device)[:numel]
    def peer_ptrs(self, t): return [t] * self.world_size
    def barrier_device(self): pass

    def all_gather(self, out, inp): pass
    def all_to_all(self, out, inp): out.copy_(inp)
    def all_reduce(self, t): return t
    def barrier(self): pass
    def broadcast(self, t, src=0): return t
    def all_gather_object(self, obj): return [obj] * self.world_size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--rank", type=int, default=0)
    ap.add_argument("--batch", type=int, default=6912)
    ap.add_argument("--cap-rows", type=int, default=0)
    ap.add_argument("--ev", type=int, default=128)
    ap.add_argument("--cpu", action="store_true", help="reference path smoke test (tiny sizes)")
    a = ap.parse_args()
    dev = torch.device("cpu" if a.cpu else "cuda")
    sizes = list(CRITEO_TB_TABLE_SIZES)
    hot = list(CRITEO_TB_MULTI_HOT)
    n, N, b = len(sizes), a.world, a.batch
    plan = generate_plan(sizes, hot, N, ev_size=a.ev)
    if a.cap_rows:
        sizes = [min(s, a.cap_rows) for s in sizes]
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig(str(i), sizes[i], a.ev) for i in range(n)],
                         [f"d{i}" for i in range(n)], "emb", ["sum"] * n)
    cfg.shard(plan[0], plan[1])
    act = torch.float32 if a.cpu else torch.bfloat16
    e = EmbeddingCollection(cfg, b, {f"d{i}": hot[i] for i in range(n)}, dev, act, EmuComm(a.rank, N, dev),
                            CreateOptimizer(Optimizer_t.AdaGrad, epsilon=1e-8), fused=True)
    g = torch.Generator().manual_seed(0)
    kc = e.key_chans[0]
    for r in range(N):                                   # every source rank's batch, dispatched into my inbox
        keys = torch.cat([power_law_keys(b * hot[i], sizes[i], 1.1, g).to(e.key_dtype) for i in range(n)])
        slab = e.key_slab if r == a.rank else torch.zeros_like(e.key_slab)
        slab[:keys.numel()].copy_(keys)
        routes = [x for x in e._build_key_routes(r)[0] if x.dst_rank == a.rank]
        E.dispatch(slab, routes, E.routes_to_device(routes, dev), kc.peers, kc.nnz_peers)
    e.grads_all.normal_(0, 0.01)
    lr = torch.tensor([0.004], device=dev)
    st = torch.ones(1, dtype=torch.int32, device=dev)
    mp = [grp for grp in e.groups if grp.kind == "mp"]

    def timeit(fn, reps=5):
        fn()
        if dev.type == "cuda":
            torch.cuda.synchronize()
            s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(reps):
                fn()
            t.record()
            torch.cuda.synchronize()
            return s.elapsed_time(t) / reps * 1e3
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e6

    def bwd():
        e.backward_index()
        e._index_done = False
        for grp in mp:
            e._accum_update(grp, lr, st)

    print(f"world {N} rank {a.rank}: local mp lookups {sum(len(g_.lookups) for g_ in mp)}, "
          f"split row-sharded lookups {sum('split_off' in gl for gl in e.glookups)}")
    print("forward (owner side, all source ranks)  us:", round(timeit(e.forward_compute), 1))
    print("backward index + reduce + update        us:", round(timeit(bwd), 1))


if __name__ == "__main__":
    main()
