"""Volumes of the embedding collection's exchanges under the benchmark's sharding plan: every owner receives
exactly the key blocks of the lookups it serves and sends exactly the pooled vectors it produces, on the
collective path (packed variable-size all-to-alls) and on the peer-memory path (dispatch and gradient push
routes).  Nothing may travel as a whole slab."""
import os
import re
import subprocess
import sys

import pytest
import torch

from hugectr_b200.embedding.collection import EmbeddingCollection, EmbeddingCollectionConfig, EmbeddingTableConfig
from hugectr_b200.enums import Optimizer_t
from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
from hugectr_b200.parallel.emu import run_ranks
from hugectr_b200.solver import CreateOptimizer
from hugectr_b200.tools.planner import generate_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")
B, EV = 8, 8
SIZES = [min(s, 4000) for s in CRITEO_TB_TABLE_SIZES]
HOT = list(CRITEO_TB_MULTI_HOT)


def _collection(comm, fused):
    """the benchmark's plan at this rank count (planned for the full tables, tables capped)"""
    n = len(SIZES)
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig(str(i), SIZES[i], EV) for i in range(n)],
                         [f"d{i}" for i in range(n)], "emb", ["sum"] * n)
    plan = generate_plan(CRITEO_TB_TABLE_SIZES, HOT, comm.world_size)
    cfg.shard(plan[0], plan[1])
    return EmbeddingCollection(cfg, B, {f"d{i}": HOT[i] for i in range(n)}, CPU, torch.float32, comm,
                               CreateOptimizer(Optimizer_t.AdaGrad), seed=1, fused=fused)


def _owners(e, gl):
    """ranks holding a shard of the table behind lookup ``gl`` (none for a data-parallel table)"""
    pl = e.placement[gl["table"]]
    return set(pl.shard_gpus) if pl.kind == "mp" else set()


def _step(e, comm):
    gen = torch.Generator().manual_seed(comm.rank)
    e.set_keys(torch.cat([torch.randint(0, SIZES[i], (B * HOT[i],), generator=gen) for i in range(len(SIZES))]).int())
    e.forward()
    e.top_grad["emb"].copy_(torch.randn(e.top_grad["emb"].shape, generator=gen))
    e.backward(torch.tensor([0.01]), torch.tensor([1], dtype=torch.int32))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_packed_exchange_moves_only_served_blocks_cpu(world):
    def body(comm):
        e = _collection(comm, fused=False)
        assert not e.fused and not e.hier
        me, W = comm.rank, comm.world_size
        # what every owner serves and produces, from the lookups alone
        keys_served = [sum(B * gl["hotness"] for gl in e.glookups if o in _owners(e, gl)) for o in range(W)]
        produced = comm.all_gather_object(sum(B * d.ev_size for grp in e.groups if grp.kind == "mp"
                                              for d in grp.lookups))
        assert sum(produced) == sum(B * gl["ev"] * len(_owners(e, gl)) for gl in e.glookups)
        pk = e.packed
        assert pk["kn"] == keys_served and pk["n"] == produced
        moved = []
        for name in ("all_gather", "all_to_all", "all_to_all_v", "hier_all_gather"):
            def rec(*a, _f=getattr(comm, name), _n=name):
                moved.append((_n, a[0].numel()))
                return _f(*a)
            setattr(comm, name, rec)
        _step(e, comm)
        # keys to every owner, pooled vectors back, gradients to every owner: nothing else moves
        assert moved == [("all_to_all_v", W * keys_served[me]), ("all_to_all_v", sum(produced)),
                         ("all_to_all_v", W * produced[me])], moved
    run_ranks(world, body, device=CPU, p2p=False)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_peer_memory_routes_move_only_served_blocks_cpu(world):
    def body(comm):
        e = _collection(comm, fused=True)
        assert e.fused and e.shard_split
        me = comm.rank
        # a whole bag (or, row-sharded, its compacted shard list of the same size) to every other owner,
        # the lookup's gradient columns back to every other owner
        remote = [len(_owners(e, gl) - {me}) for gl in e.glookups]
        assert e.dispatch_key_bytes == sum(B * gl["hotness"] * 4 * r for gl, r in zip(e.glookups, remote))
        _step(e, comm)
        assert e.push_grad_bytes == sum(B * gl["ev"] * 4 * r for gl, r in zip(e.glookups, remote))
    run_ranks(world, body, device=CPU, p2p="force")


def test_rank_emulator_runs_the_split_layout_cpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools_dev", "emb_rank_emulator.py"), "--cpu",
                        "--world", "4", "--batch", "8", "--cap-rows", "4000", "--ev", "8"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    m = re.search(r"split row-sharded lookups (\d+)", r.stdout)
    assert m and int(m.group(1)) > 0, r.stdout
    assert "forward (owner side" in r.stdout and "backward index" in r.stdout
