"""Multi-rank paths on ONE device through the in-process fabric (hugectr_b200/parallel/emu.py): the same
entry points as tests/test_dist.py (torchrun, real GPUs), run as N threads.  On a GPU the collections are in
FUSED mode: owner-side kernels read the other ranks' key slabs, write their output slabs and read their
gradient slabs through "peer" pointers (ordinary device pointers here), the device barrier and the two-shot
all-reduce kernels rendezvous across the ranks' streams -- this is the driver-visible proof for the peer
kernels on a one-GPU box.  On CPU the collective path is exercised without process spawns."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dist_worker as W  # noqa: E402
from hugectr_b200.parallel.emu import run_ranks  # noqa: E402

CPU = torch.device("cpu")


@pytest.mark.parametrize("plan", ["mixed", "column"])
def test_emu_ebc_collective_cpu(plan):
    run_ranks(2 if plan == "column" else 3, lambda c: W.run_ebc(plan, False, comm=c), device=CPU)


def test_emu_equiv_cpu():
    run_ranks(2, lambda c: W.run_equiv("adagrad", comm=c), device=CPU)


def test_emu_fuzz_cpu():
    for seed in (11, 12):
        run_ranks(2, lambda c: W.run_fuzz(seed, comm=c), device=CPU)


# ----------------------------------------------------------------------------- GPU: fused peer kernels
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("plan", ["mixed", "column"])
def test_emu_ebc_fused_gpu(plan, world):
    run_ranks(world, lambda c: W.run_ebc(plan, True, comm=c))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_emu_fuzz_fused_gpu(seed):
    run_ranks(4, lambda c: W.run_fuzz(seed, comm=c))


@pytest.mark.gpu
def test_emu_p2p_allreduce_gpu():
    run_ranks(4, lambda c: W.run_allreduce(comm=c))


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
def test_emu_model_equals_single_gpu(opt):
    run_ranks(4, lambda c: W.run_equiv(opt, comm=c))


@pytest.mark.gpu
def test_emu_model_overlap_paths_gpu():
    run_ranks(2, lambda c: W.run_model(comm=c))


@pytest.mark.gpu
def test_emu_dynamic_tables_fused_gpu():
    """dynamic (hashed) tables on the fused path: owners translate the keys that landed in their inbox"""
    run_ranks(4, lambda c: W.run_dynamic(comm=c))


def test_emu_dynamic_tables_cpu():
    run_ranks(2, lambda c: W.run_dynamic(comm=c), device=CPU)


def test_emu_dynamic_tables_grow_while_loading_cpu(monkeypatch):
    """shards start at 16 rows and grow as the (500 / 900-key) tables are loaded; results still equal the static
    reference, in the collective and in the fused data flow"""
    monkeypatch.setenv("HCTR_TEST_DYN_CAP", "16")
    run_ranks(2, lambda c: W.run_dynamic(comm=c), device=CPU)
    run_ranks(3, lambda c: W.run_dynamic(comm=c), device=CPU, p2p="force")


def test_emu_legacy_embeddings_cpu():
    run_ranks(2, lambda c: W.run_legacy(comm=c), device=CPU)


@pytest.mark.gpu
def test_emu_legacy_embeddings_fused_gpu():
    """Distributed / Localized hash embeddings on the fused path (peer-store key / gradient exchange,
    one-kernel ownership filter + hash translation): replicas stay identical, loss finite"""
    run_ranks(4, lambda c: W.run_legacy(comm=c))


def _real_plan_body(world, device, p2p, fused=True):
    """fused collection with the sharding plan the BENCHMARK uses at this GPU count (capped tables): hot table
    row-split over a subset of the ranks (requester-side shard split), table-wise giants, data-parallel small
    tables; forward and AdaGrad backward against a single-process collection"""
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    from hugectr_b200.tools.planner import generate_plan
    b, ev = 8, 8
    sizes = [min(s, 4000) for s in CRITEO_TB_TABLE_SIZES]
    hot = list(CRITEO_TB_MULTI_HOT)
    plan = generate_plan(CRITEO_TB_TABLE_SIZES, hot, world)
    n = len(sizes)

    def cfg_for(pl):
        cfg = EmbeddingCollectionConfig()
        cfg.embedding_lookup([EmbeddingTableConfig(str(i), sizes[i], ev) for i in range(n)],
                             [f"d{i}" for i in range(n)], "emb", ["sum"] * n)
        if pl:
            cfg.shard(pl[0], pl[1])
        return cfg
    gen = torch.Generator().manual_seed(0)
    full = {str(i): torch.randn(sizes[i], ev, generator=gen) * 0.1 for i in range(n)}
    keys = [torch.randint(0, sizes[i], (b * world, hot[i]), generator=gen) for i in range(n)]
    grad = torch.randn(b * world, n * ev, generator=gen) * 0.1
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1, epsilon=1e-6)
    hotd = {f"d{i}": hot[i] for i in range(n)}
    cpu = torch.device("cpu")
    ref = EmbeddingCollection(cfg_for(None), b * world, hotd, cpu, torch.float32, Comm.single(cpu), opt, seed=1)
    for nm, w in full.items():
        ref.load_table_rows(nm, torch.arange(w.shape[0]), w)
    ref.set_keys(torch.cat([k.reshape(-1) for k in keys]).int())
    ref.forward()
    ref.top_grad["emb"].copy_(grad)
    lr, st = torch.tensor([0.05]), torch.tensor([1], dtype=torch.int32)
    ref.backward(lr, st)

    def body(c):
        e = EmbeddingCollection(cfg_for(plan), b, hotd, device, torch.float32, c, opt, seed=1, fused=fused)
        assert e.fused == fused and (e.shard_split or not fused)
        for nm, w in full.items():
            e.load_table_rows(nm, torch.arange(w.shape[0]), w)
        r = c.rank
        e.set_keys(torch.cat([k[r * b:(r + 1) * b].reshape(-1) for k in keys]).int().to(device))
        e.forward()
        err = (e.top_data["emb"].float().cpu() - ref.top_data["emb"][r * b:(r + 1) * b]).abs().max().item()
        assert err < 1e-5, ("forward", r, err)
        e.top_grad["emb"].copy_(grad[r * b:(r + 1) * b].to(device))
        e.backward(lr.to(device), st.to(device))
        for nm in full:
            rk, rw = ref.dump_table_local(nm)[0][:2]
            for (k, w, c0, sts, kind) in e.dump_table_local(nm):
                if len(k):
                    assert (w - rw[k][:, c0:c0 + w.shape[1]]).abs().max().item() < 2e-4, ("table", nm, r)
    run_ranks(world, body, device=device, p2p=p2p)


@pytest.mark.parametrize("world", [4, 8])
def test_emu_fused_benchmark_plan_cpu(world):
    _real_plan_body(world, CPU, "force")


@pytest.mark.parametrize("world", [2, 4, 8])
def test_emu_collective_benchmark_plan_cpu(world):
    """the NCCL-style (stand-in baseline) exchange with the benchmark's plan"""
    _real_plan_body(world, CPU, False, fused=False)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [4, 8])
def test_emu_fused_benchmark_plan_gpu(world):
    _real_plan_body(world, torch.device("cuda"), True)


# ----------------------------------------------------------------------------- CompressionStrategy.Unique
@pytest.mark.parametrize("world,names,opt", [(2, "0,2", "adagrad"), (3, "0,1,2,3,5", "adagrad"),
                                             (4, "1,5", "sgd"), (2, "0,1,2,3,5", "adam")])
def test_emu_unique_compression_cpu(world, names, opt):
    run_ranks(world, lambda c: W.run_unique(names, opt, comm=c), device=CPU, p2p=False)


def test_emu_unique_is_left_to_the_peer_store_path_when_fused_cpu():
    """fused (peer-memory) mode keeps pooled-vector transfers: Unique tables are not rerouted"""
    run_ranks(2, lambda c: W.run_unique("0,2", "adagrad", fused=True, comm=c), device=CPU, p2p="force")


def test_emu_fuzz_with_unique_subsets_cpu(monkeypatch):
    """the randomised collection oracle with a random subset of the model-parallel tables on the Unique exchange"""
    monkeypatch.setenv("HCTR_FUZZ_UNIQUE", "1")
    for world, seeds in ((2, (9001, 9002, 9003)), (3, (9301, 9302)), (4, (9501,))):
        for sd in seeds:
            run_ranks(world, lambda c, sd=sd: W.run_fuzz(sd, comm=c), device=CPU, p2p=False)


@pytest.mark.parametrize("kind,opt,world,p2p", [("distributed", "adam", 2, False), ("localized", "adagrad", 3, False),
                                                ("distributed", "adagrad", 3, "force"), ("localized", "adam", 4, "force")])
def test_emu_legacy_embeddings_equal_single_process_cpu(kind, opt, world, p2p):
    """legacy hash embeddings, N ranks == 1 process KEY BY KEY (same start from sparse model files, random slots / bag
    lengths / combiner): collective exchange and the fused (peer-store) data flow"""
    for sd in (world * 100 + 1, world * 100 + 2):
        run_ranks(world, lambda c: W.run_legacy_equiv(kind, opt, sd, comm=c), device=CPU, p2p=p2p)


@pytest.mark.parametrize("mode", ["cached", "staged"])
def test_emu_embedding_training_cache_multi_rank_equals_single_process_cpu(mode, monkeypatch):
    """tables on the host parameter server (behind the cache / staged) on N ranks == resident tables on one process"""
    monkeypatch.setenv("HCTR_TEST_ETC", mode)
    run_ranks(2, lambda c: W.run_legacy_equiv("distributed", "adam", 201, comm=c), device=CPU, p2p=False)
    run_ranks(3, lambda c: W.run_legacy_equiv("localized", "adagrad", 303, comm=c), device=CPU, p2p=False)


@pytest.mark.parametrize("update", ["global", "lazy"])
def test_emu_legacy_global_update_equals_single_process_cpu(update, monkeypatch):
    """Update_t.Global / LazyGlobal Adam on hash embeddings: N ranks == 1 process.  (Caught a real bug: batch entries a
    rank does not own used to write `untouched` into row 0's flag, so row 0 was swept again after its real update.)"""
    monkeypatch.setenv("HCTR_TEST_UPDATE", update)
    run_ranks(2, lambda c: W.run_legacy_equiv("distributed", "adam", 201, comm=c), device=CPU, p2p=False)
    run_ranks(3, lambda c: W.run_legacy_equiv("localized", "adam", 302, comm=c), device=CPU, p2p="force")
    run_ranks(4, lambda c: W.run_legacy_equiv("distributed", "adam", 403, comm=c), device=CPU, p2p="force")


@pytest.mark.parametrize("legacy", [False, True])
def test_emu_multi_rank_exact_resume_cpu(legacy, tmp_path):
    """N ranks: snapshot after 3 steps, 2 more steps == fresh N-rank model resumed from the snapshot + the same 2 steps
    (bit-identical for static tables; to rounding for hash embeddings, whose row order a reload does not reproduce)"""
    for i, (world, p2p) in enumerate(((2, False), (4, "force"))):
        d = tmp_path / f"r{i}"
        d.mkdir()
        run_ranks(world, lambda c: W.run_resume(str(d), legacy, comm=c), device=CPU, p2p=p2p)


# ----------------------------------------------------------------------------- checkpoint re-sharding N -> M ranks
def _reshard_case(n_save, n_load, tmpdir, p2p_load=False):
    """train + snapshot on ``n_save`` ranks under plan A (row-sharded + table-wise + data-parallel tables); ``n_load``
    ranks under plan B (everything model parallel, column x row split when the rank count is even) resume from it:
    every table and its AdaGrad state must come back unchanged, key by key"""
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    cpu = CPU
    d, saved = str(tmpdir), {}
    sizes, hot = [400, 30, 50, 900, 120, 7], [3, 1, 1, 4, 2, 1]
    def mk(comm, plan_kind):
        world = comm.world_size
        if plan_kind == "a":
            sm = [[1, 1, 1, 0, 1, 1] for _ in range(world)]; sm[world - 1][3] = 1
            plan = (sm, [("mp", ["0", "3"]), ("dp", ["1", "2", "4", "5"])])
        else:       # everything model parallel: table 0 column+row split, 3 row split, rest table-wise
            sm = [[1, 0, 0, 1, 0, 0] for _ in range(world)]
            for i, t in enumerate((1, 2, 4, 5)): sm[i % world][t] = 1
            plan = (sm, [("mp", [("0", 2) if world % 2 == 0 else "0", "1", "2", "3", "4", "5"])])
        m = build_dlrm_dcnv2(batchsize=32 * world, num_gpus=world, table_sizes=sizes, multi_hot=hot, ev_size=8, lr=0.02,
                             mixed=False, optimizer="adagrad", bottom=(16, 8), top=(16, 1), cross_layers=1,
                             projection_dim=4, use_cuda_graph=False, shard_plan=plan, comm=comm, seed=5)
        m.compile(); return m
    def full_tables(m, comm):
        """gather (key -> vector, state) of every table on every rank"""
        out = {}
        for e in m.ebcs_train:
            for name in e.tmap:
                parts = comm.all_gather_object([(k, w, c0, [None if s is None else s for s in (sts or [])], kind) for (k, w, c0, sts, kind) in e.dump_table_local(name)])
                ev = e.tmap[name].ev_size; n = e.tmap[name].max_vocabulary_size
                W = torch.zeros(n, ev); S = torch.zeros(n, ev)
                for rp in parts:
                    for (k, w, c0, sts, kind) in rp:
                        if len(k):
                            W[k, c0:c0 + w.shape[1]] = w
                            if sts and sts[0] is not None: S[k, c0:c0 + w.shape[1]] = sts[0].float()
                out[name] = (W, S)
        return out
    def save_body(comm):
        m = mk(comm, "a"); pool = m.reader_train.pool
        for i in range(3): m.train_on_host_batch(pool[i])
        m.save_params_to_files(os.path.join(d, "s"), 3); comm.barrier()
        t = full_tables(m, comm)
        if comm.rank == 0: saved.update(t)
    def load_body(comm):
        m = mk(comm, "b"); m.resume(os.path.join(d, "s"))
        t = full_tables(m, comm)
        if comm.rank == 0:
            for name in saved:
                dw = float((t[name][0] - saved[name][0]).abs().max()); ds = float((t[name][1] - saved[name][1]).abs().max())
                assert dw == 0.0 and ds == 0.0, (name, dw, ds)
        return True

    run_ranks(n_save, save_body, device=CPU, p2p=False)
    run_ranks(n_load, load_body, device=CPU, p2p=p2p_load)


@pytest.mark.parametrize("n_save,n_load,p2p", [(2, 3, False), (4, 2, "force"), (3, 4, False)])
def test_emu_checkpoint_resharding_between_rank_counts_cpu(n_save, n_load, p2p, tmp_path):
    _reshard_case(n_save, n_load, tmp_path, p2p)


@pytest.mark.parametrize("world,gpus_per_node,seed", [(4, 2, 501), (6, 3, 602), (6, 2, 703)])
def test_emu_hierarchical_exchange_random_plans_cpu(world, gpus_per_node, seed, monkeypatch):
    """node-aware two-stage exchange on logical nodes (emulated intra- / inter-node communicators): whole model ==
    single process under a random placement (table / row / column-wise, dp)"""
    monkeypatch.setenv("HCTR_TEST_PLAN_SEED", str(seed))
    run_ranks(world, lambda c: W.run_equiv("adagrad" if seed % 2 else "sgd", gpus_per_node, comm=c), device=CPU, p2p=False)


# ----------------------------------------------------------------------------- epoch mode, data set not divisible by the batch
@pytest.mark.parametrize("world", [2, 4])
def test_emu_epoch_mode_with_incomplete_last_batch_equals_single_process_cpu(world, tmp_path):
    """RawAsync file of 1000 training / 333 evaluation samples, global batch 64, two epochs + a full evaluation pass:
    N ranks == 1 process (loss, AUC, dense weights).  (Caught a real bug: a rank whose own slice of the last batch was
    full reported the batch as complete, the ranks then disagreed on dropping it and met in different collectives.)"""
    import hugectr_b200 as hugectr
    from hugectr_b200.data.generator import DataGenerator, DataGeneratorParams
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    cpu, d = CPU, str(tmp_path)
    sizes, hot = [300, 40, 1000, 7], [3, 1, 5, 2]
    ntr, nev = 1000, 333                       # neither divisible by the global batch
    gp = DataGeneratorParams(hugectr.DataReaderType_t.Raw, 1, 13, 4, False, os.path.join(d, "t.bin"), os.path.join(d, "v.bin"),
                             sizes, nnz_array=hot, num_samples=ntr, eval_num_samples=nev, float_label_dense=True, num_threads=2)
    DataGenerator(gp).generate()
    def run(comm):
        world = comm.world_size
        m = build_dlrm_dcnv2(batchsize=64, batchsize_eval=64, num_gpus=world, table_sizes=sizes, multi_hot=hot, ev_size=8, mixed=False,
                             bottom=(16, 8), top=(16, 1), projection_dim=4, cross_layers=1, lr=0.05, optimizer="sgd",
                             source=[gp.source], comm=comm, use_cuda_graph=False, repeat_dataset=False, seed=2,
                             max_eval_batches=100)
        m.reader_params.eval_source = gp.eval_source
        m.reader_params.num_samples, m.reader_params.eval_num_samples = ntr, nev
        m.reader_params.float_label_dense = True
        m.compile()
        m.fit(num_epochs=2, display=1000, eval_interval=1000, snapshot=10**9)
        m.eval_all = None
        # full evaluation pass over the eval set
        m.reader_eval.set_source(None)
        n = 0
        for mt in m.metrics: mt[2].reset() if hasattr(mt[2], "reset") else None
        while m.eval():
            n += 1
            if n > 50: break
        res = dict(m.get_eval_metrics())
        return (round(m.get_current_loss(), 6), {k: round(float(v), 6) for k, v in res.items()}, n, float(m.arena.weights.double().sum()))

    one = run(Comm.single(CPU))
    res = run_ranks(world, run, device=CPU, p2p=False)
    assert res[0][0] == one[0] and res[0][1] == one[1] and res[0][2] == one[2], (one, res[0])
    assert abs(res[0][3] - one[3]) < 1e-5
    assert one[2] == 6          # 333 samples / 64 -> 6 evaluation batches, the last one incomplete


@pytest.mark.parametrize("fmt", ["parquet", "norm"])
def test_emu_file_readers_epoch_mode_equal_single_process_cpu(fmt, tmp_path):
    """Parquet / Norm readers + Distributed hash embedding, 666 training and 333 evaluation samples at global batch 64
    (incomplete last batches), two epochs and a full evaluation pass: 2 and 4 ranks == 1 process"""
    import hugectr_b200 as hugectr
    from hugectr_b200.data.generator import DataGenerator, DataGeneratorParams
    from hugectr_b200.parallel.comm import Comm
    cpu, d = CPU, str(tmp_path)
    T = hugectr.DataReaderType_t
    kind = {"parquet": T.Parquet, "norm": T.Norm}[fmt]
    slots = [50, 20, 30]
    src, ev = (os.path.join(d, "fl.txt"), os.path.join(d, "fl_test.txt"))
    gp = DataGeneratorParams(kind, 1, 3, 3, True, src, ev, slots, nnz_array=[2, 1, 3], num_files=2, eval_num_files=1,
                             num_samples_per_file=333, check_type=hugectr.Check_t.Sum, num_threads=2)
    DataGenerator(gp).generate()
    def run(comm):
        world = comm.world_size
        solver = hugectr.CreateSolver(batchsize=64, batchsize_eval=64, lr=0.05, vvgpu=[list(range(world))], repeat_dataset=False,
                                      i64_input_key=True, use_cuda_graph=False, max_eval_batches=100, seed=4)
        rp = hugectr.DataReaderParams(kind, source=[src], eval_source=ev, check_type=hugectr.Check_t.Sum if fmt == "norm" else hugectr.Check_t.Non,
                                      slot_size_array=slots)
        m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=comm)
        m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=3, dense_name="dense",
                            data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("data1", [2, 1, 3], False, 3)]))
        m.add(hugectr.SparseEmbedding(hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash, 1, 4, "sum", "emb", "data1",
                                      slot_size_array=slots))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["emb"], ["r"], leading_dim=12))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["r", "dense"], ["c"]))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
        m.compile()
        # same start for the hash embedding: all keys preloaded with fixed vectors
        import numpy as np
        allk = np.arange(sum(slots), dtype="<i8"); g = torch.Generator().manual_seed(1)
        if comm.rank == 0:
            os.makedirs(os.path.join(d, "init"), exist_ok=True)
            allk.tofile(os.path.join(d, "init", "key")); (torch.randn(len(allk), 4, generator=g) * 0.1).numpy().astype("<f4").tofile(os.path.join(d, "init", "emb_vector"))
        comm.barrier()
        m.load_sparse_weights([os.path.join(d, "init")])
        w0 = m.arena.weights.clone(); comm.broadcast(w0, 0); m.arena.weights.copy_(w0); m.arena.sync_shadow()
        torch.save(w0, os.path.join(d, "w0.pt")) if comm.rank == 0 and world == 1 else None
        if world > 1:
            m.arena.weights.copy_(torch.load(os.path.join(d, "w0.pt"))); m.arena.sync_shadow()
        m.fit(num_epochs=2, display=1000, eval_interval=1000, snapshot=10**9)
        m.reader_eval.set_source(None)
        n = 0
        while m.eval():
            n += 1
            if n > 50: break
        res = dict(m.get_eval_metrics())
        return (round(m.get_current_loss(), 5), {k: round(float(v), 5) for k, v in res.items()}, n, round(float(m.arena.weights.double().sum()), 5))

    one = run(Comm.single(CPU))
    assert one[2] == 6                       # every evaluation sample is seen: ceil(333 / 64) batches
    for w in (2, 4):
        assert run_ranks(w, run, device=CPU, p2p=False)[0] == one


def test_emu_dynamic_table_grows_on_one_rank_while_all_ranks_agree_cpu():
    """`Model.fit` with a dynamic table that lives on rank 0 only and starts far too small: the display checkpoints grow
    it, every rank learns about it (the graph re-capture is a rendezvous) and training continues in lock step"""
    import hugectr_b200 as hugectr
    cpu = CPU
    def run(comm):
        world = comm.world_size
        solver = hugectr.CreateSolver(batchsize=32 * world, batchsize_eval=32 * world, lr=0.05, vvgpu=[list(range(world))], repeat_dataset=True,
                                      max_eval_batches=2, use_cuda_graph=False)
        rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.0"], eval_source="synthetic:1.0",
                                      check_type=hugectr.Check_t.Non, slot_size_array=[5000, 300])
        m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad), comm=comm)
        m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                            data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("k", 2, False, 1), hugectr.DataReaderSparseParam("q", 1, True, 1)]))
        ebc = hugectr.EmbeddingCollectionConfig()
        ebc.embedding_lookup([hugectr.EmbeddingTableConfig("t", -1, 8, init_capacity=16), hugectr.EmbeddingTableConfig("u", 300, 8)], ["k", "q"], "emb", ["sum", "sum"])
        sm = [["t"] if g == 0 else [] for g in range(world)]; sm[world - 1] = sm[world - 1] + ["u"]
        ebc.shard(sm, [("mp", ["t", "u"])])
        m.add(ebc)
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["c"]))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
        m.compile()
        m.fit(max_iter=40, display=5, eval_interval=20, snapshot=10**9)
        rows = [sl["rows"] for g in m.ebcs_train[0].groups for sl in g.table_slices if sl["table"] == "t"]
        return rows, round(m.get_current_loss(), 4)

    for w, p2p in ((2, False), (3, "force")):
        res = run_ranks(w, run, device=CPU, p2p=p2p)
        assert res[0][0][0] > 16 and all(r[0] == [] for r in res[1:])
        assert len({r[1] for r in res}) == 1


def test_emu_checkpoint_of_a_multi_rank_run_serves_single_process_inference_cpu(tmp_path):
    """graph JSON + snapshot of a 2-rank run (row-sharded + data-parallel tables) opened by a single-process inference
    session: the stored 2-GPU plan is re-planned for one GPU and the predictions equal the training model's exactly"""
    import numpy as np
    import hugectr_b200 as hugectr
    from hugectr_b200.inference import CreateInferenceSession, InferenceParams
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    cpu, d = CPU, str(tmp_path)
    sizes, hot = [400, 30, 50, 900, 120, 7], [3, 1, 1, 4, 2, 1]
    def run(comm):
        world = comm.world_size
        sm = [[1, 1, 1, 0, 1, 1] for _ in range(world)]; sm[world - 1][3] = 1
        plan = (sm, [("mp", ["0", "3"]), ("dp", ["1", "2", "4", "5"])])
        m = build_dlrm_dcnv2(batchsize=32 * world, batchsize_eval=32 * world, num_gpus=world, table_sizes=sizes, multi_hot=hot, ev_size=8, lr=0.02,
                             mixed=False, optimizer="adagrad", bottom=(16, 8), top=(16, 1), cross_layers=1, projection_dim=4,
                             use_cuda_graph=False, shard_plan=plan, comm=comm, seed=5)
        m.compile()
        for _ in range(4): m.train()
        m.save_params_to_files(os.path.join(d, "m"), 4)
        if comm.rank == 0: m.graph_to_json(os.path.join(d, "g.json"))
        # predictions of this rank's slice of one eval batch
        hb = m.reader_eval.read_a_batch(); m._load_batch(hb, False)
        for e in m.ebcs_eval: e.forward(False)
        m.net_eval.fprop(False)
        pred = m.net_eval.loss_layers[0].pred.float().clone()
        return hb.dense.clone(), hb.keys.clone(), pred

    res = run_ranks(2, run, device=CPU, p2p=False)
    sess = CreateInferenceSession(os.path.join(d, "g.json"), InferenceParams(
        model_name="x", max_batchsize=32, dense_model_file=os.path.join(d, "m_dense_4.model"),
        embedding_collection_path=os.path.join(d, "m_ebc_4")))
    for dense, keys, pred in res:
        p = sess.predict(dense.numpy(), keys.numpy())
        assert float(np.abs(p.reshape(-1) - pred.numpy().reshape(-1)).max()) == 0.0


@pytest.mark.parametrize("n_save,n_load", [(2, 3), (4, 2)])
def test_emu_legacy_snapshot_resharding_between_rank_counts_cpu(n_save, n_load, tmp_path):
    """Distributed hash embedding (DeepFM): snapshot of N ranks resumed on M ranks -- (key -> vector) and the Adam moments
    (matched by key) are identical, and training continues"""
    import numpy as np
    import hugectr_b200 as hugectr
    from hugectr_b200.models.legacy import build_deepfm
    cpu, d, kind = CPU, str(tmp_path), "distributed"
    def mk(comm):
        world = comm.world_size
        kw = {"embedding_type": hugectr.Embedding_t.LocalizedSlotSparseEmbeddingHash} if kind == "localized" else {}
        m = build_deepfm(batchsize=24 * world, vvgpu=[list(range(world))], slot_sizes=[30, 12, 50, 7], workspace_mb=2, mixed=False, comm=comm, max_eval_batches=1, seed=5, **kw)
        m.compile(); return m
    def dump(m, comm, tag):
        out = {}
        for rt in m.legacy_train:
            p, o = os.path.join(d, f"{tag}_{rt.name}"), os.path.join(d, f"{tag}_{rt.name}_opt")
            rt.dump_parameters(p); rt.dump_opt_states(o)
            if comm.rank == 0:
                k = np.fromfile(p + "/key", "<i8"); v = np.fromfile(p + "/emb_vector", "<f4").reshape(len(k), -1)
                st = np.fromfile(o, "<f4"); ns = st.size // max(1, v.size); st = st.reshape(ns, len(k), -1)
                idx = np.argsort(k); out[rt.name] = (k[idx], v[idx], st[:, idx])
        return out
    saved = {}
    def save_body(comm):
        m = mk(comm)
        for _ in range(3): m.train()
        m.save_params_to_files(os.path.join(d, "s"), 3); comm.barrier()
        t = dump(m, comm, "a")
        if comm.rank == 0: saved.update(t)
    def load_body(comm):
        m = mk(comm); assert m.resume(os.path.join(d, "s")) == 3
        t = dump(m, comm, "b")
        if comm.rank == 0:
            for n in saved:
                assert np.array_equal(saved[n][0], t[n][0]) and np.array_equal(saved[n][1], t[n][1]), (n, "table")
                assert saved[n][2].shape == t[n][2].shape and np.array_equal(saved[n][2], t[n][2]), (n, "opt states")
                assert saved[n][2].shape[0] >= 1 and np.abs(saved[n][2]).max() > 0
        m.train(); return True

    run_ranks(n_save, save_body, device=CPU, p2p=False)
    run_ranks(n_load, load_body, device=CPU, p2p=False)


def test_emu_embedding_training_cache_snapshot_resumes_exactly_cpu(tmp_path):
    """W&D with both tables on the host parameter server (cached + staged): snapshot after 3 steps, 2 more steps == a
    fresh cached model resumed from the snapshot + the same steps, on 1 and 2 ranks (first-sight vectors are keyed by
    key, so rows created after the resume match too); a resident model resumes from the same files"""
    import hugectr_b200 as hugectr
    from hugectr_b200.models.legacy import build_wdl
    from hugectr_b200.parallel.comm import Comm
    cpu, d = CPU, str(tmp_path)
    def mk(comm, cached):
        world = comm.world_size
        etc = hugectr.CreateETC(ps_types=[hugectr.TrainPSType_t.Cached, hugectr.TrainPSType_t.Staged], sparse_models=["", ""], host_capacity_rows=8192) if cached else None
        m = build_wdl(batchsize=32 * world, vvgpu=[list(range(world))], wide_slot_sizes=[30, 12], deep_slot_sizes=[30, 12, 50, 7], workspace_mb=(1, 2), mixed=False,
                      comm=comm, max_eval_batches=1, seed=5, etc=etc)
        for c in m.dense_layers:
            if c.layer_type == hugectr.Layer_t.Dropout: c.dropout_rate = 0.0
        m.compile(); return m
    def body(comm):
        a = mk(comm, True); pool = a.reader_train.pool
        for i in range(3): a.train_on_host_batch(pool[i])
        a.save_params_to_files(os.path.join(d, "s"), 3); comm.barrier()
        for i in range(3, 5): a.train_on_host_batch(pool[i])
        # resume into a RESIDENT (no ETC) model and into another cached model: both must continue like `a`
        out = {}
        for tag, cached in (("resident", False), ("cached", True)):
            b = mk(comm, cached); assert b.resume(os.path.join(d, "s")) == 3
            for i in range(3, 5): b.train_on_host_batch(pool[i])
            out[tag] = (abs(a.get_current_loss() - b.get_current_loss()), float((a.arena.weights - b.arena.weights).abs().max()))
        return out

    one = body(Comm.single(CPU))
    assert one["cached"] == (0.0, 0.0) and one["resident"][1] < 1e-3
    two = run_ranks(2, body, device=CPU, p2p=False)[0]
    assert two["cached"][0] == 0.0 and two["cached"][1] < 1e-8 and two["resident"][1] < 1e-3


def test_emu_embedding_training_cache_from_scratch_is_rank_count_independent_cpu(tmp_path):
    """tables on the host parameter server, NO preloaded keys: the same global batches train to the same loss trace and
    dense weights on 1, 2 and 4 ranks (a key's first-sight vector depends on the key only)"""
    import hugectr_b200 as hugectr
    from hugectr_b200.data.batch import HostBatch
    from hugectr_b200.parallel.comm import Comm
    cpu, W0 = CPU, str(tmp_path / "w0.pt")
    S, H, vec, b = 3, 2, 4, 16
    vocab = [40, 25, 60]
    def build(c, world_total):
        w = c.world_size
        solver = hugectr.CreateSolver(batchsize=b * world_total, batchsize_eval=b * world_total, lr=0.05, vvgpu=[list(range(w))], repeat_dataset=True,
                                      i64_input_key=True, use_cuda_graph=False, seed=9)
        rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.Parquet, source=["synthetic"], eval_source="synthetic", check_type=hugectr.Check_t.Non, slot_size_array=vocab)
        etc = hugectr.CreateETC(ps_types=[hugectr.TrainPSType_t.Cached], sparse_models=[""], host_capacity_rows=4096)
        m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.Adam, hugectr.Update_t.Local), etc, comm=c)
        m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense", data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("data1", H, False, S)]))
        m.add(hugectr.SparseEmbedding(hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash, 1, vec, "sum", "emb", "data1", slot_size_array=vocab))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["emb"], ["r"], leading_dim=S * vec))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["r", "dense"], ["c"]))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
        m.compile(); return m
    def run(comm, W):
        m = build(comm, W)
        w0 = torch.load(W0) if os.path.exists(W0) else None
        if w0 is None:
            torch.save(m.arena.weights.clone(), W0); w0 = m.arena.weights.clone()
        m.arena.weights.copy_(w0); m.arena.sync_shadow()
        gen = torch.Generator().manual_seed(5); import numpy as np
        offs = np.concatenate([[0], np.cumsum(vocab)[:-1]])
        L = []
        for step in range(4):
            lab = torch.randint(0, 2, (b * W, 1), generator=gen).float(); den = torch.rand(b * W, 2, generator=gen)
            keys = torch.stack([torch.randint(0, vocab[s], (b * W, H), generator=gen) + int(offs[s]) for s in range(S)], 1)
            nnz = (keys >= 0).sum(-1).int()
            r, ws = comm.rank, comm.world_size; per = b * W // ws
            sl = slice(r * per, (r + 1) * per)
            m.train_on_host_batch(HostBatch(lab[sl].clone(), den[sl].clone(), keys[sl].reshape(-1).clone(), nnz[sl].t().reshape(-1).clone(), per))
            L.append(round(m.get_current_loss(), 6))
        return L, round(float(m.arena.weights.double().sum()), 6)

    W = 4
    one = run(Comm.single(CPU), W)
    for w in (2, 4):
        assert run_ranks(w, lambda c: run(c, W), device=CPU, p2p=False)[0] == one
