"""Second line of CPU tests: API corners that the end-to-end tests do not reach (found with a line
tracer over the suite)."""
import os
import time

import numpy as np
import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.parallel.comm import Comm

CPU = lambda: Comm.single(torch.device("cpu"))


def test_sok_localized_dense_lookup_filter_and_incremental_dump(tmp_path):
    from hugectr_b200 import sok
    sok.init(CPU())
    assert sok.rank() == 0 and sok.num_gpus() == 1
    lv = sok.LocalizedVariable(shape=(30, 4), gpu=0, name="loc_v")
    idx = torch.tensor([[1, 2, 3], [4, 4, 0]])
    dense = sok.all2all_dense_embedding(lv, idx)
    torch.testing.assert_close(dense, lv.weight[idx])
    sok_vars, others = sok.filter_variables([lv, torch.nn.Parameter(torch.zeros(2))])
    assert sok_vars == [lv] and len(others) == 1
    d = sok.DynamicVariable(4, name="dyn_inc", init_capacity=8)
    out = sok.lookup_sparse(d, torch.tensor([[10 ** 11, 7]]), "sum")
    out.sum().backward()
    t0 = time.time()
    time.sleep(0.01)
    sok.SGD(0.1).apply_gradients([d])                       # touches the two rows now
    sok.lookup_sparse(d, torch.tensor([[99, -1]]), "sum")   # a third row, never updated
    sok.incremental_model_dump([d], t0, str(tmp_path))
    from hugectr_b200.sok import _read
    keys = _read(str(tmp_path / "dyn_inc-key"))
    assert sorted(keys.tolist()) == [7, 10 ** 11]
    w = _read(str(tmp_path / "dyn_inc-weight"))
    assert w.reshape(-1, 4).shape == (2, 4)


def test_lr_scheduler_state_and_reset():
    from hugectr_b200.lr_scheduler import LearningRateScheduler
    s = LearningRateScheduler(1.0, warmup_steps=2, decay_start=4, decay_steps=4, decay_power=2.0, end_lr=0.1)
    seq = [s.get_next() for _ in range(10)]
    assert seq[:2] == [0.5, 1.0] and seq[2:4] == [1.0, 1.0]
    assert abs(seq[4] - max(1.0 * (3 / 4) ** 2, 0.1)) < 1e-9 and seq[-1] == 0.1
    st = s.state_dict()
    s2 = LearningRateScheduler(1.0, 2, 4, 4, 2.0, 0.1)
    s2.load_state_dict(st)
    assert s2.get_next() == s.get_next() and abs(s.get_lr() - 0.1) < 1e-12
    s.reset()
    assert s.get_next() == 0.5


def test_local_filesystem_roundtrip(tmp_path):
    from hugectr_b200.io.filesystem import FileSystemBuilder
    fs = FileSystemBuilder.build_unique_by_path(str(tmp_path))
    d = str(tmp_path / "a" / "b")
    fs.create_dir(d)
    p = os.path.join(d, "x.bin")
    fs.write(p, b"hello world", overwrite=True)
    assert fs.exists(p) and fs.get_file_size(p) == 11 and fs.read(p) == b"hello world"
    q = os.path.join(d, "y.bin")
    fs.copy(p, q)
    assert fs.read(q) == b"hello world"
    fs.delete_file(p)
    assert not fs.exists(p)
    fs.delete_dir(str(tmp_path / "a"))
    assert not fs.exists(d)


def test_hmem_cache_keyset_and_training_cache(tmp_path):
    from hugectr_b200.cache.hps import EmbeddingTrainingCache, HMemCache, HostParameterServer
    hc = HMemCache(4, capacity_rows=2)
    hc.put(1, torch.ones(4))
    hc.put(2, torch.full((4,), 2.0))
    assert torch.equal(hc.get(1), torch.ones(4))
    hc.put(3, torch.full((4,), 3.0))                         # evicts the least recently used (2)
    assert hc.get(2) is None and hc.get(3) is not None and 0 < hc.hit_rate() < 1
    ps = HostParameterServer(4, num_states=1, capacity_rows=64)
    ks = np.array([5, 6, 7], dtype="<i8")
    ks.tofile(str(tmp_path / "keyset"))
    keys = ps.load_keyset(str(tmp_path / "keyset"))
    assert keys.tolist() == [5, 6, 7] and ps.size() == 3
    etc = EmbeddingTrainingCache(ps, hugectr.TrainPSType_t.Cached, hmem_rows=8)
    table = etc.update(keys, torch.device("cpu"))
    assert table.shape == (3, 4)
    table.add_(1.0)
    etc.dump()
    w, _ = ps.pull(keys)
    torch.testing.assert_close(w, table)


def test_hashtable_set_clear_and_gather_rows_and_dense_fallbacks():
    from hugectr_b200.embedding import ops as E
    from hugectr_b200.embedding.hashtable import HashTable
    from hugectr_b200.ops import dense as D
    ht = HashTable(16, "cpu")
    ht.set(torch.tensor([10, 20]), torch.tensor([3, 1]))
    assert ht.get(torch.tensor([20, 10, 5])).tolist() == [1, 3, -1]
    ht.clear()
    assert ht.size() == 0 and ht.get(torch.tensor([10])).tolist() == [-1]
    table = torch.arange(40.).view(-1)
    out = torch.zeros(3, 4)
    E.gather_rows(table, 4, torch.tensor([2, 0, 9]), out)
    torch.testing.assert_close(out, table.view(10, 4)[[2, 0, 9]])
    src = torch.randn(3, 5)
    dst = torch.zeros(3, 8, dtype=torch.bfloat16)
    D.cast_pad(src, dst)
    torch.testing.assert_close(dst[:, :5].float(), src.bfloat16().float())
    assert float(dst[:, 5:].abs().max()) == 0.0
    a, b, c = torch.randn(2, 8).bfloat16(), torch.randn(2, 8).bfloat16(), torch.randn(2, 8)
    o = torch.zeros(2, 8, dtype=torch.bfloat16)
    D.add3(a, b, c, o)
    torch.testing.assert_close(o.float(), (a.float() + b.float() + c).bfloat16().float())


def test_model_set_source_download_and_embedding_dump(tmp_path):
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    m = build_dlrm_dcnv2(batchsize=16, num_gpus=1, table_sizes=[30, 40], multi_hot=[2, 1], ev_size=8,
                         mixed=False, bottom=(16, 8), top=(16, 1), projection_dim=4, cross_layers=1,
                         comm=CPU(), use_cuda_graph=False)
    m.compile()
    m.train()
    assert m.get_data_reader_train() is m.reader_train and m.get_data_reader_eval() is m.reader_eval
    m.set_source("synthetic:1.1", "synthetic:1.1")
    m.train()
    m.download_params_to_files(str(tmp_path / "dl"), 2)
    assert os.path.exists(str(tmp_path / "dl_dense_2.model"))
    m.embedding_dump(str(tmp_path / "ebc"), ["0"])
    before = m.ebcs_train[0].dump_table_local("0")[0][1].clone()
    m.train()
    m.embedding_load(str(tmp_path / "ebc"), ["0"])
    torch.testing.assert_close(m.ebcs_train[0].dump_table_local("0")[0][1], before)
    from hugectr_b200.utils import diagnose
    assert diagnose.verify_model(m)
    assert m.solver.num_nodes == 1 and "lr" in m.solver.to_json() if hasattr(m.solver, "to_json") else True


def test_kernel_summary_reads_static_resources_without_a_gpu():
    import shutil
    from hugectr_b200.utils.diagnose import kernel_summary
    if not (shutil.which("cuobjdump") or os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("no cuobjdump")
    ks = kernel_summary()
    assert len(ks) > 40
    gemm = {k: v for k, v in ks.items() if "gemm_tc_kernel" in k}
    assert gemm and all(v["regs"] <= 255 and v["stack"] == 0 for v in gemm.values())   # no spills
    # the register-capped (3 blocks / SM) reduce+update kernels may spill a few words, never more
    assert all(v["stack"] <= 64 for k, v in kernel_summary("emb_bwd_reduce_update").items())


def test_dynamic_variable_eviction_and_host_tier():
    """HierarchicalKV semantics of sok.DynamicVariable: bounded HBM tier, LRU / LFU eviction, rows
    demoted to the host tier come back with weights and optimizer state intact"""
    import hugectr_b200 as hugectr
    from hugectr_b200 import sok
    from hugectr_b200.parallel.comm import Comm
    sok.init(Comm.single(torch.device("cpu")))
    opt = sok.OptimizerWrapper(hugectr.Optimizer_t.AdaGrad, lr=0.1, initial_accu_value=0.0)

    def step(v, keys):
        out = sok.lookup_sparse(v, keys.view(-1, 1), combiners="sum")
        (out * torch.arange(1, out.numel() + 1).view_as(out).float()).sum().backward()
        opt.apply_gradients([v])

    def snapshot(v, keys):
        rows = v.local_rows(keys, create=False)
        assert bool((rows >= 0).all())
        return v.weight[rows].clone(), v.states["s0"][rows].clone()

    v = sok.DynamicVariable(4, var_type="hybrid", initializer=0.5, init_capacity=16, max_capacity=64)
    a, b = torch.arange(0, 48), torch.arange(100, 132)
    step(v, a)
    wa, sa = snapshot(v, a)
    assert float((wa - 0.5).abs().min()) > 0 and float(sa.min()) > 0      # trained
    step(v, b)                                    # 48 + 32 > 64: evicts 32 rows of `a` to the host tier
    assert v.size <= 64 and v.evictions == 32 and v.host is not None
    assert v.total_size == 80
    resident = v.local_rows(a, create=False) >= 0
    assert int(resident.sum()) == 16
    out = sok.lookup_sparse(v, a.view(-1, 1), combiners="sum")        # promotes the 32 demoted rows
    assert v.promotions == 32 and v.size <= 64
    wa2, sa2 = snapshot(v, a)
    assert torch.equal(wa, wa2) and torch.equal(sa, sa2)                # weights + AdaGrad state intact
    assert torch.equal(out.detach(), wa)
    v.sparse_grad = None
    # a dump contains the HBM rows AND the rows that only live in the host tier (weights + slots)
    import tempfile
    d = tempfile.mkdtemp()
    sok.dump(d, [v], opt)
    from hugectr_b200.sok import _read
    K = torch.from_numpy(_read(f"{d}/{v.name}-key").astype("int64"))
    W = torch.from_numpy(_read(f"{d}/{v.name}-weight").copy())
    S0 = torch.from_numpy(_read(f"{d}/{v.name}-slot0").copy())
    assert K.numel() == v.total_size == 80 and torch.equal(K, torch.cat([a, b]))
    assert torch.equal(W[:48], wa) and torch.equal(S0[:48], sa)
    fresh = sok.DynamicVariable(4, var_type="hbm", initializer=0.0, init_capacity=16, max_capacity=128,
                                name=v.name)
    sok.load(d, [fresh], opt)
    assert torch.equal(fresh.weight[fresh.local_rows(a, create=False)], wa)

    # pure HBM variable: evicted keys are forgotten and start from the initializer again
    h = sok.DynamicVariable(4, var_type="hbm", initializer=0.5, init_capacity=16, max_capacity=64)
    step(h, a)
    step(h, b)
    gone = a[h.local_rows(a, create=False) < 0]
    assert gone.numel() == 32 and h.host is None
    out = sok.lookup_sparse(h, gone.view(-1, 1), combiners="sum")
    assert torch.equal(out.detach(), torch.full((32, 4), 0.5))
    h.sparse_grad = None

    # LFU: frequently used keys survive a sweep of one-off keys
    f = sok.DynamicVariable(4, var_type="hbm", initializer=0.5, init_capacity=16, max_capacity=64,
                            evict_strategy="lfu")
    hot = torch.arange(0, 10)
    for _ in range(5):
        f.local_rows(hot)
    for i in range(6):
        f.local_rows(torch.arange(1000 + 20 * i, 1020 + 20 * i))
    assert f.evictions > 0 and bool((f.local_rows(hot, create=False) >= 0).all())
    with pytest.raises(RuntimeError, match="max_capacity"):
        f.local_rows(torch.arange(5000, 5100))      # one batch larger than the tier


def test_embedding_gen_tool_writes_a_loadable_checkpoint(tmp_path):
    from hugectr_b200.io.checkpoint import iter_ebc_folder, read_ebc_folder
    from hugectr_b200.tools import embedding_gen
    embedding_gen.main(["--embedding-size", "1000-37-5", "--dim", "8", "--output", str(tmp_path)])
    tabs = read_ebc_folder(str(tmp_path / "embedding_collection_0"))
    assert sorted(tabs) == [0, 1, 2]
    k, w, s = tabs[0]
    assert torch.equal(k, torch.arange(1000)) and w.shape == (1000, 8) and s is None
    assert float(w.abs().max()) <= 1 / 1000 ** 0.5 + 1e-7 and float(w.std()) > 0
    assert sum(k.numel() for _, k, _, _ in iter_ebc_folder(str(tmp_path / "embedding_collection_0"), 100)) == 1042


def test_step_watchdog_dumps_stacks_of_a_hung_step(tmp_path):
    import time
    from hugectr_b200.utils.watchdog import StepWatchdog
    log = open(tmp_path / "wd.txt", "w+")
    wd = StepWatchdog(0.2, file=log)
    with wd:
        pass                                   # fast step: nothing is written
    time.sleep(0.4)
    log.seek(0)
    assert log.read() == ""
    with wd:
        time.sleep(0.6)                        # "hung" step
    log.seek(0)
    txt = log.read()
    assert "Timeout" in txt and "test_step_watchdog" in txt
    assert StepWatchdog.from_env() is None
    os.environ["HCTR_STEP_TIMEOUT"] = "30"
    try:
        assert StepWatchdog.from_env().timeout == 30.0
        # a model step runs under the watchdog without side effects
        from hugectr_b200.models.dlrm import build_dlrm_dcnv2
        from hugectr_b200.parallel.comm import Comm
        m = build_dlrm_dcnv2(batchsize=16, num_gpus=1, table_sizes=[30, 40], multi_hot=[2, 1], ev_size=8,
                             mixed=False, bottom=(16, 8), top=(16, 1), projection_dim=4, cross_layers=1,
                             comm=Comm.single(torch.device("cpu")))
        m.compile()
        assert m.train() and m._watchdog is not None and not m._watchdog.armed
    finally:
        del os.environ["HCTR_STEP_TIMEOUT"]


def test_bucket_finality_out_of_order():
    """ADVICE r1: a bottom layer declared after a top layer must not be flushed before its bprop ran."""
    from hugectr_b200.parallel.allreduce import advance_final
    # arena: A [0,100) (top), B [100,200) (bottom, declared later), C [200,300) (top); top pass runs C then A
    f, pend = advance_final(300, [(200, 300)])
    assert (f, pend) == (200, [])
    f, pend = advance_final(f, pend + [(0, 100)])        # A done, B not yet: nothing below 200 is final
    assert f == 200 and pend == [(0, 100)]
    f, pend = advance_final(f, pend + [(100, 200)])      # bottom pass: B done -> everything final
    assert (f, pend) == (0, [])


def test_dynamic_tables_grow_when_a_shard_runs_out_of_rows():
    """DynamicEmbeddingTable semantics: no fixed vocabulary.  A shard that runs out of rows is doubled in place
    (group arrays re-laid out around it), known keys keep their vectors and optimizer state, neighbours in the same
    group are untouched, the evaluation plan follows, and the keys that were turned away are admitted afterwards."""
    import torch
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cpu = torch.device("cpu")
    b, ev = 4, 8
    cfg = EmbeddingCollectionConfig()
    tabs = [EmbeddingTableConfig("a", 50, ev), EmbeddingTableConfig("dyn", -1, ev, init_capacity=6, max_capacity=40),
            EmbeddingTableConfig("c", 30, ev)]
    cfg.embedding_lookup(tabs, ["ka", "kd", "kc"], "emb", ["sum", "sum", "sum"])
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1)
    e = EmbeddingCollection(cfg, b, {"ka": 1, "kd": 2, "kc": 1}, cpu, torch.float32, Comm.single(cpu), opt, seed=3)
    ev_plan = e.eval_clone(b)
    lr, st = torch.tensor([0.1]), torch.tensor([1], dtype=torch.int32)

    def step(plan, dyn_keys, train=True):
        keys = torch.cat([torch.arange(b), torch.as_tensor(dyn_keys).reshape(-1), torch.arange(b) + 5]).int()
        plan.set_keys(keys)
        plan.forward(train)
        out = plan.top_data["emb"].clone()
        if train:
            plan.top_grad["emb"].fill_(0.5)
            plan.backward(lr, st)
        return out
    step(e, [[1000, 1001], [1002, 1003], [1004, 1005], [1000, 1003]])        # 6 distinct keys: table full
    assert e.grow_dynamic() == []
    snap_a = e.dump_table_local("a")[0][1].clone()
    snap_c = e.dump_table_local("c")[0][1].clone()
    kd, wd = e.dump_table_local("dyn")[0][:2]
    known = {int(k): wd[i].clone() for i, k in enumerate(kd.tolist())}
    assert len(known) == 6
    out = step(e, [[2000, 2001], [1000, 2002], [2003, 2004], [2005, 1001]], train=False)      # new keys find no row
    assert float(out[0, ev:2 * ev].abs().sum()) == 0.0                   # both keys of sample 0 read as empty
    import pytest
    old_rows = e.groups[0].rows
    grown = e.grow_dynamic()
    assert grown == [("dyn", 0, 6, 13)] and e.groups[0].rows == old_rows + 7
    assert e.grow_dynamic() == []                                        # flag cleared with the new hash table
    # neighbours and known keys are bit-identical, in the training and in the evaluation plan
    assert torch.equal(e.dump_table_local("a")[0][1], snap_a) and torch.equal(e.dump_table_local("c")[0][1], snap_c)
    kd2, wd2 = e.dump_table_local("dyn")[0][:2]
    assert sorted(kd2.tolist()) == sorted(known) and all(torch.equal(wd2[i], known[int(k)]) for i, k in enumerate(kd2.tolist()))
    o_tr = step(e, [[1000, 1001]] * b, train=False)
    o_ev = step(ev_plan, [[1000, 1001]] * b, train=False)
    assert torch.equal(o_tr, o_ev) and torch.allclose(o_tr[0, ev:2 * ev], known[1000] + known[1001])
    # turned-away keys are admitted now, and train
    out = step(e, [[2000, 2001], [1000, 2002], [2003, 2004], [2005, 1001]])
    assert float(out[0, ev:2 * ev].abs().sum()) > 0.0
    assert e._dyn_tables[("dyn", 0, 0)].size() == 12
    # the cap: 13 -> 27 -> 40 (max_capacity), then the old error
    step(e, [[3000 + 2 * i, 3001 + 2 * i] for i in range(b)])
    assert e.grow_dynamic() == [("dyn", 0, 13, 27)]
    for j in range(4):
        step(e, [[4000 + 8 * j + 2 * i, 4001 + 8 * j + 2 * i] for i in range(b)])
    assert e.grow_dynamic() == [("dyn", 0, 27, 40)]
    for j in range(3):
        step(e, [[5000 + 8 * j + 2 * i, 5001 + 8 * j + 2 * i] for i in range(b)])
    with pytest.raises(RuntimeError, match="max_capacity"):
        e.grow_dynamic()


def test_model_fit_survives_a_growing_dynamic_table(monkeypatch):
    """through `Model.fit`: the display checkpoint grows the table instead of raising (HCTR_DYNAMIC_GROW=0 raises)"""
    import torch
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm

    def build():
        solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]], repeat_dataset=True,
                                      max_eval_batches=2, use_cuda_graph=False)
        rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.0"],
                                      eval_source="synthetic:1.0", check_type=hugectr.Check_t.Non,
                                      slot_size_array=[5000])          # key range of the synthetic batches
        m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(torch.device("cpu")))
        m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                            data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("k", 2, False, 1)]))
        ebc = hugectr.EmbeddingCollectionConfig()
        ebc.embedding_lookup(hugectr.EmbeddingTableConfig("t", -1, 8, init_capacity=16), "k", "emb", "sum")
        m.add(ebc)
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["emb"], ["r"], leading_dim=8))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["r", "dense"], ["c"]))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
        m.compile()
        return m
    m = build()
    m.fit(max_iter=30, display=5, eval_interval=15, snapshot=1000000)
    rows = m.ebcs_train[0].groups[0].rows
    assert rows > 16, rows
    monkeypatch.setenv("HCTR_DYNAMIC_GROW", "0")
    m2 = build()
    import pytest
    with pytest.raises(RuntimeError, match="init_capacity"):
        m2.fit(max_iter=30, display=5, eval_interval=15, snapshot=1000000)


def test_sok_export_assign_read_and_evict_group_lookup():
    """module-level SOK helpers of the reference: export / assign (dynamic_variable.py), sparse_read_and_evict
    (lookup.py:75, hybrid variables), group_lookup, set_comm_tool"""
    import pytest
    from hugectr_b200 import sok
    from hugectr_b200.parallel.comm import Comm
    sok.init(Comm.single(torch.device("cpu")))
    assert sok.set_comm_tool("horovod") == "torch.distributed" and sok.__version__
    v = sok.DynamicVariable(4, var_type="hybrid", initializer=0.25, init_capacity=8, max_capacity=16)
    keys = torch.tensor([5, 900000000007, 42])
    vals = torch.arange(12, dtype=torch.float32).view(3, 4)
    assert sok.assign(v, keys, vals) is v
    k, w = sok.export(v)
    order = torch.argsort(k)
    assert k[order].tolist() == sorted(keys.tolist())
    assert torch.equal(w[order], vals[torch.argsort(keys)])
    # read-and-evict: known keys keep their values, unseen keys are created from the initializer; beyond the HBM
    # capacity the oldest rows move to the host tier and still export
    out = sok.sparse_read_and_evict(v, torch.tensor([[42, 7], [5, 8]]))
    assert out.shape == (2, 2, 4) and torch.equal(out[0, 0], vals[2]) and torch.equal(out[1, 0], vals[0])
    assert torch.allclose(out[0, 1].abs(), torch.full((4,), 0.25)) or float(out[0, 1].abs().max()) <= 0.25
    sok.sparse_read_and_evict(v, torch.arange(1000, 1014))
    assert v.size <= 16 and v.evictions > 0 and v.total_size == 5 + 14
    k2, w2 = sok.export(v)
    assert torch.equal(w2[(k2 == 900000000007).nonzero()[0, 0]], vals[1])         # wherever the row lives now
    with pytest.raises(TypeError):
        sok.sparse_read_and_evict(sok.DynamicVariable(4, var_type="hbm"), keys)
    # group_lookup: plain local gathers with gradients
    p1 = torch.nn.Parameter(torch.randn(10, 3))
    p2 = sok.Variable(shape=[6, 2])
    p2.weight.requires_grad_(True)
    o1, o2 = sok.group_lookup([p1, p2], [torch.tensor([1, 1, 4]), torch.tensor([[0, 5]])])
    assert o1.shape == (3, 3) and o2.shape == (1, 2, 2)
    (o1.sum() + o2.sum()).backward()
    assert float(p1.grad[1].sum()) == 6.0 and float(p2.weight.grad[5].sum()) == 2.0


def test_graph_json_round_trips_collection_extras(tmp_path):
    """dynamic-table capacities, the initializer bound, the communication strategy and the per-table compression
    strategy of an embedding collection survive graph_to_json -> construct_from_json"""
    import json
    import hugectr_b200 as hugectr
    from hugectr_b200.embedding.collection import InitParams
    from hugectr_b200.parallel.comm import Comm
    cpu = Comm.single(torch.device("cpu"))

    def solver():
        return hugectr.CreateSolver(batchsize=16, batchsize_eval=16, lr=0.01, vvgpu=[[0]], use_cuda_graph=False)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic"], eval_source="synthetic",
                                  check_type=hugectr.Check_t.Non, slot_size_array=[100, 100])
    m = hugectr.Model(solver(), rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=cpu)
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("a", 2, False, 1),
                                                        hugectr.DataReaderSparseParam("b", 1, True, 1)]))
    ebc = hugectr.EmbeddingCollectionConfig(comm_strategy=hugectr.CommunicationStrategy.Hierarchical)
    ebc.embedding_lookup([hugectr.EmbeddingTableConfig("dyn", -1, 8, init_capacity=77, max_capacity=999),
                          hugectr.EmbeddingTableConfig("st", 100, 8, init_param=InitParams(up_bound=0.25))],
                         ["a", "b"], "emb", ["sum", "sum"])
    ebc.shard([["dyn", "st"]], [("mp", ["dyn", "st"])],
              compression_strategy={hugectr.CompressionStrategy.Unique: ["st"], hugectr.CompressionStrategy.Reduction: ["dyn"]})
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["c"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    m.compile()
    p = str(tmp_path / "g.json")
    m.graph_to_json(p)
    j = [l for l in json.load(open(p))["layers"] if l["type"] == "EmbeddingCollection"][0]
    assert j["comm_strategy"] == "Hierarchical" and j["compression_strategy"] == {"Unique": ["st"], "Reduction": ["dyn"]}
    m2 = hugectr.Model(solver(), rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=cpu)
    m2.construct_from_json(p)
    m2.compile()
    c2 = m2.ebc_configs[0]
    t = {x.name: x for x in c2.tables()}
    assert t["dyn"].dynamic and (t["dyn"].init_capacity, t["dyn"].max_capacity) == (77, 999)
    assert t["st"].init_param.up_bound == 0.25 and c2.comm_strategy == hugectr.CommunicationStrategy.Hierarchical
    assert c2.compression_strategy == {hugectr.CompressionStrategy.Unique: ["st"], hugectr.CompressionStrategy.Reduction: ["dyn"]}
    m2.train()
    assert m2.get_current_loss() == m2.get_current_loss()
