"""CPU tests: hash table, gpu_cache (reference impl), HPS/offload, SOK, metrics, LR schedule,
planner, logger, filesystem, DataGenerator/readers round trip."""
import os

import numpy as np
import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.parallel.comm import Comm, DeviceMap


def test_hashtable_cpu():
    from hugectr_b200.embedding.hashtable import HashTable
    ht = HashTable(100, "cpu")
    k = torch.tensor([5, 9, 5, -1, 1000000007])
    r = ht.get_insert(k)
    assert r.tolist() == [0, 1, 0, -1, 2] and ht.size() == 3
    assert ht.get(torch.tensor([9, 77])).tolist() == [1, -1]
    keys, rows = ht.dump()
    assert keys.tolist() == [5, 9, 1000000007] and rows.tolist() == [0, 1, 2]


def test_gpu_cache_reference_lru():
    from hugectr_b200.cache import GpuCache
    c = GpuCache(64, 4, "cpu", ways=32)
    keys = torch.arange(10)
    vals = torch.arange(40).float().view(10, 4)
    out, mi, mk = c.query(keys)
    assert mi.numel() == 10
    c.replace(keys, vals)
    out, mi, mk = c.query(torch.tensor([3, 99, 7]))
    assert mi.tolist() == [1] and mk.tolist() == [99]
    torch.testing.assert_close(out[0], vals[3])
    c.update(torch.tensor([3, 1234]), torch.ones(2, 4))
    torch.testing.assert_close(c.query(torch.tensor([3]))[0][0], torch.ones(4))
    assert set(c.dump().tolist()) == set(range(10))


def test_offloaded_embedding_matches_dense():
    from hugectr_b200.cache import OffloadedEmbedding
    opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad, initial_accu_value=0.0, epsilon=1e-6)
    e = OffloadedEmbedding(8, "cpu", cache_rows=64, opt=opt, num_states=1, lr=0.1)
    keys = torch.randint(0, 500, (16, 3))
    y = e.forward(keys)
    w0, _ = e.ps.pull(e.uniq)
    torch.testing.assert_close(y, w0[e.inv].view(16, 3, 8).sum(1))
    e.backward(torch.ones(16, 8))
    w1, s1 = e.ps.pull(e.uniq)
    assert (w1 - w0).abs().max() > 0 and (s1[0] > 0).all()


def test_sok_lookup_and_optimizer():
    from hugectr_b200 import sok
    sok.init(Comm.single(torch.device("cpu")))
    v = sok.Variable(shape=(50, 4), name="v_test")
    d = sok.DynamicVariable(4, name="d_test", init_capacity=8)
    ids = torch.tensor([[1, 2, -1], [3, 3, 3]])
    out = sok.lookup_sparse(v, ids, "mean")
    exp = torch.stack([(v.weight[1] + v.weight[2]) / 2, v.weight[3]])
    torch.testing.assert_close(out, exp)
    big = torch.tensor([[10 ** 12, 5], [7, 10 ** 12]])
    o2 = sok.lookup_sparse(d, big, "sum")
    assert d.size == 3
    (out.sum() + o2.sum()).backward()
    opt = sok.OptimizerWrapper(hugectr.Optimizer_t.SGD, lr=0.5)
    w_before = v.weight.clone()
    opt.apply_gradients([v, d])
    assert not torch.allclose(v.weight[3], w_before[3])
    torch.testing.assert_close(v.weight[0], w_before[0])


def test_sok_dump_load(tmp_path):
    from hugectr_b200 import sok
    sok.init(Comm.single(torch.device("cpu")))
    v = sok.Variable(shape=(20, 4), name="v_dl")
    sok.dump(str(tmp_path), [v])
    w = v.weight.clone()
    v.weight.zero_()
    sok.load(str(tmp_path), [v])
    torch.testing.assert_close(v.weight, w)


def test_metrics_auc_matches_sklearn():
    from sklearn.metrics import roc_auc_score
    from hugectr_b200.metrics import auc_exact
    g = torch.Generator().manual_seed(1)
    p = torch.rand(5000, generator=g).round(decimals=2)   # many ties
    y = (torch.rand(5000, generator=g) < p).float()
    assert abs(auc_exact(p, y) - roc_auc_score(y.numpy(), p.numpy())) < 1e-6


def test_lr_scheduler_and_device_map():
    from hugectr_b200.lr_scheduler import LearningRateScheduler
    s = LearningRateScheduler(1.0, warmup_steps=4, decay_start=6, decay_steps=4, decay_power=2.0, end_lr=0.1)
    lrs = [s.get_next() for _ in range(12)]
    assert lrs[:4] == [0.25, 0.5, 0.75, 1.0] and lrs[5] == 1.0
    assert abs(lrs[7] - 0.25) < 1e-9 and lrs[-1] == 0.1
    dm = DeviceMap([[0, 1], [0, 1]], "NodeFirst", my_node=1)
    assert dm.get_global_id(0) == 1 and dm.get_global_id(1) == 3 and dm.size() == 4
    dm2 = DeviceMap([[0, 1], [0, 1]], "LocalFirst", my_node=1)
    assert dm2.get_global_id(0) == 2


def test_planner_and_workspace():
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    from hugectr_b200.tools.planner import generate_plan
    from hugectr_b200.tools.workspace_calculator import calculate
    sm, st = generate_plan(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, 8)
    assert len(sm) == 8 and all(len(r) == 26 for r in sm)
    kinds = dict((k, v) for k, v in st)
    assert "mp" in kinds and "dp" in kinds
    assert sum(sm[g][20] for g in range(8)) > 1          # hot table split row-wise
    for t in range(26):
        assert any(sm[g][t] for g in range(8))
    assert calculate([1000] * 26, 16, hugectr.Optimizer_t.Adam) >= 1
    from hugectr_b200.tools import planner
    rep = planner.plan_report(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, sm)
    assert rep["imbalance"] < 1.6 and max(rep["memory_gb"]) < 150
    # node-aware plan: all shards of the split hot table live on one node
    sm2, _ = generate_plan(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, 16, num_nodes=2)
    owners = [g for g in range(16) if sm2[g][20]]
    assert len(owners) > 1 and len({g // 8 for g in owners}) == 1
    import os, tempfile
    pth = os.path.join(tempfile.mkdtemp(), "plan.json")
    planner.main(["--num-gpus", "8", "--out", pth])
    sm3, st3, _ = planner.load_plan(pth)
    assert sm3 == sm and [k for k, _ in st3] == [k for k, _ in st]


def test_solver_validation_and_json_optimizer():
    with pytest.raises(RuntimeError):
        hugectr.CreateSolver(use_mixed_precision=True, enable_tf32_compute=True)
    o = hugectr.CreateOptimizer(hugectr.Optimizer_t.Ftrl, beta=0.1, lambda1=0.2, lambda2=0.3)
    o2 = hugectr.OptParamsPy.from_json(o.to_json())
    assert (o2.beta, o2.lambda1, o2.lambda2) == (0.1, 0.2, 0.3)


def test_filesystem_and_logger(tmp_path, capsys):
    from hugectr_b200.io import FileSystemBuilder
    from hugectr_b200.utils import logger
    fs = FileSystemBuilder.build_by_path(str(tmp_path / "a" / "b.bin"))
    fs.write(str(tmp_path / "a" / "b.bin"), b"hello")
    assert fs.read(str(tmp_path / "a" / "b.bin"), 1, 3) == b"ell"
    assert fs.get_file_size(str(tmp_path / "a" / "b.bin")) == 5
    logger.Logger.get().level = 2
    logger.info("hi there")
    assert "[HCTR]" in capsys.readouterr().out
    with pytest.raises(logger.HctrError):
        logger.check(False, hugectr.Error_t.WrongInput, "bad")


def test_norm_checksum_detects_corruption(tmp_path):
    from hugectr_b200.data.generator import DataGenerator, DataGeneratorParams
    from hugectr_b200.data.norm_reader import DataCheckError
    from hugectr_b200.models.legacy import build_dcn
    slots = [50] * 4
    p = DataGeneratorParams(hugectr.DataReaderType_t.Norm, 1, 13, 4, False,
                            str(tmp_path / "l.txt"), str(tmp_path / "v.txt"), slots, num_files=1,
                            eval_num_files=1, num_samples_per_file=64)
    DataGenerator(p).generate()
    f = str(tmp_path / "train" / "gen_0.data")
    raw = bytearray(open(f, "rb").read())
    raw[100] ^= 0xFF
    open(f, "wb").write(raw)
    m = build_dcn(batchsize=32, source=p.source, eval_source=p.eval_source, slot_sizes=slots,
                  num_slots=4, fmt=hugectr.DataReaderType_t.Norm, workspace_mb=1,
                  comm=Comm.single(torch.device("cpu")))
    m.reader_params.check_type = hugectr.Check_t.Sum
    m.compile()
    with pytest.raises(DataCheckError):
        m.train()


def test_pipeline_and_inference(tmp_path):
    from hugectr_b200.inference import CreateInferenceSession, InferenceParams
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.pipeline import Pipeline, StreamContextScheduleable
    order = []
    a = StreamContextScheduleable(lambda: order.append("a"), "a")
    b = StreamContextScheduleable(lambda: order.append("b"), "b").wait_event([a])
    Pipeline("p", "cpu", [a, b]).run()
    assert order == ["a", "b"]
    m = build_dlrm_dcnv2(batchsize=16, num_gpus=1, table_sizes=[30, 40], multi_hot=[2, 1], ev_size=8,
                         mixed=False, bottom=(16, 8), top=(16, 1), projection_dim=4, cross_layers=1,
                         comm=Comm.single(torch.device("cpu")))
    m.compile()
    m.train()
    m.graph_to_json(str(tmp_path / "g.json"))
    m.save_params_to_files(str(tmp_path / "m"), 1)
    sess = CreateInferenceSession(str(tmp_path / "g.json"), InferenceParams(
        "dlrm", 16, dense_model_file=str(tmp_path / "m_dense_1.model"),
        embedding_collection_path=str(tmp_path / "m_ebc_1")), )
    hb = m.reader_eval.read_a_batch()
    pred = sess.predict(hb.dense.numpy(), hb.keys.numpy())
    m._load_batch(hb, False)
    for e in m.ebcs_eval:
        e.forward(False)
    m.net_eval.fprop(False)
    ref = m.net_eval.loss_layers[0].pred.numpy()
    assert np.abs(pred - ref).max() < 1e-5


def test_sparse_tensor_and_simulators():
    from hugectr_b200.utils.data_simulator import VarianceScalingSimulator, sinusoidal_init
    from hugectr_b200.utils.sparse_tensor import SparseTensor
    k = torch.tensor([[3, 4, -1], [5, -1, -1], [-1, -1, -1]])
    st = SparseTensor.from_padded(k)
    assert st.nnz == 3 and st.row_offsets.tolist() == [0, 2, 3, 3]
    assert torch.equal(st.to_padded(3), k)
    t = torch.empty(1000, 64)
    VarianceScalingSimulator(1.0, "fan_avg", "uniform", 1000, 64).fill(t)
    assert abs(t.var().item() - 1.0 / 532) < 3e-4
    assert sinusoidal_init(10, 8).shape == (10, 8)


def test_native_parameter_server_index(tmp_path):
    """csrc/host/param_server.cpp: deterministic row assignment, duplicates, capacity roll-back, SSD
    spill round trip"""
    from hugectr_b200.cache.hps import HostParameterServer
    ps = HostParameterServer(4, num_states=1, init_bound=0.1, capacity_rows=8, ssd_path=str(tmp_path / "ssd"))
    assert ps._h is not None, "native host library was not built"
    k = torch.tensor([7, 3, 7, 1 << 40, 3])
    w, (s0,) = ps.pull(k)
    assert ps.size() == 3 and w.shape == (5, 4)
    torch.testing.assert_close(w[0], w[2])
    torch.testing.assert_close(w[1], w[4])
    assert (w.abs() <= 0.1).all() and (s0 == 0).all()
    ps.push(torch.tensor([3, 1 << 40]), torch.ones(2, 4), [torch.full((2, 4), 2.0)])
    w2, (s2,) = ps.pull(torch.tensor([1 << 40, 3, 7]))
    torch.testing.assert_close(w2[:2], torch.ones(2, 4))
    torch.testing.assert_close(s2[:2], torch.full((2, 4), 2.0))
    torch.testing.assert_close(w2[2], w[0])
    keys, rows = ps.items()
    assert dict(zip(keys.tolist(), rows.tolist())) == {7: 0, 3: 1, 1 << 40: 2}
    with pytest.raises(RuntimeError):
        ps.pull(torch.arange(100, 110))            # 3 + 10 > capacity 8: nothing is inserted
    assert ps.size() == 3
    ps.flush_to_ssd()
    ps2 = HostParameterServer(4, num_states=1, capacity_rows=8, ssd_path=str(tmp_path / "ssd"))
    w3, _ = ps2.pull(torch.tensor([3]))
    torch.testing.assert_close(w3[0], torch.ones(4))


def test_native_library_abi_matches_python_mirrors():
    """the sm_90a library loads without a GPU; its struct sizes must equal the ctypes mirrors"""
    from hugectr_b200.embedding import ops as E
    from hugectr_b200.ops import dense as D
    E.lib()
    D.lib()


def test_native_raw_reader_slices_and_layout(tmp_path):
    """csrc/host/raw_reader.cpp: per-rank slice of every global batch, feature-major keys, incomplete
    last batch, log1p of integer dense features (Appendix A.6)"""
    import types
    from hugectr_b200.data.raw_reader import RawAsyncReader
    N = 20
    path = str(tmp_path / "t.bin")

    def write(dense_float):
        rec = []
        for i in range(N):
            dense = np.array([i, i + 0.5], "<f4").view("<u4") if dense_float else np.array([i, 3 * i], "<u4")
            rec.append(np.concatenate([np.array([float(i)], "<f4").view("<u4"), dense,
                                       np.array([i, i + 1, 2 * i], "<u4")]))
        np.stack(rec).astype("<u4").tofile(path)

    def stub(rank, dense_float):
        m = types.SimpleNamespace()
        m.reader_params = types.SimpleNamespace(
            source=[path], eval_source=path, async_param=hugectr.AsyncParam(2, 2, is_dense_float=dense_float),
            float_label_dense=dense_float, num_samples=N, eval_num_samples=N)
        m.b_train = m.b_eval = 4
        m.comm = types.SimpleNamespace(rank=rank)
        m.world = 2
        m.input = types.SimpleNamespace(label_dim=1, dense_dim=2)
        m.layout = types.SimpleNamespace(blocks=[("a", 1, 2, True), ("b", 1, 1, True)])
        m.solver = types.SimpleNamespace(repeat_dataset=False, i64_input_key=False)
        m.key_dtype = torch.int32
        m.device = torch.device("cpu")
        return m

    write(True)
    for rank, firsts, valid in ((0, [0, 8, 16], [4, 4, 4]), (1, [4, 12], [4, 4, 0])):
        r = RawAsyncReader(stub(rank, True), True)
        got = []
        while True:
            hb = r.read_a_batch()
            if hb is None:
                break
            got.append((hb.num_valid, hb.label.reshape(-1).clone(), hb.dense.clone(), hb.keys.clone()))
        r.stop()
        assert [g[0] for g in got] == valid
        for g, f in zip(got, firsts):
            i = torch.arange(f, f + 4)
            assert g[1].tolist() == i.float().tolist()
            torch.testing.assert_close(g[2], torch.stack([i.float(), i.float() + 0.5], 1))
            # feature-major: table a [4 samples x 2 hot] then table b [4 x 1]
            exp = torch.cat([torch.stack([i, i + 1], 1).reshape(-1), 2 * i]).int()
            assert g[3].tolist() == exp.tolist()
    write(False)
    r = RawAsyncReader(stub(0, False), True)
    hb = r.read_a_batch()
    i = torch.arange(0, 4).float()
    torch.testing.assert_close(hb.dense, torch.stack([torch.log1p(i), torch.log1p(3 * i)], 1))
    r.stop()


def test_diagnose_threadpool_mlperf_and_criteo2raw(tmp_path, capsys):
    from hugectr_b200.utils import diagnose
    from hugectr_b200.utils.thread_pool import CPUResource, ThreadPool
    from hugectr_b200.tools import criteo2raw
    good = torch.randn(100)
    assert diagnose.verify(good, "good")
    bad = good.clone()
    bad[3] = float("nan")
    assert not diagnose.verify(bad, "bad", raise_on_error=False)
    with pytest.raises(Exception):
        diagnose.verify(bad, "bad")
    h = diagnose.histogram(good, bins=8)
    assert int(h.sum()) == 100 and h.numel() == 8
    assert diagnose.sample(good, 5).numel() == 5
    tp = ThreadPool(3)
    fs = [tp.submit(lambda x: x * x, i) for i in range(10)]
    tp.await_idle(fs)
    assert [f.result() for f in fs] == [i * i for i in range(10)]
    cr = CPUResource(7, [1, 2])
    a, b = torch.rand(3, generator=cr.get_replica_uniform_generator()), torch.rand(3, generator=CPUResource(7, [1, 2]).get_replica_uniform_generator())
    assert torch.equal(a, b)
    # criteo TSV -> raw records with frequency-thresholded categorification
    lines = []
    rng = np.random.default_rng(0)
    for i in range(50):
        dense = [str(int(x)) for x in rng.integers(0, 100, 13)]
        cats = [format(int(x), "x") for x in rng.integers(0, 5, 26)]
        lines.append("\t".join([str(i % 2)] + dense + cats))
    tsv = tmp_path / "day_0.tsv"
    tsv.write_text("\n".join(lines) + "\n")
    vocabs, sizes = criteo2raw.convert(str(tsv), str(tmp_path / "out.bin"), min_freq=2)
    rec = np.fromfile(str(tmp_path / "out.bin"), dtype="<u4").reshape(50, 1 + 13 + 26)
    assert rec[:, 0].tolist() == [i % 2 for i in range(50)]
    assert all(rec[:, 14 + j].max() < sizes[j] for j in range(26)) and len(vocabs) == 26


def test_mlperf_logging_callback_emits_events(capsys):
    from hugectr_b200.utils.mlperf import LoggingCallback
    cb = LoggingCallback(auc_threshold=0.8, iter_per_epoch=100.0, batchsize=64)
    cb.on_training_start()
    assert cb.on_eval_start(50) is False
    assert cb.on_eval_end(50, {"AUC": 0.7}) is False
    assert cb.on_eval_end(100, {"AUC": 0.81}) is True          # threshold reached -> stop
    cb.on_training_end(100)
    out = capsys.readouterr()
    text = out.out + out.err
    for key in ("run_start", "eval_accuracy", "run_stop", "train_samples"):
        assert key in text


def test_hps_inference_session_matches_direct_lookup(tmp_path):
    """use_gpu_embedding_cache: tables in the host parameter server + device LRU cache; predictions
    equal the plain session, repeated batches hit the cache, unknown keys read as zeros"""
    from hugectr_b200.cache import HpsEmbedding
    from hugectr_b200.inference import CreateInferenceSession, InferenceParams
    from hugectr_b200.models import build_dcn
    m = build_dcn(batchsize=32, slot_sizes=[60] * 26, workspace_mb=1, comm=Comm.single(torch.device("cpu")),
                  max_eval_batches=1, batchsize_eval=32)
    m.compile()
    for _ in range(3):
        m.train()
    pre = str(tmp_path / "dcn")
    m.save_params_to_files(pre, 3)
    m.graph_to_json(pre + ".json")
    common = dict(dense_model_file=pre + "_dense_3.model", sparse_model_files=[pre + "0_sparse_3.model"])
    plain = CreateInferenceSession(pre + ".json", InferenceParams("dcn", 32, **common))
    hps = CreateInferenceSession(pre + ".json", InferenceParams("dcn", 32, use_gpu_embedding_cache=True,
                                                                cache_size_percentage=0.5, **common))
    assert hps.hps, "HPS path not active"
    for i in range(3):
        hb = m.reader_eval.pool[i % len(m.reader_eval.pool)]
        a = plain.predict(hb.dense.numpy(), hb.keys.numpy())
        b = hps.predict(hb.dense.numpy(), hb.keys.numpy())
        assert np.abs(a - b).max() < 1e-6
    svc = list(hps.hps.values())[0]
    r0 = svc.hit_rate()
    hb = m.reader_eval.pool[0]
    hps.predict(hb.dense.numpy(), hb.keys.numpy())          # same batch again: served from the cache
    assert svc.hit_rate() > r0
    e = HpsEmbedding(torch.tensor([5, 9]), torch.tensor([[1., 1.], [2., 2.]]), "cpu", combiner="mean")
    out = e.lookup(torch.tensor([[[5, 9, -1], [777, -1, -1]]]))
    torch.testing.assert_close(out, torch.tensor([[[1.5, 1.5], [0., 0.]]]))


def test_heterogeneous_planner_properties():
    """plan_tables: widths / combiners per table, row + column splits, memory cap, node locality"""
    from hugectr_b200.embedding.collection import (EmbeddingCollectionConfig, EmbeddingTableConfig,
                                                   resolve_placement)
    from hugectr_b200.tools.planner import HardwareModel, plan_tables
    nt = [5, 5, 5, 5, 20, 30, 10, 20, 10, 10, 10, 5, 40, 1, 1]
    vs = [10000, 4000000, 4000000, 50000000, 1000, 10000, 5000000, 4000000, 10, 1000, 10000, 100000, 4000000,
          50000000, 500000000]
    nz = [100, 50, 30, 50, 50, 30, 20, 20, 100, 10, 100, 100, 200, 100, 100]
    ev = [128, 64, 64, 32, 128, 128, 256, 128, 128, 64, 128, 64, 64, 128, 32]
    S = [v for n, v in zip(nt, vs) for _ in range(n)]
    H = [v for n, v in zip(nt, nz) for _ in range(n)]
    E = [v for n, v in zip(nt, ev) for _ in range(n)]
    for gpus, nodes in ((8, 1), (16, 2)):
        sm, st, rep = plan_tables(S, H, E, gpus, num_nodes=nodes)
        assert rep["imbalance"] < 1.15, rep["imbalance"]
        assert max(rep["memory_gb"]) <= 150.0
        # the plan is accepted by the collection as is
        cfg = EmbeddingCollectionConfig()
        ts = [EmbeddingTableConfig(str(i), S[i], E[i]) for i in range(len(S))]
        cfg.embedding_lookup(ts, [f"d{i}" for i in range(len(S))], "top", ["sum"] * len(S))
        cfg.shard(sm, st)
        place = resolve_placement(cfg, gpus)
        assert all(p is not None for p in place.values())
        for kind, items in st:
            for it in items:
                if isinstance(it, tuple):
                    t, c = int(it[0]), it[1]
                    assert E[t] % c == 0 and E[t] // c >= 32 and sum(r[t] for r in sm) % c == 0
    # a table that does not fit one GPU is split until it does; its shards stay inside one node
    hw = HardwareModel(hbm_capacity_gb=20.0)
    sm, st, rep = plan_tables([40_000_000] + [2_000_000] * 15 + [1000, 50], [3] * 16 + [1, 1], 128, 16,
                              num_nodes=2, hw=hw)
    owners = [g for g in range(16) if sm[g][0]]
    assert 4 <= len(owners) <= 8 and len({g // 8 for g in owners}) == 1, owners
    assert max(rep["memory_gb"]) <= 20.0
    assert rep["dp"] == ["16", "17"]
    # a tiny table looked up 200 times per sample with the concat combiner: never data-parallel, and
    # only row-splittable (concat outputs keep whole vectors)
    sm, st, rep = plan_tables([5000, 5000000], [200, 1], [64, 64], 8, combiners=["concat", "sum"])
    assert "0" not in rep["dp"] and all(not isinstance(x, tuple) or x[0] != "0" for x in st[0][1])
    # CLI
    from hugectr_b200.tools import planner
    sm, st = planner.main(["--num-gpus", "8", "--ev-sizes", ",".join(["128"] * 26)])
    assert len(sm) == 8 and len(sm[0]) == 26


def test_planners_property_based():
    """hypothesis: any table set -> both planners return a plan the collection accepts, every table is
    placed, column factors divide widths and shard counts, data-parallel tables sit on every GPU"""
    from hypothesis import given, settings, strategies as st
    from hugectr_b200.embedding.collection import (EmbeddingCollectionConfig, EmbeddingTableConfig,
                                                   resolve_placement)
    from hugectr_b200.tools.planner import generate_plan, plan_tables

    tables = st.lists(st.tuples(st.integers(1, 50_000_000), st.integers(1, 120), st.sampled_from([8, 16, 32, 64, 128, 256])),
                      min_size=1, max_size=40)

    @settings(max_examples=60, deadline=None)
    @given(tables, st.sampled_from([1, 2, 4, 8, 16]), st.booleans())
    def check(tabs, gpus, hetero):
        S, H, E = [t[0] for t in tabs], [t[1] for t in tabs], [t[2] for t in tabs]
        nodes = 2 if gpus == 16 else 1
        if hetero:
            sm, strat, rep = plan_tables(S, H, E, gpus, num_nodes=nodes)
            assert len(rep["step_cost_us"]) == gpus
        else:
            E = [128] * len(S)
            sm, strat = generate_plan(S, H, gpus, ev_size=128, num_nodes=nodes)
        assert len(sm) == gpus and all(len(r) == len(S) for r in sm)
        listed = set()
        for kind, items in strat:
            for it in items:
                name, c = (it[0], it[1]) if isinstance(it, tuple) else (it, 1)
                t = int(name)
                listed.add(t)
                owners = sum(r[t] for r in sm)
                assert owners >= 1
                if kind == "dp":
                    assert owners == gpus
                else:
                    assert owners % c == 0 and E[t] % c == 0
        assert listed == set(range(len(S)))
        cfg = EmbeddingCollectionConfig()
        ts = [EmbeddingTableConfig(str(i), S[i], E[i]) for i in range(len(S))]
        cfg.embedding_lookup(ts, [f"d{i}" for i in range(len(S))], "top", ["sum"] * len(S))
        cfg.shard(sm, strat)
        assert all(p is not None for p in resolve_placement(cfg, gpus).values())
    check()
