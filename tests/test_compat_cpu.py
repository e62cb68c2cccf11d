"""Drop-in compatibility of the ``hugectr`` module name with scripts written for the reference."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def test_submodule_imports_used_by_reference_scripts():
    sys.path.insert(0, ROOT)
    from hugectr.data import DataSource, DataSourceParams          # noqa: F401
    from hugectr.inference import CreateInferenceSession, InferenceParams   # noqa: F401
    from hugectr.tools import DataGenerator, DataGeneratorParams   # noqa: F401
    import hugectr
    assert hugectr.tools.DataGenerator is DataGenerator
    assert hugectr.data.DataSourceParams is DataSourceParams
    p = DataSourceParams()
    assert hasattr(p, "server") and hasattr(p, "port")


def test_lr_scheduler_accepts_zero_warmup_and_decay_steps():
    """learning_rate_scheduler.hpp:40-46 only rejects negative values; the MLPerf script passes 0"""
    from hugectr_b200.lr_scheduler import LearningRateScheduler
    s = LearningRateScheduler(0.5, warmup_steps=0, decay_start=0, decay_steps=0)
    assert [s.get_next() for _ in range(3)] == [0.5, 0.5, 0.5]
    s = LearningRateScheduler(1.0, warmup_steps=0, decay_start=2, decay_steps=0, end_lr=0.1)
    assert [s.get_next() for _ in range(4)] == [1.0, 1.0, 0.1, 0.1]
    with pytest.raises(ValueError):
        LearningRateScheduler(-1.0)


def test_hugectr2onnx_package_name():
    sys.path.insert(0, ROOT)
    import inspect
    import hugectr2onnx
    sig = inspect.signature(hugectr2onnx.converter.convert)
    assert list(sig.parameters)[:7] == ["onnx_model_path", "graph_config", "dense_model", "convert_embedding",
                                        "sparse_models", "ntp_file", "graph_name"]


def test_data_reader_handle_api():
    """model.get_data_reader_train() handle: set_source / is_started / read_a_batch_to_device / is_eof"""
    import torch
    import hugectr_b200 as hugectr
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    m = build_dlrm_dcnv2(batchsize=16, num_gpus=1, table_sizes=[30, 40], multi_hot=[2, 1], ev_size=8,
                         mixed=False, bottom=(16, 8), top=(16, 1), projection_dim=4, cross_layers=1,
                         comm=Comm.single(torch.device("cpu")))
    m.compile()
    r = m.get_data_reader_train()
    assert isinstance(r, hugectr.Core23DataReader32) and isinstance(r, hugectr.DataReader64)
    r.set_source()
    assert r.read_a_batch_to_device() == 16 and not r.is_eof()
    r.ready_to_collect()
    assert r.read_a_batch_to_device_delay_release() == 16
    lab = m.check_out_tensor("label", hugectr.Tensor_t.Train)
    assert lab.shape == (16, 1)
    assert isinstance(hugectr.CreateOptimizer(), hugectr.Optimizer)


def test_cache_eval_data_replays_the_resident_round():
    import torch
    from hugectr_b200.data.readers import CachedEvalReader
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    m = build_dlrm_dcnv2(batchsize=16, num_gpus=1, table_sizes=[30, 40], multi_hot=[2, 1], ev_size=8,
                         mixed=False, bottom=(16, 8), top=(16, 1), projection_dim=4, cross_layers=1,
                         comm=Comm.single(torch.device("cpu")), max_eval_batches=3)
    m.reader_params.cache_eval_data = 3
    m.compile()
    r = m.get_data_reader_eval()
    assert isinstance(r, CachedEvalReader)
    calls = []
    inner_read = r.inner.read_a_batch
    r.inner.read_a_batch = lambda: (calls.append(1), inner_read())[1]
    rounds = []
    for _ in range(3):
        for _ in range(3):
            assert m.eval()
        rounds.append(m.get_eval_metrics()[0][1])
    assert len(calls) == 3                       # only the first round touched the source
    assert rounds[0] == rounds[1] == rounds[2]   # identical resident data, untrained model


def test_node_first_device_layout_permutes_the_shard_matrix():
    import hugectr_b200 as hugectr
    from types import SimpleNamespace as NS
    from hugectr_b200.model import Model
    sm = [[g] for g in range(6)]                       # row g marks "global id g"
    cfg = NS(shard_matrix=sm)
    fake = NS(solver=NS(device_layout=hugectr.DeviceLayout.NodeFirst, vvgpu=[[0, 1, 2], [0, 1, 2]]))
    out = Model._apply_device_layout(fake, cfg)
    # rank r = node * 3 + local  ->  NodeFirst global id = local * 2 + node
    assert [row[0] for row in out.shard_matrix] == [0, 2, 4, 1, 3, 5]
    assert Model._apply_device_layout(fake, out) is out                         # applied once
    fake.solver.device_layout = hugectr.DeviceLayout.LocalFirst
    assert Model._apply_device_layout(fake, cfg) is cfg


def test_shard_matrix_as_lists_of_table_names():
    """the documented reference form (hugectr_layer_book.md: "each row stores the name of embedding table
    that user want to place on row-th GPU") and the 0/1 matrix resolve to the same placement"""
    from hugectr_b200.embedding.collection import (EmbeddingCollectionConfig, EmbeddingTableConfig,
                                                   resolve_placement)

    def cfg(sm):
        c = EmbeddingCollectionConfig()
        ts = [EmbeddingTableConfig(n, 100, 8) for n in ("t0", "t1", "t2", "t3")]
        c.embedding_lookup(ts, ["a", "b", "c", "d"], "top", ["sum"] * 4)
        c.shard(sm, [("mp", ["t0", ("t1", 2)]), ("dp", ["t2", "t3"])])
        return resolve_placement(c, 4)
    names = [["t0", "t1", "t2", "t3"], ["t1", "t2", "t3"], ["t3", "t2", "t1"], ["t2", "t1", "t3"]]
    ints = [[1, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1, 1]]
    pa, pb = cfg(names), cfg(ints)
    for n in ("t0", "t1", "t2", "t3"):
        assert (pa[n].kind, pa[n].shard_gpus, pa[n].col_factor) == (pb[n].kind, pb[n].shard_gpus, pb[n].col_factor)
    assert pa["t0"].shard_gpus == [0] and pa["t1"].shard_gpus == [0, 1, 2, 3] and pa["t1"].col_factor == 2
    with pytest.raises(ValueError, match="unknown tables"):
        cfg([["t0", "nope"], [], [], []])


@pytest.mark.parametrize("cfg", ["simple_sparse_embedding_fp32.json", "simple_sparse_embedding_sgd.json"])
def test_reference_graph_json_constructs_and_trains(cfg, monkeypatch):
    """graph JSON files shipped with the reference (legacy layout with solver / optimizer sections around the
    layer list) load through construct_from_json and train"""
    import torch
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    monkeypatch.setenv("HCTR_FORCE_SYNTHETIC", "1")
    solver = hugectr.CreateSolver(batchsize=64, batchsize_eval=64, vvgpu=[[0]], max_eval_batches=1)
    reader = hugectr.DataReaderParams(hugectr.DataReaderType_t.Norm, source=["x"], eval_source="x",
                                      check_type=hugectr.Check_t.Sum)
    m = hugectr.Model(solver, reader, hugectr.CreateOptimizer(hugectr.Optimizer_t.Adam),
                      comm=Comm.single(torch.device("cpu")))
    m.construct_from_json(os.path.join(GOLDEN, cfg), True)
    m.compile()
    assert m.train() and m.get_current_loss() == m.get_current_loss()
    assert len(m.legacy_train) == 2           # one Distributed + one Localized embedding in the file


def _seed_global_rngs():
    """parts of the initialisation draw from the global generators: the stored parse was taken with these seeds"""
    import random
    import torch
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)


def _onnx_family_model(family):
    import torch
    from hugectr_b200 import models
    from hugectr_b200.parallel.comm import Comm
    _seed_global_rngs()
    kw = dict(comm=Comm.single(torch.device("cpu")), max_eval_batches=1)
    return {"dcn": lambda: models.build_dcn(batchsize=32, slot_sizes=[50] * 5, num_slots=5, vec=8, workspace_mb=1, **kw),
            "deepfm": lambda: models.build_deepfm(batchsize=32, **kw),
            "wdl": lambda: models.build_wdl(batchsize=32, **kw),
            "ncf": lambda: models.build_ncf("neumf", batchsize=64, num_users=300, num_items=200, **kw),
            "mmoe": lambda: models.build_mmoe(batchsize=64, num_slots=6, vocab=100, ev=8, expert_dims=(32, 16),
                                              tower_dim=8, **kw),
            "din": lambda: models.build_din(batchsize=32, seq_len=5, item_vocab=200, cate_vocab=30, user_vocab=50,
                                            ev=6, att_dims=(16, 8), mlp_dims=(24, 12), **kw),
            "bst": lambda: models.build_bst(batchsize=32, **kw)}[family]()


def _onnx_reference_parse():
    with open(os.path.join(GOLDEN, "onnx_loader_reference_parse.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("family", ["dcn", "deepfm", "wdl", "ncf", "mmoe", "din", "bst"])
def test_reference_onnx_loader_parses_our_graph_json_and_dense_model(family, tmp_path):
    """graph_to_json + <prefix>_dense_<it>.model written here were read layer by layer by the reference's own
    converter front end (onnx_converter/hugectr2onnx/hugectr_loader.py), consuming the weight file exactly; its
    parse -- byte range and value sums of every layer's weights -- is stored in tests/golden and the files written
    now must match it"""
    ref = _onnx_reference_parse()["dense"][family]
    m = _onnx_family_model(family)
    m.compile()
    m.train()
    m.graph_to_json(str(tmp_path / "g.json"))
    m.save_params_to_files(str(tmp_path / "m"), 1)
    dense = np.fromfile(tmp_path / "m_dense_1.model", dtype=np.float32).astype(np.float64)
    assert dense.nbytes // 2 == ref["consumed"]                   # (float64 copy: 8 bytes per stored float)
    assert len(json.load(open(tmp_path / "g.json"))["layers"]) == len(ref["layers"])
    end = 0
    for lay in ref["layers"]:
        assert lay["offset"] == end and lay["bytes"] % 4 == 0, lay
        w = dense[lay["offset"] // 4:(lay["offset"] + lay["bytes"]) // 4]
        assert np.isclose(w.sum(), lay["sum"], rtol=1e-4, atol=1e-4), lay
        assert np.isclose(np.abs(w).sum(), lay["abs_sum"], rtol=1e-4, atol=1e-4), lay
        end = lay["offset"] + lay["bytes"]


def test_reference_onnx_loader_reads_our_sparse_model_directories(tmp_path):
    """<prefix><i>_sparse_<it>.model/{key, emb_vector[, slot_id]} written here loaded into the reference converter's
    embedding tables (Distributed + Localized embeddings of the W&D sample): its key -> row mapping and tables are
    stored in tests/golden; the files written now are read with the same record layout (int64 key, one fp32 row of
    the table width, rows numbered from 1) and must give the same mapping, widths and rows"""
    import torch
    from hugectr_b200 import models
    from hugectr_b200.parallel.comm import Comm
    ref = _onnx_reference_parse()["sparse"]
    _seed_global_rngs()
    m = models.build_wdl(batchsize=32, comm=Comm.single(torch.device("cpu")), max_eval_batches=1)
    m.compile()
    for _ in range(3):
        m.train()
    m.graph_to_json(str(tmp_path / "g.json"))
    m.save_params_to_files(str(tmp_path / "m"), 3)
    assert [rt.vec for rt in m.legacy_train] == ref["widths"]
    parsed = []
    for i, rt in enumerate(m.legacy_train):
        d = tmp_path / f"m{i}_sparse_3.model"
        keys = np.fromfile(d / "key", dtype=np.int64)
        vecs = np.fromfile(d / "emb_vector", dtype=np.float32).reshape(-1, rt.vec)
        assert len(keys) == len(vecs) == ref["rows"][i]
        parsed.append((keys, vecs))
    keys, vecs = parsed[0]
    row_of = {int(k): j + 1 for j, k in enumerate(keys)}      # row 0 is the converter's default row
    assert sorted(row_of) == ref["table0_keys"]
    assert [row_of[k] for k in ref["table0_keys"]] == ref["table0_rows"]
    assert np.allclose([vecs[row_of[k] - 1].astype(np.float64).sum() for k in ref["table0_keys"]],
                       ref["table0_row_sums"], rtol=1e-4, atol=1e-5)
    # every key trained here is in the mapping, with the trained row behind it
    rt = m.legacy_train[0]
    tk, rows = rt.hash.dump()
    assert sum(int(k) in row_of for k in tk.tolist()) >= tk.numel() - 1
    k0 = int(tk[0])
    assert np.allclose(vecs[row_of[k0] - 1], rt.table.view(-1, rt.vec)[int(rows[0])].numpy())


def test_workspace_calculator_matches_the_reference_tool():
    """vocabulary / workspace sizes equal what the reference's tools/embedding_workspace_calculator script computes
    for the same inputs (its outputs are stored in tests/golden)"""
    import hugectr_b200 as hugectr
    from hugectr_b200.tools import workspace_calculator as W
    with open(os.path.join(GOLDEN, "workspace_calculator_reference.json")) as f:
        ref = json.load(f)
    slots = ref["slot_sizes"]
    assert len(ref["cases"]) == 90
    for c in ref["cases"]:
        gpus, opt, upd, vec = c["gpus"], c["opt"], c["update"], c["vec"]
        vd, vl = c["vocab_distributed"], c["vocab_localized"]
        assert vd == W.cal_vocabulary_size_per_gpu_for_distributed_slot(sum(slots), gpus)
        assert vl == W.cal_vocabulary_size_per_gpu_for_localized_slot(slots, gpus)
        assert c["workspace_distributed"] == W.cal_workspace_size_per_gpu_from_vocabulary_size_per_gpu(vd, vec, gpus, opt, upd)
        assert c["workspace_localized"] == W.cal_workspace_size_per_gpu_from_vocabulary_size_per_gpu(vl, vec, gpus, opt, upd)
        assert W.calculate(slots, vec, W._OPT[opt], W._UPD[upd], gpus) == c["workspace_distributed"]
        assert W.calculate(slots, vec, W._OPT[opt], W._UPD[upd], gpus,
                           hugectr.Embedding_t.LocalizedSlotSparseEmbeddingHash) == c["workspace_localized"]


def test_python_api_names_cover_the_reference_pybind_layer():
    """every enum value, module function, class and bound member name of the reference's pybind headers (names
    stored in tests/golden) exists here"""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tools_dev", "api_parity.py"), "--json"],
                       capture_output=True, text=True, timeout=300)
    rep = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert rep["missing"] == [] and rep["enums"] >= 20 and rep["members"] >= 80, rep
