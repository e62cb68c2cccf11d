"""fp8 serving tables (InferenceParams.fp8_quant, EmbeddingCollection(fp8_quant=True)) on the CPU path: the
quantization rule by hand and against the MX block rule, whole-session predictions equal to an fp32 session over
the dequantized checkpoint, no training state, and the rejections."""
import os
import shutil

import numpy as np
import pytest
import torch

from hugectr_b200.embedding import ops as E

CPU = torch.device("cpu")


def _bytes(q):
    return q.view(torch.uint8).tolist()


# ------------------------------------------------------------------ the rule
def test_fp8_rows_rule_hand_computed_values():
    x = torch.tensor([
        [448.0, 1.0625, -3.0, 1.0],                   # amax exactly 448: e = 0; 1.0625 ties to even -> 1.0
        [1792.0, 4.25, -1792.0, 0.0],                 # amax 448 * 2^2: e = 2; 4.25 / 4 ties to even -> 1.0
        [448.0, 3 * 2.0 ** -9, 2.0 ** -10, 1.5 * 2.0 ** -9],   # e4m3 subnormals: 3, 0 (tie), 2 (tie) x 2^-9
        [0.0, 0.0, 0.0, 0.0],                         # all zero: e = -127, zero bytes
        [-0.5, 0.25, 0.125, -0.0625],                 # amax 0.5: 0.5 / 448 = 0.56 * 2^-9 -> e = -9
    ])
    q, e = E.fp8_rows_quantize(x)
    assert (e.to(torch.int32) - 127).tolist() == [0, 2, 0, -127, -9]
    assert _bytes(q) == [
        [0x7E, 0x38, 0xC4, 0x38],
        [0x7E, 0x38, 0xFE, 0x00],
        [0x7E, 0x03, 0x00, 0x02],
        [0x00, 0x00, 0x00, 0x00],
        [0xF8, 0x70, 0x68, 0xE0],                     # -256, 128, 64, -32 at 2^-9
    ]
    # one column: 5 / 448 = 0.714 * 2^-6 -> e = -6, q = 320 = 1.25 * 2^8
    q1, e1 = E.fp8_rows_quantize(torch.tensor([[5.0]]))
    assert _bytes(q1) == [[0x7A]] and int(e1[0]) == 127 - 6
    d = E.fp8_rows_dequantize(q, e)
    assert d[0].tolist() == [448.0, 1.0, -3.0, 1.0] and d[4].tolist() == [-0.5, 0.25, 0.125, -0.0625]
    assert d[3].tolist() == [0.0] * 4 and E.fp8_rows_dequantize(q1, e1).tolist() == [[5.0]]


def test_fp8_rows_rule_is_the_mx_block_rule_on_32_wide_rows():
    from hugectr_b200.ops.mxfp8 import mx_quantize_reference
    g = torch.Generator().manual_seed(3)
    x = torch.randn(128, 128, generator=g) * torch.exp2(torch.randint(-20, 20, (128, 4, 1), generator=g).float()) \
        .expand(128, 4, 32).reshape(128, 128)
    x[5, 32:64] = 0.0
    mq, msf = mx_quantize_reference(x)
    sfb = msf.view(1, 1, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(128, 4)      # [row, 32-wide block]
    q, e = E.fp8_rows_quantize(x.reshape(-1, 32))
    assert torch.equal(q.view(torch.uint8), mq.reshape(-1, 32))
    assert torch.equal(e, sfb.reshape(-1))


# ------------------------------------------------------------------ sessions
def build_serving_test_model(tmp_path, device, iters=4, seed=5):
    """A small model over one collection covering every storage class a serving collection quantizes: sum over
    variable hotness (model parallel), mean (data parallel), concat, a growing dynamic table and an evicting
    table.  Trains ``iters`` steps, saves graph JSON + snapshot under ``tmp_path`` and returns (model, paths)."""
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]], repeat_dataset=True,
                                  max_eval_batches=2, use_cuda_graph=False, seed=seed)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.0"],
                                  eval_source="synthetic:1.0", check_type=hugectr.Check_t.Non,
                                  slot_size_array=[400, 300, 50, 500, 500])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad), comm=Comm.single(device))
    sp = hugectr.DataReaderSparseParam
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=3, dense_name="dense",
                        data_reader_sparse_param_array=[sp("a", 4, False, 1), sp("b", 3, False, 1), sp("c", 2, True, 1),
                                                        sp("d", 2, True, 1), sp("e", 3, False, 1)]))
    T = hugectr.EmbeddingTableConfig
    tabs = [T("ts", 400, 8), T("tm", 300, 8), T("tc", 50, 8), T("tg", -1, 8, init_capacity=1024),
            T("tv", -1, 8, evict_strategy="lru", max_capacity=64)]
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup(tabs, ["a", "b", "c", "d", "e"], "emb", ["sum", "mean", "concat", "sum", "mean"])
    ebc.shard([[t.name for t in tabs]], [("mp", ["ts", "tc", "tg", "tv"]), ("dp", ["tm"])])
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["x"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["x"], ["fc1"], num_output=16))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.ReLU, ["fc1"], ["r1"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["r1"], ["fc2"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc2", "label"], ["loss"]))
    m.compile()
    for _ in range(iters):
        m.train()
    d = str(tmp_path)
    m.save_params_to_files(os.path.join(d, "m"), iters)
    m.graph_to_json(os.path.join(d, "g.json"))
    return m, dict(graph=os.path.join(d, "g.json"), dense=os.path.join(d, f"m_dense_{iters}.model"),
                   ebc=os.path.join(d, f"m_ebc_{iters}"))


def rewrite_ebc_weights(src: str, dst: str, fn):
    """copy the collection snapshot ``src`` to ``dst`` with every table's weights [n, ev] replaced by fn(W)"""
    from hugectr_b200.io.checkpoint import FILE_HEAD_NBYTES
    shutil.copytree(src, dst)
    for root, _, files in os.walk(dst):
        for f in files:
            if not f.startswith("weight"):
                continue
            p = os.path.join(root, f)
            raw = open(p, "rb").read()
            tid = int(f[len("weight"):])
            ev = _ev_of(root, tid)
            W = torch.from_numpy(np.frombuffer(raw[FILE_HEAD_NBYTES:], dtype="<f4").copy()).view(-1, ev)
            with open(p, "wb") as fh:
                fh.write(raw[:FILE_HEAD_NBYTES] + fn(W).numpy().astype("<f4").tobytes())


def _ev_of(folder, tid):
    from hugectr_b200.io.checkpoint import META_HEAD_NBYTES
    meta = open(os.path.join(folder, "meta_data"), "rb").read()
    n = int(np.frombuffer(meta[:META_HEAD_NBYTES], dtype="<i4")[0])
    off = META_HEAD_NBYTES
    ids = np.frombuffer(meta[off:off + 4 * n], dtype="<i4").tolist()
    evs = np.frombuffer(meta[off + 12 * n:off + 16 * n], dtype="<i4").tolist()
    return int(evs[ids.index(tid)])


def fp8_round_trip(W):
    return E.fp8_rows_dequantize(*E.fp8_rows_quantize(W))


def session_predictions_match(m, paths, tmp_path, device):
    """fp8 session over the snapshot vs fp32 session over the dequantized snapshot: equal predictions"""
    from hugectr_b200.inference import InferenceModel, InferenceParams
    oracle = os.path.join(str(tmp_path), "oracle_ebc")
    rewrite_ebc_weights(paths["ebc"], oracle, fp8_round_trip)
    dev = str(device)
    mk = lambda ebc, fp8: InferenceModel(paths["graph"], InferenceParams(  # noqa: E731
        model_name="x", max_batchsize=32, dense_model_file=paths["dense"], embedding_collection_path=ebc,
        fp8_quant=fp8), device=dev)
    s8, s32 = mk(paths["ebc"], True), mk(oracle, False)
    assert all(g.wdtype == "fp8" for e in s8.model.ebcs_eval for g in e.groups)
    assert {g.kind for e in s8.model.ebcs_eval for g in e.groups} == {"mp", "dp"}
    n = 0
    for _ in range(3):
        hb = m.reader_eval.read_a_batch()
        dense, keys = hb.dense.cpu().numpy(), hb.keys.cpu().numpy()
        p8, p32 = s8.predict(dense, keys), s32.predict(dense, keys)
        assert float(np.abs(p8 - p32).max()) == 0.0
        n += p8.size
    assert n == 96
    return s8, s32


def test_fp8_session_predicts_as_fp32_session_on_dequantized_checkpoint_cpu(tmp_path):
    m, paths = build_serving_test_model(tmp_path, CPU)
    s8, s32 = session_predictions_match(m, paths, tmp_path, CPU)
    # the fp8 collection dumps the dequantized values
    e8, e32 = s8.model.ebcs_train[0], s32.model.ebcs_train[0]
    for t in ("ts", "tm", "tc", "tg", "tv"):
        (k8, w8, *_), = e8.dump_table_local(t)
        (k32, w32, *_), = e32.dump_table_local(t)
        assert torch.equal(k8, k32) and torch.equal(w8, w32)


def test_fp8_serving_collection_holds_no_training_state_cpu():
    import hugectr_b200 as hugectr
    from hugectr_b200.embedding.collection import EmbeddingCollection
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import OptParamsPy
    T = hugectr.EmbeddingTableConfig
    tabs = [T("s", 100, 12), T("d", 30, 12), T("g", -1, 8, init_capacity=64, admit_threshold=2)]
    cfg = hugectr.EmbeddingCollectionConfig()
    cfg.embedding_lookup(tabs, ["a", "b", "c"], "emb", ["sum", "mean", "sum"])
    cfg.shard([["s", "d", "g"]], [("mp", ["s", "g"]), ("dp", ["d"])])
    hot = {"a": 2, "b": 1, "c": 3}
    args = (cfg, 16, hot, CPU, torch.float32, Comm.single(CPU), OptParamsPy())
    with pytest.raises(ValueError, match="is_train=False"):
        EmbeddingCollection(*args, is_train=True, fp8_quant=True)
    e = EmbeddingCollection(*args, is_train=False, fp8_quant=True)
    assert e.grad_slab is None and not e.top_grad
    total = 0
    for g in e.groups:
        assert g.wdtype == "fp8" and g.table.dtype == torch.float8_e4m3fn and g.exps.dtype == torch.uint8
        assert g.s0 is None and g.s1 is None and getattr(g, "ws", None) is None
        assert getattr(g, "dense_wgrad", None) is None
        total += max(g.rows, 1) * (g.pitch + 1)
    sketches = sum(sk.nbytes() for sk in e._admit_sketches())
    assert sketches > 0 and e.memory_bytes() == total + sketches
    # the initial fill of the static tables went through the quantizer
    for name in ("s", "d"):
        (_, w, *_), = e.dump_table_local(name)
        assert bool(torch.isfinite(w).all()) and float(w.abs().max()) > 0


def test_fp8_load_rejects_a_nan_row_naming_the_table_cpu(tmp_path):
    from hugectr_b200.inference import InferenceModel, InferenceParams
    _, paths = build_serving_test_model(tmp_path, CPU, iters=1)
    bad = os.path.join(str(tmp_path), "bad_ebc")

    def poison(W):
        W = W.clone()
        W[W.shape[0] // 2, 3] = float("nan")
        return W
    rewrite_ebc_weights(paths["ebc"], bad, poison)
    with pytest.raises(ValueError, match="table ts"):
        InferenceModel(paths["graph"], InferenceParams(model_name="x", max_batchsize=32, dense_model_file=paths["dense"],
                                                       embedding_collection_path=bad, fp8_quant=True), device="cpu")


def test_fp8_quant_rejects_a_model_without_collection_tables_cpu(tmp_path):
    from hugectr_b200.inference import InferenceModel, InferenceParams
    from hugectr_b200.models.legacy import build_deepfm
    m = build_deepfm(batchsize=16, vvgpu=[[0]], slot_sizes=[30, 12, 50, 7], workspace_mb=2, mixed=False,
                     max_eval_batches=1, seed=5)
    g = os.path.join(str(tmp_path), "deepfm.json")
    m.graph_to_json(g)
    with pytest.raises(ValueError, match="fp8_quant"):
        InferenceModel(g, InferenceParams(model_name="x", max_batchsize=16, fp8_quant=True), device="cpu")


def grown_fp8_table_matches_fp32(device):
    """A growing table (init_capacity 16) loads 12 keys, then 88 more: it grows, the fp8 arena's rows and exponents
    are re-laid out and the new rows filled through the quantizer.  Lookups and dumps equal an fp32 serving table
    loaded with the dequantized values."""
    import hugectr_b200 as hugectr
    from hugectr_b200.embedding.collection import EmbeddingCollection
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import OptParamsPy
    cfg = hugectr.EmbeddingCollectionConfig()
    cfg.embedding_lookup([hugectr.EmbeddingTableConfig("g", -1, 16, init_capacity=16)], ["a"], "emb", ["sum"])
    mk = lambda fp8: EmbeddingCollection(cfg, 20, {"a": 3}, device, torch.float32, Comm.single(device),  # noqa: E731
                                         OptParamsPy(), is_train=False, fp8_quant=fp8)
    e8, e32 = mk(True), mk(False)
    g = torch.Generator().manual_seed(4)
    keys = torch.randperm(1000, generator=g)[:100] * 3 + 1
    W = torch.randn(100, 16, generator=g) * torch.exp2(torch.randint(-8, 8, (100, 1), generator=g).float())
    for lo, hi in ((0, 12), (12, 100)):
        e8.load_table_rows("g", keys[lo:hi], W[lo:hi])
        e32.load_table_rows("g", keys[lo:hi], fp8_round_trip(W[lo:hi]))
    e8.check_quantized()
    assert [sl["rows"] for gr in e8.groups for sl in gr.table_slices][0] >= 100
    assert e8.groups[0].exps.numel() == e8.groups[0].rows
    batch = torch.where(torch.rand(20, 3, generator=g) < 0.8, keys[torch.randint(0, 100, (20, 3), generator=g)],
                        torch.randint(3000, 4000, (20, 3), generator=g))      # some unseen keys
    for e in (e8, e32):
        e.set_keys(batch.reshape(-1).to(device, e.key_dtype))
        e.forward(False)
    assert torch.equal(e8.top_data["emb"], e32.top_data["emb"])
    (k8, w8, *_), = e8.dump_table_local("g")
    (k32, w32, *_), = e32.dump_table_local("g")
    assert torch.equal(k8, k32) and torch.equal(w8, w32) and k8.numel() == 100


def test_fp8_growing_table_grows_through_the_quantizer_cpu():
    grown_fp8_table_matches_fp32(CPU)
