"""fp8 serving tables on the H100: the quantize kernel against the CPU rule, the fp8 lookup against the fp32 lookup
over the dequantized table (bit for bit, every path of the kernel), whole sessions, and a streamed load that never
holds an fp32 copy of the table on the device."""
import os

import numpy as np
import pytest
import torch

from hugectr_b200.embedding import ops as E

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
PITCHES = [1, 3, 6, 11, 64, 128, 132, 256, 258, 1023, 1024]


def _rows(n, pitch, seed):
    """random fp32 rows of widely varying magnitude plus the rule's edge rows"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, pitch, generator=g) * torch.exp2(torch.randint(-30, 30, (n, 1), generator=g).float())
    edge = torch.zeros(6, pitch)
    edge[0, 0] = 448.0                                   # amax exactly 448 * 2^0
    edge[0, 1:] = 1.0625                                 # ties to even
    edge[1, :] = -1792.0                                 # amax 448 * 2^2, negative
    edge[2, 0] = 448.0
    edge[2, 1:] = 3 * 2.0 ** -9                          # e4m3 subnormals
    edge[4, :] = torch.linspace(-1e-3, 2e-3, pitch)      # row 3: all zero
    edge[5, :] = 1e30
    return torch.cat([x, edge])


@pytest.mark.parametrize("pitch", PITCHES)
def test_quantize_rows_kernel_matches_cpu_rule(pitch):
    x = _rows(200, pitch, pitch)
    n = x.shape[0]
    R = n + 17
    perm = torch.randperm(R, generator=torch.Generator().manual_seed(1))[:n]
    table = torch.zeros(R * pitch, dtype=torch.float8_e4m3fn, device=DEV)
    exps = torch.zeros(R, dtype=torch.uint8, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    E.quantize_rows(x, perm, table, exps, bad)
    q, e = E.fp8_rows_quantize(x)
    assert int(bad.item()) == 0
    assert torch.equal(table.view(R, pitch)[perm.to(DEV)].view(torch.uint8).cpu(), q.view(torch.uint8))
    assert torch.equal(exps[perm.to(DEV)].cpu(), e)
    x[7, pitch // 2] = float("inf")
    E.quantize_rows(x, perm, table, exps, bad)
    assert int(bad.item()) == 1


def _lookup_case(pitch, out_dtype, combiner, weighted, variable, shards, key_dtype, seed):
    g = torch.Generator().manual_seed(seed)
    rows, B, H = 300, 37, 5
    x = _rows(rows - 6, pitch, seed)
    q, e = E.fp8_rows_quantize(x)
    deq = E.fp8_rows_dequantize(q, e)
    k = shards
    keys = torch.randint(-1, rows * k, (B, H), generator=g).to(key_dtype)
    nnz = torch.randint(0, H + 1, (B,), generator=g).to(torch.int32)
    w = torch.rand(B, H, generator=g) * 4 - 1
    lk = E.LookupDesc(table_row_off=0, key_off=0, out_off=0, grad_off=0, hotness=H, key_stride=H, num_shards=k,
                      shard_idx=k - 1, out_stride=pitch, grad_stride=pitch, combiner=combiner, ev_size=pitch,
                      rows=rows, nnz_off=0 if variable else -1, weighted=int(weighted))
    ldev = E.lookups_to_device([lk], DEV)
    outs = []
    for table, rexp in ((q.view(-1).to(DEV), e.to(DEV)), (deq.reshape(-1).to(DEV), None)):
        out = torch.full((B, pitch), 7.0, dtype=out_dtype, device=DEV)
        E.forward([lk], ldev, table, pitch, [keys.to(DEV)], [out], B, 0, nnz_bufs=[nnz.to(DEV)] if variable else None,
                  key_bytes=keys.element_size(), act_bf16=out_dtype == torch.bfloat16,
                  weight_bufs=[w.to(DEV)] if weighted else None, row_exp=rexp)
        outs.append(out)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("pitch", PITCHES)
def test_fp8_lookup_equals_fp32_lookup_over_dequantized_table(pitch):
    n = 0
    for out_dtype in (torch.float32, torch.bfloat16):
        for combiner in (0, 1):
            for weighted in (False, True):
                for variable in (False, True):
                    for shards in (1, 3):
                        for key_dtype in (torch.int32, torch.int64):
                            o8, o32 = _lookup_case(pitch, out_dtype, combiner, weighted, variable, shards, key_dtype,
                                                   seed=pitch * 131 + n)
                            assert torch.equal(o8, o32), (out_dtype, combiner, weighted, variable, shards, key_dtype)
                            n += 1
    assert n == 64


def test_fp8_lookup_at_the_bottom_of_the_exponent_range():
    """the boundary of the exactness above (docs/embedding.md): a row at e = -126 whose dequantized values are
    normal fp32 numbers still looks up bit for bit as the fp32 table; a row with exponent byte 0 (e = -127, nonzero
    codes) pools to zero in the device fp8 lookup, where the fp32 lookup over the dequantized table and the CPU fp8
    lookup keep its values"""
    pitch, n = 64, 4
    g = torch.Generator().manual_seed(3)
    x = torch.zeros(n, pitch)
    x[0] = torch.randn(pitch, generator=g)
    x[1] = torch.rand(pitch, generator=g) * 2.0 ** -120                 # amax < 448 * 2^-127: byte 0
    x[1, 0] = 2.0 ** -120
    codes = torch.randint(0x38, 0x7F, (pitch,), generator=g).to(torch.uint8)   # e4m3 values 1 .. 448
    codes[0] = 0x7E
    x[2] = codes.view(torch.float8_e4m3fn).float() * 2.0 ** -126       # amax 448 * 2^-126: e = -126, all normal
    table = torch.zeros(n * pitch, dtype=torch.float8_e4m3fn, device=DEV)
    exps = torch.zeros(n, dtype=torch.uint8, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    E.quantize_rows(x, torch.arange(n), table, exps, bad)
    q, e = E.fp8_rows_quantize(x)
    assert torch.equal(table.view(torch.uint8).view(n, pitch).cpu(), q.view(torch.uint8))
    assert torch.equal(exps.cpu(), e) and e.tolist() == [e[0].item(), 0, 1, 0]
    deq = E.fp8_rows_dequantize(q, e)
    assert bool((deq[2].abs() >= 2.0 ** -126).all()) and bool((deq[1] != 0).any())
    keys = torch.arange(n, dtype=torch.int64).view(n, 1)
    lk = E.LookupDesc(table_row_off=0, key_off=0, out_off=0, grad_off=0, hotness=1, key_stride=1, num_shards=1,
                      shard_idx=0, out_stride=pitch, grad_stride=pitch, combiner=0, ev_size=pitch, rows=n,
                      nnz_off=-1, weighted=0)
    outs = []
    for dev in (DEV, "cpu"):
        for tab, rexp in ((table.to(dev), exps.to(dev)), (deq.reshape(-1).to(dev), None)):
            out = torch.full((n, pitch), 7.0, device=dev)
            E.forward([lk], E.lookups_to_device([lk], dev) if dev == DEV else None, tab, pitch, [keys.to(dev)],
                      [out], n, 0, key_bytes=8, act_bf16=False, row_exp=rexp)
            outs.append(out.cpu())
    o8, o32, c8, c32 = outs
    for r in (0, 2, 3):
        assert torch.equal(o8[r], o32[r]), r
    assert bool((o8[1] == 0).all())
    assert torch.equal(o32[1], deq[1] * (deq[1].abs() >= 2.0 ** -126))     # the fp32 kernel flushes subnormals
    assert torch.equal(c8, deq) and torch.equal(c32, deq)


def test_fp8_session_predicts_as_fp32_session_on_dequantized_checkpoint_gpu(tmp_path):
    from test_embedding_fp8_serving_cpu import build_serving_test_model, session_predictions_match
    m, paths = build_serving_test_model(tmp_path, DEV)
    s8, _ = session_predictions_match(m, paths, tmp_path, DEV)
    assert s8.model.ebcs_train[0] is s8.model.ebcs_eval[0]


def test_fp8_session_rejects_a_nan_row_naming_the_table_gpu(tmp_path):
    from test_embedding_fp8_serving_cpu import build_serving_test_model, rewrite_ebc_weights
    from hugectr_b200.inference import InferenceModel, InferenceParams
    _, paths = build_serving_test_model(tmp_path, DEV, iters=1)
    bad = os.path.join(str(tmp_path), "bad_ebc")

    def poison(W):
        W = W.clone()
        W[1, 2] = float("-inf")
        return W
    rewrite_ebc_weights(paths["ebc"], bad, poison)
    with pytest.raises(ValueError, match="table t"):
        InferenceModel(paths["graph"], InferenceParams(model_name="x", max_batchsize=32, dense_model_file=paths["dense"],
                                                       embedding_collection_path=bad, fp8_quant=True), device="cuda")


def test_fp8_streaming_load_stays_below_the_fp32_table_size(tmp_path, monkeypatch):
    """a 2 GiB fp32 table (4M rows x 128) streamed in chunks of 2^18 rows into an fp8 session: the peak device
    allocation while the session is created and loaded stays below 40% of the fp32 table"""
    import hugectr_b200 as hugectr
    from hugectr_b200.inference import InferenceModel, InferenceParams
    from hugectr_b200.io.checkpoint import FILE_HEAD_NBYTES, _file_head
    from hugectr_b200.parallel.comm import Comm
    rows, ev, d = 1 << 22, 128, str(tmp_path)
    solver = hugectr.CreateSolver(batchsize=64, batchsize_eval=64, lr=0.05, vvgpu=[[0]], use_cuda_graph=False)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.0"],
                                  eval_source="synthetic:1.0", check_type=hugectr.Check_t.Non, slot_size_array=[rows])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.Adam), comm=Comm.single(DEV))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=1, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("a", 2, True, 1)]))
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup([hugectr.EmbeddingTableConfig("big", rows, ev)], ["a"], "emb", ["sum"])
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["x"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["x"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    graph = os.path.join(d, "g.json")
    m.graph_to_json(graph)                       # (never compiled: no training copy of the table)
    folder = os.path.join(d, "ebc", "embedding_collection_0")
    os.makedirs(folder)
    head = np.zeros(5, dtype="<i4")
    head[0] = 1
    with open(os.path.join(folder, "meta_data"), "wb") as f:
        f.write(head.tobytes() + np.asarray([0], "<i4").tobytes() + np.asarray([rows], "<u8").tobytes()
                + np.asarray([ev], "<i4").tobytes())
    with open(os.path.join(folder, "key0"), "wb") as f:
        f.write(_file_head(1, 0) + np.arange(rows, dtype="<u4").tobytes())
    g = np.random.default_rng(0)
    with open(os.path.join(folder, "weight0"), "wb") as f:
        f.write(_file_head(2, 0))
        for lo in range(0, rows, 1 << 18):
            f.write((g.standard_normal((1 << 18, ev), dtype=np.float32) * 0.01).astype("<f4").tobytes())
    monkeypatch.setenv("HCTR_EBC_LOAD_CHUNK_ROWS", str(1 << 18))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    sess = InferenceModel(graph, InferenceParams(model_name="x", max_batchsize=64, fp8_quant=True,
                                                 embedding_collection_path=os.path.join(d, "ebc")), device="cuda")
    torch.cuda.synchronize()
    fp32_bytes = rows * ev * 4
    peak = torch.cuda.max_memory_allocated(DEV) - base
    e = sess.model.ebcs_eval[0]
    assert e.memory_bytes() == rows * (ev + 1)
    assert peak < 0.4 * fp32_bytes, (peak, fp32_bytes)
    # rows at both ends of the stream were quantized as the CPU rule does
    W = np.memmap(os.path.join(folder, "weight0"), dtype="<f4", mode="r", offset=FILE_HEAD_NBYTES, shape=(rows, ev))
    grp = e.groups[0]
    for lo in (0, rows - 1000):
        q, ex = E.fp8_rows_quantize(torch.from_numpy(np.array(W[lo:lo + 1000])))
        assert torch.equal(grp.table.view(-1, ev)[lo:lo + 1000].view(torch.uint8).cpu(), q.view(torch.uint8))
        assert torch.equal(grp.exps[lo:lo + 1000].cpu(), ex)


def test_fp8_growing_table_grows_through_the_quantizer_gpu():
    from test_embedding_fp8_serving_cpu import grown_fp8_table_matches_fp32
    grown_fp8_table_matches_fp32(DEV)
