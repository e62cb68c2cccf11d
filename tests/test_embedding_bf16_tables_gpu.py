"""bf16 weight storage of model-parallel embedding tables (EmbeddingTableConfig(weight_dtype="bf16")).

The kernels read bf16 rows, pool / reduce / run the optimizer in fp32 and store every updated weight
with stochastic rounding: the upper 16 bits of (fp32 bits + r), r = 16 bits of a hash of (seed,
device step, arena index).  ``ops.sr_round_bf16`` mirrors that bit for bit.

The GPU tests reuse the fp64 oracle of test_embedding_kernels_gpu.py on the bf16 weights upcast to
fp64: a stored weight must lie within one bf16 ulp of the oracle's result (plus the oracle's fp32
bound), i.e. be the oracle's value rounded either way.  A case whose pre-rounding fp32 values are
exact (SGD, power-of-two learning rate, small dyadic gradients) pins the kernels' bits to the mirror.
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_embedding_kernels_gpu as K  # noqa: E402
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.enums import Optimizer_t as O  # noqa: E402

BF = torch.bfloat16
ULP1 = 2.0 ** -7          # bf16 ulp in [1, 2)
N_UNBIASED = 1 << 20


# ------------------------------------------------------------------------------------ mirror (CPU)
def _fmix64_int(k):
    """MurmurHash3 fmix64 on Python ints, written out independently of the numpy mirror"""
    m = (1 << 64) - 1
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & m
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & m
    return k ^ (k >> 33)


def _bits(t):
    return t.view(torch.int16).int() & 0xFFFF


def test_mirror_matches_hand_computed_bits():
    seed, step = 0x1234ABCD, 7
    key = _fmix64_int((seed << 32) | step)
    assert E.sr_step_key(seed, step) == key
    idx = [0, 1, 5, 127, 1 << 20, (1 << 40) + 3]
    r = [(_fmix64_int(key ^ (i >> 2)) >> (16 * (i & 3))) & 0xFFFF for i in idx]
    assert E.sr_bits(key, torch.tensor(idx)).tolist() == r
    # fp32 patterns: 1 + 2^-8 (half an ulp), -(1 + 2^-8), 1 + 2^-7 (exact in bf16), a subnormal-free small
    # value with a full low half, +inf, -inf
    pats = [0x3F808000, 0xBF808000, 0x3F810000, 0x3A83FFFF, 0x7F800000, 0xFF800000]
    x = torch.tensor(pats, dtype=torch.int64).to(torch.int32).view(torch.float32)
    got = _bits(E.sr_round_bf16(x, seed, step, torch.tensor(idx))).tolist()
    exp = [((p + ri) >> 16) & 0xFFFF for p, ri in zip(pats, r)]
    exp[4], exp[5] = 0x7F80, 0xFF80
    assert got == exp
    assert got[2] == 0x3F81                           # a bf16 value is stored unchanged whatever r
    nan = E.sr_round_bf16(torch.tensor([float("nan")]), seed, step, torch.tensor([3]))
    assert torch.isnan(nan.float()).all()


def test_mirror_is_deterministic_and_keyed_by_step():
    x = torch.rand(4096) + 1.0
    idx = torch.arange(4096) + 12345
    a = E.sr_round_bf16(x, 5, 11, idx)
    assert torch.equal(_bits(a), _bits(E.sr_round_bf16(x, 5, 11, idx)))
    for other in (E.sr_round_bf16(x, 5, 12, idx), E.sr_round_bf16(x, 6, 11, idx),
                  E.sr_round_bf16(x, 5, 11, idx + 1)):
        assert not torch.equal(_bits(a), _bits(other))


def _unbiased(got, what):
    """one update of 0.3 ulp from 1.0: mean moves by 0.3 ulp within 5 sigma, ~30 % round up"""
    d = (got.double() - 1.0) / ULP1
    assert set(torch.unique(d).tolist()) <= {0.0, 1.0}, what
    n, p = d.numel(), 0.3
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(float(d.mean()) - p) < 5 * sigma, f"{what}: mean {float(d.mean())}"


def test_mirror_is_unbiased_cpu_update_rows():
    """update_rows (the CPU path) on a bf16 table of 2^20 ones: SGD step of 0.3 ulp"""
    pitch = 1024
    rows = N_UNBIASED // pitch
    tab = torch.ones(rows * pitch, dtype=BF)
    g = torch.full((rows, pitch), -0.3 * ULP1)
    E.update_rows(O.SGD, tab, None, None, pitch, torch.arange(rows), g, {"sr_seed": 9},
                  torch.tensor([1.0]), torch.tensor([1], dtype=torch.int32))
    _unbiased(tab, "cpu")
    assert bool(((1.0 + 0.3 * ULP1) * torch.ones(8)).to(BF).eq(1.0).all())   # to nearest: none moves


# ------------------------------------------------------------------------------------ model (CPU)
def _tiny_model(tmp_path, wdt, seed=7):
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    sizes, hot = [50, 40, 30], [2, 1, 1]
    solver = hugectr.CreateSolver(model_name="bf16tables", seed=seed, batchsize=32, batchsize_eval=32,
                                  vvgpu=[[0]], lr=0.05, use_mixed_precision=False, use_cuda_graph=False,
                                  use_embedding_collection=True, warmup_steps=1, max_eval_batches=1)
    reader = hugectr.DataReaderParams(
        data_reader_type=hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.1"], eval_source="synthetic:1.1",
        check_type=hugectr.Check_t.Non, slot_size_array=sizes,
        async_param=hugectr.AsyncParam(1, 16, shuffle=False, multi_hot_reader=True, is_dense_float=True))
    opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad, hugectr.Update_t.Global, initial_accu_value=0.0,
                                  epsilon=1e-8)
    m = hugectr.Model(solver, reader, opt, comm=Comm.single(torch.device("cpu")))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=13, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam(f"data{i}", hot[i], True, 1)
                                                        for i in range(3)]))
    tables = [hugectr.EmbeddingTableConfig(name=str(i), max_vocabulary_size=sizes[i], ev_size=8, weight_dtype=wdt)
              for i in range(3)]
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup(table_config=tables, bottom_name=[f"data{i}" for i in range(3)],
                         top_name="sparse_embedding", combiner=["sum"] * 3)
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["dense"], ["mlp1"], num_outputs=[16, 8],
                             act_type=hugectr.Activation_t.Relu))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["sparse_embedding", "mlp1"], ["concat1"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["concat1"], ["mlp2"], num_outputs=[16, 1],
                             activations=[hugectr.Activation_t.Relu, hugectr.Activation_t.Non]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["mlp2", "label"], ["loss"]))
    m.compile()
    return m


def test_config_rejects_unknown_weight_dtype():
    from hugectr_b200.embedding.collection import EmbeddingTableConfig
    assert EmbeddingTableConfig("t", 10, 8).weight_dtype == "fp32"
    with pytest.raises(ValueError, match="weight_dtype"):
        EmbeddingTableConfig("t", 10, 8, weight_dtype="fp16")


def test_bf16_model_trains_round_trips_and_resumes(tmp_path):
    a = _tiny_model(tmp_path, "bf16")
    e = a.ebcs_train[0]
    assert all(g.table.dtype == BF and g.wdtype == "bf16" for g in e.groups)
    pool = a.reader_train.pool
    t0 = [g.table.clone() for g in e.groups]
    losses = []
    pre = str(tmp_path / "snap")
    for i in range(7):
        a.train_on_host_batch(pool[i % len(pool)])
        losses.append(a.get_current_loss())
        if i == 4:
            a.save_params_to_files(pre, 5)
    assert all(math.isfinite(x) for x in losses)
    assert any(not torch.equal(x, g.table) for x, g in zip(t0, e.groups)), "tables did not train"
    # half the table bytes of the fp32 model (AdaGrad state stays fp32 in both)
    f = _tiny_model(tmp_path, "fp32")
    tb = sum(g.table.numel() for g in f.ebcs_train[0].groups)
    assert f.ebcs_train[0].memory_bytes() - e.memory_bytes() == 2 * tb
    # graph JSON round trip: the bf16 tables come back as bf16
    a.graph_to_json(str(tmp_path / "g.json"))
    import json
    tj = [l for l in json.load(open(tmp_path / "g.json"))["layers"] if l["type"] == "EmbeddingCollection"][0]
    assert [t["weight_dtype"] for t in tj["tables"]] == ["bf16"] * 3
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]],
                                  use_embedding_collection=True, use_cuda_graph=False)
    m2 = hugectr.Model(solver, a.reader_params, a.opt_params, comm=Comm.single(torch.device("cpu")))
    m2.construct_from_json(str(tmp_path / "g.json"))
    assert all(t.weight_dtype == "bf16" for t in m2.ebc_configs[0].tables())
    # dump -> load -> dump is byte-identical (bf16 -> fp32 is exact, fp32 -> bf16 of those is too)
    d1 = [e.dump_table_local(str(i)) for i in range(3)]
    b = _tiny_model(tmp_path, "bf16", seed=99)
    for i in range(3):
        for keys, w, col0, sts, kind in d1[i]:
            assert w.dtype == torch.float32
            b.ebcs_train[0].load_table_rows(str(i), keys, w, sts)
    d2 = [b.ebcs_train[0].dump_table_local(str(i)) for i in range(3)]
    for p1, p2 in zip(d1, d2):
        for x, y in zip(p1, p2):
            assert x[1].numpy().tobytes() == y[1].numpy().tobytes()
    # resume from the step-5 snapshot: bit-identical continuation (same stochastic-rounding bits)
    c = _tiny_model(tmp_path, "bf16")
    assert c.resume(pre) == 5
    for i in range(5, 7):
        c.train_on_host_batch(pool[i % len(pool)])
    assert float((a.arena.weights - c.arena.weights).abs().max()) == 0.0
    for name in ("0", "1", "2"):
        for pa, pc in zip(e.dump_table_local(name), c.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pa[1], pc[1]) and torch.equal(pa[3][0], pc[3][0])
    assert a.get_current_loss() == c.get_current_loss()


def test_bf16_checkpoint_loads_into_fp32_model_and_back(tmp_path):
    a = _tiny_model(tmp_path, "bf16")
    a.train_on_host_batch(a.reader_train.pool[0])
    pre = str(tmp_path / "x")
    a.save_params_to_files(pre, 1)
    f = _tiny_model(tmp_path, "fp32", seed=5)
    f.embedding_load(pre + "_ebc_1")
    for name in ("0", "1", "2"):
        for pa, pf in zip(a.ebcs_train[0].dump_table_local(name), f.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pa[1], pf[1])
    f.save_params_to_files(pre + "f", 1)
    b = _tiny_model(tmp_path, "bf16", seed=6)
    b.embedding_load(pre + "f_ebc_1")
    for name in ("0", "1", "2"):
        for pa, pb in zip(a.ebcs_train[0].dump_table_local(name), b.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pa[1], pb[1])


def test_fp32_graph_json_is_unchanged(tmp_path):
    """no weight_dtype key for fp32 tables: the graph JSON of the fp32 model is byte-identical to the
    one written before bf16 tables existed (tests/golden/bf16_tables_fp32_graph.json)"""
    f = _tiny_model(tmp_path, "fp32")
    f.graph_to_json(str(tmp_path / "f.json"))
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bf16_tables_fp32_graph.json")
    assert open(tmp_path / "f.json", "rb").read() == open(golden, "rb").read()


def test_dp_tables_stay_fp32_and_groups_split_by_dtype(capsys):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    ts = [EmbeddingTableConfig("a", 100, 16, weight_dtype="bf16"), EmbeddingTableConfig("b", 80, 16),
          EmbeddingTableConfig("c", 60, 16, weight_dtype="bf16")]
    cfg.embedding_lookup(ts, ["d0", "d1", "d2"], "emb", ["sum"] * 3)
    cfg.shard([[1, 1, 1]], [("mp", ["a", "b"]), ("dp", ["c"])])
    cpu = torch.device("cpu")
    e = EmbeddingCollection(cfg, 4, {"d0": 1, "d1": 1, "d2": 1}, cpu, torch.float32, Comm.single(cpu),
                            CreateOptimizer(O.SGD), seed=1)
    kinds = sorted((g.kind, g.wdtype, g.table.dtype == BF) for g in e.groups)
    assert kinds == [("dp", "fp32", False), ("mp", "bf16", True), ("mp", "fp32", False)]
    assert "tables ['c'] keep fp32 weights" in capsys.readouterr().out


# ======================================================================================== GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("odt", [torch.float32, BF])
@pytest.mark.parametrize("pitch", [1, 3, 6, 11, 64, 128, 132, 256, 258, 1023, 1024])
def test_bf16_forward_widths(pitch, odt):
    """the lookup on a bf16 arena: scalar and vector widths, wide rows, scalar passes past 256
    columns, sum / mean / a row-sharded lookup, int32 and int64 keys"""
    gen = torch.Generator().manual_seed(pitch)
    case = K.features_case(pitch, torch.float32, gen, batch=257)
    tab = (torch.randn(case.rows * pitch, generator=gen)).to(BF)
    n = case.grads[0].numel()
    ref, tol, hit = K.oracle_forward(case, tab.double(), n)
    dev = torch.device("cuda")
    keys, _, nnz = K._dev(case, torch.int64 if pitch % 2 else torch.int32)
    outs = [torch.full((n,), 7.0, dtype=odt, device=dev) for _ in keys]
    E.forward(case.lookups, E.lookups_to_device(case.lookups, dev), tab.to(dev), pitch, keys, outs,
              case.batch, nnz_bufs=nnz)
    got = torch.stack([o.cpu() for o in outs])
    K.assert_close_bound(f"bf16 forward ev={pitch}", got[hit], ref[hit], tol[hit], bf16=odt == BF)
    assert bool((got[~hit] == 7.0).all())


def check_bf16_update(what, case, opt, tab, s0, s1, new, hp=K.HP, lr=K.LR, step=1, grad_scale=1.0):
    """every stored bf16 weight within one bf16 ulp of the oracle (its fp32 result rounded either
    way); states as in the fp32 tests; untouched rows unchanged"""
    uniq, old, ref, tol = K.oracle_update(opt, hp, lr, step, tab, s0, s1, K.oracle_reduce(case, grad_scale))
    P = case.pitch
    for j, (name, before, after) in enumerate(zip(("w", "s0", "s1"), (tab, s0, s1), new)):
        if before is None:
            continue
        after = after.cpu()
        assert after.dtype == before.dtype
        K.assert_close_bound(f"{what} {name}", after.view(-1, P)[uniq], ref[j], tol[j],
                             bf16=after.dtype == BF)
        keep = torch.ones(after.numel() // P, dtype=torch.bool)
        keep[uniq] = False
        assert torch.equal(after.view(-1, P)[keep], before.view(-1, P)[keep]), f"{what}: untouched {name} rows changed"


def bf16_step(what, case, opt, sdt, gen, **kw):
    tab, s0, s1 = K.init_state(opt, case.rows, case.pitch, sdt, gen)
    tab = tab.to(BF)
    new, ws = K.run_step(case, opt, tab, s0, s1, **kw)
    assert new[0].dtype == BF
    check_bf16_update(what, case, opt, tab, s0, s1, new, hp=kw.get("hp", K.HP), step=kw.get("step", 1),
                      grad_scale=kw.get("grad_scale", 1.0))
    K.assert_ws_clean(ws)


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", [128, 516])
@pytest.mark.parametrize("sdt", [torch.float32, BF])
@pytest.mark.parametrize("opt", K.OPTS, ids=[o.name for o in K.OPTS])
def test_bf16_fused_row_classes_all_optimizers(opt, sdt, pitch):
    """light, medium and heavy rows (1-3 chunks) of the fused backward on a bf16 arena, seven
    optimizers, fp32 and bf16 state, G = 8 and G = 32 with two passes"""
    gen = torch.Generator().manual_seed(21 + pitch)
    case = K.single_case(K.class_keys(512, 8, 3000, gen), 512, 8, pitch, 3000, BF, gen)
    hp = dict(K.HP, sr_seed=77)
    bf16_step(f"{opt.name} {sdt} ev={pitch}", case, opt, sdt, gen, hp=hp, step=3)


@pytest.mark.gpu
@pytest.mark.parametrize("sdt", [torch.float32, BF])
@pytest.mark.parametrize("opt", K.OPTS, ids=[o.name for o in K.OPTS])
@pytest.mark.parametrize("pitch", [6, 128])
def test_bf16_accumulate_update_misaligned(pitch, opt, sdt):
    """the accumulate + update path (scalar at ev 6, a misaligned layout; vector at ev 128) on a bf16
    arena with every lookup feature"""
    gen = torch.Generator().manual_seed(31 + pitch)
    case = K.features_case(pitch, torch.float32, gen, batch=200)
    bf16_step(f"accum {opt.name} {sdt} ev={pitch}", case, opt, sdt, gen, path="accum",
              hp=dict(K.HP, scaler=4.0, sr_seed=5), grad_scale=0.5, step=2)


@pytest.mark.gpu
def test_bf16_row_with_more_than_4096_chunks():
    """a 2.1 M-occurrence row (warp-per-row fallback past 4096 chunks) next to ordinary rows"""
    gen = torch.Generator().manual_seed(6)
    batch, hot, pitch = 16500, 128, 4
    keys = torch.full((batch * hot,), 7, dtype=torch.int64)
    keys[torch.randperm(keys.numel(), generator=gen)[:3000]] = torch.randint(8, 900, (3000,), generator=gen)
    grads = torch.randint(-2, 3, (batch * pitch,), generator=gen).float() / 16
    case = K.Case([K.lookup(0, 1000, 0, 0, hot, pitch, pitch)], pitch, batch, [keys], [grads])
    bf16_step("bf16 2.1 M-occurrence row", case, O.SGD, torch.float32, gen)


# ------------------------------------------------------------------------------- exact stochastic rounding
def _exact_case(pitch, heavy):
    """rows occurring once (and optionally one 1025-occurrence row), gradients k / 256 with
    |k| <= 32 and weights that are multiples of 2^-12 in [-1/2, 1/2]: every partial sum and
    w - lr * g (lr = 2^-4) is exact in fp32"""
    gen = torch.Generator().manual_seed(pitch + heavy)
    rows, batch, hot = 4000, 1500, 2
    counts = [1] * 1800 + ([1025] if heavy else [])
    keys = K.class_keys(batch, hot, rows, gen, counts)
    grads = (torch.randint(-32, 33, (batch * pitch,), generator=gen).float() / 256)
    case = K.single_case(keys, batch, hot, pitch, rows, torch.float32, gen)
    case.grads = [grads]
    tab = (torch.randint(-2048, 2049, (rows * pitch,), generator=gen).float() / 4096).to(BF)
    return case, tab


@pytest.mark.gpu
@pytest.mark.parametrize("path,pitch,heavy", [("fused", 128, True), ("fused", 516, True), ("accum", 128, True),
                                              ("accum", 6, False)])
def test_stochastic_rounding_bits_match_the_mirror(path, pitch, heavy):
    lr, seed, step = 2.0 ** -4, 0xC0FFEE, 13
    case, tab = _exact_case(pitch, heavy)
    uniq, G, _, n = K.oracle_reduce(case)
    w = tab.double().view(-1, pitch)[uniq] - lr * G
    assert torch.equal(w.float().double(), w), "case is not exact in fp32"
    idx = uniq.view(-1, 1) * pitch + torch.arange(pitch).view(1, -1)
    exp = tab.clone().view(-1, pitch)
    exp[uniq] = E.sr_round_bf16(w.float(), seed, step, idx)
    (t, _, _), _ = K.run_step(case, O.SGD, tab, None, None, path=path, hp=dict(K.HP, sr_seed=seed), lr=lr,
                              step=step)
    got = t.cpu().view(-1, pitch)
    bad = (_bits(got) != _bits(exp)).any(1)
    assert not bool(bad.any()), f"{path} ev={pitch}: {int(bad.sum())} rows differ from the mirror, " \
                                f"occurrences {n[torch.isin(uniq, bad.nonzero().view(-1))].tolist()[:5]}"
    # the rounding did something: not all values are round-to-nearest
    assert not torch.equal(_bits(exp[uniq]), _bits(w.float().to(BF)))


@pytest.mark.gpu
def test_stochastic_rounding_unbiased_on_device():
    """one fused SGD step of 0.3 ulp on 2^20 bf16 ones"""
    pitch = 1024
    rows = N_UNBIASED // pitch
    keys = torch.randperm(rows)
    grads = torch.full((rows * pitch,), -0.3 * ULP1)
    case = K.Case([K.lookup(0, rows, 0, 0, 1, pitch, pitch)], pitch, rows, [keys], [grads])
    tab = torch.ones(rows * pitch, dtype=BF)
    (t, _, _), _ = K.run_step(case, O.SGD, tab, None, None, hp=dict(K.HP, sr_seed=3), lr=1.0)
    _unbiased(t.cpu(), "device")


# ------------------------------------------------------------------------------- collection on the GPU
def _collection(dev, dyn_cap=16):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    ts = [EmbeddingTableConfig("s", 500, 32, weight_dtype="bf16"),
          EmbeddingTableConfig("f", 300, 32),
          EmbeddingTableConfig("dyn", -1, 32, weight_dtype="bf16", init_capacity=dyn_cap)]
    cfg.embedding_lookup(ts, ["d0", "d1", "d2"], "emb", ["sum", "mean", "sum"])
    return EmbeddingCollection(cfg, 64, {"d0": 3, "d1": 2, "d2": 2}, dev, torch.float32, Comm(dev),
                               CreateOptimizer(O.AdaGrad, initial_accu_value=0.1), seed=4)


def _keys(gen, dyn_vocab):
    return torch.cat([torch.randint(0, 500, (64 * 3,), generator=gen), torch.randint(0, 300, (64 * 2,), generator=gen),
                      torch.randint(0, dyn_vocab, (64 * 2,), generator=gen) * 1000003]).long()


def _dumps(e):
    return {n: e.dump_table_local(n)[0] for n in ("s", "f", "dyn")}


@pytest.mark.gpu
def test_bf16_collection_matches_cpu_and_survives_growth():
    gen = torch.Generator().manual_seed(0)
    g = _collection(torch.device("cuda"), dyn_cap=64)
    c = _collection(torch.device("cpu"), dyn_cap=64)
    assert sorted(gg.wdtype for gg in g.groups) == ["bf16", "fp32"]
    keys = _keys(gen, 40)
    # same weights on both sides (the dynamic rows exist after the first lookup)
    for e in (g, c):
        e.set_keys(keys.to(e.device))
        e.forward()
    for name, (k, w, col0, sts, kind) in _dumps(g).items():
        c.load_table_rows(name, k, w, sts)
    lr_c, st_c = torch.tensor([0.05]), torch.tensor([2], dtype=torch.int32)
    lr_g, st_g = lr_c.cuda(), st_c.cuda()
    for e in (g, c):
        e.set_keys(keys.to(e.device))
        e.forward()
    torch.testing.assert_close(g.top_data["emb"].cpu(), c.top_data["emb"], rtol=2e-4, atol=2e-4)
    grad = torch.randn(c.top_grad["emb"].shape, generator=gen) * 0.1
    g.top_grad["emb"].copy_(grad.cuda())
    c.top_grad["emb"].copy_(grad)
    g.backward(lr_g, st_g)
    c.backward(lr_c, st_c)
    dg, dc = _dumps(g), _dumps(c)
    for name in dg:
        kg, wg = dg[name][0], dg[name][1].double()
        kc, wc = dc[name][0], dc[name][1].double()
        assert torch.equal(kg, kc)
        tol = K.bf16_ulp(torch.maximum(wg.abs(), wc.abs())) if name != "f" else 2e-4 + 1e-3 * wc.abs()
        assert bool(((wg - wc).abs() <= tol + 1e-7).all()), f"table {name}: GPU and CPU steps disagree"
    g.check_overflow()
    # an eval clone shares the arenas; more distinct dynamic keys than rows make the table grow
    ev = g.eval_clone(64)
    before = _dumps(g)["dyn"]
    big = _keys(gen, 100)           # ~70 new distinct keys: past the 64 rows, within the grown 129
    g.set_keys(big.cuda())
    g.forward()
    with pytest.raises(RuntimeError, match="init_capacity"):
        g.check_overflow()
    grown = g.grow_dynamic()
    assert grown and grown[0][0] == "dyn"
    gd = [gg for gg in g.groups if gg.wdtype == "bf16"][0]
    assert gd.table.dtype == BF and ev.groups[g.groups.index(gd)].table is gd.table
    after = _dumps(g)["dyn"]
    pos = torch.searchsorted(after[0], before[0])
    assert torch.equal(after[0][pos], before[0])
    assert torch.equal(after[1][pos], before[1]), "rows changed when the table grew"
    for e in (g, ev):
        e.set_keys(big.cuda())
        e.forward()
    torch.testing.assert_close(ev.top_data["emb"], g.top_data["emb"], rtol=0, atol=0)
    g.check_overflow()
