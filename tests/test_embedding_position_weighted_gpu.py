"""Position-weighted inputs on the device: the fill and weight-gradient kernels against the fp64 oracle of
test_embedding_position_weighted_cpu.py (fp32 and bf16 arenas, widths 4 to 1024, static, growing and evicting tables,
data-parallel tables), a CUDA-graph model against eager steps and against a second replay, and an fp8 serving
session over a trained model."""
import os
import sys

import numpy as np
import pytest
import torch

from hugectr_b200.enums import Optimizer_t
from hugectr_b200.parallel.comm import Comm

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_embedding_position_weighted_cpu import (PW, _model, bound, check_dP, load_tables, make_batch,
                                                  make_collection, make_P, make_tables, oracle, position_batches,
                                                  step)  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


@pytest.mark.parametrize("ev", [4, 6, 128, 1024])
@pytest.mark.parametrize("wdtype", ["fp32", "bf16"])
@pytest.mark.parametrize("combiner", ["sum", "mean"])
@pytest.mark.parametrize("table", ["static", "grow", "lru"])
def test_weight_gradient_kernel_matches_fp64_oracle(ev, wdtype, combiner, table):
    gen = torch.Generator().manual_seed(ev)
    B = 24
    tables = make_tables(gen, ev=ev, shared=True)
    if wdtype == "bf16":
        tables = {n: t.to(torch.bfloat16).double() for n, t in tables.items()}   # the rows the arena holds
    P = make_P(gen, zero_bag=True)
    e, params = make_collection(DEV, Comm.single(DEV), B, combiner=combiner, P=P, shared=True, ev=ev,
                                weight_dtype=wdtype, dynamic=None if table == "static" else table)
    load_tables(e, tables)
    keys = make_batch(gen, B, zero_bag=True)
    grads = {"emb": torch.randn(B, 3 * ev, generator=gen) * 0.1, "emb2": torch.randn(B, ev, generator=gen) * 0.1}
    outs = step(e, keys, grads)
    exp_out, dP, S = oracle(tables, keys, P, combiner, grads, shared=True)
    for t in outs:
        assert (outs[t].double() - exp_out[t]).abs().max().item() < 1e-5
    bd = bound(S, B, 1, ev)
    for n in PW:
        err = (params[n][1].double().cpu() - dP[n]).abs()
        assert bool((err <= bd[n] + 1e-12).all()), f"{n}: err {err.max().item()} bound {bd[n].max().item()}"


def test_weight_gradient_matches_cpu_path_data_parallel():
    gen = torch.Generator().manual_seed(2)
    B = 32
    tables = make_tables(gen)
    P = make_P(gen)
    keys = make_batch(gen, B)
    grads = {"emb": torch.randn(B, 48, generator=gen) * 0.1}
    _, dP, S = oracle(tables, keys, P, "mean", grads)
    res = {}
    for dev in (torch.device("cpu"), DEV):
        e, params = make_collection(dev, Comm.single(dev), B, plan="dp", combiner="mean", P=P)
        assert any(g.kind == "dp" and g.pw_sel for g in e.groups)
        load_tables(e, tables)
        step(e, keys, grads)
        check_dP(params, dP, S, B)
        res[dev.type] = {n: params[n][1].cpu() for n in PW}
    for n in PW:
        assert (res["cpu"][n] - res["cuda"][n]).abs().max().item() < 1e-6


def _train(cuda_graph, steps=12):
    gen = torch.Generator().manual_seed(3)
    m = _model(lr=0.05, opt=Optimizer_t.Adam, device=DEV, cuda_graph=cuda_graph)
    m.compile()
    for hb in position_batches(m, steps, gen):
        m.train_on_host_batch(hb)
    torch.cuda.synchronize()
    return m


def test_cuda_graph_equals_eager_and_replays_reproduce_bits():
    g1, g2, eager = _train(True), _train(True), _train(False)
    assert g1._graph is not None and eager._graph is None
    p1, p2, pe = (m.position_weights["a"].w.detach().cpu() for m in (g1, g2, eager))
    assert not torch.equal(p1, torch.ones_like(p1))
    assert torch.equal(p1, p2)                       # two replays from one state: the same bits
    assert torch.equal(p1, pe)
    # (the dense network's GEMMs may pick other algorithms under capture than eagerly: its weights agree to rounding)
    torch.testing.assert_close(g1.arena.weights, eager.arena.weights, rtol=0, atol=1e-6)


def test_fp8_serving_session_over_the_trained_model(tmp_path):
    from hugectr_b200.inference import InferenceModel, InferenceParams
    from hugectr_b200.io.checkpoint import dense_paths
    m = _train(True)
    pre = str(tmp_path / "m")
    m.save_params_to_files(pre)
    m.graph_to_json(str(tmp_path / "g.json"))
    m.embedding_dump(str(tmp_path / "emb"))
    mk = lambda fp8: InferenceModel(str(tmp_path / "g.json"), InferenceParams(
        "m", 32, dense_model_file=dense_paths(pre, 0)[0], embedding_collection_path=str(tmp_path / "emb"),
        fp8_quant=fp8), device="cuda:0")
    s32, s8 = mk(False), mk(True)
    assert torch.equal(s8.model.position_weights["a"].w, m.position_weights["a"].w)
    hb = position_batches(m, 1, torch.Generator().manual_seed(8))[0]
    p32 = s32.predict(hb.dense.numpy(), hb.keys.numpy())
    p8 = s8.predict(hb.dense.numpy(), hb.keys.numpy())
    m._load_batch(hb, False)
    for e in m.ebcs_eval:
        e.forward(False)
    m.net_eval.fprop(False)
    exp = m.net_eval.loss_layers[0].pred[:32].float().cpu().numpy()
    np.testing.assert_allclose(p32, exp, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(p8, exp, atol=2e-2)
