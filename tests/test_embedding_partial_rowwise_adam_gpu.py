"""Partial row-wise Adam on the GPU: the fused sparse-update kernels (light, medium and heavy rows), the accumulate
path, the data-parallel kernel and the evict reinit kernel against the fp64 oracle of
test_embedding_partial_rowwise_adam_cpu.py, whose module docstring states the rule and the fp32 error bound;
then collections and models on the GPU against the CPU path, eager runs and one process."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_embedding_kernels_gpu as K  # noqa: E402
import test_embedding_partial_rowwise_adam_cpu as P  # noqa: E402
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.enums import Optimizer_t as O  # noqa: E402

PRA, BF, HP, LR = P.PRA, P.BF, P.HP, P.LR
DEV = torch.device("cuda")
pytestmark = pytest.mark.gpu


def run_prow(case, tab, m, v, path="fused", step=3, hp=HP, grad_scale=1.0, ws=None, dev_state=None, **ws_kw):
    return K.run_step(case, PRA, tab, m, v, path=path, hp=hp, lr=LR, step=step, grad_scale=grad_scale, ws=ws,
                      dev_state=dev_state, **ws_kw)


WIDTHS = [4, 8, 124, 128, 132, 256, 512, 516, 1024]


@pytest.mark.parametrize("pitch", WIDTHS)
@pytest.mark.parametrize("mdt", [torch.float32, BF])
@pytest.mark.parametrize("wdt", [torch.float32, BF])
def test_fused_row_classes_and_widths(pitch, mdt, wdt):
    """rows occurring 1..5, 64, 65, 512, 513 and 1025 times (light, medium and heavy rows with 1-3 chunks)
    at every width class of the fused kernels, bf16 gradients, fp32 / bf16 weights and first moments"""
    gen = torch.Generator().manual_seed(pitch)
    case = K.single_case(K.class_keys(512, 8, 4000, gen), 512, 8, pitch, 4000, BF, gen)
    tab, m, v = P.init_prow(case.rows, pitch, gen, wdt, mdt)
    new, ws = run_prow(case, tab, m, v)
    P.check_prow(f"fused ev={pitch}", case, tab, m, v, new, 3, bf16=wdt == BF)
    K.assert_ws_clean(ws)


@pytest.mark.parametrize("wdt", [torch.float32, BF])
@pytest.mark.parametrize("pitch", [1, 3, 6, 11, 128, 258])
def test_accumulate_path_with_lookup_features(pitch, wdt):
    """emb_update_kernel (float4 and scalar widths) after backward_accum: mean combiners with variable nnz and
    padding, a row-sharded lookup, two source buffers, grad_scale and scaler != 1, steps 1 and 2"""
    gen = torch.Generator().manual_seed(pitch)
    case = K.features_case(pitch, torch.float32, gen)
    tab, m, v = P.init_prow(case.rows, pitch, gen, wdt, BF if pitch % 2 else torch.float32)
    hp = dict(HP, scaler=4.0)
    for step in (1, 2):
        new, ws = run_prow(case, tab, m, v, path="accum", step=step, hp=hp, grad_scale=0.5)
        P.check_prow(f"accum ev={pitch} t={step}", case, tab, m, v, new, step, hp=hp, grad_scale=0.5,
                     bf16=wdt == BF)
        K.assert_ws_clean(ws)
        tab, m, v = (x.cpu() for x in new)


@pytest.mark.parametrize("pitch", [128, 516])
def test_fused_lookup_features(pitch):
    gen = torch.Generator().manual_seed(pitch + 1)
    case = K.features_case(pitch, BF, gen)
    tab, m, v = P.init_prow(case.rows, pitch, gen)
    hp = dict(HP, scaler=4.0)
    new, ws = run_prow(case, tab, m, v, hp=hp, grad_scale=0.5, key_dtype=torch.int64)
    P.check_prow(f"fused features ev={pitch}", case, tab, m, v, new, 3, hp=hp, grad_scale=0.5)
    K.assert_ws_clean(ws)


def test_small_heavy_caps_fall_back_to_the_medium_list():
    """heavy rows beyond 2 scratch rows / 3 chunk items take the warp-per-row kernel; two steps (t = 1, 2) on
    one workspace, clean after each"""
    gen = torch.Generator().manual_seed(4)
    pitch = 516
    tab, m, v = P.init_prow(3000, pitch, gen)
    ws, state = None, None
    for step, counts in ((1, [70, 65, 1100, 66, 5, 3, 1]), (2, [1025, 600, 65, 70, 64, 2])):
        case = K.single_case(K.class_keys(512, 16, 3000, gen, counts), 512, 16, pitch, 3000, torch.float32, gen)
        state, ws = run_prow(case, tab, m, v, step=step, ws=ws, dev_state=state, max_heavy_rows=2,
                             max_heavy_items=3)
        P.check_prow("small caps", case, tab, m, v, state, step)
        K.assert_ws_clean(ws)
        tab, m, v = (x.cpu() for x in state)


def test_row_with_more_than_4096_chunks():
    gen = torch.Generator().manual_seed(6)
    batch, hot, pitch = 16500, 128, 4
    keys = torch.full((batch * hot,), 7, dtype=torch.int64)
    keys[torch.randperm(keys.numel(), generator=gen)[:3000]] = torch.randint(8, 900, (3000,), generator=gen)
    grads = torch.randint(-2, 3, (batch * pitch,), generator=gen).float() / 16
    case = K.Case([K.lookup(0, 1000, 0, 0, hot, pitch, pitch)], pitch, batch, [keys], [grads])
    tab, m, v = P.init_prow(1000, pitch, gen)
    new, ws = run_prow(case, tab, m, v)
    P.check_prow("2.1 M-occurrence row", case, tab, m, v, new, 3)
    K.assert_ws_clean(ws)


@pytest.mark.parametrize("pitch", [6, 128])
def test_dp_update_against_the_oracle(pitch):
    """the rule on an all-reduced dense gradient: touched rows against the oracle, all-zero rows skipped (weights
    and both moments unchanged), the gradient zeroed"""
    gen = torch.Generator().manual_seed(pitch)
    rows = 300
    G = torch.randn(rows, pitch, generator=gen).double() * 0.1
    G[torch.randperm(rows, generator=gen)[:100]] = 0
    tab, m, v = P.init_prow(rows, pitch, gen)
    uniq = (G != 0).any(1).nonzero().view(-1)
    wg = G.float().reshape(-1).cuda()
    t, a, b = tab.cuda(), m.cuda(), v.cuda()
    hp = dict(HP, scaler=2.0)
    E.dp_prow_adam_update(t, a, b, wg, pitch, hp, torch.tensor([LR], device=DEV),
                          torch.tensor([4], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    red = (uniq, G[uniq], G.abs()[uniq], torch.zeros(uniq.numel(), dtype=torch.long))
    P.check_red("dp", red, pitch, tab, m, v, (t, a, b), 4, hp=hp)
    assert int((wg != 0).sum()) == 0
    # the CPU path does the same
    tc, ac, bc, gc = tab.clone(), m.clone(), v.clone(), G.float().reshape(-1).clone()
    E.dp_prow_adam_update(tc, ac, bc, gc, pitch, hp, torch.tensor([LR]), torch.tensor([4], dtype=torch.int32))
    P.check_red("dp cpu", red, pitch, tab, m, v, (tc, ac, bc), 4, hp=hp)


def test_evict_reinit_kernel():
    """admitted ways start with m = 0 (bf16) and v = 0 (fp32) on the device as on the CPU path; Adam (bf16 state)
    and AdaGrad tables reinitialise on the device exactly as on the CPU path"""
    from hugectr_b200.solver import CreateOptimizer
    for opt, sdt in ((P._opt(), BF), (P._opt(), torch.float32), (CreateOptimizer(O.Adam), BF),
                     (CreateOptimizer(O.AdaGrad, initial_accu_value=0.25), torch.float32)):
        got = []
        for dev in (DEV, P.CPU):
            e = P.evicting_collection(dev, opt, sdt)
            rows, g = P.admit_with_stale_state(e)
            torch.cuda.synchronize()
            got.append([x.cpu() for x in (g.s0, g.s1) if x is not None])
        for a, b in zip(*got):
            assert a.dtype == b.dtype and torch.equal(a, b), opt.optimizer_type
        if opt.optimizer_type == PRA:
            rows = rows.cpu()
            s0, s1 = got[0]
            assert s0.dtype == sdt and s1.dtype == torch.float32
            assert not bool(s0.view(-1, 8)[rows].any()) and not bool(s1[rows].any())
            assert int((s1 == 0.375).sum()) == s1.numel() - rows.numel()


def test_collection_steps_match_the_cpu_path():
    """model- and data-parallel partial row-wise Adam tables beside Adam and row-wise AdaGrad ones: five GPU steps
    (t = 1..5) equal the CPU collection's within tolerance, and a CUDA-graph replay equals the eager step"""
    g, c = P._mixed_collection(DEV), P._mixed_collection(P.CPU)
    for gg, cg in zip(g.groups, c.groups):
        cg.table.copy_(gg.table.cpu())
    gen = torch.Generator().manual_seed(0)
    lr_c, lr_g = torch.tensor([LR]), torch.tensor([LR], device=DEV)
    for t in range(1, 6):
        keys, grad = P._batch(c, gen)
        st = torch.tensor([t], dtype=torch.int32)
        P._step(g, keys, grad, lr_g, st.cuda())
        P._step(c, keys, grad, lr_c, st)
        torch.cuda.synchronize()
        for gg, cg in zip(g.groups, c.groups):
            torch.testing.assert_close(gg.table.cpu(), cg.table, rtol=1e-3, atol=2e-5)
            for a, b in zip((gg.s0, gg.s1), (cg.s0, cg.s1)):
                if a is not None:
                    torch.testing.assert_close(a.cpu(), b, rtol=1e-3, atol=1e-7)
    keys, grad = P._batch(c, gen)
    st = torch.tensor([6], dtype=torch.int32, device=DEV)
    arrays = lambda: [x for gg in g.groups for x in (gg.table, gg.s0, gg.s1) if x is not None]  # noqa: E731
    snap = [x.clone() for x in arrays()]
    P._step(g, keys, grad, lr_g, st)
    torch.cuda.synchronize()
    eager = [x.clone() for x in arrays()]
    for x, s in zip(arrays(), snap):
        x.copy_(s)
    g.set_keys(keys.cuda())
    g.top_grad["emb"].copy_(grad.cuda())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            g.forward()
            g.backward(lr_g, st)
    torch.cuda.current_stream().wait_stream(side)
    for x, s in zip(arrays(), snap):
        x.copy_(s)
    g.top_grad["emb"].copy_(grad.cuda())
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(arrays(), eager):
        assert torch.equal(x, y)
    g.check_overflow()


@pytest.mark.parametrize("wdt", ["fp32", "bf16"])
def test_model_cuda_graph_equals_eager(wdt):
    """DLRM-DCNv2 with partial row-wise Adam tables: six CUDA-graph training steps equal six eager ones, the bias
    correction reading the step counter that advances inside the graph"""
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    kw = dict(batchsize=128, num_gpus=1, table_sizes=[5000, 300], multi_hot=[3, 1], ev_size=128,
              bottom=(64, 128), top=(128, 1), projection_dim=64, cross_layers=1, lr=0.01, mixed=True,
              embedding_optimizer="partial_rowwise_adam", weight_dtype=wdt)
    a = build_dlrm_dcnv2(use_cuda_graph=True, comm=Comm(DEV), **kw)
    b = build_dlrm_dcnv2(use_cuda_graph=False, comm=Comm(DEV), **kw)
    a.compile(); b.compile()
    b.arena.load_flat(a.arena.dump_flat())
    for ga, gb in zip(a.ebcs_train[0].groups, b.ebcs_train[0].groups):
        assert ga.prow_adam and ga.s1.dtype == torch.float32 and ga.s1.numel() == ga.rows
        gb.table.copy_(ga.table)
    for i in range(6):
        hb = a.reader_train.pool[i % 4]
        a.train_on_host_batch(hb); b.train_on_host_batch(hb)
    torch.cuda.synchronize()
    assert int(a.step_t.item()) == int(b.step_t.item()) >= 6
    torch.testing.assert_close(a.arena.weights, b.arena.weights, rtol=1e-3, atol=1e-4)
    for ga, gb in zip(a.ebcs_train[0].groups, b.ebcs_train[0].groups):
        assert bool((ga.s1 > 0).any())
        torch.testing.assert_close(ga.s1, gb.s1, rtol=1e-3, atol=1e-12)
        torch.testing.assert_close(ga.s0.float(), gb.s0.float(), rtol=1e-2, atol=1e-6)
        torch.testing.assert_close(ga.table.float(), gb.table.float(), rtol=2e-2, atol=1e-4)


@pytest.mark.parametrize("plan,world", [("mixed", 2), ("mixed", 4), ("column", 2)])
def test_emu_ranks_fused_gpu(plan, world):
    """the kernels fed through the fused peer data flow (world > 1) on the GPU equal one process"""
    from hugectr_b200.parallel.emu import run_ranks
    run_ranks(world, lambda c: P.emu_body(plan, True, False, c))


def test_fp8_serving_session_loads_a_checkpoint_of_the_optimizer(tmp_path):
    """a model trained on the GPU with partial row-wise Adam tables writes a checkpoint that an fp8 session loads;
    it predicts as an fp32 session over the dequantized checkpoint"""
    from test_embedding_fp8_serving_cpu import session_predictions_match
    m = P.tiny_model("bf16", dev=DEV)
    for i in range(4):
        m.train_on_host_batch(m.reader_train.pool[i])
    d = str(tmp_path)
    m.save_params_to_files(os.path.join(d, "m"), 4)
    m.graph_to_json(os.path.join(d, "g.json"))
    paths = dict(graph=os.path.join(d, "g.json"), dense=os.path.join(d, "m_dense_4.model"),
                 ebc=os.path.join(d, "m_ebc_4"))
    s8, _ = session_predictions_match(m, paths, tmp_path, DEV)
    assert all(g.s0 is None and g.s1 is None for e in s8.model.ebcs_eval for g in e.groups)
