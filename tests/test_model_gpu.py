"""GPU: native embedding kernels + full DLRM-DCNv2 step vs the fp32 PyTorch/CPU oracle."""

import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk_ebc(device, act, opt_type, ev=128):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    sizes = [1000, 37, 5000]
    hot = {"d0": 3, "d1": 1, "d2": 20}
    ts = [EmbeddingTableConfig(str(i), sizes[i], ev) for i in range(3)]
    cfg.embedding_lookup(ts, ["d0", "d1", "d2"], "emb", ["sum", "mean", "sum"])
    comm = Comm(device)
    opt = CreateOptimizer(opt_type, initial_accu_value=0.1, epsilon=1e-6)
    return EmbeddingCollection(cfg, 64, hot, device, act, comm, opt, seed=3), sizes, hot


@pytest.mark.parametrize("opt", ["SGD", "AdaGrad", "Adam", "Ftrl", "MomentumSGD", "Nesterov"])
@pytest.mark.parametrize("ev", [128, 16])
def test_ebc_fwd_bwd_matches_cpu(opt, ev):
    from hugectr_b200.enums import Optimizer_t
    o = Optimizer_t[opt]
    g, sizes, hot = _mk_ebc(torch.device("cuda"), torch.float32, o, ev)
    c, _, _ = _mk_ebc(torch.device("cpu"), torch.float32, o, ev)
    for gg, cg in zip(g.groups, c.groups):
        cg.table.copy_(gg.table.cpu())
    gen = torch.Generator().manual_seed(0)
    keys = torch.cat([torch.randint(0, sizes[i], (64 * h,), generator=gen)
                      for i, h in enumerate(hot.values())]).int()
    lr_c, st_c = torch.tensor([0.05]), torch.tensor([1], dtype=torch.int32)
    lr_g, st_g = lr_c.cuda(), st_c.cuda()
    for it in range(3):
        g.set_keys(keys.cuda()); c.set_keys(keys)
        g.forward(); c.forward()
        torch.testing.assert_close(g.top_data["emb"].cpu(), c.top_data["emb"], rtol=2e-4, atol=2e-4)
        grad = torch.randn(64, 3 * ev, generator=gen) * 0.1
        g.top_grad["emb"].copy_(grad.cuda()); c.top_grad["emb"].copy_(grad)
        st_c.fill_(it + 1); st_g.fill_(it + 1)
        g.backward(lr_g, st_g); c.backward(lr_c, st_c)
        for gg, cg in zip(g.groups, c.groups):
            torch.testing.assert_close(gg.table.cpu(), cg.table, rtol=1e-3, atol=2e-4)


# bf16 activations and gradients against the fp32 CPU path: the per-step gradients differ by ~1% of their
# norm (see test_dense_path_fp64_gpu.py); 0.1 leaves margin for four steps and stays far below the 1.0 of
# a step whose dense gradients are lost
DELTA_REL = 0.1


def test_dcnv2_step_matches_cpu_reference():
    """bf16 wgmma path vs fp32 CPU path: same init, same batch -> close loss and weights."""
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    kw = dict(batchsize=256, num_gpus=1, table_sizes=[5000, 300, 20000, 40], multi_hot=[3, 1, 10, 2],
              ev_size=128, bottom=(64, 128), top=(256, 128, 1), projection_dim=64, cross_layers=2,
              lr=0.01, use_cuda_graph=False, optimizer="sgd")
    mg = build_dlrm_dcnv2(mixed=True, comm=Comm(torch.device("cuda")), **kw)
    mc = build_dlrm_dcnv2(mixed=False, comm=Comm(torch.device("cpu")), **kw)
    mg.compile(); mc.compile()
    w0 = mg.arena.dump_flat()
    mc.arena.load_flat(w0)
    for gg, cg in zip(mg.ebcs_train[0].groups, mc.ebcs_train[0].groups):
        cg.table.copy_(gg.table.cpu())
    hb = mc.reader_train.pool[0]
    lg, lc = [], []
    for i in range(4):
        mg.train_on_host_batch(hb); mc.train_on_host_batch(hb)
        lg.append(mg.get_current_loss()); lc.append(mc.get_current_loss())
    for a, b in zip(lg, lc):
        assert abs(a - b) < 0.03 * max(1.0, abs(b)), (lg, lc)
    # four SGD steps at lr 0.01 move the dense weights by ~0.02% of their norm, so the weights themselves
    # cannot show a wrong gradient: compare what the steps changed, relative to the size of that change
    dg, dc = mg.arena.dump_flat() - w0, mc.arena.dump_flat() - w0
    rel = ((dg - dc).norm() / dc.norm()).item()
    assert rel < DELTA_REL, rel


def test_cuda_graph_equals_eager():
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    kw = dict(batchsize=128, num_gpus=1, table_sizes=[5000, 300], multi_hot=[3, 1], ev_size=128,
              bottom=(64, 128), top=(128, 1), projection_dim=64, cross_layers=1, lr=0.01, mixed=True)
    a = build_dlrm_dcnv2(use_cuda_graph=True, comm=Comm(torch.device("cuda")), **kw)
    b = build_dlrm_dcnv2(use_cuda_graph=False, comm=Comm(torch.device("cuda")), **kw)
    a.compile(); b.compile()
    b.arena.load_flat(a.arena.dump_flat())
    for ga, gb in zip(a.ebcs_train[0].groups, b.ebcs_train[0].groups):
        gb.table.copy_(ga.table)
    for i in range(6):
        hb = a.reader_train.pool[i % 4]
        a.train_on_host_batch(hb); b.train_on_host_batch(hb)
    torch.cuda.synchronize()
    torch.testing.assert_close(a.arena.weights, b.arena.weights, rtol=1e-3, atol=1e-4)
