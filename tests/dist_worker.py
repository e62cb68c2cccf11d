"""Worker run under torch.distributed.run by the dist tests (gloo on CPU, nccl on GPU)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,  # noqa: E402
                                               EmbeddingTableConfig)
from hugectr_b200.enums import Optimizer_t  # noqa: E402
from hugectr_b200.parallel.comm import Comm  # noqa: E402
from hugectr_b200.solver import CreateOptimizer  # noqa: E402


def dsync(comm=None):
    """wait for my work: the whole device in a real rank; only my stream in an emulated rank (ranks are
    threads of one process there, and another rank's kernel may be spinning on a flag I have yet to set)"""
    if torch.cuda.is_available():
        if comm is not None and getattr(comm, "emulated", False):
            torch.cuda.current_stream().synchronize()
        else:
            torch.cuda.synchronize()


def make_cfg(world, plan):
    sizes = [1000, 37, 5000, 64, 3000]
    hot = {"d0": 3, "d1": 1, "d2": 12, "d3": 2, "d4": 4}
    ev = 16
    ts = [EmbeddingTableConfig(str(i), sizes[i], ev) for i in range(5)]
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(ts, list(hot), "emb", ["sum", "mean", "sum", "sum", "mean"])
    if plan == "mixed":
        sm = [[0] * 5 for _ in range(world)]
        for g in range(world):
            sm[g][2] = 1            # table 2 row-sharded over all GPUs
            sm[g][3] = 1            # table 3 data parallel
        sm[0][0] = 1
        sm[world - 1][1] = 1
        sm[(world // 2)][4] = 1
        cfg.shard(sm, [("mp", ["0", "1", "2", "4"]), ("dp", ["3"])])
    elif plan == "column":
        sm = [[1] * 5 for _ in range(world)]
        cfg.shard(sm, [("mp", ["0", "1", ("2", world), "3", "4"])])
    return cfg, sizes, hot, ev


def run_ebc(plan, fused, comm=None):
    comm = comm or Comm.init_from_env()
    dev = comm.device
    world, rank = comm.world_size, comm.rank
    b = 32
    cfg, sizes, hot, ev = make_cfg(world, plan)
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1, epsilon=1e-6)
    act = torch.float32
    e = EmbeddingCollection(cfg, b, hot, dev, act, comm, opt, seed=1, fused=fused)
    cfg1, _, _, _ = make_cfg(1, "none")
    ref = EmbeddingCollection(cfg1, b * world, hot, torch.device("cpu"), act,
                              Comm.single(torch.device("cpu")), opt, seed=1)
    gen = torch.Generator().manual_seed(5)
    full = {str(i): torch.randn(sizes[i], ev, generator=gen) * 0.1 for i in range(5)}
    for n, w in full.items():
        k = torch.arange(w.shape[0])
        e.load_table_rows(n, k, w)
        ref.load_table_rows(n, k, w)
    lr = torch.tensor([0.05])
    st = torch.tensor([1], dtype=torch.int32)
    lr_d, st_d = lr.to(dev), st.to(dev)
    if os.environ.get("HCTR_TEST_DYN_CAP"):
        assert max(sl["rows"] for g in e.groups for sl in g.table_slices if sl.get("dynamic")) > \
            int(os.environ["HCTR_TEST_DYN_CAP"]), "no shard grew"
    for it in range(3):
        gk = [torch.randint(0, sizes[i], (b * world, h), generator=gen) for i, h in enumerate(hot.values())]
        keys_ref = torch.cat([k.reshape(-1) for k in gk]).int()
        keys_loc = torch.cat([k[rank * b:(rank + 1) * b].reshape(-1) for k in gk]).int()
        grad = torch.randn(b * world, 5 * ev, generator=gen) * 0.1
        e.set_keys(keys_loc.to(dev)); ref.set_keys(keys_ref)
        e.forward(); ref.forward()
        if dev.type == "cuda":
            dsync(comm)
        out = e.top_data["emb"].float().cpu()
        exp = ref.top_data["emb"][rank * b:(rank + 1) * b]
        err = (out - exp).abs().max().item()
        assert err < 1e-4, f"rank {rank} it {it} fwd err {err}"
        e.top_grad["emb"].copy_(grad[rank * b:(rank + 1) * b].to(dev))
        ref.top_grad["emb"].copy_(grad)
        e.backward(lr_d, st_d); ref.backward(lr, st)
        if dev.type == "cuda":
            dsync(comm)
    # compare every local shard with the reference table
    for n in full:
        rk, rw = ref.dump_table_local(n)[0][:2]
        for (k, w, c0, sts, kind) in e.dump_table_local(n):
            exp = rw[k][:, c0:c0 + w.shape[1]]
            err = (w - exp).abs().max().item()
            assert err < 2e-4, f"rank {rank} table {n} err {err}"
    comm.barrier()
    if rank == 0:
        print(f"EBC_OK plan={plan} fused={fused} world={world}")


def run_dynamic(comm=None):
    """dynamic (hashed) tables inside the collection: arbitrary 64-bit keys, rows assigned on first
    sight; must behave like the static tables they shadow (same values under a key bijection)"""
    comm = comm or Comm.init_from_env()
    dev = comm.device
    world, rank = comm.world_size, comm.rank
    b, ev = 16, 8
    sizes = [500, 40, 900]
    hot = {"d0": 3, "d1": 1, "d2": 5}
    scramble = lambda k: k * 1000003 + 17

    def cfg_for(w, dynamic):
        # HCTR_TEST_DYN_CAP: start far below the number of keys -- the shards grow while the tables are loaded
        cap = int(os.environ.get("HCTR_TEST_DYN_CAP", "1024"))
        ts = [EmbeddingTableConfig(str(i), -1 if (dynamic and i != 1) else sizes[i], ev, init_capacity=cap)
              for i in range(3)]
        cfg = EmbeddingCollectionConfig()
        cfg.embedding_lookup(ts, list(hot), "emb", ["sum", "sum", "mean"])
        sm = [[0] * 3 for _ in range(w)]
        for g in range(w):
            sm[g][2] = 1                # table 2 row-sharded over every rank
        sm[0][0] = 1
        sm[w - 1][1] = 1
        cfg.shard(sm, [("mp", ["0", "1", "2"])])
        return cfg
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1, epsilon=1e-6)
    e = EmbeddingCollection(cfg_for(world, True), b, hot, dev, torch.float32, comm, opt, key_dtype=torch.int64,
                            seed=1)
    assert e.has_dynamic
    ref = EmbeddingCollection(cfg_for(1, False), b * world, hot, torch.device("cpu"), torch.float32,
                              Comm.single(torch.device("cpu")), opt, key_dtype=torch.int64, seed=1)
    gen = torch.Generator().manual_seed(9)
    full = {str(i): torch.randn(sizes[i], ev, generator=gen) * 0.1 for i in range(3)}
    for n, w in full.items():
        k = torch.arange(w.shape[0])
        ref.load_table_rows(n, k, w)
        e.load_table_rows(n, scramble(k) if n != "1" else k, w)
    lr, st = torch.tensor([0.05]), torch.tensor([1], dtype=torch.int32)
    if os.environ.get("HCTR_TEST_DYN_CAP"):
        assert max(sl["rows"] for g in e.groups for sl in g.table_slices if sl.get("dynamic")) > \
            int(os.environ["HCTR_TEST_DYN_CAP"]), "no shard grew"
    for it in range(3):
        gk = [torch.randint(0, sizes[i], (b * world, h), generator=gen) for i, h in enumerate(hot.values())]
        keys_ref = torch.cat([k.reshape(-1) for k in gk])
        gk2 = [scramble(k) if i != 1 else k for i, k in enumerate(gk)]
        keys_loc = torch.cat([k[rank * b:(rank + 1) * b].reshape(-1) for k in gk2])
        grad = torch.randn(b * world, 3 * ev, generator=gen) * 0.1
        e.set_keys(keys_loc.to(dev)); ref.set_keys(keys_ref)
        e.forward(); ref.forward()
        err = (e.top_data["emb"].float().cpu() - ref.top_data["emb"][rank * b:(rank + 1) * b]).abs().max().item()
        assert err < 1e-5, f"rank {rank} it {it} fwd err {err}"
        e.top_grad["emb"].copy_(grad[rank * b:(rank + 1) * b].to(dev))
        ref.top_grad["emb"].copy_(grad)
        e.backward(lr.to(dev), st.to(dev)); ref.backward(lr, st)
    for n in full:
        rk, rw = ref.dump_table_local(n)[0][:2]
        for (k, w, c0, sts, kind) in e.dump_table_local(n):
            if len(k) == 0:
                continue
            orig = (k - 17) // 1000003 if n != "1" else k
            err = (w - rw[orig][:, c0:c0 + w.shape[1]]).abs().max().item()
            assert err < 1e-5, f"rank {rank} table {n} err {err}"
    # evaluation plan: unknown keys read as zero vectors
    ev_e = e.eval_clone(b)
    unk = torch.full((b * sum(hot.values()),), 987654321987, dtype=torch.int64)
    ev_e.set_keys(unk.to(dev))
    ev_e.forward(False)
    assert float(ev_e.top_data["emb"][:, :ev].abs().max()) == 0.0
    comm.barrier()
    if rank == 0:
        print("DYNAMIC_OK")


def run_sok(comm=None):
    """sok.lookup_sparse over a distributed variable (rows sharded by key %% world): forward, sparse
    backward and optimizer step must equal a dense single-process embedding"""
    import hugectr_b200 as hugectr
    from hugectr_b200 import sok
    comm = comm or Comm.init_from_env()
    world, rank = comm.world_size, comm.rank
    sok.init(comm)
    torch.manual_seed(0)
    full = torch.randn(40, 4)                               # same on every rank
    v = sok.Variable(initial_value=full.clone(), name="dist_v")
    gen = torch.Generator().manual_seed(11)
    b = 6
    ids_all = torch.randint(0, 40, (b * world, 3), generator=gen)
    ids_all[0, 2] = -1
    ids = ids_all[rank * b:(rank + 1) * b]
    out = sok.lookup_sparse(v, ids, "mean")
    W = full.clone().requires_grad_(True)
    m = (ids_all >= 0).unsqueeze(-1).float()
    ref = (W[ids_all.clamp(min=0)] * m).sum(1) / m.sum(1).clamp(min=1)
    torch.testing.assert_close(out, ref[rank * b:(rank + 1) * b].detach(), atol=1e-6, rtol=1e-5)
    gout = torch.randn(b * world, 4, generator=gen)
    (out * gout[rank * b:(rank + 1) * b]).sum().backward()
    (ref * gout).sum().backward()
    sok.OptimizerWrapper(hugectr.Optimizer_t.SGD, lr=0.1).apply_gradients([v])
    W2 = (W - 0.1 * W.grad).detach()
    keys = v.global_keys()
    torch.testing.assert_close(v.weight.float().cpu(), W2[keys.cpu()], atol=1e-6, rtol=1e-5)
    # weighted lookups (sp_weights): mean = weighted sum / sum of weights, gradients scale with the weight
    for comb in ("sum", "mean"):
        full2 = torch.randn(40, 4, generator=gen)
        v2 = sok.Variable(initial_value=full2.clone(), name="dist_w_" + comb)
        w_all = torch.rand(b * world, 3, generator=gen) + 0.1
        out = sok.lookup_sparse(v2, ids, sp_weights=w_all[rank * b:(rank + 1) * b], combiners=comb)
        W = full2.clone().requires_grad_(True)
        wm = w_all * (ids_all >= 0).float()
        ref = (W[ids_all.clamp(min=0)] * wm.unsqueeze(-1)).sum(1)
        if comb == "mean":
            ref = ref / wm.sum(1, keepdim=True)
        torch.testing.assert_close(out, ref[rank * b:(rank + 1) * b].detach(), atol=1e-5, rtol=1e-5)
        (out * gout[rank * b:(rank + 1) * b]).sum().backward()
        (ref * gout).sum().backward()
        sok.OptimizerWrapper(hugectr.Optimizer_t.SGD, lr=0.1).apply_gradients([v2])
        keys = v2.global_keys()
        torch.testing.assert_close(v2.weight.float().cpu(), (W - 0.1 * W.grad).detach()[keys.cpu()],
                                   atol=1e-5, rtol=1e-5)
    comm.barrier()
    if rank == 0:
        print("SOK_OK")


def run_sok_fuzz(seed, comm=None):
    """sok.lookup_sparse over a random mix of variables (distributed / localized / dynamic with scrambled 64-bit keys),
    random hotness, combiners, optional per-id weights, padded bags: forward, sparse backward and an AdaGrad step must
    equal dense single-process embeddings"""
    import random
    import hugectr_b200 as hugectr
    from hugectr_b200 import sok
    comm = comm or Comm.init_from_env()
    world, rank = comm.world_size, comm.rank
    sok.init(comm)
    rnd = random.Random(int(seed))
    gen = torch.Generator().manual_seed(int(seed))
    b = 5
    nv = rnd.randint(1, 3)
    scramble = lambda k: k * 1000003 + 17
    vars_, fulls, kinds, ids_all, wts_all, combs = [], [], [], [], [], []
    for i in range(nv):
        vocab, dim = rnd.randint(6, 40), rnd.choice([4, 8])
        full = torch.randn(vocab, dim, generator=gen)
        kind = rnd.choice(["distributed", "localized", "dynamic"])
        if kind == "distributed":
            v = sok.Variable(initial_value=full.clone(), name=f"fz{seed}_{i}")
        elif kind == "localized":
            v = sok.Variable(initial_value=full.clone(), mode=f"localized:{rnd.randrange(world)}", name=f"fz{seed}_{i}")
        else:
            v = sok.DynamicVariable(dim, var_type="hbm", init_capacity=64, max_capacity=256, name=f"fz{seed}_{i}")
            sok.assign(v, scramble(torch.arange(vocab)), full)
        H = rnd.randint(1, 4)
        ids = torch.randint(0, vocab, (b * world, H), generator=gen)
        if H > 1:
            n = torch.randint(1, H + 1, (b * world,), generator=gen)
            ids = torch.where(torch.arange(H).view(1, -1) < n.view(-1, 1), ids, torch.full_like(ids, -1))
        w = torch.rand(b * world, H, generator=gen) + 0.1 if rnd.random() < 0.4 else None
        vars_.append(v); fulls.append(full); kinds.append(kind); ids_all.append(ids); wts_all.append(w)
        combs.append(rnd.choice(["sum", "mean"]))
    use_w = all(w is not None for w in wts_all)
    loc = lambda t: t[rank * b:(rank + 1) * b]
    feed = [loc(scramble(i_) * (i_ >= 0) + (-1) * (i_ < 0)) if k == "dynamic" else loc(i_) for i_, k in zip(ids_all, kinds)]
    outs = sok.lookup_sparse(vars_, feed, sp_weights=[loc(w) for w in wts_all] if use_w else None, combiners=combs)
    gouts = [torch.randn(b * world, f.shape[1], generator=gen) for f in fulls]
    loss = sum((o * loc(g)).sum() for o, g in zip(outs, gouts))
    loss.backward()
    opt = sok.OptimizerWrapper(hugectr.Optimizer_t.AdaGrad, lr=0.1, initial_accu_value=0.0)
    opt.apply_gradients(vars_)
    for i in range(nv):
        Wt = fulls[i].clone().requires_grad_(True)
        ids = ids_all[i]
        m = (ids >= 0).float()
        wm = m * wts_all[i] if use_w else m
        ref = (Wt[ids.clamp(min=0)] * wm.unsqueeze(-1)).sum(1)
        if combs[i] == "mean":
            ref = ref / wm.sum(1, keepdim=True).clamp(min=1e-12)
        torch.testing.assert_close(outs[i].detach(), loc(ref).detach(), atol=1e-5, rtol=1e-5)
        (ref * gouts[i]).sum().backward()
        g = Wt.grad
        W2 = Wt.detach() - 0.1 * g / ((g * g).sqrt() + 1e-7)        # first AdaGrad step from a zero accumulator
        if kinds[i] == "dynamic":
            k, wv = sok.export(vars_[i])
            orig = (k - 17) // 1000003
        else:
            k = vars_[i].global_keys().cpu()
            wv, orig = vars_[i].weight.float().cpu(), k
        touched = (g.abs().sum(1) > 0)
        sel = touched[orig]
        torch.testing.assert_close(wv[sel], W2[orig][sel], atol=2e-5, rtol=1e-4)
        torch.testing.assert_close(wv[~sel], fulls[i][orig][~sel], atol=0, rtol=0)       # untouched rows did not move
    comm.barrier()
    if rank == 0:
        print("SOK_FUZZ_OK", seed)


def run_fuzz(seed, comm=None):
    """randomised collection: random tables / hotness / combiners (sum, mean, concat) / batch- or
    feature-major tops / padded bags / random sharding plan (table-wise, row-wise, column-wise, dp),
    compared with a brute-force gather oracle (forward) and a scatter oracle (SGD backward)"""
    import random
    comm = comm or Comm.init_from_env()
    dev = comm.device
    world, rank = comm.world_size, comm.rank
    rnd = random.Random(int(seed))
    b = 8
    nt = rnd.randint(3, 5)
    ev = [rnd.choice([4, 8]) for _ in range(nt)]
    vocab = [rnd.randint(5, 60) for _ in range(nt)]
    hot = [rnd.randint(1, 4) for _ in range(nt)]
    comb = [rnd.choice(["sum", "mean", "concat"]) for _ in range(nt)]
    ts = [EmbeddingTableConfig(str(i), vocab[i], ev[i]) for i in range(nt)]
    cfg = EmbeddingCollectionConfig()
    split = rnd.randint(1, nt - 1)
    # first `split` lookups share one batch-major top, the rest are feature-major tops of their own
    cfg.embedding_lookup(ts[:split], [f"d{i}" for i in range(split)], "bm", comb[:split])
    for i in range(split, nt):
        cfg.embedding_lookup(ts[i], f"d{i}", f"fm{i}", comb[i])
    if world > 1:
        sm = [[0] * nt for _ in range(world)]
        strat_mp, strat_dp = [], []
        for i in range(nt):
            kind = rnd.choice(["table", "row", "dp", "col"])
            if kind == "dp":
                for g in range(world):
                    sm[g][i] = 1
                strat_dp.append(str(i))
            elif kind == "table":
                sm[rnd.randrange(world)][i] = 1
                strat_mp.append(str(i))
            elif kind == "row" or ev[i] % world:
                for g in range(world):
                    sm[g][i] = 1
                strat_mp.append(str(i))
            else:
                for g in range(world):
                    sm[g][i] = 1
                strat_mp.append((str(i), world))
        st = ([("mp", strat_mp)] if strat_mp else []) + ([("dp", strat_dp)] if strat_dp else [])
        if rnd.random() < 0.5:          # the reference's form: per GPU the list of table NAMES it holds
            sm = [[str(i) for i in range(nt) if row[i]] for row in sm]
        comp = None
        if os.environ.get("HCTR_FUZZ_UNIQUE") and strat_mp:
            # a random subset of the model-parallel tables on the Unique-compression exchange (column-split ones
            # fall back to Reduction inside the collection; the fused data flow keeps its own exchange)
            from hugectr_b200.enums import CompressionStrategy
            names_mp = [x[0] if isinstance(x, tuple) else x for x in strat_mp]
            comp = {CompressionStrategy.Unique: [n_ for n_ in names_mp if rnd.random() < 0.6]}
        cfg.shard(sm, st, compression_strategy=comp)
    adagrad = rnd.random() < 0.5          # non-linear rule: exercises the reduce-then-update order and
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.0, epsilon=1e-7) if adagrad \
        else CreateOptimizer(Optimizer_t.SGD)    # the optimizer-state windows of column / row shards
    S = [torch.zeros(vocab[i], ev[i]) for i in range(nt)]
    hotd = {f"d{i}": hot[i] for i in range(nt)}
    e = EmbeddingCollection(cfg, b, hotd, dev, torch.float32, comm, opt, key_dtype=torch.int64, seed=3)
    gen = torch.Generator().manual_seed(int(seed))
    W = [torch.randn(vocab[i], ev[i], generator=gen) for i in range(nt)]
    for i in range(nt):
        e.load_table_rows(str(i), torch.arange(vocab[i]), W[i])
    lr = 0.1
    for it in range(2):
        keys = []
        for i in range(nt):
            k = torch.randint(0, vocab[i], (b * world, hot[i]), generator=gen)
            if comb[i] != "concat" and hot[i] > 1:          # padded (shorter) bags
                n = torch.randint(1, hot[i] + 1, (b * world,), generator=gen)
                k = torch.where(torch.arange(hot[i]).view(1, -1) < n.view(-1, 1), k, torch.full_like(k, -1))
            keys.append(k)
        loc = torch.cat([k[rank * b:(rank + 1) * b].reshape(-1) for k in keys])
        e.set_keys(loc.to(dev))
        e.forward()

        def pooled(i):
            k = keys[i]
            v = W[i][k.clamp(min=0)] * (k >= 0).unsqueeze(-1)
            if comb[i] == "concat":
                return v.reshape(b * world, -1)
            s_ = v.sum(1)
            return s_ / (k >= 0).sum(1, keepdim=True).clamp(min=1) if comb[i] == "mean" else s_
        exp_bm = torch.cat([pooled(i) for i in range(split)], 1)
        got = e.top_data["bm"].float().cpu().reshape(b, -1)
        assert (got - exp_bm[rank * b:(rank + 1) * b]).abs().max() < 1e-5, ("bm", seed, it)
        for i in range(split, nt):
            got = e.top_data[f"fm{i}"].float().cpu().reshape(b, -1)
            assert (got - pooled(i)[rank * b:(rank + 1) * b]).abs().max() < 1e-5, (f"fm{i}", seed, it)
        # backward: random top grads, SGD update == scatter of (scaled) grads
        G = {}
        gb = torch.randn(b * world, exp_bm.shape[1], generator=gen)
        e.top_grad["bm"].copy_(gb[rank * b:(rank + 1) * b].view_as(e.top_grad["bm"]).to(dev))
        off = 0
        for i in range(split):
            w_ = ev[i] * (hot[i] if comb[i] == "concat" else 1)
            G[i] = gb[:, off:off + w_]
            off += w_
        for i in range(split, nt):
            w_ = ev[i] * (hot[i] if comb[i] == "concat" else 1)
            G[i] = torch.randn(b * world, w_, generator=gen)
            e.top_grad[f"fm{i}"].copy_(G[i][rank * b:(rank + 1) * b].view_as(e.top_grad[f"fm{i}"]).to(dev))
        e.backward(torch.tensor([lr], device=dev), torch.tensor([1], dtype=torch.int32, device=dev))
        for i in range(nt):
            k = keys[i]
            valid = (k >= 0)
            if comb[i] == "concat":
                g_ = G[i].view(b * world, hot[i], ev[i])
            else:
                g_ = G[i].unsqueeze(1).expand(b * world, hot[i], ev[i])
                if comb[i] == "mean":
                    g_ = g_ / valid.sum(1).clamp(min=1).view(-1, 1, 1)
            if not adagrad:
                W[i].index_add_(0, k[valid], -lr * g_[valid])
            else:
                Gr = torch.zeros_like(W[i]).index_add_(0, k[valid], g_[valid])      # reduce per row first
                S[i] += Gr * Gr
                W[i] -= lr * Gr / (S[i].sqrt() + 1e-7)
    for i in range(nt):
        for (k, w, c0, sts, kind) in e.dump_table_local(str(i)):
            if len(k):
                err = (w[:, :min(w.shape[1], ev[i] - c0)] - W[i][k][:, c0:c0 + w.shape[1]]).abs().max().item()
                assert err < 1e-4, (seed, "table", i, err)
    comm.barrier()
    if rank == 0:
        print("FUZZ_OK", seed)


def run_ebcio(tmpdir, seed, comm=None):
    """parallel (every rank writes its windows) vs gather (rank 0 writes) collection dumps hold the same
    key -> (row, optimizer state) content for a random plan incl. column-wise, data-parallel and dynamic
    tables; a chunked load of the parallel dump restores every shard bit-exactly"""
    import random
    from types import SimpleNamespace as NS
    from hugectr_b200.io.checkpoint import embedding_dump, embedding_load, read_ebc_folder
    comm = comm or Comm.init_from_env()
    dev, world, rank = comm.device, comm.world_size, comm.rank
    rnd = random.Random(int(seed))
    b, nt = 8, 5
    ev = [rnd.choice([4, 8]) for _ in range(nt)]
    vocab = [rnd.randint(5, 60) for _ in range(nt)]
    ts = [EmbeddingTableConfig(str(i), vocab[i], ev[i]) for i in range(nt - 1)]
    ts.append(EmbeddingTableConfig(str(nt - 1), -1, ev[nt - 1], init_capacity=128))     # dynamic
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(ts, [f"d{i}" for i in range(nt)], "bm", ["sum"] * nt)
    if world > 1:
        sm = [[0] * nt for _ in range(world)]
        mp, dp = [], []
        for i in range(nt):
            kind = rnd.choice(["table", "row", "dp", "col"]) if i < nt - 1 else "row"
            if kind == "table":
                sm[rnd.randrange(world)][i] = 1
            else:
                for g in range(world):
                    sm[g][i] = 1
            if kind == "dp":
                dp.append(str(i))
            elif kind == "col" and ev[i] % world == 0:
                mp.append((str(i), world))
            else:
                mp.append(str(i))
        cfg.shard(sm, ([("mp", mp)] if mp else []) + ([("dp", dp)] if dp else []))
    opt = CreateOptimizer(Optimizer_t.AdaGrad)
    e = EmbeddingCollection(cfg, b, {f"d{i}": 2 for i in range(nt)}, dev, torch.float32, comm, opt,
                            key_dtype=torch.int64, seed=5)
    gen = torch.Generator().manual_seed(int(seed))
    for it in range(3):
        keys = [torch.randint(0, vocab[i] if i < nt - 1 else 1000, (b * world, 2), generator=gen) for i in range(nt)]
        e.set_keys(torch.cat([k[rank * b:(rank + 1) * b].reshape(-1) for k in keys]).to(dev))
        e.forward()
        e.top_grad["bm"].copy_(torch.randn(e.top_grad["bm"].shape, generator=gen).to(dev))
        e.backward(torch.tensor([0.1], device=dev), torch.tensor([1], dtype=torch.int32, device=dev))
    model = NS(comm=comm, world=world, ebcs_train=[e], key_dtype=torch.int64, reader_params=None)
    pa, ga = os.path.join(tmpdir, "par"), os.path.join(tmpdir, "gat")
    embedding_dump(model, pa)
    os.environ["HCTR_EBC_DUMP"] = "gather"
    embedding_dump(model, ga)
    os.environ.pop("HCTR_EBC_DUMP")
    comm.barrier()
    A, B = read_ebc_folder(pa + "/embedding_collection_0"), read_ebc_folder(ga + "/embedding_collection_0")
    assert sorted(A) == sorted(B) == list(range(nt))
    for tid in A:
        (ka, wa, sa), (kb, wb, sb) = A[tid], B[tid]
        oa, ob = torch.argsort(ka), torch.argsort(kb)
        assert torch.equal(ka[oa], kb[ob]) and ka.unique().numel() == ka.numel(), tid
        assert torch.equal(wa[oa], wb[ob]), tid
        assert (sa is None) == (sb is None)
        for x, y in zip(sa or [], sb or []):
            assert torch.equal(x[oa], y[ob]), tid
        assert sa is not None and float(sa[0].abs().sum()) > 0       # AdaGrad accumulators travelled
    before = {str(i): e.dump_table_local(str(i)) for i in range(nt)}
    for grp in e.groups:
        grp.table.zero_()
        if grp.s0 is not None:
            grp.s0.zero_()
    os.environ["HCTR_EBC_LOAD_CHUNK_ROWS"] = "7"
    embedding_load(model, pa)
    for n_, parts in before.items():
        for (k0, w0, c0, s0, _), (k1, w1, c1, s1, _) in zip(parts, e.dump_table_local(n_)):
            assert torch.equal(k0, k1) and torch.equal(w0, w1) and c0 == c1, n_
            assert torch.equal(s0[0], s1[0]), n_
    comm.barrier()
    if rank == 0:
        print("EBCIO_OK", seed)


def run_symmfail(comm=None):
    """a peer-mapping failure on ONE rank makes EVERY rank raise (agreement before the error), so the
    job falls back to NCCL collectives as a whole instead of deadlocking in mismatched collectives"""
    import ctypes as C
    from hugectr_b200.parallel import symm
    comm = comm or Comm.init_from_env()

    class FakeLib:
        freed = closed = 0
        def hctr_ipc_alloc(self, n): return 0x1000 * (comm.rank + 1)
        def hctr_ipc_get_handle(self, p, h): return 0
        def hctr_ipc_open(self, h): return 0 if comm.rank == 1 else 0x9000
        def hctr_ipc_close(self, q): FakeLib.closed += 1; return 0
        def hctr_ipc_free(self, p): FakeLib.freed += 1; return 0
        def hctr_last_cuda_error(self): return b"peer access unsupported"
    fake = FakeLib()
    symm.lib = lambda: fake
    heap = symm.SymmetricHeap.__new__(symm.SymmetricHeap)
    heap.comm, heap.rank, heap.world, heap.device, heap._allocs = comm, comm.rank, comm.world_size, comm.device, {}
    try:
        heap.alloc(64, torch.int32)
        raise SystemExit("alloc did not fail")
    except RuntimeError as e:
        assert "rank(s) 1:" in str(e) and "peer access unsupported" in str(e), str(e)
    assert FakeLib.freed == 1 and not heap._allocs
    comm.barrier()                       # the collective sequence is still aligned on all ranks
    if comm.rank == 0:
        print("SYMMFAIL_OK")


def run_allreduce(comm=None):
    comm = comm or Comm.init_from_env()
    from hugectr_b200.parallel.p2p import P2PAllReduce
    n = 4 * comm.world_size * 100003
    buf = comm.symm_alloc(n, torch.float32)
    ar = P2PAllReduce(comm, buf)
    for it in range(5):
        g = torch.Generator(device="cuda").manual_seed(it * 10 + comm.rank)
        x = torch.randn(n, device="cuda", generator=g)
        exp = x.clone()
        comm.all_reduce(exp)
        buf.copy_(x)
        ar.run()
        dsync(comm)
        err = (buf - exp).abs().max().item()
        assert err < 1e-4, f"allreduce err {err}"
    comm.barrier()
    if comm.rank == 0:
        print("ALLREDUCE_OK")


def run_model(comm=None):
    """whole-model data-parallel step: (NCCL all-reduce, no overlap, eager) vs (bucketed P2P
    all-reduce overlapped with backward, side streams, CUDA graph) must train to the same weights"""
    import hugectr_b200 as hugectr
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    comm = comm or Comm.init_from_env()
    world = comm.world_size
    cuda = comm.device.type == "cuda"
    sizes = [4000, 300, 50, 9000, 1200, 77]
    hot = [3, 1, 1, 8, 2, 1]

    def build(algo):
        m = build_dlrm_dcnv2(batchsize=256 * world, num_gpus=world, table_sizes=sizes, multi_hot=hot,
                             ev_size=16, lr=0.05, mixed=cuda, optimizer="sgd", bottom=(64, 32, 16),
                             top=(64, 32, 1), cross_layers=2, projection_dim=16, comm=comm,
                             all_reduce_algo=algo,
                             use_cuda_graph=cuda and not getattr(comm, "emulated", False))
        m.compile()
        return m

    flags = ("HCTR_DISABLE_AR_OVERLAP", "HCTR_DISABLE_OVERLAP", "HCTR_DISABLE_CUDA_GRAPH")
    comm.barrier()
    for f in flags:
        os.environ[f] = "1"
    ma = build(hugectr.AllReduceAlgo.NCCL)
    pool = ma.reader_train.pool
    for i in range(5):
        ma.train_on_host_batch(pool[i % len(pool)])
    wa = ma.arena.weights.clone()
    la = ma.get_current_loss()
    comm.barrier()                      # (emulated ranks share the process environment)
    for f in flags:
        os.environ[f] = "0"
    mb = build(hugectr.AllReduceAlgo.OneShot if cuda else hugectr.AllReduceAlgo.NCCL)
    for i in range(5):
        mb.train_on_host_batch(pool[i % len(pool)])
    wb = mb.arena.weights
    lb = mb.get_current_loss()
    err = float((wa - wb).abs().max())
    moved = float((wa - ma.arena.weights * 0).abs().max())
    assert err < 2e-3 * max(1.0, moved), f"weights differ: {err} (loss {la} vs {lb})"
    assert abs(la - lb) < 2e-2 * max(1.0, abs(la)), (la, lb)
    # replicas stay identical across ranks
    ref = wb.clone()
    comm.broadcast(ref, 0)
    assert float((ref - wb).abs().max()) == 0.0, "dense replicas diverged across ranks"
    comm.barrier()
    if comm.rank == 0:
        print("MODEL_OK", err, la, lb)


def run_equiv(optimizer="sgd", gpus_per_node=0, comm=None):
    """N-rank training (data-parallel dense, model-parallel / data-parallel embeddings) must equal
    single-process training on the concatenation of the ranks' batches."""
    import hugectr_b200 as hugectr
    from hugectr_b200.data.batch import HostBatch
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    comm = comm or Comm.init_from_env()
    world, rank = comm.world_size, comm.rank
    cuda = comm.device.type == "cuda"
    sizes = [4000, 300, 50, 9000, 1200, 77]
    hot = [3, 1, 1, 8, 2, 1]
    b = 128
    kw = dict(table_sizes=sizes, multi_hot=hot, ev_size=16, lr=0.05 if optimizer == "sgd" else 0.01,
              mixed=False, optimizer=optimizer,
              bottom=(64, 32, 16), top=(64, 32, 1), cross_layers=2, projection_dim=16,
              use_cuda_graph=False)
    # table 0 row-sharded over every rank, table 3 on the last rank, the small tables data-parallel
    sm = [[1, 1, 1, 0, 1, 1] for _ in range(world)]
    sm[world - 1][3] = 1
    plan = (sm, [("mp", ["0", "3"]), ("dp", ["1", "2", "4", "5"])])
    if os.environ.get("HCTR_TEST_PLAN_SEED"):
        # random placement per table: table-wise, row-wise, column-wise (x row-wise) or data-parallel
        import random
        rnd = random.Random(int(os.environ["HCTR_TEST_PLAN_SEED"]))
        sm = [[0] * len(sizes) for _ in range(world)]
        mp, dp = [], []
        for t in range(len(sizes)):
            kind = rnd.choice(["table", "row", "col", "dp"])
            if kind == "table":
                sm[rnd.randrange(world)][t] = 1
            else:
                for g in range(world):
                    sm[g][t] = 1
            if kind == "dp":
                dp.append(str(t))
            elif kind == "col" and world % 2 == 0:
                mp.append((str(t), 2))
            else:
                mp.append(str(t))
        plan = (sm, ([("mp", mp)] if mp else []) + ([("dp", dp)] if dp else []))
    hkw = {}
    if gpus_per_node:
        # logical nodes: hierarchical two-stage exchange (intra-node reduce, inter-node same-local-id)
        hkw = dict(gpus_per_node=gpus_per_node, comm_strategy=hugectr.CommunicationStrategy.Hierarchical,
                   fused_embedding_comm=False)
    if os.environ.get("HCTR_TEST_UNIQUE"):
        # every model-parallel table on the Unique-compression exchange (collective path)
        mp_names = [x[0] if isinstance(x, tuple) else x for (k_, items) in plan[1] if k_ == "mp" for x in items]
        hkw.update(compression_strategy={hugectr.CompressionStrategy.Unique: mp_names}, fused_embedding_comm=False)
    m = build_dlrm_dcnv2(batchsize=b * world, num_gpus=world, comm=comm, shard_plan=plan, **kw, **hkw)
    m.compile()
    if os.environ.get("HCTR_TEST_UNIQUE"):
        assert m.ebcs_train[0]._uniq is not None and not m._graph_safe()
    if gpus_per_node:
        assert m.ebcs_train[0].hier and comm.num_nodes == world // gpus_per_node
    single = Comm.single(comm.device)
    ref = build_dlrm_dcnv2(batchsize=b * world, num_gpus=1, comm=single, **kw)
    ref.compile()
    # identical initial embedding tables: copy the reference's rows into the sharded model
    for e_ref, e in zip(ref.ebcs_train, m.ebcs_train):
        for name in list(e_ref.tmap.keys()):
            ev = e_ref.tmap[name].ev_size
            for keys, vals, col0, _, _ in e_ref.dump_table_local(name):
                e.load_table_rows(name, keys, vals[:, :ev].cpu())
    m.arena.weights.copy_(ref.arena.weights)
    m.arena.sync_shadow()
    pool = m.reader_train.pool
    blocks = m.layout.blocks
    for step in range(3):
        hb = pool[step % len(pool)]
        allb = comm.all_gather_object((hb.label.clone(), hb.dense.clone(), hb.keys.clone()))
        labels = torch.cat([x[0] for x in allb])
        dense = torch.cat([x[1] for x in allb])
        keys, off = [], 0
        for (_, S, H, _) in blocks:
            n = b * S * H
            keys.append(torch.cat([x[2][off:off + n] for x in allb]))
            off += n
        big = HostBatch(labels, dense, torch.cat(keys), None, b * world)
        m.train_on_host_batch(hb)
        ref.train_on_host_batch(big)
        l_m, l_r = m.get_current_loss(), ref.get_current_loss()
        assert abs(l_m - l_r) < 2e-3 * max(1.0, abs(l_r)), (step, l_m, l_r)
    err = float((m.arena.weights - ref.arena.weights).abs().max())
    assert err < 2e-3, f"dense weights differ from the single-process run: {err}"
    # embedding rows: gather every local shard and compare with the reference table
    for e_ref, e in zip(ref.ebcs_train, m.ebcs_train):
        for name in list(e_ref.tmap.keys()):
            ev = e_ref.tmap[name].ev_size
            rk, rv = None, None
            for keys, vals, col0, _, _ in e_ref.dump_table_local(name):
                rk, rv = keys.cpu(), vals[:, :ev].cpu()
            for keys, vals, col0, _, _ in e.dump_table_local(name):
                if len(keys) == 0:
                    continue
                idx = torch.searchsorted(rk, keys.cpu())
                w = min(vals.shape[1], ev - col0)
                d = (rv[idx][:, col0:col0 + w] - vals[:, :w].cpu()).abs().max().item()
                assert d < 2e-3, f"table {name} differs: {d}"
    comm.barrier()
    if rank == 0:
        print("EQUIV_OK", err)


def run_legacy(comm=None):
    """legacy embeddings (Distributed = row-sharded over all ranks, Localized = slot s on rank s % N)
    trained data-parallel: replicas stay identical and the loss is finite"""
    import hugectr_b200 as hugectr
    from hugectr_b200.models import build_dcn, build_deepfm
    comm = comm or Comm.init_from_env()
    world = comm.world_size
    slots = [120] * 26
    for build, kw in ((build_dcn, {}),
                      (build_deepfm, {"embedding_type": hugectr.Embedding_t.LocalizedSlotSparseEmbeddingHash})):
        m = build(batchsize=64 * world, vvgpu=[list(range(world))], slot_sizes=slots, workspace_mb=2,
                  comm=comm, max_eval_batches=1, **kw)
        m.compile()
        for _ in range(4):
            assert m.train()
        loss = m.get_current_loss()
        assert loss == loss and abs(loss) < 1e4, loss
        w = m.arena.weights.clone()
        comm.broadcast(w, 0)
        assert float((w - m.arena.weights).abs().max()) < 1e-6, "dense replicas diverged"
        m.eval()
        m.get_eval_metrics()
    comm.barrier()
    if comm.rank == 0:
        print("LEGACY_OK")


def run_legacy_equiv(kind="distributed", optimizer="adam", seed=0, comm=None):
    """Legacy hash embeddings: N-rank training must equal single-process training on the concatenated batches, KEY BY
    KEY (rows are handed out in arrival order, so tables are compared through their (key -> vector) dumps).  Both
    models start from the same sparse model files and dense weights; random slots / bag lengths / combiner."""
    import random
    import tempfile
    import numpy as np
    import hugectr_b200 as hugectr
    from hugectr_b200.data.batch import HostBatch
    comm = comm or Comm.init_from_env()
    world, rank = comm.world_size, comm.rank
    rnd = random.Random(int(seed))
    S = rnd.randint(2, 5)
    H = rnd.choice([1, 2, 4])
    vec = rnd.choice([4, 8])
    comb = rnd.choice(["sum", "mean"])
    vocab = [rnd.randint(5, 40) for _ in range(S)]
    offs = np.concatenate([[0], np.cumsum(vocab)[:-1]])
    b = 16
    et = hugectr.Embedding_t.LocalizedSlotSparseEmbeddingHash if kind == "localized" \
        else hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash
    opt_t = {"adam": hugectr.Optimizer_t.Adam, "sgd": hugectr.Optimizer_t.SGD, "adagrad": hugectr.Optimizer_t.AdaGrad}[optimizer]

    def build(c, w):
        solver = hugectr.CreateSolver(batchsize=b * world, batchsize_eval=b * world, lr=0.05, vvgpu=[list(range(w))],
                                      repeat_dataset=True, i64_input_key=True, use_cuda_graph=False)
        rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.Parquet, source=["synthetic"], eval_source="synthetic",
                                      check_type=hugectr.Check_t.Non, slot_size_array=vocab)
        etc = None
        if w > 1 and os.environ.get("HCTR_TEST_ETC"):
            # the N-rank model keeps its table on the host parameter server (behind the cache / staged)
            ps_t = hugectr.TrainPSType_t.Cached if os.environ["HCTR_TEST_ETC"] == "cached" else hugectr.TrainPSType_t.Staged
            etc = hugectr.CreateETC(ps_types=[ps_t], sparse_models=[""], host_capacity_rows=4096)
        upd = {"global": hugectr.Update_t.Global, "lazy": hugectr.Update_t.LazyGlobal}.get(
            os.environ.get("HCTR_TEST_UPDATE", ""), hugectr.Update_t.Local)
        m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(opt_t, upd), etc, comm=c)
        m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                            data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("data1", H, H == 1, S)]))
        m.add(hugectr.SparseEmbedding(et, 1, vec, comb, "emb", "data1", slot_size_array=vocab))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["emb"], ["r"], leading_dim=S * vec))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["r", "dense"], ["c"]))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
        m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
        m.compile()
        return m
    m = build(comm, world)
    if world > 1 and os.environ.get("HCTR_TEST_ETC"):
        assert type(m.legacy_train[0]).__name__ == "CachedSparseEmbeddingRuntime", type(m.legacy_train[0])
    ref = build(Comm.single(comm.device), 1) if rank == 0 else None
    # identical start: every key of every slot with a known vector, identical dense weights
    gen = torch.Generator().manual_seed(int(seed) + 1)
    allk = torch.cat([torch.arange(vocab[s]) + int(offs[s]) for s in range(S)])
    allv = torch.randn(allk.numel(), vec, generator=gen) * 0.1
    slot_of = torch.cat([torch.full((vocab[s],), s) for s in range(S)])
    d = comm.all_gather_object(tempfile.mkdtemp() if rank == 0 else None)[0]
    if rank == 0:
        sm = os.path.join(d, "init")
        os.makedirs(sm, exist_ok=True)
        allk.numpy().astype("<i8").tofile(os.path.join(sm, "key"))
        allv.numpy().astype("<f4").tofile(os.path.join(sm, "emb_vector"))
        if kind == "localized":
            slot_of.numpy().astype("<u8").tofile(os.path.join(sm, "slot_id"))
    comm.barrier()
    m.load_sparse_weights([os.path.join(d, "init")])
    w0 = m.arena.weights.clone()
    comm.broadcast(w0, 0)
    m.arena.weights.copy_(w0)
    m.arena.sync_shadow()
    if ref is not None:
        ref.load_sparse_weights([os.path.join(d, "init")])
        ref.arena.weights.copy_(w0)
        ref.arena.sync_shadow()
    for step in range(3):
        lab = torch.randint(0, 2, (b * world, 1), generator=gen).float()
        den = torch.rand(b * world, 2, generator=gen)
        keys = torch.stack([torch.randint(0, vocab[s], (b * world, H), generator=gen) + int(offs[s]) for s in range(S)], 1)
        if H > 1:                                   # shorter bags: padding -1 behind the first n keys
            n = torch.randint(1, H + 1, (b * world, S), generator=gen)
            keys = torch.where(torch.arange(H).view(1, 1, H) < n.unsqueeze(-1), keys, torch.full_like(keys, -1))
        nnz = (keys >= 0).sum(-1).int()             # [B, S]

        def batch(lo, hi):
            k = keys[lo:hi].reshape(-1)
            z = nnz[lo:hi].t().reshape(-1)          # [S, b] layout of the nnz block
            return HostBatch(lab[lo:hi].clone(), den[lo:hi].clone(), k.clone(), z.clone(), hi - lo)
        m.train_on_host_batch(batch(rank * b, (rank + 1) * b))
        if ref is not None:
            ref.train_on_host_batch(batch(0, b * world))
    lm = m.get_current_loss()
    out = os.path.join(d, "out_n")
    m.legacy_train[0].dump_parameters(out)
    if ref is not None:
        lr_ = ref.get_current_loss()
        assert abs(lm - lr_) < 1e-4 * max(1.0, abs(lr_)), (seed, kind, optimizer, lm, lr_)
        err = float((m.arena.weights - ref.arena.weights).abs().max())
        assert err < 1e-4, (seed, kind, optimizer, "dense", err)
        ref.legacy_train[0].dump_parameters(os.path.join(d, "out_1"))
        tabs = []
        for o in ("out_n", "out_1"):
            k = np.fromfile(os.path.join(d, o, "key"), dtype="<i8")
            v = np.fromfile(os.path.join(d, o, "emb_vector"), dtype="<f4").reshape(-1, vec)
            order = np.argsort(k)
            tabs.append((k[order], v[order]))
        assert (tabs[0][0] == tabs[1][0]).all() and len(tabs[0][0]) == allk.numel(), (seed, "key sets differ")
        diff = float(np.abs(tabs[0][1] - tabs[1][1]).max())
        moved = float(np.abs(tabs[1][1] - allv.numpy()[np.argsort(allk.numpy())]).max())
        assert diff < 1e-4 and moved > 1e-6, (seed, kind, optimizer, "table", diff, moved)
    # ---- snapshot written by N ranks, loaded by ONE process (re-sharding + optimizer states matched by key), dumped
    # again: (key -> vector, key -> states) must survive unchanged
    ost = os.path.join(d, "out_n_opt")
    m.legacy_train[0].dump_opt_states(ost)
    comm.barrier()
    if ref is not None:
        fresh = build(Comm.single(comm.device), 1)
        fresh.load_sparse_weights([out])
        fresh.load_sparse_optimizer_states([ost])
        fresh.legacy_train[0].dump_parameters(os.path.join(d, "re"))
        fresh.legacy_train[0].dump_opt_states(os.path.join(d, "re_opt"))

        def by_key(pd, po):
            k = np.fromfile(os.path.join(d, pd, "key"), dtype="<i8")
            v = np.fromfile(os.path.join(d, pd, "emb_vector"), dtype="<f4").reshape(-1, vec)
            st = np.fromfile(os.path.join(d, po), dtype="<f4")
            ns = st.size // max(1, k.size * vec)
            st = st.reshape(ns, k.size, vec) if ns else st.reshape(0, k.size, vec)
            o = np.argsort(k)
            return k[o], v[o], st[:, o]
        a_, b_ = by_key("out_n", "out_n_opt"), by_key("re", "re_opt")
        assert (a_[0] == b_[0]).all() and np.array_equal(a_[1], b_[1]), (seed, "reloaded table differs")
        assert a_[2].shape == b_[2].shape and np.array_equal(a_[2], b_[2]), (seed, "optimizer states scrambled on reload")
        if optimizer != "sgd":
            assert a_[2].shape[0] >= 1 and float(np.abs(a_[2]).max()) > 0, "no optimizer state was written"
    comm.barrier()
    if rank == 0:
        print("LEGACY_EQUIV_OK", seed)


def run_resume(tmpdir, legacy=False, comm=None):
    """multi-rank exact resume: N ranks train 3 steps, snapshot, train 2 more; a fresh N-rank model resumes from the
    snapshot and trains the same 2 steps -- dense weights, embedding tables and the loss must be BIT-identical"""
    import hugectr_b200 as hugectr
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.models.legacy import build_deepfm
    comm = comm or Comm.init_from_env()
    world, rank = comm.world_size, comm.rank

    def mk():
        if legacy:
            m = build_deepfm(batchsize=32 * world, vvgpu=[list(range(world))], slot_sizes=[30, 12, 50, 7], workspace_mb=2,
                             mixed=False, comm=comm, max_eval_batches=1, seed=5)
            for c in m.dense_layers:
                if c.layer_type == hugectr.Layer_t.Dropout:
                    c.dropout_rate = 0.0
        else:
            sizes, hot = [400, 30, 50, 900, 120, 7], [3, 1, 1, 4, 2, 1]
            sm = [[1, 1, 1, 0, 1, 1] for _ in range(world)]
            sm[world - 1][3] = 1
            plan = (sm, [("mp", ["0", "3"]), ("dp", ["1", "2", "4", "5"])])
            m = build_dlrm_dcnv2(batchsize=32 * world, num_gpus=world, table_sizes=sizes, multi_hot=hot, ev_size=8, lr=0.02,
                                 mixed=False, optimizer="adagrad", bottom=(16, 8), top=(16, 1), cross_layers=1,
                                 projection_dim=4, use_cuda_graph=False, shard_plan=plan, comm=comm, seed=5)
        m.compile()
        return m
    a = mk()
    pool = a.reader_train.pool
    for i in range(3):
        a.train_on_host_batch(pool[i % len(pool)])
    pre = os.path.join(tmpdir, "snap")
    a.save_params_to_files(pre, 3)
    comm.barrier()
    for i in range(3, 5):
        a.train_on_host_batch(pool[i % len(pool)])
    b = mk()
    assert b.resume(pre) == 3
    for i in range(3, 5):
        b.train_on_host_batch(pool[i % len(pool)])
    # static tables: bit-identical.  Hash embeddings hand out rows in arrival order, which a reload does not reproduce;
    # reductions over duplicate keys then add in another order -> equal to rounding, not to the bit
    tol = 1e-5 if legacy else 0.0
    err = float((a.arena.weights - b.arena.weights).abs().max())
    assert err <= tol, f"dense weights differ after resume: {err}"
    assert abs(a.get_current_loss() - b.get_current_loss()) <= tol
    if legacy:
        for ra, rb in zip(a.legacy_train, b.legacy_train):
            da, db = os.path.join(tmpdir, f"a_{ra.name}"), os.path.join(tmpdir, f"b_{rb.name}")
            ra.dump_parameters(da)
            rb.dump_parameters(db)
            if rank == 0:
                import numpy as np
                ka, kb = np.fromfile(da + "/key", "<i8"), np.fromfile(db + "/key", "<i8")
                va = np.fromfile(da + "/emb_vector", "<f4").reshape(len(ka), -1)[np.argsort(ka)]
                vb = np.fromfile(db + "/emb_vector", "<f4").reshape(len(kb), -1)[np.argsort(kb)]
                assert np.array_equal(np.sort(ka), np.sort(kb)) and float(np.abs(va - vb).max()) <= 1e-5, \
                    "legacy table differs after resume"
    else:
        for ea, eb in zip(a.ebcs_train, b.ebcs_train):
            for name in ea.tmap:
                for pa_, pb_ in zip(ea.dump_table_local(name), eb.dump_table_local(name)):
                    assert torch.equal(pa_[0], pb_[0]) and torch.equal(pa_[1], pb_[1]), f"table {name} differs after resume"
                    for sa, sb in zip(pa_[3] or [], pb_[3] or []):
                        assert (sa is None and sb is None) or torch.equal(sa, sb), \
                            f"optimizer state of table {name} differs after resume"
    comm.barrier()
    if rank == 0:
        print("RESUME_OK")


def run_ckpt(tmpdir, comm=None):
    """train on N ranks (row-sharded + table-wise + dp tables), save dense + embedding-collection
    checkpoints, load them into a SINGLE-process model (different sharding) and compare weights,
    tables and the loss on the same data (parameter_IO.cpp:262-350 re-sharding on load)"""
    import hugectr_b200 as hugectr
    from hugectr_b200.data.batch import HostBatch
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    comm = comm or Comm.init_from_env()
    world, rank = comm.world_size, comm.rank
    sizes = [4000, 300, 50, 9000, 1200, 77]
    hot = [3, 1, 1, 8, 2, 1]
    b = 64
    kw = dict(table_sizes=sizes, multi_hot=hot, ev_size=16, lr=0.02, mixed=False, optimizer="adagrad",
              bottom=(32, 16), top=(32, 1), cross_layers=1, projection_dim=8, use_cuda_graph=False)
    sm = [[1, 1, 1, 0, 1, 1] for _ in range(world)]
    sm[world - 1][3] = 1
    plan = (sm, [("mp", ["0", "3"]), ("dp", ["1", "2", "4", "5"])])
    m = build_dlrm_dcnv2(batchsize=b * world, num_gpus=world, comm=comm, shard_plan=plan, **kw)
    m.compile()
    for _ in range(4):
        m.train()
    prefix = os.path.join(tmpdir, "ck")
    m.save_params_to_files(prefix, 4)
    m.embedding_dump(os.path.join(tmpdir, "ebc"))
    comm.barrier()
    single = Comm.single(comm.device)
    ref = build_dlrm_dcnv2(batchsize=b * world, num_gpus=1, comm=single, **kw)
    ref.compile()
    ref.load_dense_weights(prefix + "_dense_4.model")
    ref.embedding_load(os.path.join(tmpdir, "ebc"))
    err = float((ref.arena.weights - m.arena.weights).abs().max())
    assert err == 0.0, f"dense weights differ after load: {err}"
    for e_ref, e in zip(ref.ebcs_train, m.ebcs_train):
        for name in list(e_ref.tmap.keys()):
            ev = e_ref.tmap[name].ev_size
            rk, rv = None, None
            for keys, vals, col0, _, _ in e_ref.dump_table_local(name):
                rk, rv = keys.cpu(), vals[:, :ev].cpu()
            for keys, vals, col0, _, _ in e.dump_table_local(name):
                if len(keys):
                    idx = torch.searchsorted(rk, keys.cpu())
                    assert float((rv[idx] - vals[:, :ev].cpu()).abs().max()) == 0.0, f"table {name}"
    # same data -> same loss (eval forward of the global batch vs the ranks' shards)
    pool = m.reader_train.pool
    hb = pool[0]
    allb = comm.all_gather_object((hb.label.clone(), hb.dense.clone(), hb.keys.clone()))
    keys, off = [], 0
    for (_, S, H, _) in m.layout.blocks:
        n = b * S * H
        keys.append(torch.cat([x[2][off:off + n] for x in allb]))
        off += n
    big = HostBatch(torch.cat([x[0] for x in allb]), torch.cat([x[1] for x in allb]), torch.cat(keys),
                    None, b * world)
    m.train_on_host_batch(hb)
    ref.train_on_host_batch(big)
    l_m, l_r = m.get_current_loss(), ref.get_current_loss()
    assert abs(l_m - l_r) < 1e-4 * max(1.0, abs(l_r)), (l_m, l_r)
    comm.barrier()
    if rank == 0:
        print("CKPT_OK", l_m, l_r)


def run_unique(names="0,2", opt_name="adagrad", fused=False, comm=None):
    """collective path with some tables on the Unique exchange (distinct keys travel once, rows return once per
    distinct key, owners de-duplicate across requesters) against a single-process collection"""
    c = comm or Comm.init_from_env()
    world, device = c.world_size, c.device
    unique_names = [x for x in str(names).split(",") if x]
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import CompressionStrategy, Optimizer_t
    from hugectr_b200.solver import CreateOptimizer
    b, ev = 6, 8
    sizes = [40, 1000, 64, 300, 17, 90]
    hot = [5, 3, 4, 2, 1, 6]
    comb = ["sum", "mean", "concat", "sum", "sum", "mean"]
    n = len(sizes)
    # table 0: row-sharded over ranks {0, 1}; 1, 2, 3, 5: table-wise; 4: data parallel
    sm = [[0] * n for _ in range(world)]
    sm[0][0] = sm[1 % world][0] = 1
    for i in (1, 2, 3, 5):
        sm[i % world][i] = 1
    for g in range(world):
        sm[g][4] = 1
    strat = [("mp", ["0", "1", "2", "3", "5"]), ("dp", ["4"])]

    def cfg_for(sharded):
        cfg = EmbeddingCollectionConfig()
        cfg.embedding_lookup([EmbeddingTableConfig(str(i), sizes[i], ev) for i in range(n)],
                             [f"d{i}" for i in range(n)], "emb", comb)
        if sharded:
            cfg.shard(sm, strat, compression_strategy={CompressionStrategy.Unique: list(unique_names),
                                                       CompressionStrategy.Reduction: []})
        return cfg
    gen = torch.Generator().manual_seed(3)
    full = {str(i): torch.randn(sizes[i], ev, generator=gen) * 0.1 for i in range(n)}
    keys = [torch.randint(0, max(2, sizes[i] // 3), (b * world, hot[i]), generator=gen) for i in range(n)]
    keys[1][::3, -1] = -1                               # short bags (mean over the actual bag)
    keys[5][1::4, 2:] = -1
    width = sum(ev * (hot[i] if comb[i] == "concat" else 1) for i in range(n))
    grad = torch.randn(b * world, width, generator=gen) * 0.1
    kind = {"adagrad": Optimizer_t.AdaGrad, "sgd": Optimizer_t.SGD, "adam": Optimizer_t.Adam}[opt_name]
    opt = CreateOptimizer(kind, **({"initial_accu_value": 0.1, "epsilon": 1e-6} if opt_name == "adagrad" else {}))
    hotd = {f"d{i}": hot[i] for i in range(n)}
    cpu = torch.device("cpu")
    ref = EmbeddingCollection(cfg_for(False), b * world, hotd, cpu, torch.float32, Comm.single(cpu), opt, seed=1)
    for nm, w in full.items():
        ref.load_table_rows(nm, torch.arange(w.shape[0]), w)
    lr, st = torch.tensor([0.05]), torch.tensor([1], dtype=torch.int32)
    steps = 2
    ref_out = []
    for it in range(steps):
        ref.set_keys(torch.cat([k.roll(it, 0).reshape(-1) for k in keys]).int())
        ref.forward()
        ref_out.append(ref.top_data["emb"].clone())
        ref.top_grad["emb"].copy_(grad)
        ref.backward(lr, st + it)
    e = EmbeddingCollection(cfg_for(True), b, hotd, device, torch.float32, c, opt, seed=1, fused=fused)
    uq = {gl["table"] for gl in e.glookups if gl.get("unique")}
    assert uq == (set(unique_names) if not fused else set()), uq
    for nm, w in full.items():
        e.load_table_rows(nm, torch.arange(w.shape[0]), w)
    r = c.rank
    for it in range(steps):
        e.set_keys(torch.cat([k.roll(it, 0)[r * b:(r + 1) * b].reshape(-1) for k in keys]).int().to(device))
        e.forward()
        err = (e.top_data["emb"].float().cpu() - ref_out[it][r * b:(r + 1) * b]).abs().max().item()
        assert err < 1e-5, ("forward", it, r, err)
        if e._uniq is not None and it == 0:
            sent, _ = e._uniq.wire_elems()
            total = sum(b * hot[int(t)] for t in unique_names)
            assert 0 < sent < total, (sent, total)        # repeated ids: fewer codes than key slots
        e.top_grad["emb"].copy_(grad[r * b:(r + 1) * b].to(device))
        e.backward(lr.to(device), (st + it).to(device))
    for nm in full:
        rk, rw = ref.dump_table_local(nm)[0][:2]
        for (k, w, c0, sts, kind_) in e.dump_table_local(nm):
            if len(k):
                d = (w - rw[k][:, c0:c0 + w.shape[1]]).abs().max().item()
                assert d < 2e-5, ("table", nm, r, d)
    dsync(c)
    c.barrier()
    if c.rank == 0:
        print("UNIQUE_OK", flush=True)


def dispatch(what, a):
    """one worker mode with its positional arguments (strings)"""
    if what == "unique":
        run_unique(a[0], a[1] if len(a) > 1 else "adagrad")
    elif what == "ckpt":
        run_ckpt(a[0])
    elif what == "dynamic":
        run_dynamic()
    elif what == "sok":
        run_sok()
    elif what == "sok_fuzz":
        for sd in a[0].split(","):
            run_sok_fuzz(sd)
    elif what == "ebcio":
        for sd in a[1].split(","):
            d = os.path.join(a[0], sd)
            os.makedirs(d, exist_ok=True)
            run_ebcio(d, sd)
    elif what == "symmfail":
        run_symmfail()
    elif what == "fuzz":
        for sd in a[0].split(","):
            run_fuzz(sd)
    elif what == "legacy":
        run_legacy()
    elif what == "resume":
        run_resume(a[0], a[1] == "legacy")
    elif what == "legacy_equiv":
        for sd in a[2].split(","):
            run_legacy_equiv(a[0], a[1], sd)
    elif what == "equiv":
        run_equiv(a[0] if a else "sgd", int(a[1]) if len(a) > 1 else 0)
    elif what == "model":
        run_model()
    elif what == "ebc":
        run_ebc(a[0], {"fused": True, "collective": False}[a[1]])
    elif what == "allreduce":
        run_allreduce()
    else:
        raise SystemExit(f"unknown worker mode {what}")


if __name__ == "__main__":
    if sys.argv[1] == "multi":
        # several modes in ONE process group (interpreter start-up dominates a gloo test): "mode;arg;arg" each;
        # a failing mode stops the session, the markers printed so far tell which ones passed
        for spec in sys.argv[2:]:
            parts = spec.split(";")
            dispatch(parts[0], parts[1:])
            if int(os.environ.get("RANK", "0")) == 0:
                print("MULTI_DONE", spec, flush=True)
    else:
        dispatch(sys.argv[1], sys.argv[2:])
    if dist.is_initialized():
        dist.destroy_process_group()
