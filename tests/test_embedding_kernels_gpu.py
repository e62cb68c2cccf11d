"""Model-parallel embedding kernels against an fp64 oracle: the lookup (emb_fwd_kernel), the fused
backward (index + counting sort + light / medium / heavy classification + reduce + optimizer,
csrc/embedding_bwd.cu) and the accumulate + update path, at their row-class, width and capacity edges.

The oracle is written from the definition of the operation, not from the package's CPU path:
  * a (source, lookup, sample, h) pair contributes when h < min(nnz, hotness), key >= 0,
    key % shards == shard and key // shards < rows; its gradient row is scaled by 1/nnz for mean
    and by grad_scale, and summed per distinct arena row in float64;
  * the optimizer is ``ops.sparse_opt_reference`` on float64 copies (test_optim_cpu.py pins it to
    torch.optim and the FTRL closed form); it divides by hp["scaler"] itself.

Error bounds (stated once, used everywhere): the kernels add a row's n gradient rows in fp32 in any
order -- the heavy-row kernel with atomics -- so their sum lies within E = (n + 4) u sum|g| of the
exact one (u = 2^-24; the n u summation bound plus the fp32 scale factors).  E is carried through
the optimizer by evaluating the oracle at G - E and G + E; 16 u of the magnitudes of the old and
new values covers the fp32 evaluation of the update formula.  Updates are compared as w_new - w_old.
A bf16 state is stored rounded to nearest even (pack_bf16x2 / __float2bfloat16 round to nearest)
from an fp32 value, so it may differ from the rounded fp64 value by one bf16 ulp.  Rows that no pair
touches must not change at all.
"""
import pytest
import torch

from hugectr_b200.data.batch import power_law_keys
from hugectr_b200.embedding import ops as E
from hugectr_b200.enums import Optimizer_t as O

U = 2.0 ** -24
OPTS = [O.SGD, O.AdaGrad, O.Adam, O.Ftrl, O.MomentumSGD, O.Nesterov, O.RMSProp]
# non-default hyper-parameters; FTRL with lambda1 > 0 so that the shrinkage branch is exercised
HP = dict(scaler=1.0, beta1=0.875, beta2=0.9375, epsilon=2.0 ** -20, lambda1=0.015625, lambda2=0.125,
          ftrl_beta=0.5, momentum=0.9)
LR = 0.0625


def n_states(opt):
    return {O.SGD: 0, O.Adam: 2, O.Ftrl: 2}.get(opt, 1)


# ------------------------------------------------------------------------------------------ cases
class Case:
    """Lookups of ``batch`` samples from R source buffers (flat CPU tensors: keys, gradient rows in
    their final dtype, optional nnz) into one arena of ``rows`` rows of width ``pitch``."""

    def __init__(self, lookups, pitch, batch, keys, grads, nnz=None):
        self.lookups, self.pitch, self.batch = lookups, pitch, batch
        self.keys, self.grads, self.nnz = keys, grads, nnz
        po = 0
        for lk in lookups:
            lk.pair_off = po
            po += len(keys) * batch * lk.hotness
        self.pairs = po
        self.rows = max(lk.table_row_off + lk.rows for lk in lookups)
        self.mean = any(lk.combiner == 1 for lk in lookups)


def lookup(row_off, rows, key_off, goff, hot, stride, ev, comb=0, ns=1, shard=0, nnz_off=-1):
    return E.LookupDesc(table_row_off=row_off, key_off=key_off, out_off=goff, grad_off=goff, hotness=hot,
                        key_stride=hot, num_shards=ns, shard_idx=shard, out_stride=stride,
                        grad_stride=stride, combiner=comb, ev_size=ev, rows=rows, nnz_off=nnz_off)


def single_case(keys, batch, hot, pitch, rows, gdt, gen):
    """one sum lookup of [batch, hot] keys, gradient rows [batch, pitch]"""
    grads = (torch.randn(batch * pitch, generator=gen) * 0.1).to(gdt)
    return Case([lookup(0, rows, 0, 0, hot, pitch, pitch)], pitch, batch, [keys], [grads])


# occurrences per row: around the light (<= 4), medium (<= 64) and heavy (> 64, 512-entry chunks)
# thresholds, and three chunks with a partial last one
CLASS_COUNTS = [1] * 40 + [2, 3, 4] * 4 + [4, 5] * 3 + [64, 65] * 3 + [512, 513, 1025]


def class_keys(batch, hot, rows, gen, counts=CLASS_COUNTS):
    """keys where distinct random rows occur exactly ``counts`` times, scattered over all positions
    (so one row's pairs fall into several 1024-pair index blocks); the rest is padding (-1)"""
    ids = torch.randperm(rows, generator=gen)[:len(counts)]
    occ = torch.cat([ids[i].repeat(c) for i, c in enumerate(counts)])
    flat = torch.full((batch * hot,), -1, dtype=torch.int64)
    flat[torch.randperm(batch * hot, generator=gen)[:occ.numel()]] = occ
    return flat


def features_case(pitch, gdt, gen, batch=300):
    """four lookups, two source buffers, one launch: sum and mean with variable nnz (0 and above the
    hotness included), padding keys and keys >= rows, a row-sharded lookup (shard 2 of 3) and a
    fixed-hotness mean lookup"""
    specs = [  # rows, hotness, combiner, shards, variable nnz, key range
        (700, 5, 0, 1, True, 800), (300, 7, 1, 1, True, 360), (500, 4, 0, 3, False, 1650),
        (50, 3, 1, 1, False, 60)]
    lookups, roff, koff, nslot = [], 0, 0, 0
    width = pitch * len(specs)
    for i, (rows, hot, comb, ns, var, _) in enumerate(specs):
        lookups.append(lookup(roff, rows, koff, i * pitch, hot, width, pitch, comb, ns, ns - 1,
                              nslot * batch if var else -1))
        roff += rows
        koff += batch * hot
        nslot += var
    keys, grads, nnz = [], [], []
    for _ in range(2):
        keys.append(torch.cat([torch.randint(-1, kr, (batch * h,), generator=gen)
                               for _, h, _, _, _, kr in specs]))
        grads.append((torch.randn(batch * width, generator=gen) * 0.1).to(gdt))
        nnz.append(torch.randint(0, 10, (nslot * batch,), generator=gen, dtype=torch.int32))
    return Case(lookups, pitch, batch, keys, grads, nnz)


# ------------------------------------------------------------------------------------------ oracle
def _bags(case, src, lk):
    """(owned [B, H], local row [B, H], clamped nnz [B]) of one lookup of one source"""
    B, H = case.batch, lk.hotness
    k = case.keys[src].long().as_strided((B, H), (lk.key_stride, 1), lk.key_off)
    nnz = torch.full((B,), H, dtype=torch.long)
    if lk.nnz_off >= 0:
        nnz = case.nnz[src].long()[lk.nnz_off:lk.nnz_off + B].clamp(max=H)
    own = (torch.arange(H).view(1, -1) < nnz.view(-1, 1)) & (k >= 0)
    r = k
    if lk.num_shards > 1:
        own &= (k % lk.num_shards) == lk.shard_idx
        r = torch.div(k, lk.num_shards, rounding_mode="floor")
    own &= r < lk.rows
    return own, torch.where(own, r, torch.zeros_like(r)), nnz


def oracle_reduce(case, grad_scale=1.0):
    """distinct arena rows, their fp64 gradient sums G, sums of magnitudes A and occurrence counts"""
    rows_l, g_l = [], []
    for src in range(len(case.keys)):
        gbuf = case.grads[src].double()
        for lk in case.lookups:
            own, r, nnz = _bags(case, src, lk)
            g = gbuf.as_strided((case.batch, lk.ev_size), (lk.grad_stride, 1), lk.grad_off) * grad_scale
            if lk.combiner == 1:
                g = g / nnz.clamp(min=1).view(-1, 1)
            g = torch.nn.functional.pad(g, (0, case.pitch - lk.ev_size))
            b_i, h_i = own.nonzero(as_tuple=True)
            rows_l.append(lk.table_row_off + r[b_i, h_i])
            g_l.append(g[b_i])
    rows, g = torch.cat(rows_l), torch.cat(g_l)
    uniq, inv = torch.unique(rows, return_inverse=True)
    G = torch.zeros(uniq.numel(), case.pitch, dtype=torch.float64).index_add_(0, inv, g)
    A = torch.zeros_like(G).index_add_(0, inv, g.abs())
    return uniq, G, A, torch.bincount(inv, minlength=uniq.numel())


def oracle_update(opt, hp, lr, step, tab, s0, s1, red, exact_sums=False):
    """expected (w, s0, s1) of the updated rows in fp64 and their error bounds (module docstring).
    ``exact_sums``: every partial gradient sum is representable in fp32 (small multiples of a power
    of two), so the kernels' sums are exact whatever their order and only the optimizer rounds"""
    uniq, G, A, n = red
    P = G.shape[1]
    old = [None if x is None else x.view(-1, P)[uniq].double() for x in (tab, s0, s1)]

    def run(g):
        v = [None if x is None else x.clone() for x in old]
        E.sparse_opt_reference(opt, v[0], v[1], v[2], g, hp, lr, step)
        return v

    err = torch.zeros_like(A) if exact_sums else (n.view(-1, 1) + 4).double() * U * A
    ref, lo, hi = run(G), run(G - err), run(G + err)
    tol = [None if r is None else
           torch.maximum((a - r).abs(), (b - r).abs()) + 16 * U * (o.abs() + r.abs())
           for r, a, b, o in zip(ref, lo, hi, old)]
    if opt == O.Ftrl:
        # z_new = z + g + (sqrt(n + beta) - sqrt(n_new + beta)) w / lr cancels: its rounding is
        # relative to the terms, not to the result; w_new = (+-lambda1 - z_new) / q inherits it
        fb = hp["ftrl_beta"]
        mag = old[1].abs() + (G / hp["scaler"]).abs() + \
            ((old[2] + fb).sqrt() + (ref[2] + fb).sqrt()) * old[0].abs() / lr
        tol[1] += 16 * U * mag
        tol[0] += 16 * U * mag / ((ref[2] + fb).sqrt() / lr + hp["lambda2"])
    return uniq, old, ref, tol


def bf16_ulp(x):
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -100))
    return torch.ldexp(torch.ones_like(x), e.to(torch.int32) - 8)


def assert_close_bound(what, got, ref, tol, bf16=False):
    got = got.double()
    if bf16:
        tol = tol + bf16_ulp(ref)
    bad = (got - ref).abs() > tol
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; "
                             f"first at {i}: got {got[tuple(i)].item()!r} expected {ref[tuple(i)].item()!r} "
                             f"bound {tol[tuple(i)].item()!r}")


def init_state(opt, rows, pitch, sdt, gen):
    """fp32 weights and optimizer state as after some training: positive second moments, and state
    rounded to its storage type before use"""
    tab = torch.randn(rows * pitch, generator=gen) * 0.1
    ns = n_states(opt)
    s = [None, None]
    for j in range(ns):
        r = torch.rand(rows * pitch, generator=gen)
        if opt == O.Adam:
            v = torch.randn(rows * pitch, generator=gen) * 0.01 if j == 0 else r * 1e-2 + 1e-4
        elif opt == O.Ftrl:
            v = torch.randn(rows * pitch, generator=gen) if j == 0 else r + 0.01
        elif opt in (O.MomentumSGD, O.Nesterov):
            v = torch.randn(rows * pitch, generator=gen) * 0.01
        else:   # AdaGrad accumulator, RMSProp second moment
            v = r * 0.5 + 0.01
        s[j] = v.to(sdt)
    return tab, s[0], s[1]


def check_update(what, case, opt, tab, s0, s1, new, hp=HP, lr=LR, step=1, grad_scale=1.0,
                 exact_sums=False):
    """compare the kernels' (w, s0, s1) = ``new`` with the oracle; returns nothing"""
    uniq, old, ref, tol = oracle_update(opt, hp, lr, step, tab, s0, s1, oracle_reduce(case, grad_scale),
                                        exact_sums)
    P = case.pitch
    for j, (name, before, after) in enumerate(zip(("w", "s0", "s1"), (tab, s0, s1), new)):
        if before is None:
            continue
        after = after.cpu()
        bf = after.dtype == torch.bfloat16
        if j == 0:   # the update, w_new - w_old
            assert_close_bound(f"{what} dw", after.view(-1, P)[uniq].double() - old[0], ref[0] - old[0], tol[0])
        else:
            assert_close_bound(f"{what} {name}", after.view(-1, P)[uniq], ref[j], tol[j], bf16=bf)
        keep = torch.ones(after.numel() // P, dtype=torch.bool)
        keep[uniq] = False
        assert torch.equal(after.view(-1, P)[keep], before.view(-1, P)[keep]), f"{what}: untouched {name} rows changed"


# ------------------------------------------------------------------------------------------ device runs
def _dev(case, key_dtype):
    dev = torch.device("cuda")
    keys = [k.to(key_dtype).to(dev) for k in case.keys]
    grads = [g.to(dev) for g in case.grads]
    nnz = [n.to(dev) for n in case.nnz] if case.nnz is not None else None
    return keys, grads, nnz


def run_step(case, opt, tab, s0, s1, path="fused", key_dtype=torch.int32, hp=HP, lr=LR, step=1,
             grad_scale=1.0, ws=None, dev_state=None, **ws_kw):
    """one backward step on the GPU; returns ((w, s0, s1) on the device, workspace)"""
    dev = torch.device("cuda")
    t, a, b = dev_state if dev_state is not None else \
        [None if x is None else x.to(dev) for x in (tab, s0, s1)]
    keys, grads, nnz = _dev(case, key_dtype)
    ld = E.lookups_to_device(case.lookups, dev)
    lr_t = torch.tensor([lr], device=dev)
    st_t = torch.tensor([step], dtype=torch.int32, device=dev)
    if path == "fused":
        if ws is None:
            ws = E.UniqueWorkspace(case.pairs, case.pitch, dev, indexed=True, need_scale=case.mean, **ws_kw)
        E.bwd_index(case.lookups, ld, t, case.pitch, keys, case.batch, ws, nnz_bufs=nnz)
        E.bwd_reduce_update(opt, case.lookups, ld, t, a, b, case.pitch, keys, grads, case.batch, ws, hp,
                            lr_t, st_t, grad_scale=grad_scale, nnz_bufs=nnz)
    else:
        if ws is None:
            ws = E.UniqueWorkspace(case.pairs, case.pitch, dev)
        E.backward_accum(case.lookups, ld, t, case.pitch, keys, grads, case.batch, ws, grad_scale,
                         nnz_bufs=nnz)
        E.update(opt, t, a, b, case.pitch, ws, hp, lr_t, st_t)
    torch.cuda.synchronize()
    return (t, a, b), ws


def assert_ws_clean(ws):
    """a step leaves the transient hash empty and the heavy-row scratch / tickets zeroed"""
    assert bool((ws.keys == -1).all()) and bool((ws.vals == -1).all()), "hash slots left occupied"
    assert int(ws.counter.item()) == 0
    assert int(ws.overflow.item()) == 0
    if ws.indexed:
        assert int(ws.heavy_ticket.abs().sum().item()) == 0, "heavy tickets not reset"
        assert int((ws.heavy_scratch != 0).sum().item()) == 0, "heavy scratch rows not reset"


def fused_check(what, case, opt, sdt=torch.float32, gen=None, exact_sums=False, **kw):
    """one step from a fresh workspace, compared with the oracle; the workspace must end clean"""
    tab, s0, s1 = init_state(opt, case.rows, case.pitch, sdt, gen)
    new, ws = run_step(case, opt, tab, s0, s1, **kw)
    check_update(what, case, opt, tab, s0, s1, new, hp=kw.get("hp", HP), step=kw.get("step", 1),
                 grad_scale=kw.get("grad_scale", 1.0), exact_sums=exact_sums)
    assert_ws_clean(ws)
    return ws


# ========================================================================================== CPU tests
@pytest.mark.parametrize("opt", OPTS)
def test_oracle_matches_package_cpu_path(opt):
    """the fp64 oracle and the package's CPU path (backward_accum + update) agree on a small case
    with every lookup feature, so the oracle can be trusted before it judges a kernel"""
    gen = torch.Generator().manual_seed(1)
    case = features_case(8, torch.float32, gen, batch=40)
    tab, s0, s1 = init_state(opt, case.rows, case.pitch, torch.float32, gen)
    hp = dict(HP, scaler=4.0)
    t, a, b = [None if x is None else x.clone() for x in (tab, s0, s1)]
    ws = E.UniqueWorkspace(case.pairs, case.pitch, torch.device("cpu"))
    E.backward_accum(case.lookups, None, t, case.pitch, case.keys, case.grads, case.batch, ws, 0.5,
                     nnz_bufs=case.nnz)
    E.update(opt, t, a, b, case.pitch, ws, hp, torch.tensor([LR]), torch.tensor([7], dtype=torch.int32))
    check_update(f"cpu {opt.name}", case, opt, tab, s0, s1, (t, a, b), hp=hp, step=7, grad_scale=0.5)


def test_oracle_rejects_a_wrong_update():
    """the bound is tight enough to see one occurrence of a row dropped or a mis-scaled row"""
    gen = torch.Generator().manual_seed(2)
    case = single_case(class_keys(512, 8, 3000, gen), 512, 8, 16, 3000, torch.float32, gen)
    tab = torch.randn(case.rows * 16, generator=gen)
    uniq, G, A, n = oracle_reduce(case)
    good = tab.clone().view(-1, 16)
    good[uniq] -= (LR * G).float()
    check_update("exact", case, O.SGD, tab, None, None, (good.view(-1), None, None))
    # one of the five occurrences of a medium row missing
    r = uniq[(n == 5).nonzero()[0, 0]]
    s = (case.keys[0].view(-1, 8) == r).any(1).nonzero()[0, 0]
    bad = good.clone()
    bad[r] += LR * case.grads[0].view(-1, 16)[s]
    with pytest.raises(AssertionError, match="outside the bound"):
        check_update("dropped", case, O.SGD, tab, None, None, (bad.view(-1), None, None))
    # every update 0.1 % too large
    bad = good.clone()
    bad[uniq] -= (LR * 1e-3 * G).float()
    with pytest.raises(AssertionError, match="outside the bound"):
        check_update("scaled", case, O.SGD, tab, None, None, (bad.view(-1), None, None))
    # a row that no pair touches changed
    bad = good.clone()
    keep = torch.ones(case.rows, dtype=torch.bool)
    keep[uniq] = False
    bad[keep.nonzero()[0, 0]] += 1e-3
    with pytest.raises(AssertionError, match="untouched"):
        check_update("untouched", case, O.SGD, tab, None, None, (bad.view(-1), None, None))


def _layout_collection(layout, batch):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    t6, t128 = EmbeddingTableConfig("n6", 100, 6), EmbeddingTableConfig("w128", 500, 128)
    if layout == "concat":       # one top [ev-6 | ev-128]: the wide table's columns start at 6 of 134
        cfg.embedding_lookup([t6, t128], ["d0", "d1"], "emb", ["sum", "mean"])
    else:                        # a width-6 top, then another top: at an odd batch it starts at 6 b
        cfg.embedding_lookup([t6], ["d0"], "a", ["sum"])
        cfg.embedding_lookup([t128], ["d1"], "b", ["mean"])
    return lambda dev: EmbeddingCollection(cfg, batch, {"d0": 3, "d1": 2}, dev, torch.float32, Comm(dev),
                                           CreateOptimizer(O.AdaGrad, initial_accu_value=0.1), seed=3)


@pytest.mark.parametrize("layout,batch,aligned", [("concat", 64, False), ("odd_batch", 63, False),
                                                  ("odd_batch", 64, True)])
def test_vec4_guard_on_collection_layouts(layout, batch, aligned):
    """the group of the ev-128 table may use the fused backward (and the vector lookup stores) only
    when its columns in the top are 4-element aligned"""
    from hugectr_b200.embedding.collection import fused_backward_ok
    e = _layout_collection(layout, batch)(torch.device("cpu"))
    grp = [g for g in e.groups if g.pitch == 128][0]
    assert E.vec4_aligned(grp.lookups, grp.pitch) == aligned
    assert E.vec4_aligned(grp.lookups, grp.pitch, grad=False) == aligned
    assert fused_backward_ok(grp) == aligned
    narrow = [g for g in e.groups if g.pitch == 6][0]
    assert not fused_backward_ok(narrow)


def test_width_limit_is_a_clear_error():
    E.check_ev_size(E.MAX_EV_SIZE)
    with pytest.raises(ValueError, match="exceeds"):
        E.check_ev_size(E.MAX_EV_SIZE + 4)


# ========================================================================================== GPU tests
WIDTHS = [4, 16, 124, 128, 132, 512, 516, 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", WIDTHS)
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("opt", [O.SGD, O.AdaGrad])
def test_fused_row_classes_and_widths(pitch, gdt, opt):
    """rows occurring 1..4 | 5..64 | 65, 512, 513, 1025 times (light, medium, heavy with 1-3 chunks)
    at every width class of the fused kernels (G = 8 up to 128, G = 32 above, 1-2 passes of four
    chunks)"""
    gen = torch.Generator().manual_seed(pitch)
    case = single_case(class_keys(512, 8, 4000, gen), 512, 8, pitch, 4000, gdt, gen)
    fused_check(f"classes ev={pitch}", case, opt, gen=gen)


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", [128, 132])
def test_fused_power_law_batch(pitch):
    """one batch from the data generator's power-law sampler (alpha 1.1): a heavy head, a long tail"""
    gen = torch.Generator().manual_seed(0)
    keys = power_law_keys(2048 * 16, 20000, 1.1, gen)
    case = single_case(keys, 2048, 16, pitch, 20000, torch.bfloat16, gen)
    uniq, _, _, n = oracle_reduce(case)
    assert int((n > 64).sum()) >= 3 and int((n > 512).sum()) >= 1
    fused_check(f"power law ev={pitch}", case, O.AdaGrad, gen=gen)


OPT_STEPS = [(o, 1) for o in OPTS] + [(O.Adam, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", [128, 516])
@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("opt,step", OPT_STEPS, ids=[f"{o.name}-t{s}" for o, s in OPT_STEPS])
def test_fused_optimizers(opt, step, sdt, pitch):
    """all seven optimizers, fp32 and bf16 state, in the light, medium and heavy kernels; Adam reads its
    bias-correction step from the device step tensor"""
    gen = torch.Generator().manual_seed(11 + step)
    case = single_case(class_keys(512, 8, 3000, gen), 512, 8, pitch, 3000, torch.bfloat16, gen)
    fused_check(f"{opt.name} {sdt} ev={pitch}", case, opt, sdt=sdt, gen=gen, step=step)


FEATURE_RUNS = [("fused", 128), ("fused", 516), ("accum", 1), ("accum", 6), ("accum", 11),
                ("accum", 128), ("accum", 258)]


@pytest.mark.gpu
@pytest.mark.parametrize("key_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("path,pitch", FEATURE_RUNS)
def test_lookup_features_in_one_launch(path, pitch, key_dtype):
    """sum / mean with variable nnz, padding keys, keys >= rows, a row-sharded lookup, two source
    buffers, int32 / int64 keys, grad_scale and loss scaler != 1 -- fused and accumulate + update"""
    gen = torch.Generator().manual_seed(pitch)
    gdt = torch.bfloat16 if key_dtype == torch.int64 and pitch % 4 == 0 else torch.float32
    case = features_case(pitch, gdt, gen)
    hp = dict(HP, scaler=4.0)
    fused_check(f"{path} ev={pitch}", case, O.AdaGrad, gen=gen, path=path, key_dtype=key_dtype, hp=hp,
                grad_scale=0.5)


def oracle_forward(case, tab, out_elems):
    """pooled outputs in fp64 (layout of the gradient rows), their bounds and the written mask"""
    R, P = len(case.keys), case.pitch
    tab64 = tab.double().view(-1, P)
    ref = torch.zeros(R, out_elems, dtype=torch.float64)
    tol = torch.zeros_like(ref)
    hit = torch.zeros(R, out_elems, dtype=torch.bool)
    for src in range(R):
        for lk in case.lookups:
            own, r, nnz = _bags(case, src, lk)
            v = tab64[lk.table_row_off + r][..., :lk.ev_size] * own.unsqueeze(-1)
            pooled, mag = v.sum(1), v.abs().sum(1)
            if lk.combiner == 1:
                pooled, mag = pooled / nnz.clamp(min=1).view(-1, 1), mag / nnz.clamp(min=1).view(-1, 1)
            view = lambda x: x[src].as_strided((case.batch, lk.ev_size), (lk.out_stride, 1),
                                               src * out_elems + lk.out_off)
            view(ref).copy_(pooled)
            view(tol).copy_((lk.hotness + 2) * U * mag)
            view(hit).fill_(True)
    return ref, tol, hit


@pytest.mark.gpu
@pytest.mark.parametrize("odt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("pitch", [1, 3, 6, 11, 64, 128, 132, 256, 258, 1023, 1024])
def test_forward_widths(pitch, odt):
    """emb_fwd_kernel at the scalar (VEC = 1) widths, the narrow U = 4 launch (64..128), wide rows, and
    scalar rows past 256 columns, which take passes of 256 columns (258: two, 1023: four); outside
    the lookups' columns the output stays untouched"""
    gen = torch.Generator().manual_seed(pitch)
    case = features_case(pitch, torch.float32, gen, batch=257)
    tab = torch.randn(case.rows * pitch, generator=gen)
    n = case.grads[0].numel()
    ref, tol, hit = oracle_forward(case, tab, n)
    dev = torch.device("cuda")
    keys, _, nnz = _dev(case, torch.int64 if pitch % 2 else torch.int32)
    outs = [torch.full((n,), 7.0, dtype=odt, device=dev) for _ in keys]
    E.forward(case.lookups, E.lookups_to_device(case.lookups, dev), tab.to(dev), pitch, keys, outs,
              case.batch, nnz_bufs=nnz)
    got = torch.stack([o.cpu() for o in outs])
    assert_close_bound(f"forward ev={pitch}", got[hit], ref[hit], tol[hit], bf16=odt == torch.bfloat16)
    assert bool((got[~hit] == 7.0).all())


@pytest.mark.gpu
def test_width_past_limit_is_rejected():
    """1028 columns: the lookup, the fused backward and the accumulate path refuse instead of
    truncating the row at 1024"""
    gen = torch.Generator().manual_seed(0)
    case = single_case(torch.randint(0, 50, (64 * 2,), generator=gen), 64, 2, 1028, 50, torch.float32, gen)
    dev = torch.device("cuda")
    keys, grads, _ = _dev(case, torch.int32)
    tab = torch.zeros(50 * 1028, device=dev)
    ld = E.lookups_to_device(case.lookups, dev)
    with pytest.raises(ValueError, match="exceeds"):
        E.forward(case.lookups, ld, tab, 1028, keys, [torch.zeros_like(grads[0])], 64)
    with pytest.raises(ValueError, match="exceeds"):
        run_step(case, O.SGD, tab.cpu(), None, None, path="fused")
    with pytest.raises(ValueError, match="exceeds"):
        run_step(case, O.SGD, tab.cpu(), None, None, path="accum")


@pytest.mark.gpu
def test_workspace_reuse_and_small_heavy_caps():
    """three steps on one workspace with tiny heavy caps (4 scratch rows, 4 chunk items) and a
    different heavy set each step: every row is updated exactly once and the workspace is clean
    after each step.
      step 0: four 1-chunk heavy rows fill all four items with valid entries;
      step 1: three 3-chunk rows reserve items 0-2, 3-5 and 6-8: the second row fits only partly,
              its in-range item 3 (holding a valid entry of step 0) must be marked invalid and
              skipped, and the second and third row fall back to the warp-per-row kernel;
      step 2: eight heavy rows of 1-3 chunks for four scratch rows."""
    gen = torch.Generator().manual_seed(4)
    light = [5, 3, 1, 1, 64, 2]
    steps = [[70, 65, 100, 66] + light, [1025, 1100, 1500] + light,
             [70, 65, 600, 1025, 513, 100, 66, 300] + light]
    pitch = 128
    tab, s0, s1 = init_state(O.AdaGrad, 3000, pitch, torch.float32, gen)
    ws, state = None, None
    for it, counts in enumerate(steps):
        case = single_case(class_keys(512, 16, 3000, gen, counts), 512, 16, pitch, 3000, torch.float32, gen)
        state, ws = run_step(case, O.AdaGrad, tab, s0, s1, ws=ws, dev_state=state, max_heavy_rows=4,
                             max_heavy_items=4)
        check_update(f"step {it}", case, O.AdaGrad, tab, s0, s1, state)
        assert_ws_clean(ws)
        items_uid = ws.heavy_items.view(-1, 2)[:, 0].cpu()
        if it == 0:
            assert int(ws.heavy_count.item()) == 4 and bool((items_uid >= 0).all())
        elif it == 1:
            assert int(ws.heavy_count.item()) == 9 > ws.max_heavy_items   # the item cap overflowed
            assert bool((items_uid[:3] >= 0).all()) and int(items_uid[3]) == -1
        else:
            assert int(ws.heavy_slot.item()) > ws.max_heavy_rows          # the row cap overflowed
        tab, s0, s1 = [None if x is None else x.cpu() for x in state]


@pytest.mark.gpu
def test_more_than_8192_heavy_rows_at_default_sizing():
    """8 310 rows of 65 occurrences each (540 k pairs at ev 16) on a fresh workspace of default
    size: the caps sized from the pair count hold every heavy row (no warp-per-row fallback)"""
    gen = torch.Generator().manual_seed(5)
    nrows, batch, hot = 8310, 4220, 128
    case = single_case(class_keys(batch, hot, 20000, gen, [65] * nrows), batch, hot, 16, 20000,
                       torch.float32, gen)
    ws = fused_check("8310 heavy rows", case, O.SGD, gen=gen)
    assert int(ws.heavy_slot.item()) == nrows <= ws.max_heavy_rows
    assert int(ws.heavy_count.item()) <= ws.max_heavy_items


@pytest.mark.gpu
def test_row_with_more_than_4096_chunks():
    """one row occurring 2.1 M times (over 4 096 chunks of 512, past the 12-bit chunk field) next to
    ordinary rows, ev 4.  The gradients are multiples of 1/16 in [-1/8, 1/8], so every partial sum
    is exact in fp32 and the row's update is checked to the optimizer's rounding"""
    gen = torch.Generator().manual_seed(6)
    batch, hot, pitch = 16500, 128, 4
    keys = torch.full((batch * hot,), 7, dtype=torch.int64)
    keys[torch.randperm(keys.numel(), generator=gen)[:3000]] = torch.randint(8, 900, (3000,), generator=gen)
    grads = torch.randint(-2, 3, (batch * pitch,), generator=gen).float() / 16
    case = Case([lookup(0, 1000, 0, 0, hot, pitch, pitch)], pitch, batch, [keys], [grads])
    assert int((keys == 7).sum()) > 4096 * 512
    fused_check("2.1 M-occurrence row", case, O.SGD, gen=gen, exact_sums=True)


@pytest.mark.gpu
@pytest.mark.parametrize("layout,batch", [("concat", 64), ("odd_batch", 63)])
def test_misaligned_collection_matches_cpu(layout, batch):
    """collections whose ev-128 columns are not 4-aligned in their top run on the scalar lookup and
    accumulate + update paths and match the CPU collection"""
    mk = _layout_collection(layout, batch)
    g, c = mk(torch.device("cuda")), mk(torch.device("cpu"))
    assert not any(getattr(gg, "indexed", False) for gg in g.groups)
    for gg, cg in zip(g.groups, c.groups):
        cg.table.copy_(gg.table.cpu())
    gen = torch.Generator().manual_seed(0)
    keys = torch.cat([torch.randint(0, 100, (batch * 3,), generator=gen),
                      torch.randint(0, 500, (batch * 2,), generator=gen)]).int()
    lr_c, st_c = torch.tensor([0.05]), torch.tensor([1], dtype=torch.int32)
    lr_g, st_g = lr_c.cuda(), st_c.cuda()
    for it in range(2):
        g.set_keys(keys.cuda()); c.set_keys(keys)
        g.forward(); c.forward()
        for name in c.top_data:
            torch.testing.assert_close(g.top_data[name].cpu(), c.top_data[name], rtol=2e-4, atol=2e-4)
            grad = torch.randn(c.top_grad[name].shape, generator=gen) * 0.1
            g.top_grad[name].copy_(grad.cuda()); c.top_grad[name].copy_(grad)
        g.backward(lr_g, st_g); c.backward(lr_c, st_c)
        for gg, cg in zip(g.groups, c.groups):
            torch.testing.assert_close(gg.table.cpu(), cg.table, rtol=1e-3, atol=2e-4)
    g.check_overflow()
