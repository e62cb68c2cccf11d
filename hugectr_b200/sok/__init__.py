"""Sparse Operation Kit, PyTorch flavour.

API parity with ``sparse_operation_kit`` (sparse_operation_kit/sparse_operation_kit/*.py):
``init``, ``Variable`` / ``DistributedVariable`` (row-wise key % N sharding), ``LocalizedVariable``
(whole table on one GPU), ``DynamicVariable`` (hash-backed, unbounded vocabulary; the role of
HKV / DET), ``lookup_sparse`` (lookup.py:425-541), ``all2all_dense_embedding``,
``OptimizerWrapper`` / ``SGD``, ``dump`` / ``load`` / ``incremental_model_dump`` (dump_load.py),
``filter_variables``.  The reference is a TensorFlow plugin that communicates through Horovod
(allgather of keys, alltoall of vectors); here variables are sharded torch tensors, communication is
``torch.distributed`` and the backward is a custom autograd Function that hands *sparse* gradients
(unique rows + reduced grads) to the optimizer wrapper.
"""
from __future__ import annotations

import os
import struct
import time
from typing import List, Optional, Sequence, Union

import numpy as np
import torch

from ..embedding.hashtable import HashTable
from ..ops.optim import opt_reference
from ..enums import Optimizer_t
from ..parallel.comm import Comm

_comm: Optional[Comm] = None
_variables: List["Variable"] = []


def init(comm: Optional[Comm] = None, device: Optional[str] = None):
    """sok.init(): bind to the process group (one process per GPU)."""
    global _comm
    _comm = comm or Comm.init_from_env(device)
    return _comm


def _c() -> Comm:
    if _comm is None:
        init()
    return _comm


def core():
    """the backend-neutral resource view SOK runs on (core.py; reference core::CoreResourceManager)"""
    from ..core import as_core
    return as_core(_c())


def rank(): return core().get_global_gpu_id()
def num_gpus(): return core().get_global_gpu_count()


class Variable:
    """Static-shape embedding variable. mode='distributed': row r lives on rank r % N at local row
    r // N; mode='localized:<gpu>': the whole table lives on one GPU."""

    def __init__(self, initial_value=None, shape=None, dtype=torch.float32, mode: str = "distributed",
                 name: Optional[str] = None, initializer: str = "uniform", trainable: bool = True):
        c = _c()
        self.name = name or f"sok_var_{len(_variables)}"
        self.mode = mode
        self.trainable = trainable
        if initial_value is not None:
            full = torch.as_tensor(initial_value, dtype=dtype)
            shape = tuple(full.shape)
        else:
            full = None
        self.shape = tuple(shape)
        self.vocab, self.dim = self.shape
        self.world, self.rank = c.world_size, c.rank
        self.device = c.device
        if mode.startswith("localized"):
            self.owner = int(mode.split(":")[1]) if ":" in mode else 0
            rows = self.vocab if self.rank == self.owner else 0
            keys = torch.arange(self.vocab)
        else:
            self.owner = -1
            keys = torch.arange(self.rank, self.vocab, self.world)
            rows = keys.numel()
        if full is not None:
            local = full[keys] if rows else torch.zeros(0, self.dim)
        else:
            import zlib
            g = torch.Generator().manual_seed(zlib.crc32(self.name.encode()) & 0xFFFF)
            allv = (torch.rand(self.vocab, self.dim, generator=g) * 2 - 1) * 0.05
            local = allv[keys] if rows else torch.zeros(0, self.dim)
        self.weight = local.to(self.device, dtype).contiguous()
        self.states = {}
        self.sparse_grad = None
        self.last_touch = torch.zeros(self.weight.shape[0], dtype=torch.float64)
        _variables.append(self)

    # key -> (owner rank, local row)
    def locate(self, keys: torch.Tensor):
        if self.owner >= 0:
            return torch.full_like(keys, self.owner), keys
        return keys % self.world, torch.div(keys, self.world, rounding_mode="floor")

    def local_rows(self, keys: torch.Tensor, create: bool = True) -> torch.Tensor:
        _, r = self.locate(keys)
        return r

    def global_keys(self) -> torch.Tensor:
        n = self.weight.shape[0]
        if self.owner >= 0:
            return torch.arange(n)
        return torch.arange(n) * self.world + self.rank


DistributedVariable = Variable


def LocalizedVariable(*a, gpu: int = 0, **kw):
    kw["mode"] = f"localized:{gpu}"
    return Variable(*a, **kw)


class DynamicVariable(Variable):
    """Hash-backed variable with unbounded key space (sok.DynamicVariable over HKV/DET):
    rows are created on first lookup; capacity grows geometrically up to ``max_capacity`` rows of HBM.

    HierarchicalKV semantics (third_party/HierarchicalKV, kit_src/variable/impl/hkv_variable.cu): when
    the HBM tier is full the least recently (``evict_strategy="lru"``) or least frequently (``"lfu"``)
    used rows are evicted -- a quarter of the table at a time, keys of the running batch are never
    evicted.  With ``var_type="hybrid"`` evicted rows (weights and optimizer states) are demoted to a
    host-memory tier (native key index, csrc/host/param_server.cpp) and promoted back, values intact,
    the next time their key is looked up; with ``"hbm"`` they are dropped and a returning key starts
    from the initializer again."""

    def __init__(self, dimension: int, var_type: str = "hbm", initializer: Union[str, float] = "uniform",
                 init_capacity: int = 1 << 16, max_capacity: int = 1 << 26, name: Optional[str] = None,
                 key_type=torch.int64, dtype=torch.float32, trainable: bool = True,
                 evict_strategy: str = "lru", host_capacity: int = 1 << 24):
        c = _c()
        self.name = name or f"sok_dynvar_{len(_variables)}"
        self.mode = "dynamic"
        self.owner = -1
        self.trainable = trainable
        self.dim = int(dimension)
        self.world, self.rank, self.device = c.world_size, c.rank, c.device
        self.var_type = var_type
        self.initializer = initializer
        self.max_capacity = max_capacity
        self.hash = HashTable(max_capacity, self.device)
        self.weight = torch.zeros(init_capacity, self.dim, dtype=dtype, device=self.device)
        self._init_rows(0, init_capacity)
        self.states = {}
        self.sparse_grad = None
        self.last_touch = torch.zeros(init_capacity, dtype=torch.float64)
        init_capacity = min(init_capacity, max_capacity)
        if self.weight.shape[0] > init_capacity:
            self.weight = self.weight[:init_capacity].clone()
            self.last_touch = self.last_touch[:init_capacity].clone()
        assert evict_strategy in ("lru", "lfu") and var_type in ("hbm", "hybrid")
        self.evict_strategy, self.host_capacity = evict_strategy, host_capacity
        self.last_used = torch.zeros(init_capacity, dtype=torch.int64)   # lookup clock per row
        self.freq = torch.zeros(init_capacity, dtype=torch.int64)
        self.clock = 0
        self.host = None            # host tier, created at the first eviction of a hybrid variable
        self.evictions = 0
        self.promotions = 0
        self.vocab = -1
        self.shape = (-1, self.dim)
        _variables.append(self)

    def _init_rows(self, lo, hi):
        if isinstance(self.initializer, (int, float)):
            self.weight[lo:hi] = float(self.initializer)
        else:
            self.weight[lo:hi].uniform_(-0.05, 0.05)

    def _grow(self, need: int):
        cap = self.weight.shape[0]
        if need <= cap:
            return
        new = cap
        while new < need:
            new *= 2
        w = torch.zeros(new, self.dim, dtype=self.weight.dtype, device=self.device)
        w[:cap] = self.weight
        old = self.weight
        self.weight = w
        self._init_rows(cap, new)
        for k, s in list(self.states.items()):
            ns = torch.zeros(new, self.dim, dtype=s.dtype, device=self.device)
            ns[:cap] = s
            self.states[k] = ns
        lt = torch.zeros(new, dtype=torch.float64)
        lt[:cap] = self.last_touch
        self.last_touch = lt
        for nm in ("last_used", "freq"):
            t = torch.zeros(new, dtype=torch.int64)
            t[:cap] = getattr(self, nm)
            setattr(self, nm, t)
        del old

    def _state_names(self):
        return sorted(self.states.keys())

    def _evict(self, n_new: int, protect: torch.Tensor):
        """make room for ``n_new`` rows: keep the best-scored 3/4 of the capacity (minus the incoming
        rows), demote / drop the rest and rebuild the key index compactly"""
        if self.sparse_grad is not None:
            raise RuntimeError(f"{self.name}: gradients of an earlier lookup are pending; apply them before a "
                               "lookup that has to evict rows (row ids change on eviction)")
        keys_all, rows_all = self.hash.dump()                      # CPU, ordered by row
        n = keys_all.numel()
        score = (self.last_used if self.evict_strategy == "lru" else self.freq)[rows_all].clone().double()
        score += self.last_used[rows_all].double() * 1e-12          # lfu ties: older first
        prot = torch.isin(keys_all, protect.cpu())
        score[prot] = float("inf")
        target = max(int(prot.sum()), min(n, int(self.max_capacity * 0.75) - n_new))
        if target + n_new > self.max_capacity:
            raise RuntimeError(f"{self.name}: one batch needs {target + n_new} rows, max_capacity is {self.max_capacity}")
        order = torch.argsort(score, descending=True, stable=True)
        keep, gone = order[:target], order[target:]
        dev_rows = lambda idx: rows_all[idx].to(self.device)
        if gone.numel() and self.var_type == "hybrid":
            names = self._state_names()
            if self.host is None:
                from ..cache.hps import HostParameterServer
                self.host = HostParameterServer(self.dim, num_states=len(names), capacity_rows=self.host_capacity)
                self._host_states = names
            self.host.push(keys_all[gone], self.weight[dev_rows(gone)].float().cpu(),
                           [self.states[nm][dev_rows(gone)].float().cpu() for nm in self._host_states
                            if nm in self.states])
        self.evictions += int(gone.numel())
        old_rows = dev_rows(keep)
        w_keep = self.weight[old_rows].clone()
        s_keep = {nm: st[old_rows].clone() for nm, st in self.states.items()}
        meta = {nm: getattr(self, nm)[rows_all[keep]].clone() for nm in ("last_used", "freq", "last_touch")}
        self.hash.clear()
        new_rows = self.hash.get_insert(keys_all[keep].to(self.device))
        self._init_rows(0, self.weight.shape[0])
        self.weight[new_rows] = w_keep
        for nm, st in self.states.items():
            st.zero_()
            st[new_rows] = s_keep[nm]
        for nm, val in meta.items():
            t = getattr(self, nm)
            t.zero_()
            t[new_rows.cpu()] = val

    def local_rows(self, keys: torch.Tensor, create: bool = True) -> torch.Tensor:
        k = keys.to(self.device).to(torch.int64)
        if not create:
            return self.hash.get(k)
        fresh = None
        if self.hash.size() + k.numel() > self.max_capacity or self.host is not None:
            known = self.hash.get(k)
            fresh = torch.unique(k[(known < 0) & (k >= 0)])
            if self.hash.size() + fresh.numel() > self.max_capacity:
                self._evict(int(fresh.numel()), torch.unique(k[k >= 0]))
        rows = self.hash.get_insert(k)
        self._grow(self.hash.size())
        if self.host is not None and fresh is not None and fresh.numel():
            hrows = self.host._rows(fresh.cpu(), create=False)        # promote demoted rows, values intact
            hit = hrows >= 0
            if bool(hit.any()):
                dst = self.hash.get(fresh[hit.to(fresh.device)])
                self.weight[dst] = self.host._gather(self.host.w, hrows[hit]).to(self.device, self.weight.dtype)
                for j, nm in enumerate(self._host_states):
                    if nm in self.states:
                        self.states[nm][dst] = self.host._gather(self.host.s[j], hrows[hit]).to(
                            self.device, self.states[nm].dtype)
                self.promotions += int(hit.sum())
        self.clock += 1
        r = rows[rows >= 0].cpu()
        self.last_used[r] = self.clock
        self.freq.index_add_(0, r, torch.ones_like(r))
        return rows

    def locate(self, keys):
        return keys % self.world, keys

    def global_keys(self):
        k, r = self.hash.dump()
        return k

    @property
    def size(self):
        return self.hash.size()

    def export(self):
        """-> (keys, weights, {state name: rows}) of every row this rank holds: the HBM tier plus the rows
        that currently live only in the host tier"""
        k, r = self.hash.dump()
        rd = r.to(self.device)
        w = self.weight[rd].float().cpu()
        sts = {nm: st[rd].float().cpu() for nm, st in self.states.items()}
        if self.host is not None:
            hk, hr = self.host.items()
            only = ~torch.isin(hk, k)
            if bool(only.any()):
                hk, hr = hk[only], hr[only]
                k = torch.cat([k, hk])
                w = torch.cat([w, self.host._gather(self.host.w, hr)])
                for j, nm in enumerate(self._host_states):
                    if nm in sts:
                        sts[nm] = torch.cat([sts[nm], self.host._gather(self.host.s[j], hr)])
                for nm in sts:
                    if nm not in self._host_states:      # state created after the tier: demoted rows have none
                        sts[nm] = torch.cat([sts[nm], torch.zeros(int(only.sum()), self.dim)])
        return k, w, sts

    @property
    def total_size(self):
        """rows in HBM + rows that only live in the host tier"""
        if self.host is None:
            return self.hash.size()
        hk, _ = self.host.items()
        in_hbm, _ = self.hash.dump()
        return int(self.hash.size() + (~torch.isin(hk, in_hbm)).sum())


# ----------------------------------------------------------------------------- lookup
def _to_csr(sp_ids):
    """accept [b, H] padded (-1), or (values, row_lengths)"""
    if isinstance(sp_ids, (tuple, list)) and len(sp_ids) == 2 and sp_ids[0].dim() == 1:
        vals, lens = sp_ids
        return vals.to(torch.int64), lens.to(torch.int64)
    t = sp_ids.to(torch.int64)
    mask = t >= 0
    return t[mask], mask.sum(1)


class _Lookup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, var, vals, lens, combiner, wts=None):
        c = _c()
        dev = var.device
        vals = vals.to(dev)
        lens = lens.to(dev)
        b = lens.numel()
        seg = torch.repeat_interleave(torch.arange(b, device=dev), lens)
        wts = None if wts is None else wts.to(dev).float().reshape(-1)
        ctx.w_own = None
        if c.world_size == 1:
            rows = var.local_rows(vals)
            vec = var.weight[rows].float()
            if wts is not None:
                vec = vec * wts.unsqueeze(1)
                ctx.w_own = wts
            out = torch.zeros(b, var.dim, device=dev).index_add_(0, seg, vec)
            ctx.rows, ctx.seg_owner = rows, None
        else:
            # allgather keys (+segment ids, + source rank), local lookup of owned keys, alltoall back
            n_loc = torch.tensor([vals.numel()], device=dev)
            ns = [torch.zeros_like(n_loc) for _ in range(c.world_size)]
            torch.distributed.all_gather(ns, n_loc)
            ns = [int(x) for x in ns]
            mx = max(ns + [1])
            pad_v = torch.full((mx,), -1, dtype=torch.int64, device=dev)
            pad_v[:vals.numel()] = vals
            pad_s = torch.zeros(mx, dtype=torch.int64, device=dev)
            pad_s[:vals.numel()] = seg
            gv = torch.zeros(c.world_size, mx, dtype=torch.int64, device=dev)
            gs = torch.zeros(c.world_size, mx, dtype=torch.int64, device=dev)
            c.all_gather(gv, pad_v)
            c.all_gather(gs, pad_s)
            gw = None
            if wts is not None:
                pad_w = torch.zeros(mx, device=dev)
                pad_w[:vals.numel()] = wts
                gw = torch.zeros(c.world_size, mx, device=dev)
                c.all_gather(gw, pad_w)
            owner, _ = var.locate(gv.clamp(min=0))
            mine = (owner == c.rank) & (gv >= 0)
            partial = torch.zeros(c.world_size, b_max(c, b), var.dim, device=dev)
            rows_all = torch.full_like(gv, -1)
            if bool(mine.any()):
                rws = var.local_rows(gv[mine])
                rows_all[mine] = rws
                src = torch.nonzero(mine)[:, 0]
                vec = var.weight[rws].float()
                if gw is not None:
                    vec = vec * gw[mine].unsqueeze(1)
                    ctx.w_own = gw[mine]
                partial.view(-1, var.dim).index_add_(0, src * partial.shape[1] + gs[mine], vec)
            recv = torch.zeros_like(partial)
            c.all_to_all(recv, partial)
            out = recv.sum(0)[:b]
            ctx.rows, ctx.seg_owner = rows_all, (gs, mine)
        if wts is None:
            cnt = lens.clamp(min=1).float().unsqueeze(1)
        else:      # weighted mean = weighted sum / sum of weights (tf.nn.embedding_lookup_sparse)
            cnt = torch.zeros(b, device=dev).index_add_(0, seg, wts).unsqueeze(1)
            cnt = torch.where(cnt == 0, torch.ones_like(cnt), cnt)
        if combiner == "mean":
            out = out / cnt
        ctx.var, ctx.seg, ctx.cnt, ctx.combiner, ctx.b = var, seg, cnt, combiner, b
        return out

    @staticmethod
    def backward(ctx, g):
        var, c = ctx.var, _c()
        g = g.float()
        if ctx.combiner == "mean":
            g = g / ctx.cnt
        if c.world_size == 1:
            rows, grads = ctx.rows, g[ctx.seg]
        else:
            gs, mine = ctx.seg_owner
            bm = b_max(c, ctx.b)
            gpad = torch.zeros(bm, var.dim, device=g.device)
            gpad[:ctx.b] = g
            gall = torch.zeros(c.world_size, bm, var.dim, device=g.device)
            c.all_gather(gall, gpad)
            src = torch.nonzero(mine)[:, 0]
            rows = ctx.rows[mine]
            grads = gall[src, gs[mine]]
        if ctx.w_own is not None and rows.numel():
            grads = grads * ctx.w_own.unsqueeze(1)
        if rows.numel():
            u, inv = torch.unique(rows, return_inverse=True)
            red = torch.zeros(u.numel(), var.dim, device=g.device).index_add_(0, inv, grads)
            if var.sparse_grad is None:
                var.sparse_grad = (u, red)
            else:
                var.sparse_grad = (torch.cat([var.sparse_grad[0], u]), torch.cat([var.sparse_grad[1], red]))
        return torch.zeros((), device=g.device), None, None, None, None, None


def b_max(c: Comm, b: int) -> int:
    t = torch.tensor([b], device=c.device)
    if c.world_size > 1:
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
    return int(t.item())


_anchor = None


def lookup_sparse(params, sp_ids, sp_weights=None, combiners: Union[str, Sequence[str], None] = None,
                  use_low_frequency_filter: bool = False):
    """sok.lookup_sparse(params, sp_ids, sp_weights=None, combiners=None) -> pooled embeddings
    [b, dim] per variable (reference lookup.py:543).  ``sp_weights``: per-id weights in the same layout
    as ``sp_ids`` (padded [b, H] or (values, row_lengths)); ``mean`` then divides by the sum of weights.
    A combiner (or list of combiners) passed in the third position is accepted as ``combiners``."""
    if isinstance(sp_weights, str) or (isinstance(sp_weights, (list, tuple)) and sp_weights
                                       and all(isinstance(x, str) for x in sp_weights)):
        sp_weights, combiners = None, sp_weights
    single = not isinstance(params, (list, tuple))
    ps = [params] if single else list(params)
    ids = [sp_ids] if single else list(sp_ids)
    ws = [None] * len(ps) if sp_weights is None or (isinstance(sp_weights, (list, tuple)) and not sp_weights) \
        else ([sp_weights] if single else list(sp_weights))
    combiners = combiners or "sum"
    cs = [combiners] * len(ps) if isinstance(combiners, str) else list(combiners)
    outs = []
    for p, i, w, cb in zip(ps, ids, ws, cs):
        vals, lens = _to_csr(i)
        wv = None
        if w is not None:
            if isinstance(w, (tuple, list)):
                wv = w[0].float().reshape(-1)
            else:
                wv = w.float()[i.to(torch.int64) >= 0] if w.dim() == 2 else w.float().reshape(-1)
            if wv.numel() != vals.numel():
                raise ValueError("sp_ids and sp_weights must have the same shape")
        anchor = torch.zeros((), device=p.device, requires_grad=True)
        outs.append(_Lookup.apply(anchor, p, vals, lens, cb, wv))
    return outs[0] if single else outs


def all2all_dense_embedding(param: Variable, indices: torch.Tensor) -> torch.Tensor:
    """dense (no pooling) lookup: [b, n] indices -> [b, n, dim]"""
    b, n = indices.shape
    out = lookup_sparse(param, indices.reshape(-1, 1), "sum")
    return out.view(b, n, param.dim)


# ----------------------------------------------------------------------------- optimizers
class OptimizerWrapper:
    """Applies sparse updates to SOK variables (sok.OptimizerWrapper over a tf optimizer): holds
    per-variable slot tensors, consumes ``var.sparse_grad``."""

    def __init__(self, optimizer: Optimizer_t = Optimizer_t.SGD, lr: float = 0.01, **hp):
        from ..solver import check_not_rowwise
        check_not_rowwise(optimizer, "sok.OptimizerWrapper")
        self.opt, self.lr, self.hp = optimizer, lr, hp
        self.step = 0

    def apply_gradients(self, variables: Sequence[Variable]):
        self.step += 1
        for v in variables:
            if v.sparse_grad is None or not v.trainable:
                v.sparse_grad = None
                continue
            rows, g = v.sparse_grad
            u, inv = torch.unique(rows, return_inverse=True)
            gg = torch.zeros(u.numel(), v.dim, device=g.device).index_add_(0, inv, g)
            for k in ("s0", "s1"):
                if k not in v.states:
                    v.states[k] = torch.full_like(v.weight, self.hp.get("initial_accu_value", 0.0)
                                                  if (k == "s0" and self.opt == Optimizer_t.AdaGrad) else 0.0,
                                                  dtype=torch.float32)
                elif v.states[k].shape[0] < v.weight.shape[0]:
                    ns = torch.zeros(v.weight.shape[0], v.dim, device=v.device)
                    ns[:v.states[k].shape[0]] = v.states[k]
                    v.states[k] = ns
            w = v.weight[u].float()
            a, b = v.states["s0"][u].clone(), v.states["s1"][u].clone()
            opt_reference(self.opt, w, a, b, gg, self.hp, self.lr, self.step)
            v.weight[u] = w.to(v.weight.dtype)
            v.states["s0"][u], v.states["s1"][u] = a, b
            v.last_touch[u.cpu()] = time.time()
            v.sparse_grad = None


def SGD(lr: float = 0.01):
    return OptimizerWrapper(Optimizer_t.SGD, lr)


def filter_variables(vars_):
    """split a variable list into (sok variables, others)"""
    sok_v = [v for v in vars_ if isinstance(v, Variable)]
    other = [v for v in vars_ if not isinstance(v, Variable)]
    return sok_v, other


# ----------------------------------------------------------------------------- dump / load
_MAGIC = b"SOKB200\0"


def _write(path, arr: np.ndarray, kind: int):
    with open(path, "wb") as f:
        f.write(_MAGIC + struct.pack("<iiqq", kind, arr.dtype.itemsize, arr.shape[0],
                                     arr.shape[1] if arr.ndim > 1 else 1))
        f.write(arr.tobytes())


def _read(path):
    raw = open(path, "rb").read()
    assert raw[:8] == _MAGIC, f"{path}: not a SOK dump"
    kind, isz, n, d = struct.unpack("<iiqq", raw[8:32])
    dt = {1: "<i8", 2: "<f4", 3: "<f4"}[kind]
    a = np.frombuffer(raw[32:], dtype=dt)
    return a.reshape(n, d) if kind != 1 else a


def dump(path: str, variables: Sequence[Variable], optimizer: Optional[OptimizerWrapper] = None):
    """<path>/<name>-key, <name>-weight (+ -slot0/-slot1), keys sorted, gathered on rank 0."""
    c = _c()
    os.makedirs(path, exist_ok=True)
    for v in variables:
        keys = v.global_keys()
        if isinstance(v, DynamicVariable):
            keys, w, sts = v.export()
            sts = [sts[s] for s in ("s0", "s1") if s in sts]
        else:
            w = v.weight.float().cpu()
            sts = [v.states[s].cpu() for s in ("s0", "s1") if s in v.states]
        parts = c.all_gather_object((keys, w, sts))
        if c.rank == 0:
            K = torch.cat([p[0] for p in parts])
            W = torch.cat([p[1] for p in parts])
            order = torch.argsort(K)
            _write(os.path.join(path, f"{v.name}-key"), K[order].numpy().astype("<i8"), 1)
            _write(os.path.join(path, f"{v.name}-weight"), W[order].numpy().astype("<f4"), 2)
            if optimizer is not None:
                for i in range(len(parts[0][2])):
                    S = torch.cat([p[2][i] for p in parts])
                    _write(os.path.join(path, f"{v.name}-slot{i}"), S[order].numpy().astype("<f4"), 3)
        c.barrier()


def load(path: str, variables: Sequence[Variable], optimizer: Optional[OptimizerWrapper] = None):
    for v in variables:
        K = torch.from_numpy(_read(os.path.join(path, f"{v.name}-key")).astype("int64"))
        W = torch.from_numpy(_read(os.path.join(path, f"{v.name}-weight")).copy())
        owner, _ = v.locate(K)
        m = owner == v.rank
        rows = v.local_rows(K[m])
        v.weight[rows] = W[m].to(v.device, v.weight.dtype)
        if optimizer is not None:
            for i, s in enumerate(("s0", "s1")):
                p = os.path.join(path, f"{v.name}-slot{i}")
                if os.path.exists(p):
                    S = torch.from_numpy(_read(p).copy())
                    if s not in v.states:
                        v.states[s] = torch.zeros_like(v.weight, dtype=torch.float32)
                    v.states[s][rows] = S[m].to(v.device)


def incremental_model_dump(variables: Sequence[DynamicVariable], time_threshold: float, path: str):
    """export only the rows touched after ``time_threshold`` (dump_load.py:1343-1500)."""
    os.makedirs(path, exist_ok=True)
    for v in variables:
        if isinstance(v, DynamicVariable):
            k, r = v.hash.dump()
        else:
            k, r = v.global_keys(), torch.arange(v.weight.shape[0])
        m = v.last_touch[r] > time_threshold
        _write(os.path.join(path, f"{v.name}-key"), k[m].numpy().astype("<i8"), 1)
        _write(os.path.join(path, f"{v.name}-weight"),
               v.weight[r[m].to(v.device)].float().cpu().numpy().astype("<f4"), 2)


# ----------------------------------------------------------------------------- dynamic-variable utilities
__version__ = "2.0.0.b200"


def set_comm_tool(tool: str = "torch.distributed"):
    """sok.set_comm_tool("horovod" | "tf.distribute") of the reference: there is one communication layer here
    (torch.distributed, one process per GPU); the call is accepted so that scripts keep working."""
    return "torch.distributed"


def export(var):
    """sok.export(var) -> (indices, values) of a DynamicVariable (dynamic_variable.py:465-491): the keys this rank
    holds and their vectors, HBM tier and host tier, on the CPU"""
    if not isinstance(var, DynamicVariable):
        raise TypeError("sok.export takes a sok.DynamicVariable")
    k, w, _ = var.export()
    return k, w


def assign(var, indices: torch.Tensor, values: torch.Tensor):
    """sok.assign(var, indices, values) (dynamic_variable.py:494-517): insert or overwrite the rows of ``indices``
    (this rank keeps the keys it owns, ``key % world == rank``)"""
    if not isinstance(var, DynamicVariable):
        raise TypeError("sok.assign takes a sok.DynamicVariable")
    k = torch.as_tensor(indices).reshape(-1).to(torch.int64)
    v = torch.as_tensor(values).reshape(k.numel(), var.dim)
    mine = (k % var.world) == var.rank
    if bool(mine.any()):
        rows = var.local_rows(k[mine], create=True)
        ok = rows >= 0
        var.weight[rows[ok]] = v[mine][ok.cpu()].to(var.device, var.weight.dtype)
    return var


def sparse_read_and_evict(var, indices: torch.Tensor):
    """sok.sparse_read_and_evict(var, indices) (lookup.py:75-80, hybrid variables only): the rows of ``indices`` with
    unseen keys created; when the HBM tier is full the least recently / least frequently used rows are demoted to
    the host tier first.  Local read: every key is served by this rank's table."""
    if not isinstance(var, DynamicVariable) or var.var_type != "hybrid":
        raise TypeError("sparse_read_and_evict only works on hybrid DynamicVariables")
    k = torch.as_tensor(indices).to(torch.int64)
    rows = var.local_rows(k.reshape(-1), create=True)
    out = var.weight[rows.clamp(min=0)] * (rows >= 0).unsqueeze(-1).to(var.weight.dtype)
    return out.view(*k.shape, var.dim)


def group_lookup(params, indices):
    """sok.group_lookup (lookup.py:83-96): several single-GPU embedding lookups in one call; every ``params[i]`` is a
    local [rows, dim] tensor / Parameter or a sok.Variable whose rows live on this rank, gradients flow to it"""
    single = not isinstance(params, (list, tuple))
    ps = [params] if single else list(params)
    ids = [indices] if not isinstance(indices, (list, tuple)) else list(indices)
    outs = []
    for p_, i_ in zip(ps, ids):
        w = p_.weight if isinstance(p_, Variable) else p_
        outs.append(torch.nn.functional.embedding(torch.as_tensor(i_).to(w.device).long(), w))
    return outs[0] if single else outs
