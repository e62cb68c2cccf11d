"""Host parameter server tier: HostParameterServer (pinned host table, optional SSD spill file),
HMemCache (host-memory block cache with a target hit rate), SparseModelFile,
EmbeddingTrainingCache (TrainPSType_t Staged / Cached) and OffloadedEmbedding (GPU hot-row cache in
front of a host-resident table: Query -> miss fetch -> Replace, write-back of updated rows).

Re-created from the interfaces that survive in the reference
(HugeCTR/include/embedding_training_cache/*.hpp: ParameterServer{pull,push,load_keyset,flush_to_ssd},
HMemCache, SparseModelFile(TS), EmbeddingTrainingCache; the wiring was deleted upstream).
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import numpy as np
import torch

from ..enums import TrainPSType_t
from ..ops.optim import opt_hp, opt_reference
from .gpu_cache import GpuCache


class SparseModelFile:
    """On-disk sparse model in the legacy format: <dir>/key (int64), <dir>/emb_vector (fp32)."""

    def __init__(self, path: str, ev: int):
        self.path, self.ev = path, ev
        os.makedirs(path, exist_ok=True)
        self.kf, self.vf = os.path.join(path, "key"), os.path.join(path, "emb_vector")
        self.index: Dict[int, int] = {}
        if os.path.exists(self.kf):
            keys = np.fromfile(self.kf, dtype="<i8")
            self.index = {int(k): i for i, k in enumerate(keys)}

    def load(self, keys):
        if not self.index:
            return {}
        mm = np.memmap(self.vf, dtype="<f4", mode="r").reshape(-1, self.ev)
        return {int(k): torch.from_numpy(np.array(mm[self.index[int(k)]]))
                for k in keys if int(k) in self.index}

    def dump(self, keys: torch.Tensor, values: torch.Tensor):
        """append new keys, overwrite existing ones"""
        new_k, new_v = [], []
        if self.index:
            mm = np.memmap(self.vf, dtype="<f4", mode="r+").reshape(-1, self.ev)
        for k, v in zip(keys.tolist(), values):
            if k in self.index:
                mm[self.index[k]] = v.numpy()
            else:
                self.index[k] = len(self.index)
                new_k.append(k)
                new_v.append(v.numpy())
        if new_k:
            with open(self.kf, "ab") as f:
                f.write(np.asarray(new_k, dtype="<i8").tobytes())
            with open(self.vf, "ab") as f:
                f.write(np.stack(new_v).astype("<f4").tobytes())


class HMemCache:
    """Host-memory block cache in front of the SSD file (target hit rate controls its size)."""

    def __init__(self, ev: int, capacity_rows: int):
        from collections import OrderedDict
        self.ev, self.cap = ev, capacity_rows
        self.d = OrderedDict()
        self.hits = self.reqs = 0

    def get(self, k):
        self.reqs += 1
        if k in self.d:
            self.d.move_to_end(k)
            self.hits += 1
            return self.d[k]
        return None

    def put(self, k, v):
        self.d[k] = v
        self.d.move_to_end(k)
        evicted = []
        while len(self.d) > self.cap:
            evicted.append(self.d.popitem(last=False))
        return evicted

    def hit_rate(self):
        return self.hits / max(1, self.reqs)


class HostParameterServer:
    """Whole table (weights + optimizer states) in (pinned) host memory; rows are created lazily with
    the embedding initializer; optional SSD spill (`flush_to_ssd`)."""

    def __init__(self, ev: int, num_states: int = 0, init_bound: float = 0.05,
                 ssd_path: Optional[str] = None, capacity_rows: int = 1 << 20, seed: int = 0):
        self.ev, self.ns = ev, num_states
        self.bound = init_bound
        self.cap = capacity_rows
        pin = torch.cuda.is_available()
        self.w = torch.zeros(self.cap, ev)
        self.s = [torch.zeros(self.cap, ev) for _ in range(num_states)]
        if pin:
            self.w = self.w.pin_memory()
            self.s = [t.pin_memory() for t in self.s]
        self._stage: Dict[int, torch.Tensor] = {}
        self.gen = torch.Generator().manual_seed(seed)
        self._seed = (int(seed) * 0x9E3779B97F4A7C15 + 0x1234567) & 0xFFFFFFFFFFFFFFFF
        self.ssd = SparseModelFile(ssd_path, ev) if ssd_path else None
        # key -> row index: native sharded hash maps + OpenMP row movers (csrc/host/param_server.cpp);
        # a Python dict when the host library cannot be built
        self._h = None
        self.index: Dict[int, int] = {}
        try:
            import ctypes as C
            from .. import _native
            lib = _native.host_lib()
            vp, ll = C.c_void_p, C.c_longlong
            lib.hctr_ps_create.restype = vp
            lib.hctr_ps_destroy.argtypes = [vp]
            lib.hctr_ps_size.argtypes = [vp]
            lib.hctr_ps_size.restype = ll
            lib.hctr_ps_lookup.argtypes = [vp, vp, ll, vp, vp, C.c_int, ll]
            lib.hctr_ps_lookup.restype = ll
            lib.hctr_ps_dump.argtypes = [vp, vp, vp]
            lib.hctr_ps_dump.restype = ll
            lib.hctr_ps_gather.argtypes = [vp, vp, ll, ll, vp]
            lib.hctr_ps_scatter.argtypes = [vp, vp, ll, ll, vp]
            lib.hctr_ps_init_rows.argtypes = [vp, vp, vp, ll, C.c_int, C.c_float, C.c_ulonglong]
            self._lib = lib
            self._h = lib.hctr_ps_create()
        except Exception:  # pragma: no cover - no compiler available
            self._h = None

    def __del__(self):
        if getattr(self, "_h", None):
            try:
                self._lib.hctr_ps_destroy(self._h)
            except Exception:
                pass
            self._h = None

    def _rows(self, keys, create=True):
        keys = keys.reshape(-1).to(torch.int64).contiguous()
        if self._h is not None:
            n = keys.numel()
            rows = torch.empty(n, dtype=torch.int64)
            is_new = torch.zeros(n, dtype=torch.uint8)
            created = self._lib.hctr_ps_lookup(self._h, keys.data_ptr(), n, rows.data_ptr(),
                                               is_new.data_ptr(), int(create), self.cap)
            if created < 0:
                raise RuntimeError("HostParameterServer capacity exceeded")
            if created > 0:
                nr = rows[is_new.bool()].contiguous()
                nk = keys[is_new.bool()].contiguous()
                # counter-based initializer in the row movers' thread pool (value of a cell = f(seed, key, column))
                self._lib.hctr_ps_init_rows(self.w.data_ptr(), nr.data_ptr(), nk.data_ptr(), nr.numel(), self.ev,
                                            float(self.bound), int(self._seed) & 0xFFFFFFFFFFFFFFFF)
                if self.ssd:
                    newk = keys[is_new.bool()].tolist()
                    loaded = self.ssd.load(newk)
                    for j, k in enumerate(newk):
                        if k in loaded:
                            self.w[nr[j]] = loaded[k]
            return rows
        rows = []
        for k in keys.tolist():
            r = self.index.get(k)
            if r is None and create:
                r = len(self.index)
                if r >= self.cap:
                    raise RuntimeError("HostParameterServer capacity exceeded")
                self.index[k] = r
                loaded = self.ssd.load([k]) if self.ssd else {}
                self.w[r] = loaded.get(k, (torch.rand(self.ev, generator=self.gen) * 2 - 1) * self.bound)
            rows.append(-1 if r is None else r)
        return torch.tensor(rows, dtype=torch.int64)

    def _gather(self, table: torch.Tensor, rows: torch.Tensor, reuse: Optional[int] = None) -> torch.Tensor:
        """out[i] = table[rows[i]] (rows[i] < 0 -> zeros).  ``reuse=<slot>``: gather into this server's reusable
        (pinned on a GPU box) staging buffer ``slot`` and return a view of it -- no allocation / first-touch page
        faults per step, fast H2D; the caller must be done with the previous result of the same slot."""
        if self._h is None:
            return table[rows.clamp(min=0)] * (rows >= 0).unsqueeze(1)
        n = rows.numel()
        if reuse is None:
            out = torch.empty(n, self.ev)
        else:
            buf = self._stage.get(reuse)
            if buf is None or buf.shape[0] < n:
                buf = torch.empty(max(n, 1024) * 5 // 4, self.ev)
                if torch.cuda.is_available():
                    buf = buf.pin_memory()
                self._stage[reuse] = buf
            out = buf[:n]
        rows = rows.contiguous()
        self._lib.hctr_ps_gather(table.data_ptr(), rows.data_ptr(), n, self.ev * 4, out.data_ptr())
        return out

    def _scatter(self, table: torch.Tensor, rows: torch.Tensor, src: torch.Tensor):
        src = src.detach().cpu().float().contiguous()
        if self._h is None:
            table[rows] = src
            return
        self._lib.hctr_ps_scatter(table.data_ptr(), rows.data_ptr(), rows.numel(), self.ev * 4, src.data_ptr())

    def pull(self, keys: torch.Tensor):
        rows = self._rows(keys.cpu())
        return self._gather(self.w, rows), [self._gather(s, rows) for s in self.s]

    def push(self, keys: torch.Tensor, w: torch.Tensor, states=()):
        rows = self._rows(keys.cpu())
        self._scatter(self.w, rows, w)
        for dst, src in zip(self.s, states):
            self._scatter(dst, rows, src)

    def items(self):
        """-> (keys int64 [n], rows int64 [n]) of every stored row"""
        if self._h is not None:
            n = int(self._lib.hctr_ps_size(self._h))
            k, r = torch.empty(n, dtype=torch.int64), torch.empty(n, dtype=torch.int64)
            c = self._lib.hctr_ps_dump(self._h, k.data_ptr(), r.data_ptr()) if n else 0
            return k[:c], r[:c]
        return (torch.tensor(list(self.index.keys()), dtype=torch.int64),
                torch.tensor(list(self.index.values()), dtype=torch.int64))

    def load_keyset(self, keyset_file: str):
        keys = torch.from_numpy(np.fromfile(keyset_file, dtype="<i8").astype("int64"))
        self._rows(keys)
        return keys

    def flush_to_ssd(self):
        if self.ssd is None:
            return
        keys, rows = self.items()
        self.ssd.dump(keys, self.w[rows])

    def size(self):
        if self._h is not None:
            return int(self._lib.hctr_ps_size(self._h))
        return len(self.index)


class EmbeddingTrainingCache:
    """Train models larger than HBM pass by pass: ``update(keyset)`` loads the rows of the next
    keyset from the parameter server into a device table, training runs on it, ``dump()`` writes
    them back (Staged = straight from host/SSD, Cached = through HMemCache)."""

    def __init__(self, ps: HostParameterServer, ps_type: TrainPSType_t = TrainPSType_t.Staged,
                 hmem_rows: int = 1 << 16):
        self.ps, self.type = ps, ps_type
        self.hmem = HMemCache(ps.ev, hmem_rows) if ps_type == TrainPSType_t.Cached else None
        self.keys = None
        self.device_table = None

    def update(self, keyset: torch.Tensor, device):
        self.keys = keyset.to(torch.int64).cpu()
        w, _ = self.ps.pull(self.keys)
        self.device_table = w.to(device, non_blocking=True)
        return self.device_table

    def dump(self):
        if self.keys is not None:
            self.ps.push(self.keys, self.device_table.cpu())


class OffloadedEmbedding:
    """Table on the host parameter server, hot rows in the HBM GpuCache.

    forward(keys [b, H]) -> pooled [b, ev]:  unique keys -> cache.Query -> fetch misses from the host
    -> cache.Replace -> pool;   backward(grad [b, ev]) : per-unique-row reduce + optimizer on the
    staged rows -> cache.Update + write-through to the host server.
    """

    def __init__(self, ev: int, device, cache_rows: int, opt, num_states: int = 1, lr: float = 0.01,
                 host_capacity: int = 1 << 20, combiner: str = "sum", ssd_path: Optional[str] = None):
        self.ev, self.device, self.opt, self.lr, self.combiner = ev, torch.device(device), opt, lr, combiner
        self.ps = HostParameterServer(ev, num_states, ssd_path=ssd_path, capacity_rows=host_capacity)
        self.cache = GpuCache(cache_rows, ev, device)
        self.state_cache = [GpuCache(cache_rows, ev, device) for _ in range(num_states)]

    def _fetch(self, uniq):
        vals, mi, mk = self.cache.query(uniq)
        st = [c.query(uniq)[0] for c in self.state_cache]
        if mk.numel():
            w, s = self.ps.pull(mk)
            vals[mi] = w.to(self.device)
            self.cache.replace(mk.to(self.device), vals[mi])
            for c, sv, t in zip(self.state_cache, s, st):
                t[mi] = sv.to(self.device)
                c.replace(mk.to(self.device), t[mi])
        return vals, st

    def forward(self, keys: torch.Tensor) -> torch.Tensor:
        b, H = keys.shape
        k = keys.to(self.device).to(torch.int64)
        self.uniq, self.inv = torch.unique(k.reshape(-1), return_inverse=True)
        self.vals, self.states = self._fetch(self.uniq)
        out = self.vals[self.inv].view(b, H, self.ev).sum(1)
        if self.combiner == "mean":
            out = out / H
        self._shape = (b, H)
        return out

    def backward(self, grad: torch.Tensor, step: int = 1):
        b, H = self._shape
        g = grad.float().unsqueeze(1).expand(b, H, self.ev).reshape(-1, self.ev)
        if self.combiner == "mean":
            g = g / H
        gu = torch.zeros(self.uniq.numel(), self.ev, device=self.device).index_add_(0, self.inv, g)
        w = self.vals
        s0 = self.states[0] if len(self.states) > 0 else None
        s1 = self.states[1] if len(self.states) > 1 else None
        o = self.opt
        opt_reference(o.optimizer_type, w, s0, s1, gu, opt_hp(o), self.lr, step)
        self.cache.update(self.uniq, w)
        for c, s in zip(self.state_cache, (s0, s1)):
            if s is not None:
                c.update(self.uniq, s)
        self.ps.push(self.uniq, w, [s for s in (s0, s1) if s is not None])


class HpsEmbedding:
    """Inference-time embedding service in the shape of the reference's (removed) Hierarchical
    Parameter Server: the full table lives in the host parameter server, a set-associative LRU cache
    in device memory serves the hot rows; a lookup de-duplicates the batch's keys, queries the cache,
    pulls the misses from the host table and inserts them (gpu_cache Query / Replace).  Unknown keys
    read as zero vectors."""

    def __init__(self, keys: torch.Tensor, vectors: torch.Tensor, device, cache_fraction: float = 0.2,
                 combiner: str = "sum", min_cache_rows: int = 64):
        from .gpu_cache import GpuCache
        self.device = torch.device(device)
        self.ev = int(vectors.shape[1])
        n = int(keys.numel())
        self.ps = HostParameterServer(self.ev, 0, capacity_rows=max(n, 1))
        if n:
            self.ps.push(keys.to(torch.int64), vectors.float())
        rows = max(int(min_cache_rows), int(cache_fraction * n))
        self.cache = GpuCache(rows, self.ev, self.device)
        self.combiner = combiner
        self.lookups = 0

    def hit_rate(self) -> float:
        return self.cache.hit_rate()

    def lookup(self, keys: torch.Tensor) -> torch.Tensor:
        """keys [b, S, H] (int64, -1 padded) -> pooled vectors [b, S, ev] on the cache's device"""
        b, S, H = keys.shape
        flat = keys.reshape(-1).to(torch.int64)
        valid = flat >= 0
        vec = torch.zeros(flat.numel(), self.ev, device=self.device)
        if bool(valid.any()):
            uniq, inv = torch.unique(flat[valid].to(self.device), return_inverse=True)
            vals, miss_idx, miss_keys = self.cache.query(uniq)
            if miss_idx.numel():
                mk = miss_keys.cpu()
                rows = self.ps._rows(mk, create=False)
                w = self.ps._gather(self.ps.w, rows)             # absent keys -> zero rows
                vals[miss_idx.to(self.device)] = w.to(self.device)
                known = rows >= 0
                if bool(known.any()):
                    self.cache.replace(mk[known].to(self.device), w[known].to(self.device))
            vec[valid.to(self.device)] = vals[inv]
        self.lookups += 1
        out = vec.view(b, S, H, self.ev).sum(2)
        if self.combiner == "mean":
            out = out / (keys.to(self.device) >= 0).sum(2, keepdim=True).clamp(min=1)
        return out
