"""HashTable: key -> dense row index with insertion on first sight (legacy SparseEmbedding
semantics).  GPU: csrc/hashtable.cu (open addressing, atomicCAS); CPU: python dict reference.
Parity: HugeCTR/src/hashtable/nv_hashtable.cu:36-306 (get_insert / get(get_mark) / set / dump /
get_size), capacity = max_vocabulary_size / 0.75 (nv_hashtable.hpp:179).

SetAssocTable: the fixed-capacity, evicting key -> row map of a dynamic table with an
``evict_strategy`` (LRU / LFU over 32-way sets).  GPU: csrc/evict_table.cu; CPU: the same rules
in Python, the oracle of the tests.

AdmitSketch: the count-min admission sketch of a dynamic table with ``admit_threshold`` > 1, used by
both tables above.  GPU: csrc/admit_sketch.cuh (+ the count / filter kernels of csrc/hashtable.cu and
the folded ones of csrc/evict_table.cu); CPU: the same rules in Python.
"""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native
from ..ops import dense as D

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = _native.cuda_lib()
        vp, ull, ll, i = C.c_void_p, C.c_ulonglong, C.c_longlong, C.c_int
        l.hctr_ht_get_insert.argtypes = [vp, vp, vp, ull, ll, vp, vp, ll, i, vp, vp]
        l.hctr_ht_set.argtypes = [vp, vp, vp, ull, vp, vp, ll, vp]
        l.hctr_ht_dump.argtypes = [vp, vp, ull, vp, vp, vp, vp]
        l.hctr_ht_translate.argtypes = [vp, vp, vp, ull, ll, vp, vp, ll, i, vp, ll, i, i, i, i, vp]
        l.hctr_ht_translate.restype = i
        for n in ("hctr_ht_get_insert", "hctr_ht_set", "hctr_ht_dump"):
            getattr(l, n).restype = i
        l.hctr_evict_touch.argtypes = [vp, vp, vp, vp]
        l.hctr_evict_insert.argtypes = [vp, vp, vp, vp, i, vp, vp]
        l.hctr_ht_admit.argtypes = [vp, ull, vp, ll, vp, i, vp]
        l.hctr_admit_decay.argtypes = [vp, ll, vp, ull, vp]
        l.hctr_evict_get.argtypes = [vp, vp, vp]
        l.hctr_evict_dump.argtypes = [vp, ll, vp, vp, vp, vp]
        l.hctr_evict_reinit.argtypes = [vp, ll, i, vp]
        for n in ("hctr_evict_touch", "hctr_evict_insert", "hctr_evict_get", "hctr_evict_dump",
                  "hctr_evict_reinit", "hctr_ht_admit", "hctr_admit_decay"):
            getattr(l, n).restype = i
        _lib = l
    return _lib


class HashTable:
    LOAD_FACTOR = 0.75

    def __init__(self, max_rows: int, device):
        self.max_rows = int(max_rows)
        self.device = torch.device(device)
        cap = 1
        while cap < max(16, int(self.max_rows / self.LOAD_FACTOR)):
            cap <<= 1
        self.capacity = cap
        # admission sketch of an admitting growing table (set by the owner; kept when the shard grows)
        self.sketch: "AdmitSketch | None" = None
        if self.device.type == "cuda":
            self.keys = torch.full((cap,), -1, dtype=torch.int64, device=self.device)
            self.vals = torch.full((cap,), -1, dtype=torch.int64, device=self.device)
            self.counter = torch.zeros(1, dtype=torch.int64, device=self.device)
            self.overflow = torch.zeros(1, dtype=torch.int32, device=self.device)   # sticky device flag
        else:
            self.map = {}
            self._overflowed = False

    def _st(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def get_insert(self, keys: torch.Tensor) -> torch.Tensor:
        """rows for keys; unseen keys get the next free row. keys < 0 -> -1. Overflow -> -1 and
        size() > max_rows (check_overflow raises)."""
        return self._lookup(keys, True)

    def get(self, keys: torch.Tensor) -> torch.Tensor:
        """lookup only (get_mark): missing keys -> -1 (treated as zero vectors by the lookup)."""
        return self._lookup(keys, False)

    def _lookup(self, keys, insert):
        k = keys.reshape(-1).to(torch.int64)
        if self.device.type == "cuda":
            out = torch.empty_like(k)
            rc = lib().hctr_ht_get_insert(self.keys.data_ptr(), self.vals.data_ptr(),
                                          self.counter.data_ptr(), self.capacity, self.max_rows,
                                          k.data_ptr(), out.data_ptr(), k.numel(), int(insert),
                                          self._st(), self.overflow.data_ptr())
            if rc:
                raise RuntimeError("hash get_insert failed")
            D._count()
            return out.view(keys.shape)
        out = torch.empty_like(k)
        kl = k.tolist()
        res = []
        for x in kl:
            if x < 0:
                res.append(-1)
            elif x in self.map:
                v = self.map[x]
                res.append(v if v < self.max_rows else -1)
            elif insert:
                v = len(self.map)
                if v >= self.max_rows:          # rows exhausted: no insertion, sticky overflow
                    self._overflowed = True
                    res.append(-1)
                    continue
                self.map[x] = v
                res.append(v)
            else:
                res.append(-1)
        return torch.tensor(res, dtype=torch.int64).view(keys.shape)

    def translate(self, keys: torch.Tensor, out: torch.Tensor, insert: bool, n_per_rank: int, key_mod: int = 1,
                  key_rem: int = 0, slot_div: int = 1, slot_num: int = 0):
        """out = row of every OWNED key of ``keys`` (int64, any shape; -1 elsewhere) in one launch, no host
        sync.  Ownership: ``key % key_mod == key_rem`` or, with ``slot_num`` > 0, the slot of the key's
        position ``((pos % n_per_rank) // slot_div) % slot_num) % key_mod == key_rem``."""
        k = keys.reshape(-1)
        if self.device.type == "cuda":
            rc = lib().hctr_ht_translate(self.keys.data_ptr(), self.vals.data_ptr(), self.counter.data_ptr(),
                                         self.capacity, self.max_rows, k.data_ptr(), out.data_ptr(), k.numel(),
                                         int(insert), self.overflow.data_ptr(), int(n_per_rank), int(key_mod),
                                         int(key_rem), int(slot_div), int(slot_num), self._st())
            if rc:
                raise RuntimeError("hash translate failed")
            D._count()
            return out
        pos = torch.arange(k.numel()) % max(int(n_per_rank), 1)
        own = k >= 0
        if slot_num > 0:
            own &= ((pos // slot_div) % slot_num) % key_mod == key_rem
        elif key_mod > 1:
            own &= (k % key_mod) == key_rem
        kk = torch.where(own, k, torch.full_like(k, -1))
        out.reshape(-1).copy_(self._lookup(kk, insert))
        return out

    def admit_count(self, keys: torch.Tensor):
        """count, in the sketch, every occurrence of a key >= 0 of ``keys`` (int64, 1-D) that has no row: one
        training lookup calls this on every key region of the table before any ``admit_filter`` / ``get_insert``"""
        sk = self.sketch
        if self.device.type == "cuda":
            if lib().hctr_ht_admit(self.keys.data_ptr(), self.capacity, keys.data_ptr(), keys.numel(),
                                   C.byref(sk.view()), 0, self._st()):
                raise RuntimeError("hash admit count failed")
            D._count()
            return
        sk.count([x for x in keys.tolist() if x >= 0 and x not in self.map])

    def admit_filter(self, keys: torch.Tensor):
        """in place: every key >= 0 without a row whose sketch count is below the threshold becomes -1
        (rejected: no row, counted in the sketch's ``rejected``)"""
        sk = self.sketch
        if self.device.type == "cuda":
            if lib().hctr_ht_admit(self.keys.data_ptr(), self.capacity, keys.data_ptr(), keys.numel(),
                                   C.byref(sk.view()), 1, self._st()):
                raise RuntimeError("hash admit filter failed")
            D._count()
            return
        kl = keys.tolist()
        miss = [i for i, x in enumerate(kl) if x >= 0 and x not in self.map]
        if miss:
            ok = sk.admits([kl[i] for i in miss])
            rej = [i for i, a in zip(miss, ok) if not a]
            keys[rej] = -1
            sk.stats[1] += len(rej)

    def set(self, keys: torch.Tensor, vals: torch.Tensor):
        k, v = keys.reshape(-1).to(torch.int64), vals.reshape(-1).to(torch.int64)
        if self.device.type == "cuda":
            k, v = k.to(self.device), v.to(self.device)
            rc = lib().hctr_ht_set(self.keys.data_ptr(), self.vals.data_ptr(), self.counter.data_ptr(),
                                   self.capacity, k.data_ptr(), v.data_ptr(), k.numel(), self._st())
            if rc:
                raise RuntimeError("hash set failed")
            self.counter.fill_(max(int(self.counter.item()), int(v.max().item()) + 1 if v.numel() else 0))
        else:
            for a, b in zip(k.tolist(), v.tolist()):
                self.map[a] = b

    def overflowed(self) -> bool:
        """True once a key could not get a row (host sync on CUDA: call it outside the step)."""
        if self.device.type == "cuda":
            return bool(int(self.overflow.item()))
        return self._overflowed

    def size(self) -> int:
        if self.device.type == "cuda":
            return int(self.counter.item())
        return len(self.map)

    def dump(self):
        """-> (keys int64 [n], rows int64 [n]) on CPU"""
        if self.device.type == "cuda":
            n = self.capacity
            ok = torch.empty(n, dtype=torch.int64, device=self.device)
            ov = torch.empty(n, dtype=torch.int64, device=self.device)
            cnt = torch.zeros(1, dtype=torch.int64, device=self.device)
            lib().hctr_ht_dump(self.keys.data_ptr(), self.vals.data_ptr(), self.capacity,
                               ok.data_ptr(), ov.data_ptr(), cnt.data_ptr(), self._st())
            c = int(cnt.item())
            k, v = ok[:c].cpu(), ov[:c].cpu()
        else:
            k = torch.tensor(list(self.map.keys()), dtype=torch.int64)
            v = torch.tensor(list(self.map.values()), dtype=torch.int64)
        order = torch.argsort(v)
        return k[order], v[order]

    def clear(self):
        if self.device.type == "cuda":
            self.keys.fill_(-1)
            self.vals.fill_(-1)
            self.counter.zero_()
            self.overflow.zero_()
        else:
            self.map = {}
            self._overflowed = False


# ------------------------------------------------------------------------- evicting tables
EVICT_STRATEGIES = ("lru", "lfu")
WAYS = 32
COUNT_MAX = (1 << 32) - 1


class _EvictTableView(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("stamps", C.c_void_p), ("counts", C.c_void_p), ("locks", C.c_void_p),
                ("clock", C.c_void_p), ("stats", C.c_void_p), ("num_sets", C.c_int), ("lfu", C.c_int)]


class _KeyRegion(C.Structure):
    _fields_ = [("base", C.c_void_p), ("n", C.c_longlong), ("stride", C.c_longlong), ("ranks", C.c_int),
                ("key_mod", C.c_int), ("key_rem", C.c_int), ("key_bytes", C.c_int)]


class _EvictReinit(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("adm", C.c_void_p), ("adm_n", C.c_void_p), ("table", C.c_void_p),
                ("s0", C.c_void_p), ("s1", C.c_void_p), ("row_off", C.c_longlong), ("init_key", C.c_ulonglong),
                ("bound", C.c_float), ("s0_init", C.c_float), ("pitch", C.c_int), ("col0", C.c_int),
                ("s0_pitch", C.c_int), ("state_bf16", C.c_int), ("s1_row", C.c_int)]


def evict_set_of(keys, num_sets: int):
    """set of every key: the low 32 bits of fmix64(key), modulo the number of sets (hash64 in
    csrc/embedding.cuh); int64 numpy array"""
    import numpy as np
    from .ops import _fmix64
    h = _fmix64(np.asarray(keys, dtype=np.int64).astype(np.uint64)) & np.uint64(0xFFFFFFFF)
    return (h % np.uint64(num_sets)).astype(np.int64)


class SetAssocTable:
    """One evicting shard: ``capacity`` (``max_capacity`` rounded up to 32) ways in sets of 32.  A key
    lives only in set ``evict_set_of(key)``; its local row is ``set * 32 + way``.  ``clock`` is the
    collection's device clock (int64 [1]), ticked once per training step by the caller.

    A training lookup of a table calls ``touch`` on every key region of the table, then ``insert`` on
    every region (rows written in place over the keys), then ``reinit`` on the admitted ways; an
    evaluation lookup calls ``get``.  Regions are 2-D slabs [ranks, stride]: columns
    [key_off, key_off + n) of every row, keys with key >= 0 and key % key_mod == key_rem are handled,
    the others become -1.  Rules in docs/embedding.md; the CPU implementation is the reference."""

    def __init__(self, max_capacity: int, strategy: str, clock: torch.Tensor, device, sketch=None):
        """``sketch``: the shard's AdmitSketch (admitting tables), else None"""
        if strategy not in EVICT_STRATEGIES:
            raise ValueError(f"evict_strategy must be one of {EVICT_STRATEGIES}, not {strategy!r}")
        self.capacity = (int(max_capacity) + WAYS - 1) // WAYS * WAYS
        self.num_sets = self.capacity // WAYS
        self.strategy, self.clock = strategy, clock
        self.device = torch.device(device)
        dev = self.device
        self.keys = torch.full((self.capacity,), -1, dtype=torch.int64, device=dev)
        self.stamps = torch.zeros(self.capacity, dtype=torch.int64, device=dev)
        self.counts = torch.zeros(self.capacity, dtype=torch.int64, device=dev)
        self.locks = torch.zeros(self.num_sets, dtype=torch.int32, device=dev)
        self.stats = torch.zeros(3, dtype=torch.int64, device=dev)      # admitted, evicted, dropped
        self.sketch = sketch

    # ---- device plumbing
    def _view(self, stats=None):
        return _EvictTableView(self.keys.data_ptr(), self.stamps.data_ptr(), self.counts.data_ptr(),
                               self.locks.data_ptr(), self.clock.data_ptr(),
                               (self.stats if stats is None else stats).data_ptr(), self.num_sets,
                               int(self.strategy == "lfu"))

    @staticmethod
    def _region(buf, key_off, n, key_mod, key_rem):
        assert buf.dim() == 2 and buf.stride(1) == 1 and buf.dtype in (torch.int32, torch.int64)
        return _KeyRegion(buf.data_ptr() + key_off * buf.element_size(), int(n), buf.stride(0), buf.shape[0],
                          int(key_mod), int(key_rem), buf.element_size())

    def _st(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _call(self, name, *args):
        if getattr(lib(), name)(*args):
            raise RuntimeError(f"{name} failed")
        D._count()

    # ---- CPU rules (the reference the kernels are tested against)
    def _owned_keys(self, region, key_mod, key_rem):
        k = region.to(torch.int64).contiguous()
        own = k >= 0
        if key_mod > 1:
            own &= (k % key_mod) == key_rem
        return k, own

    def _find(self, base, key):
        hit = (self.keys[base:base + WAYS] == key).nonzero()
        return int(hit[0, 0]) if hit.numel() else -1

    def _insert_one(self, key, now, evict, adm, stats):
        import numpy as np
        base = int(evict_set_of([key], self.num_sets)[0]) * WAYS
        slot = self._find(base, key)
        if slot >= 0:
            return base + slot
        k = self.keys[base:base + WAYS].numpy()
        empty = np.nonzero(k < 0)[0]
        if empty.size:
            slot, victim = int(empty[0]), False
        else:
            st = self.stamps[base:base + WAYS].numpy()
            cand = [w for w in range(WAYS) if evict and st[w] != now]
            if not cand:
                stats[2] += 1
                return -1
            lfu = self.strategy == "lfu"
            cnt = self.counts[base:base + WAYS].numpy()
            slot = min(cand, key=lambda w: ((min(int(cnt[w]), COUNT_MAX) if lfu else 0), int(st[w]), int(k[w])))
            victim = True
        g = base + slot
        stats[0] += 1
        stats[1] += int(victim)
        self.keys[g], self.stamps[g], self.counts[g] = key, now, 1
        if adm is not None:
            adm.append(g)
        return g

    # ---- lookups
    def touch(self, buf, key_off: int, n: int, key_mod: int = 1, key_rem: int = 0):
        """stamp the ways of the present keys with the clock, count the occurrences"""
        if self.device.type == "cuda":
            sk = None if self.sketch is None else C.byref(self.sketch.view())
            self._call("hctr_evict_touch", C.byref(self._view()),
                       C.byref(self._region(buf, key_off, n, key_mod, key_rem)), sk, self._st())
            return
        now = int(self.clock[0])
        k, own = self._owned_keys(buf[:, key_off:key_off + n], key_mod, key_rem)
        missing = []
        for key in k[own].tolist():
            base = int(evict_set_of([key], self.num_sets)[0]) * WAYS
            slot = self._find(base, key)
            if slot >= 0:
                g = base + slot
                self.stamps[g] = now
                self.counts[g] += 1
            else:
                missing.append(key)
        if self.sketch is not None:
            self.sketch.count(missing)

    def insert(self, buf, key_off: int, n: int, key_mod: int = 1, key_rem: int = 0, adm=None, evict=True,
               stats=None):
        """rows of the keys written in place over them: present keys keep their way, missing keys are
        admitted (an empty way, else the victim of the strategy among the unprotected ways) or dropped
        (-1).  With a sketch, a missing key below the admission threshold is rejected first (-1).
        ``adm``: (list [m] int64, count [1] int32) collecting the admitted ways.  ``evict=False`` takes
        empty ways only and skips admission (checkpoint load)."""
        stats = self.stats if stats is None else stats
        sk = self.sketch if evict else None
        if self.device.type == "cuda":
            a, an = (adm[0].data_ptr(), adm[1].data_ptr()) if adm is not None else (None, None)
            self._call("hctr_evict_insert", C.byref(self._view(stats)),
                       C.byref(self._region(buf, key_off, n, key_mod, key_rem)), a, an, int(evict),
                       None if sk is None else C.byref(sk.view()), self._st())
            return
        now = int(self.clock[0])
        region = buf[:, key_off:key_off + n]
        k, own = self._owned_keys(region, key_mod, key_rem)
        out = torch.full_like(k, -1)
        got = [] if adm is not None else None
        for idx in own.reshape(-1).nonzero()[:, 0].tolist():
            key = int(k.view(-1)[idx])
            if sk is not None and self._find(int(evict_set_of([key], self.num_sets)[0]) * WAYS, key) < 0 \
                    and not sk.admits([key])[0]:
                sk.stats[1] += 1
                continue
            out.view(-1)[idx] = self._insert_one(key, now, evict, got, stats)
        region.copy_(out.to(region.dtype))
        if adm is not None and got:
            m = int(adm[1][0])
            adm[0][m:m + len(got)] = torch.tensor(got, dtype=torch.int64)
            adm[1][0] = m + len(got)

    def get(self, buf, key_off: int, n: int, key_mod: int = 1, key_rem: int = 0):
        """rows of the present keys in place, -1 for the others (no touch, no insert)"""
        if self.device.type == "cuda":
            self._call("hctr_evict_get", C.byref(self._view()),
                       C.byref(self._region(buf, key_off, n, key_mod, key_rem)), self._st())
            return
        region = buf[:, key_off:key_off + n]
        k, own = self._owned_keys(region, key_mod, key_rem)
        out = torch.full_like(k, -1)
        for idx in own.reshape(-1).nonzero()[:, 0].tolist():
            key = int(k.view(-1)[idx])
            base = int(evict_set_of([key], self.num_sets)[0]) * WAYS
            slot = self._find(base, key)
            out.view(-1)[idx] = base + slot if slot >= 0 else -1
        region.copy_(out.to(region.dtype))

    def reinit(self, adm, max_adm: int, table, s0, s1, row_off: int, pitch: int, s0_pitch: int, s0_init: float,
               bound: float, init_key: int, col0: int = 0, s1_row: bool = False):
        """fresh weights (ops.evict_init_rows) and initial optimizer state for the admitted ways; ``s1_row``:
        ``s1`` holds one fp32 value per row (partial row-wise Adam), otherwise it has the row pitch and the
        dtype of ``s0``"""
        s1_row = bool(s1_row) and s1 is not None
        if self.device.type == "cuda":
            sbf = int(any(s is not None and s.dtype == torch.bfloat16 for s in (s0, s1)))
            p = _EvictReinit(self.keys.data_ptr(), adm[0].data_ptr(), adm[1].data_ptr(), table.data_ptr(),
                             None if s0 is None else s0.data_ptr(), None if s1 is None else s1.data_ptr(),
                             int(row_off), int(init_key) & ((1 << 64) - 1), float(bound), float(s0_init),
                             int(pitch), int(col0), int(s0_pitch), sbf, int(s1_row))
            from .ops import table_type
            self._call("hctr_evict_reinit", C.byref(p), int(max_adm), table_type(table), self._st())
            return
        from .ops import evict_init_rows
        ways = adm[0][:int(adm[1][0])]
        if ways.numel() == 0:
            return
        rows = ways + row_off
        table.view(-1, pitch)[rows] = evict_init_rows(init_key, self.keys[ways], col0, pitch, bound, table.dtype)
        if s0 is not None:
            s0.view(-1, s0_pitch)[rows] = s0_init
        if s1 is not None:
            s1.view(-1, 1 if s1_row else pitch)[rows] = 0

    # ---- whole-table views (host synchronisation: outside the step)
    def dump(self):
        """-> (keys int64 [n], local rows int64 [n]) of the live keys, by key, on CPU"""
        if self.device.type == "cuda":
            ok = torch.empty(self.capacity, dtype=torch.int64, device=self.device)
            os_ = torch.empty(self.capacity, dtype=torch.int64, device=self.device)
            cnt = torch.zeros(1, dtype=torch.int64, device=self.device)
            self._call("hctr_evict_dump", self.keys.data_ptr(), self.capacity, ok.data_ptr(), os_.data_ptr(),
                       cnt.data_ptr(), self._st())
            c = int(cnt.item())
            k, s = ok[:c].cpu(), os_[:c].cpu()
        else:
            s = (self.keys >= 0).nonzero()[:, 0]
            k = self.keys[s].clone()
        order = torch.argsort(k)
        return k[order], s[order]

    def live(self) -> torch.Tensor:
        """number of live keys, as a device scalar"""
        return (self.keys >= 0).sum()


# ------------------------------------------------------------------------- admission sketch
SKETCH_ROWS = 4
SKETCH_MAX = (1 << 32) - 1
SKETCH_SALT = 0x9E3779B97F4A7C15


class _AdmitSketch(C.Structure):
    _fields_ = [("counters", C.c_void_p), ("stats", C.c_void_p), ("width_mask", C.c_uint),
                ("threshold", C.c_uint)]


def sketch_width(rows: int) -> int:
    """counters per sketch row: the smallest power of two >= 2 * rows, at least 1024"""
    w = 1024
    while w < 2 * int(rows):
        w <<= 1
    return w


def sketch_slots(keys, width: int):
    """flat counter index [n, 4] of every key, row r at r * width + (lo32(h) + r * (hi32(h) | 1)) mod width,
    h = fmix64(key ^ SKETCH_SALT) (sketch_counter in csrc/admit_sketch.cuh); int64 numpy array"""
    import numpy as np
    from .ops import _fmix64
    h = _fmix64(np.asarray(keys, dtype=np.int64).reshape(-1).astype(np.uint64) ^ np.uint64(SKETCH_SALT))
    lo, hi = h & np.uint64(0xFFFFFFFF), (h >> np.uint64(32)) | np.uint64(1)
    r = np.arange(SKETCH_ROWS, dtype=np.uint64)
    with np.errstate(over="ignore"):
        col = (lo[:, None] + r[None, :] * hi[:, None]) & np.uint64(width - 1)
    return (r[None, :] * np.uint64(width) + col).astype(np.int64)


class AdmitSketch:
    """Count-min admission sketch of one row shard of a dynamic table with ``admit_threshold`` > 1: 4 rows
    of ``sketch_width(rows)`` uint32 counters that saturate at 2**32 - 1, allocated once.  A training lookup
    counts every owned occurrence of a key without a row (all counts of the table before any insert), and a
    missing key may take a row only when the minimum of its four counters is >= ``threshold``.  With
    ``decay_steps`` P > 0, ``decay`` (called once per training step, after the clock tick) halves every
    counter when the clock is a multiple of P.  ``stats``: counted occurrences and rejected positions.
    Rules in docs/embedding.md; the CPU implementation is the reference."""

    def __init__(self, rows: int, threshold: int, decay_steps: int, clock: torch.Tensor, device):
        self.width = sketch_width(rows)
        self.threshold, self.decay_steps, self.clock = int(threshold), int(decay_steps), clock
        self.device = torch.device(device)
        # uint32 counters stored in int32 words (torch has no general uint32 arithmetic)
        self.counters = torch.zeros(SKETCH_ROWS * self.width, dtype=torch.int32, device=self.device)
        self.stats = torch.zeros(2, dtype=torch.int64, device=self.device)      # counted, rejected

    def view(self):
        return _AdmitSketch(self.counters.data_ptr(), self.stats.data_ptr(), self.width - 1, self.threshold)

    def values(self) -> torch.Tensor:
        """the counters as int64 [4, width] on CPU (host synchronisation)"""
        return (self.counters.cpu().to(torch.int64) & SKETCH_MAX).view(SKETCH_ROWS, self.width)

    def nbytes(self) -> int:
        return self.counters.numel() * self.counters.element_size()

    # ---- CPU rules (the reference the kernels are tested against)
    def _u32(self):
        import numpy as np
        return self.counters.numpy().view(np.uint32)

    def count(self, keys):
        """one occurrence of every key in ``keys`` (a list of missing keys, repeats counted)"""
        import numpy as np
        if not len(keys):
            return
        c = self._u32()
        v = c.astype(np.int64)
        np.add.at(v, sketch_slots(keys, self.width).reshape(-1), 1)
        c[:] = np.minimum(v, SKETCH_MAX).astype(np.uint32)          # saturating adds commute
        self.stats[0] += len(keys)

    def admits(self, keys):
        """bool numpy array: the minimum of each key's counters reaches the threshold"""
        c = self._u32()
        return c[sketch_slots(keys, self.width)].min(axis=1).astype("int64") >= self.threshold

    def decay(self):
        """halve every counter (rounding down) when the clock is a multiple of ``decay_steps`` (no host read
        on CUDA: the kernel tests the clock)"""
        if self.decay_steps <= 0:
            return
        if self.device.type == "cuda":
            if lib().hctr_admit_decay(self.counters.data_ptr(), self.counters.numel(), self.clock.data_ptr(),
                                      self.decay_steps, torch.cuda.current_stream(self.device).cuda_stream):
                raise RuntimeError("hctr_admit_decay failed")
            D._count()
            return
        if int(self.clock[0]) % self.decay_steps == 0:
            c = self._u32()
            c >>= 1
