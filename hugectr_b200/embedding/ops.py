"""Embedding kernels: ctypes bindings for csrc/embedding.cu + PyTorch reference implementations.

The reference implementations define the semantics (they are the CPU path and the test oracle):
  forward   pooled[src, lookup, sample] = combiner( w * table[row_off + key // k] for owned keys ),
            w the key's weight for a weighted lookup, else 1
  backward  per unique arena row: g = sum of bucket gradients times w (scaled 1/nnz for mean);
            then the sparse optimizer of Appendix A.3 on that row.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List

import torch

from .. import _native
from ..enums import Optimizer_t
from ..ops import dense as D
from ..ops.optim import OPT_CODE, COptHyper, opt_hyper, sr_seed
from ..ops.optim import opt_reference as sparse_opt_reference

MAX_RANKS = 16


class CEmbLookup(C.Structure):
    _fields_ = [("table_row_off", C.c_longlong), ("key_off", C.c_longlong),
                ("nnz_off", C.c_longlong), ("out_off", C.c_longlong), ("grad_off", C.c_longlong),
                ("hotness", C.c_int), ("key_stride", C.c_int), ("num_shards", C.c_int),
                ("shard_idx", C.c_int), ("out_stride", C.c_int), ("grad_stride", C.c_int),
                ("combiner", C.c_int), ("ev_size", C.c_int), ("rows", C.c_int), ("weighted", C.c_int),
                ("pair_off", C.c_longlong)]


class CEmbParams(C.Structure):
    _fields_ = [("num_ranks", C.c_int), ("my_rank", C.c_int), ("batch", C.c_int),
                ("num_lookups", C.c_int), ("keys", C.c_void_p * MAX_RANKS),
                ("nnz", C.c_void_p * MAX_RANKS), ("out", C.c_void_p * MAX_RANKS),
                ("grad", C.c_void_p * MAX_RANKS), ("lookups", C.c_void_p), ("table", C.c_void_p),
                ("ev_size", C.c_int), ("weights", C.c_void_p * MAX_RANKS)]


class CUniqueTable(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("vals", C.c_void_p), ("counter", C.c_void_p),
                ("rows", C.c_void_p), ("slots", C.c_void_p), ("mask", C.c_uint),
                ("max_unique", C.c_uint)]


class CBwdIndex(C.Structure):
    _fields_ = [("count", C.c_void_p), ("offsets", C.c_void_p), ("block_sums", C.c_void_p),
                ("pair_uid", C.c_void_p), ("bucket_list", C.c_void_p), ("bucket_scale", C.c_void_p),
                ("heavy_items", C.c_void_p),
                ("heavy_count", C.c_void_p), ("heavy_scratch", C.c_void_p),
                ("heavy_ticket", C.c_void_p), ("heavy_slot", C.c_void_p),
                ("max_heavy_rows", C.c_uint), ("max_heavy_items", C.c_uint),
                ("light_list", C.c_void_p), ("medium_list", C.c_void_p), ("class_count", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        l = _native.cuda_lib()
        vp, i, f, ll = C.c_void_p, C.c_int, C.c_float, C.c_longlong
        l.hctr_emb_forward.argtypes = [C.POINTER(CEmbParams), i, i, i, i, i, vp]
        l.hctr_emb_backward_accum.argtypes = [C.POINTER(CEmbParams), C.POINTER(CUniqueTable), vp, f,
                                              i, i, i, i, vp]
        l.hctr_emb_update.argtypes = [vp, vp, vp, vp, C.POINTER(CUniqueTable), i, i, i,
                                      C.POINTER(COptHyper), vp, i, i, vp]
        l.hctr_emb_gather_rows.argtypes = [vp, vp, vp, ll, i, i, i, vp]
        l.hctr_emb_bwd_index.argtypes = [C.POINTER(CEmbParams), C.POINTER(CUniqueTable),
                                         C.POINTER(CBwdIndex), ll, i, vp]
        l.hctr_emb_bwd_reduce_update.argtypes = [C.POINTER(CEmbParams), C.POINTER(CUniqueTable),
                                                 C.POINTER(CBwdIndex), vp, vp, i, i,
                                                 C.POINTER(COptHyper), f, i, vp, i, i, vp]
        l.hctr_emb_dp_rowwise_update.argtypes = [vp, vp, vp, ll, i, C.POINTER(COptHyper), i, vp]
        for n in ("hctr_emb_forward", "hctr_emb_backward_accum", "hctr_emb_update",
                  "hctr_emb_gather_rows", "hctr_emb_bwd_index", "hctr_emb_bwd_reduce_update",
                  "hctr_emb_dp_rowwise_update"):
            getattr(l, n).restype = i
        # ABI self-check: ctypes mirrors vs the structs the kernels were compiled with
        if hasattr(l, "hctr_abi_sizes_emb"):
            sz = (C.c_int * 8)()
            l.hctr_abi_sizes_emb(sz)
            mine = [C.sizeof(CEmbLookup), C.sizeof(CEmbParams), C.sizeof(CUniqueTable),
                    C.sizeof(CBwdIndex), C.sizeof(COptHyper)]
            if list(sz[:5]) != mine:
                raise RuntimeError(f"libhctr_cuda.so struct layout {list(sz[:5])} != python mirrors {mine}: "
                                   "rebuild the library (python -m hugectr_b200._native)")
        _lib = l
    return _lib


@dataclass
class LookupDesc:
    """Python mirror of EmbLookup (one owner-side lookup)."""
    table_row_off: int
    key_off: int
    out_off: int
    grad_off: int
    hotness: int
    key_stride: int
    num_shards: int
    shard_idx: int
    out_stride: int
    grad_stride: int
    combiner: int
    ev_size: int
    rows: int
    nnz_off: int = -1
    pair_off: int = 0
    weighted: int = 0    # 1: every key has an fp32 weight at the same element offset of the weight buffers

    def to_c(self) -> CEmbLookup:
        return CEmbLookup(self.table_row_off, self.key_off, self.nnz_off, self.out_off,
                          self.grad_off, self.hotness, self.key_stride, self.num_shards,
                          self.shard_idx, self.out_stride, self.grad_stride, self.combiner,
                          self.ev_size, self.rows, int(self.weighted), self.pair_off)


def lookups_to_device(lookups: List[LookupDesc], device) -> torch.Tensor:
    arr = (CEmbLookup * max(1, len(lookups)))()
    for i, l in enumerate(lookups):
        arr[i] = l.to_c()
    raw = bytes(arr)
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8).clone()
    return t.to(device)


def _st(dev):
    return torch.cuda.current_stream(dev).cuda_stream


# widest embedding row the CUDA lookup / accumulate / fused-update kernels cover (kMaxEmbWidth in
# csrc/embedding.cuh); wider tables are rejected rather than truncated
MAX_EV_SIZE = 1024


def check_ev_size(ev_size: int, what: str = "embedding vector"):
    if ev_size > MAX_EV_SIZE:
        raise ValueError(f"{what} size {ev_size} exceeds the widest row the embedding kernels support "
                         f"({MAX_EV_SIZE}); split the table's columns (column-wise sharding) or use a "
                         f"narrower ev_size")


def vec4_aligned(lookups, ev_pitch, bufs=(), grad: bool = True) -> bool:
    """True when the kernels may move 4 consecutive elements as one vector for every lookup: ev_size,
    pitch and the gradient (``grad``) or output offsets and strides are multiples of 4 elements and
    every base pointer in ``bufs`` (tensors or int device pointers) is 16-byte aligned.  Collections
    that concatenate a narrow table in front of another one (column 6 of a 134-wide top), or odd
    batches behind a width-6 top, break this; the kernels then take their scalar paths."""
    def ptr(b):
        return b if isinstance(b, int) else b.data_ptr()
    if ev_pitch % 4:
        return False
    for l in lookups:
        off, stride = (l.grad_off, l.grad_stride) if grad else (l.out_off, l.out_stride)
        if l.ev_size % 4 or off % 4 or stride % 4:
            return False
    return all(ptr(b) % 16 == 0 for b in bufs if b is not None)


# ----------------------------------------------------------------------------- dispatch (peer stores)
class CDispatchRoute(C.Structure):
    _fields_ = [("src_off", C.c_longlong), ("dst_off", C.c_longlong), ("nnz_off", C.c_longlong),
                ("rows", C.c_int), ("row_elems", C.c_int), ("src_stride", C.c_int),
                ("dst_stride", C.c_int), ("dst_rank", C.c_int), ("kind", C.c_int), ("k", C.c_int),
                ("shard", C.c_int)]


@dataclass
class Route:
    """One block a rank sends to one destination rank's inbox (csrc/emb_dispatch.cu).  kind 0: 2-D
    copy of [rows, row_elems]; kind 1: key-bag split for shard ``shard`` of ``k`` (+ list lengths)."""
    src_off: int
    dst_off: int
    rows: int
    row_elems: int
    src_stride: int
    dst_stride: int
    dst_rank: int
    kind: int = 0
    k: int = 1
    shard: int = 0
    nnz_off: int = 0


def routes_to_device(routes: List[Route], device) -> torch.Tensor:
    arr = (CDispatchRoute * max(1, len(routes)))()
    for i, r in enumerate(routes):
        arr[i] = CDispatchRoute(r.src_off, r.dst_off, r.nnz_off, r.rows, r.row_elems, r.src_stride,
                                r.dst_stride, r.dst_rank, r.kind, r.k, r.shard)
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).clone().to(device)


def dispatch(src: torch.Tensor, routes: List[Route], routes_dev, dst_bufs, nnz_bufs=None, blocks_x: int = 8):
    """Scatter blocks of the local 1-D buffer ``src`` into the per-rank inboxes ``dst_bufs`` (tensor or
    int peer pointer per destination rank; element type of ``src``).  Posted peer stores on CUDA."""
    if not routes:
        return
    if src.is_cuda:
        l = lib()
        if not hasattr(l, "_dispatch_ready"):
            l.hctr_emb_dispatch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_void_p),
                                            C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_void_p]
            l.hctr_emb_dispatch.restype = C.c_int
            if l.hctr_abi_size_dispatch_route() != C.sizeof(CDispatchRoute):
                raise RuntimeError("libhctr_cuda.so DispatchRoute layout differs from the python mirror: rebuild")
            l._dispatch_ready = True
        n = len(dst_bufs)
        dp = (C.c_void_p * n)(*[d if isinstance(d, int) else d.data_ptr() for d in dst_bufs])
        np_ = None
        if nnz_bufs is not None:
            np_ = (C.c_void_p * n)(*[d if isinstance(d, int) else d.data_ptr() for d in nnz_bufs])
        rc = l.hctr_emb_dispatch(src.data_ptr(), routes_dev.data_ptr(), len(routes), dp, np_, n,
                                 src.element_size(), blocks_x, _st(src.device))
        if rc:
            raise RuntimeError(f"hctr_emb_dispatch failed rc={rc}")
        D._count()
        return
    for r in routes:
        dst = dst_bufs[r.dst_rank].reshape(-1)
        if r.kind == 0:
            s2 = torch.as_strided(src, (r.rows, r.row_elems), (r.src_stride, 1), src.storage_offset() + r.src_off)
            d2 = torch.as_strided(dst, (r.rows, r.row_elems), (r.dst_stride, 1), dst.storage_offset() + r.dst_off)
            d2.copy_(s2)
            continue
        keys = torch.as_strided(src, (r.rows, r.row_elems), (r.src_stride, 1),
                                src.storage_offset() + r.src_off).long()
        m = (keys >= 0) & (keys % r.k == r.shard)
        order = torch.argsort((~m).to(torch.int8), dim=1, stable=True)
        rows = torch.div(keys, r.k, rounding_mode="floor").gather(1, order)
        cnt = m.sum(1)
        pos = torch.arange(r.row_elems).view(1, -1)
        d2 = torch.as_strided(dst, (r.rows, r.row_elems), (r.dst_stride, 1), dst.storage_offset() + r.dst_off)
        d2.copy_(torch.where(pos < cnt.view(-1, 1), rows, torch.full_like(rows, -1)).to(dst.dtype))
        nn = nnz_bufs[r.dst_rank].reshape(-1)
        nn[r.nnz_off:r.nnz_off + r.rows].copy_(cnt.to(torch.int32))


# ----------------------------------------------------------------------------- forward
def _params(lookups, lookups_dev, table, ev_pitch, key_bufs, batch, my_rank, key_bytes, act_bf16,
            nnz_bufs=None, weight_bufs=None, out_bufs=None, grad_bufs=None):
    """CEmbParams of a launch over one source rank per entry of ``key_bufs`` (tensors, or int device
    pointers for peers), with the key width and whether the outputs / gradients are bf16: read from the
    buffers that are tensors, ``key_bytes`` / ``act_bf16`` where every one is a pointer.  The weight
    pointers stay null without a weighted lookup (the kernels' unweighted instantiations)."""
    def ptr(x):
        return x if isinstance(x, int) else x.data_ptr()
    p = CEmbParams()
    p.num_ranks, p.my_rank, p.batch, p.num_lookups = len(key_bufs), my_rank, batch, len(lookups)
    kb, abf = key_bytes, int(act_bf16)
    weighted = weight_bufs is not None and any(l.weighted for l in lookups)
    for r, k in enumerate(key_bufs):
        p.keys[r] = ptr(k)
        if not isinstance(k, int):
            kb = k.element_size()
        if nnz_bufs is not None:
            p.nnz[r] = ptr(nnz_bufs[r])
        if weighted:
            p.weights[r] = ptr(weight_bufs[r])
        for dst, bufs in ((p.out, out_bufs), (p.grad, grad_bufs)):
            if bufs is not None:
                dst[r] = ptr(bufs[r])
                if not isinstance(bufs[r], int):
                    abf = int(bufs[r].dtype == torch.bfloat16)
    p.lookups = lookups_dev.data_ptr()
    p.table = table.data_ptr()
    p.ev_size = ev_pitch
    return p, kb, abf


def _key_weights(lk, weight_bufs, src, batch, own):
    """[batch, hotness] fp32 weights of the owned keys of lookup ``lk`` (1 for an unweighted lookup,
    0 where a key is not owned, whatever the stored weight)"""
    if not lk.weighted:
        return own.float()
    wbuf = weight_bufs[src].reshape(-1)
    w = torch.as_strided(wbuf, (batch, lk.hotness), (lk.key_stride, 1), wbuf.storage_offset() + lk.key_off)
    return torch.where(own, w.float(), torch.zeros((), device=w.device))


def forward(lookups, lookups_dev, table, ev_pitch, key_bufs, out_bufs, batch, my_rank=0,
            nnz_bufs=None, key_bytes=4, act_bf16=True, weight_bufs=None):
    """key_bufs / out_bufs (/ weight_bufs, fp32 per-key weights of weighted lookups): one entry per
    source rank (tensor, or int device pointer for peers)."""
    if table.is_cuda:
        p, kb, out_bf16 = _params(lookups, lookups_dev, table, ev_pitch, key_bufs, batch, my_rank, key_bytes,
                                  act_bf16, nnz_bufs, weight_bufs, out_bufs=out_bufs)
        max_ev = max((l.ev_size for l in lookups), default=ev_pitch)
        check_ev_size(max_ev)
        al4 = int(vec4_aligned(lookups, ev_pitch, [table, *out_bufs], grad=False))
        rc = lib().hctr_emb_forward(C.byref(p), max_ev, kb, out_bf16, al4, table_bf16(table),
                                    _st(table.device))
        if rc:
            raise RuntimeError(f"hctr_emb_forward failed rc={rc}")
        D._count()
        return
    forward_reference(lookups, table, ev_pitch, key_bufs, out_bufs, batch, nnz_bufs, weight_bufs)


def _bag(lk: LookupDesc, key_bufs, nnz_bufs, src, batch):
    """(owned [batch, hotness], arena rows, bag lengths [batch]) of lookup ``lk`` over source rank
    ``src``'s keys: a key is owned when valid, of this shard, inside the table and -- for a split list
    -- inside its bag length"""
    kbuf = key_bufs[src].reshape(-1)
    keys = torch.as_strided(kbuf, (batch, lk.hotness), (lk.key_stride, 1), kbuf.storage_offset() + lk.key_off).long()
    own = keys >= 0
    if lk.num_shards > 1:
        own &= (keys % lk.num_shards) == lk.shard_idx
    r = torch.div(keys, lk.num_shards, rounding_mode="floor")
    own &= r < lk.rows
    nnz = torch.full((batch,), lk.hotness, device=keys.device)
    if lk.nnz_off >= 0 and nnz_bufs is not None:
        nnz = nnz_bufs[src].reshape(-1)[lk.nnz_off:lk.nnz_off + batch].long().clamp(max=lk.hotness)
        own &= torch.arange(lk.hotness, device=keys.device).view(1, -1) < nnz.view(-1, 1)
    return own, lk.table_row_off + torch.where(own, r, torch.zeros_like(r)), nnz


def forward_reference(lookups, table, ev_pitch, key_bufs, out_bufs, batch, nnz_bufs=None, weight_bufs=None):
    tab = table.view(-1, ev_pitch)
    for src in range(len(key_bufs)):
        obuf = out_bufs[src].reshape(-1)
        for lk in lookups:
            own, rows, nnz = _bag(lk, key_bufs, nnz_bufs, src, batch)
            v = tab[rows][..., :lk.ev_size].float() * _key_weights(lk, weight_bufs, src, batch, own).unsqueeze(-1)
            pooled = v.sum(1)
            if lk.combiner == 1:
                pooled = pooled / nnz.clamp(min=1).view(-1, 1).float()
            o = torch.as_strided(obuf, (batch, lk.ev_size), (lk.out_stride, 1),
                                 obuf.storage_offset() + lk.out_off)
            o.copy_(pooled.to(o.dtype))


# ----------------------------------------------------------------------------- backward
HEAVY_MIN_COUNT = 65   # occurrences in one step from which a row is reduced block-per-chunk (kHeavy + 1)


class UniqueWorkspace:
    """Transient hash + fp32 per-unique-row gradient accumulator (device)."""

    def __init__(self, max_pairs: int, ev_pitch: int, device, unique_ratio: float = 1.0,
                 indexed: bool = False, need_scale: bool = False, max_heavy_rows: int = None,
                 max_heavy_items: int = None):
        """``max_heavy_rows`` / ``max_heavy_items`` (indexed path) size the scratch rows and the
        512-entry chunk work items of the block-per-chunk kernel for rows with more than 64
        occurrences in a step; heavy rows beyond them, and rows of more than 4096 chunks, are
        reduced by the warp-per-row kernel (correct, but one warp per row).  By default they are
        sized from ``max_pairs`` so that every heavy row fits -- at most max_pairs / 65 rows and
        max_pairs / 512 + rows chunks -- with the scratch rows capped at 64 MiB (and >= 8192)."""
        self.device = device
        self.ev = ev_pitch
        self.max_unique = max(16, int(max_pairs * unique_ratio))
        cap = 1
        while cap < 2 * self.max_unique:
            cap <<= 1
        self.capacity = cap
        if device.type == "cuda":
            self.keys = torch.full((cap,), -1, dtype=torch.int64, device=device)
            self.vals = torch.full((cap,), -1, dtype=torch.int32, device=device)
            self.counter = torch.zeros(1, dtype=torch.int32, device=device)
            self.rows = torch.zeros(self.max_unique, dtype=torch.int64, device=device)
            self.slots = torch.zeros(self.max_unique, dtype=torch.int32, device=device)
            self.wgrad = None if indexed else torch.zeros(self.max_unique, ev_pitch,
                                                          dtype=torch.float32, device=device)
            self.overflow = torch.zeros(1, dtype=torch.int32, device=device)
            self.c = CUniqueTable(self.keys.data_ptr(), self.vals.data_ptr(),
                                  self.counter.data_ptr(), self.rows.data_ptr(),
                                  self.slots.data_ptr(), cap - 1, self.max_unique)
            self.indexed = indexed
            if indexed:
                # counting-sort index (csrc/embedding_bwd.cu); the fp32 per-row accumulator is
                # not needed on this path
                self.wgrad = None
                mu, mp = self.max_unique, max(int(max_pairs), 1)
                i32 = dict(dtype=torch.int32, device=device)
                self.count = torch.zeros(mu, **i32)
                self.offsets = torch.zeros(mu + 1, **i32)
                self.block_sums = torch.zeros((mu + 1023) // 1024 + 1, **i32)
                self.pair_uid = torch.full((mp,), -1, **i32)
                self.bucket_list = torch.zeros(mp, **i32)
                self.bucket_scale = torch.ones(mp, dtype=torch.float32, device=device) if need_scale else None
                if max_heavy_rows is None:
                    max_heavy_rows = min(max(mp // HEAVY_MIN_COUNT, 1),
                                         max(8192, (1 << 24) // max(ev_pitch, 1)), 1 << 20)
                if max_heavy_items is None:
                    max_heavy_items = mp // 512 + max_heavy_rows
                if not 1 <= max_heavy_rows <= (1 << 20) or max_heavy_items < 1:
                    raise ValueError("max_heavy_rows must be in [1, 2^20] and max_heavy_items >= 1")
                self.max_heavy_rows = int(max_heavy_rows)
                self.max_heavy_items = int(max_heavy_items)
                self.heavy_items = torch.zeros(2 * self.max_heavy_items, **i32)
                self.heavy_count = torch.zeros(1, **i32)
                self.heavy_slot = torch.zeros(1, **i32)
                self.heavy_scratch = torch.zeros(self.max_heavy_rows, ev_pitch, dtype=torch.float32,
                                                 device=device)
                self.heavy_ticket = torch.zeros(self.max_heavy_rows, **i32)
                self.light_list = torch.zeros(2 * mu, **i32)
                self.medium_list = torch.zeros(2 * mu, **i32)
                self.class_count = torch.zeros(2, **i32)
                self.ix = CBwdIndex(self.count.data_ptr(), self.offsets.data_ptr(),
                                    self.block_sums.data_ptr(), self.pair_uid.data_ptr(),
                                    self.bucket_list.data_ptr(),
                                    0 if self.bucket_scale is None else self.bucket_scale.data_ptr(),
                                    self.heavy_items.data_ptr(),
                                    self.heavy_count.data_ptr(), self.heavy_scratch.data_ptr(),
                                    self.heavy_ticket.data_ptr(), self.heavy_slot.data_ptr(),
                                    self.max_heavy_rows, self.max_heavy_items,
                                    self.light_list.data_ptr(), self.medium_list.data_ptr(),
                                    self.class_count.data_ptr())
        else:
            self.ref_rows = None
            self.ref_grads = None


def check_workspace_overflow(ws, what: str):
    """Raise if a backward step found more distinct rows than ``ws`` holds (their updates were
    dropped).  Reads the workspace's sticky device flag: a host sync."""
    flag = getattr(ws, "overflow", None)
    if flag is not None and int(flag.item()) != 0:
        raise RuntimeError(f"embedding backward workspace of {what} overflowed: "
                           f"{int(flag.item()) & 0xFFFFFFFF} distinct rows in one step, room for "
                           f"{ws.max_unique}")


def backward_accum(lookups, lookups_dev, table, ev_pitch, key_bufs, grad_bufs, batch, ws, grad_scale=1.0,
                   my_rank=0, nnz_bufs=None, dense_wgrad=None, key_bytes=4, act_bf16=True, weight_bufs=None):
    """Accumulate bucket gradients (times the key's weight for weighted lookups) per unique row (or
    into a dense wgrad for DP tables)."""
    if table.is_cuda:
        p, kb, gbf = _params(lookups, lookups_dev, table, ev_pitch, key_bufs, batch, my_rank, key_bytes, act_bf16,
                             nnz_bufs, weight_bufs, grad_bufs=grad_bufs)
        max_ev = max((l.ev_size for l in lookups), default=ev_pitch)
        if dense_wgrad is not None:
            ut = CUniqueTable(0, 0, 0, 0, 0, 0, 0xFFFFFFFF)
            dst = dense_wgrad.data_ptr()
        else:
            ut, dst = ws.c, ws.wgrad.data_ptr()
        if dense_wgrad is None:
            check_ev_size(max_ev)
        ev4 = int(vec4_aligned(lookups, ev_pitch, [dst, *grad_bufs], grad=True))
        rc = lib().hctr_emb_backward_accum(C.byref(p), C.byref(ut), dst, float(grad_scale), max_ev,
                                           kb, gbf, ev4, _st(table.device))
        if rc:
            raise RuntimeError(f"hctr_emb_backward_accum failed rc={rc}")
        D._count()
        return
    rows_all, grads_all = [], []
    for src in range(len(key_bufs)):
        gbuf = grad_bufs[src].reshape(-1)
        for lk in lookups:
            own, rows, nnz = _bag(lk, key_bufs, nnz_bufs, src, batch)
            g = torch.as_strided(gbuf, (batch, lk.ev_size), (lk.grad_stride, 1),
                                 gbuf.storage_offset() + lk.grad_off)
            g = g.float() * grad_scale
            if lk.combiner == 1:
                g = g / nnz.clamp(min=1).view(-1, 1).float()
            gg = g.unsqueeze(1).expand(batch, lk.hotness, lk.ev_size)
            if lk.weighted:
                gg = gg * _key_weights(lk, weight_bufs, src, batch, own).unsqueeze(-1)
            gg = gg[own]
            if lk.ev_size < ev_pitch:
                gg = torch.nn.functional.pad(gg, (0, ev_pitch - lk.ev_size))
            rows_all.append(rows[own])
            grads_all.append(gg)
    rows = torch.cat(rows_all) if rows_all else torch.zeros(0, dtype=torch.long)
    grads = torch.cat(grads_all) if grads_all else torch.zeros(0, ev_pitch)
    if dense_wgrad is not None:
        dense_wgrad.view(-1, ev_pitch).index_add_(0, rows, grads)
        return
    if ws.ref_rows is not None:
        rows = torch.cat([ws.ref_rows, rows])
        grads = torch.cat([ws.ref_grads, grads])
    ws.ref_rows, ws.ref_grads = rows, grads


# ----------------------------------------------------------------------------- bf16 weights
def table_bf16(table) -> int:
    """1 when the arena stores bf16 weights (the kernels' WT = __nv_bfloat16), 0 for fp32"""
    if table.dtype not in (torch.float32, torch.bfloat16):
        raise TypeError(f"embedding tables are fp32 or bf16, not {table.dtype}")
    return int(table.dtype == torch.bfloat16)


_M64 = (1 << 64) - 1


def _fmix64(k):
    """MurmurHash3 64-bit finaliser on uint64 numpy arrays (fmix64 in csrc/embedding.cuh)"""
    import numpy as np
    with np.errstate(over="ignore"):
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(0xff51afd7ed558ccd)
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(0xc4ceb9fe1a85ec53)
        return k ^ (k >> np.uint64(33))


def sr_step_key(seed: int, step: int) -> int:
    """per-(seed, step) key of the stochastic rounding (sr_step_key in csrc/embedding.cuh)"""
    import numpy as np
    k = np.array([((int(seed) & 0xFFFFFFFF) << 32) | (int(step) & 0xFFFFFFFF)], dtype=np.uint64)
    return int(_fmix64(k)[0])


def sr_bits(key: int, idx):
    """the 16 random bits r of the elements at arena indices ``idx`` (int tensor / array of
    row * pitch + col) under the step key ``key``: 16-bit lane idx % 4 of fmix64(key ^ idx // 4)
    (one hash per four consecutive elements); uint32 numpy array in [0, 65536)"""
    import numpy as np
    i = np.asarray(idx.cpu().numpy() if torch.is_tensor(idx) else idx, dtype=np.int64).astype(np.uint64)
    h = _fmix64(np.uint64(key & _M64) ^ (i >> np.uint64(2)))
    return ((h >> (np.uint64(16) * (i & np.uint64(3)))) & np.uint64(0xFFFF)).astype(np.uint32)


def sr_round_bf16(x, seed: int, step: int, idx):
    """bf16 values of the fp32 tensor ``x`` stored with stochastic rounding, bit for bit as the
    kernels store a bf16 weight: the upper 16 bits of (fp32 bits + r), r = sr_bits of (seed, step,
    arena index ``idx``, same shape as ``x``); inf / NaN round to nearest.  Unbiased: the expected
    stored value is ``x``."""
    import numpy as np
    xf = x.detach().float().contiguous()
    b = xf.cpu().numpy().view(np.uint32).reshape(-1)
    r = sr_bits(sr_step_key(seed, step), torch.as_tensor(idx).reshape(-1))
    out = ((b.astype(np.uint64) + r) >> np.uint64(16)).astype(np.uint16)
    res = torch.from_numpy(out.view(np.int16).copy()).view(torch.bfloat16).view(xf.shape)
    special = torch.from_numpy((b & 0x7f800000) == 0x7f800000).view(xf.shape)
    if bool(special.any()):
        res = torch.where(special, xf.cpu().to(torch.bfloat16), res)
    return res.to(x.device)


def evict_init_key(seed: int, table_id: int) -> int:
    """key of the stateless initializer of an evicting table's admitted rows (EvictReinit::init_key)"""
    return sr_step_key(seed, table_id)


def evict_init_rows(init_key: int, keys, col0: int, width: int, bound: float, dtype=torch.float32):
    """initial weights [n, width] of the admitted ``keys`` of an evicting table, bit for bit as
    evict_init_value in csrc/evict_table.cu: bound * (2u - 1) in fp32, u = the top 24 bits of
    fmix64(fmix64(init_key ^ key) ^ global column) / 2^24; a bf16 arena rounds to nearest"""
    import numpy as np
    k = np.asarray(keys.cpu().numpy() if torch.is_tensor(keys) else keys, dtype=np.int64).astype(np.uint64)
    cols = np.arange(col0, col0 + width, dtype=np.uint64)
    h = _fmix64(_fmix64(np.uint64(init_key & _M64) ^ k)[:, None] ^ cols[None, :])
    u = (h >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    w = np.float32(bound) * (np.float32(2.0) * u - np.float32(1.0))
    return torch.from_numpy(w.astype(np.float32)).to(dtype)


def update(opt: Optimizer_t, table, s0, s1, ev_pitch, ws: UniqueWorkspace, hp: dict, lr_t, step_t,
           num_sms: int = 132):
    """Fused per-unique-row optimizer; consumes and clears the workspace."""
    if table.is_cuda:
        h = opt_hyper(hp, lr_t, step_t)
        sbf = int(s0 is not None and s0.dtype == torch.bfloat16)
        rc = lib().hctr_emb_update(table.data_ptr(), 0 if s0 is None else s0.data_ptr(),
                                   0 if s1 is None else s1.data_ptr(), ws.wgrad.data_ptr(),
                                   C.byref(ws.c), ev_pitch, OPT_CODE[opt], sbf, C.byref(h),
                                   ws.overflow.data_ptr(), num_sms, table_bf16(table),
                                   _st(table.device))
        if rc:
            raise RuntimeError("hctr_emb_update failed")
        D._count(2)
        return
    if ws.ref_rows is None or ws.ref_rows.numel() == 0:
        ws.ref_rows = ws.ref_grads = None
        return
    update_rows(opt, table, s0, s1, ev_pitch, ws.ref_rows, ws.ref_grads, hp, lr_t, step_t)
    ws.ref_rows = ws.ref_grads = None


def update_rows(opt: Optimizer_t, table, s0, s1, ev_pitch, rows, grads, hp: dict, lr_t, step_t):
    """One optimizer application per DISTINCT row (``rows`` [n] may repeat, ``grads`` [n, pitch] fp32 are
    summed per row first).  Plain tensor ops on the tables' device: the CPU path of ``update`` and the
    owner side of the Unique-compression exchange (embedding/unique_exchange.py).  A bf16 table is
    updated in fp32 and stored with the kernels' stochastic rounding (sr_round_bf16)."""
    if rows.numel() == 0:
        return
    uniq, inv = torch.unique(rows, return_inverse=True)
    g = torch.zeros(uniq.numel(), ev_pitch, dtype=torch.float32, device=grads.device).index_add_(0, inv, grads.float())
    tab = table.view(-1, ev_pitch)
    w = tab[uniq].float().clone()
    # row-wise state: s0 [rows], one accumulator per row
    rowwise = opt == Optimizer_t.RowWiseAdaGrad
    spitch = 1 if rowwise else ev_pitch
    a = None if s0 is None else s0.view(-1, spitch)[uniq].float().clone()
    b = None if s1 is None else s1.view(-1, ev_pitch)[uniq].float().clone()
    if rowwise and a is not None:
        a = a.view(-1)
    step = int(step_t.item())
    sparse_opt_reference(opt, w, a, b, g, hp, float(lr_t.item()), step)
    if table_bf16(table):
        idx = uniq.view(-1, 1) * ev_pitch + torch.arange(ev_pitch, device=uniq.device).view(1, -1)
        w = sr_round_bf16(w, sr_seed(hp), step, idx)
    tab[uniq] = w
    if a is not None:
        s0.view(-1, spitch)[uniq] = a.view(-1, spitch).to(s0.dtype)
    if b is not None:
        s1.view(-1, ev_pitch)[uniq] = b.to(s1.dtype)


def dp_rowwise_update(table, s0, wgrad, pitch, hp: dict, lr_t, num_sms: int = 132):
    """Row-wise AdaGrad of a data-parallel table from its all-reduced dense gradient ``wgrad``
    ([rows * pitch] fp32, zeroed on return): every row takes the row rule; an all-zero row keeps its
    weights and accumulator (``s0`` [rows] fp32)."""
    rows = table.numel() // pitch
    if table.is_cuda:
        h = opt_hyper(hp, lr_t, None)
        rc = lib().hctr_emb_dp_rowwise_update(table.data_ptr(), s0.data_ptr(), wgrad.data_ptr(), rows,
                                              pitch, C.byref(h), num_sms, _st(table.device))
        if rc:
            raise RuntimeError(f"hctr_emb_dp_rowwise_update failed rc={rc}")
        D._count()
        return
    g = wgrad[:rows * pitch].view(rows, pitch)
    w = table.view(rows, pitch).clone()
    a = s0.clone()
    sparse_opt_reference(Optimizer_t.RowWiseAdaGrad, w, a, None, g.clone(), hp, float(lr_t.item()), 1)
    table.view(rows, pitch).copy_(w)
    s0.copy_(a)
    wgrad.zero_()


def gather_rows(table, ev_pitch, rows, out):
    """out[i] = table[rows[i]] (rows < 0 -> zeros)."""
    if table.is_cuda and rows.dtype == torch.int64:
        rc = lib().hctr_emb_gather_rows(table.data_ptr(), rows.data_ptr(), out.data_ptr(),
                                        rows.numel(), ev_pitch, int(out.dtype == torch.bfloat16),
                                        table_bf16(table), _st(table.device))
        if rc:
            raise RuntimeError("hctr_emb_gather_rows failed")
        D._count()
        return
    v = table.view(-1, ev_pitch)[rows.clamp(min=0)] * (rows >= 0).unsqueeze(-1)
    out.copy_(v.to(out.dtype))


def bwd_index(lookups, lookups_dev, table, ev_pitch, key_bufs, batch, ws, my_rank=0, nnz_bufs=None,
              key_bytes=4, weight_bufs=None):
    """Gradient-independent part of the backward: unique rows + per-row bucket lists (with the
    per-entry scales: 1/nnz of mean bags, times the key's weight of weighted lookups)."""
    check_ev_size(ev_pitch)
    if not vec4_aligned(lookups, ev_pitch, [table], grad=True):
        raise ValueError("the fused backward needs 4-element aligned gradient rows and pitch "
                         "(see vec4_aligned); use backward_accum + update")
    if any(l.weighted for l in lookups) and (weight_bufs is None or ws.bucket_scale is None):
        raise ValueError("weighted lookups need their weight buffers and a workspace built with need_scale")
    p, kb, _ = _params(lookups, lookups_dev, table, ev_pitch, key_bufs, batch, my_rank, key_bytes, True,
                       nnz_bufs, weight_bufs)
    total_pairs = len(key_bufs) * batch * sum(l.hotness for l in lookups)
    rc = lib().hctr_emb_bwd_index(C.byref(p), C.byref(ws.c), C.byref(ws.ix), total_pairs, kb,
                                  _st(table.device))
    if rc:
        raise RuntimeError("hctr_emb_bwd_index failed")
    D._count(6)


def bwd_reduce_update(opt: Optimizer_t, lookups, lookups_dev, table, s0, s1, ev_pitch, key_bufs,
                      grad_bufs, batch, ws, hp: dict, lr_t, step_t, grad_scale=1.0, my_rank=0,
                      nnz_bufs=None, num_sms: int = 132, key_bytes=4, act_bf16=True):
    """Fused gradient gather (local / peer loads) + duplicate reduction + optimizer."""
    check_ev_size(ev_pitch)
    if not vec4_aligned(lookups, ev_pitch, [table, *grad_bufs], grad=True):
        raise ValueError("the fused backward needs 4-element aligned gradient rows and pitch "
                         "(see vec4_aligned); use backward_accum + update")
    p, kb, gbf = _params(lookups, lookups_dev, table, ev_pitch, key_bufs, batch, my_rank, key_bytes, act_bf16,
                         nnz_bufs, grad_bufs=grad_bufs)
    h = opt_hyper(hp, lr_t, step_t)
    sbf = int(s0 is not None and s0.dtype == torch.bfloat16)
    rc = lib().hctr_emb_bwd_reduce_update(C.byref(p), C.byref(ws.c), C.byref(ws.ix),
                                          0 if s0 is None else s0.data_ptr(),
                                          0 if s1 is None else s1.data_ptr(), OPT_CODE[opt], sbf,
                                          C.byref(h), float(grad_scale), gbf, ws.overflow.data_ptr(),
                                          num_sms, table_bf16(table), _st(table.device))
    if rc:
        raise RuntimeError(f"hctr_emb_bwd_reduce_update failed rc={rc}")
    D._count(3)
