"""Parquet reader (C12): file list + _metadata.json schema, worker threads decode row groups with
pyarrow into the common feature-major HostBatch; label/dense float32, categorical columns int64
scalars (one-hot) or lists (multi-hot).  ``slot_size_array`` adds per-slot key offsets so one hash
table can hold all slots (HugeCTR/src/pybind/add_input.cpp:314-318,
docs/source/api/python_interface.md:397-473).  Reference pipeline: DataReader<T> +
DataReaderWorkerGroupParquet (HugeCTR/src/data_readers/*.cpp) with cuDF decode; here decode is on
CPU worker threads (no cuDF in this environment) and the batch lands in pinned memory.
"""
from __future__ import annotations

import json
import os
import queue
import threading

import numpy as np
import torch

from .batch import HostBatch
from .readers import IDataReader


def read_file_list(path: str):
    with open(path) as f:
        lines = [l.strip() for l in f if l.strip()]
    n = int(lines[0])
    files = lines[1:1 + n]
    if len(files) != n:
        raise RuntimeError(f"file list {path} announces {n} files but lists {len(files)}")
    return files


def _csr_to_padded(offs, vals, n, H, add, blk, s, nz):
    """blk[i, s, :min(len_i, H)] = vals[offs[i]:...] + add ; nz[s, i] = min(len_i, H)  (native, OpenMP)"""
    import ctypes as C
    from .. import _native
    L = _native.host_lib()
    L.hctr_csr_to_padded.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_longlong,
                                     C.c_void_p, C.c_longlong, C.c_void_p]
    offs = np.ascontiguousarray(offs)
    if offs.dtype not in (np.int32, np.int64):
        offs = offs.astype(np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.int64)
    S, Hb = blk.shape[1], blk.shape[2]
    L.hctr_csr_to_padded(offs.ctypes.data, offs.dtype.itemsize, vals.ctypes.data, int(n), int(H), int(add),
                         blk.ctypes.data + 8 * s * Hb, S * Hb, nz.ctypes.data + 4 * s * nz.shape[1])


def _csr_to_padded_f32(offs, vals, n, H, wblk, s):
    """wblk[i, s, :min(len_i, H)] = vals[offs[i]:...]: the weights of a multi-hot slot where _csr_to_padded puts
    its keys (native, OpenMP)"""
    import ctypes as C
    from .. import _native
    L = _native.host_lib()
    L.hctr_csr_to_padded_f32.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                         C.c_longlong]
    offs = np.ascontiguousarray(offs)
    if offs.dtype not in (np.int32, np.int64):
        offs = offs.astype(np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.float32)
    S, Hb = wblk.shape[1], wblk.shape[2]
    L.hctr_csr_to_padded_f32(offs.ctypes.data, offs.dtype.itemsize, vals.ctypes.data, int(n), int(H),
                             wblk.ctypes.data + 4 * s * Hb, S * Hb)


def _onehot_block(cols, add, lo, nloc, b, blk, nz):
    """blk[i, s, 0] = cols[s][lo + i] + add[s] (i < nloc; -1 behind), nz[s, i] = 1 / 0 -- native, GIL released"""
    import ctypes as C
    from .. import _native
    L = _native.host_lib()
    L.hctr_onehot_block.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_longlong, C.c_longlong,
                                    C.c_longlong, C.c_void_p, C.c_int, C.c_void_p]
    S = len(cols)
    cols = [np.ascontiguousarray(c, dtype=np.int64) for c in cols]
    ptrs = (C.c_void_p * S)(*[c.ctypes.data for c in cols])
    addp = None
    if add is not None:
        add = np.ascontiguousarray(add, dtype=np.int64)
        addp = add.ctypes.data
    L.hctr_onehot_block(ptrs, addp, S, int(lo), int(nloc), int(b), blk.ctypes.data, blk.dtype.itemsize,
                        nz.ctypes.data)


class ParquetReader(IDataReader):
    def __init__(self, model, is_train: bool):
        rp = model.reader_params
        b = model.b_train if is_train else model.b_eval
        super().__init__(b, model.comm.rank, model.world, repeat=model.solver.repeat_dataset)
        self.file_list = rp.source[0] if is_train else rp.eval_source
        self.inp = model.input
        self.layout = model.layout
        self.key_dtype = model.key_dtype
        self.slot_offsets = None
        n_slots = model.layout.total_slots
        if rp.slot_size_array and len(rp.slot_size_array) >= n_slots and model.sparse_embeddings:
            self.slot_offsets = np.concatenate([[0], np.cumsum(rp.slot_size_array[:n_slots])[:-1]]).astype("int64")
        self.num_workers = max(1, min(int(rp.num_workers), 8))      # row-group decode threads
        self.q: "queue.Queue" = queue.Queue(maxsize=4)
        self.thread = None
        self._stop = threading.Event()
        # the incomplete last batch of an epoch is always DELIVERED (evaluation counts every sample; for training
        # `Solver.drop_incomplete_batch` is applied by Model._train_step, like for the Raw / Norm readers)
        self.drop_incomplete = False
        self._device = getattr(model, "device", None)
        # per block: does the input carry weights (weight_index columns of its slots)
        self.weighted = list(getattr(self.layout, "weighted", None) or [False] * len(self.layout.blocks))
        if any(self.weighted):
            self._columns(read_file_list(self.file_list))     # a weighted slot without a weight column raises here

    # -------------------------------------------------------------- producer
    def _columns(self, files):
        d = os.path.dirname(files[0])
        meta_path = os.path.join(d, "_metadata.json")
        inp = self.inp
        nl, nd, ns = inp.label_dim, inp.dense_dim, self.layout.total_slots
        wgt = [None] * ns
        if os.path.exists(meta_path):
            m = json.load(open(meta_path))
            lab = [c["index"] for c in m["labels"]][:nl]
            con = [c["index"] for c in m["conts"]][:nd]
            cat = [c["index"] for c in m["cats"]][:ns]
            wgt = [c.get("weight_index") for c in m["cats"]][:ns]
        else:
            lab, con, cat = list(range(nl)), list(range(nl, nl + nd)), list(range(nl + nd, nl + nd + ns))
        # weight columns of the slots of weighted inputs only (an unweighted input ignores a weight_index)
        si = 0
        for (name, S, _, _), w in zip(self.layout.blocks, self.weighted):
            for s in range(S):
                if not w:
                    wgt[si] = None
                elif wgt[si] is None:
                    raise ValueError(f"weighted input {name}: slot {s} (cats entry {si} of {meta_path}) has no "
                                     "weight_index")
                si += 1
        return lab, con, (cat, wgt)

    def _decode_row_group(self, fp, rg, lab_i, con_i, cat_i):
        """one row group -> (label [n, L], dense [n, D], per-slot (offsets|None, values, weights|None), n); runs
        on the row-group worker threads (reference RowGroupReadingThread, row_group_reading_thread.cpp)"""
        import pyarrow as pa
        import pyarrow.parquet as pq
        from ..utils.diagnose import nvtx_range
        tl = self._tls
        if getattr(tl, "path", None) != fp:
            tl.path, tl.pf = fp, pq.ParquetFile(fp)
        with nvtx_range("parquet_read_row_group"):      # the reference annotates its reader threads too
            tbl = tl.pf.read_row_group(rg)
        cols = [tbl.column(i) for i in range(tbl.num_columns)]
        n = tbl.num_rows
        lab = np.stack([cols[i].to_numpy().astype("float32", copy=False) for i in lab_i], 1) \
            if lab_i else np.zeros((n, 0), "float32")
        den = np.stack([cols[i].to_numpy().astype("float32", copy=False) for i in con_i], 1) \
            if con_i else np.zeros((n, 0), "float32")
        cats = []
        is_list = lambda c: pa.types.is_list(c.type) or pa.types.is_large_list(c.type)
        for i, wi in zip(*cat_i):
            c = cols[i].combine_chunks()
            wv = None
            if wi is not None:
                w = cols[wi].combine_chunks()
                same = is_list(w) == is_list(c) and (not is_list(c) or np.array_equal(
                    np.diff(w.offsets.to_numpy()), np.diff(c.offsets.to_numpy())))
                if not same:
                    raise ValueError(f"{fp} row group {rg}: weight column {tbl.column_names[wi]} does not have the "
                                     f"list lengths of key column {tbl.column_names[i]}")
                if is_list(w):
                    # indexed like the key values: both columns' offsets may start anywhere in their buffers
                    ko, wo = c.offsets.to_numpy(), w.offsets.to_numpy()
                    wv = np.zeros(len(c.values), dtype="float32")
                    wv[ko[0]:ko[-1]] = w.values.to_numpy(zero_copy_only=False)[wo[0]:wo[-1]]
                else:
                    wv = w.to_numpy(zero_copy_only=False).astype("float32", copy=False)
            if is_list(c):
                cats.append((c.offsets.to_numpy(), c.values.to_numpy().astype("int64", copy=False), wv))
            else:
                cats.append((None, c.to_numpy().astype("int64", copy=False), wv))
        return (lab, den, cats, n)

    def _row_groups(self, files):
        import pyarrow.parquet as pq
        counts = {}
        while not self._stop.is_set():
            for fp in files:
                if fp not in counts:
                    counts[fp] = pq.ParquetFile(fp).num_row_groups
                for rg in range(counts[fp]):
                    yield fp, rg
            if not self.repeat:
                return

    def _bind_device(self):
        """reader threads pin host memory: bind them to this rank's GPU, not to device 0"""
        d = self._device
        if d is not None and d.type == "cuda":
            torch.cuda.set_device(d)

    def _produce(self):
        """``num_workers`` threads decode row groups ahead of the batch assembler, which consumes them
        strictly in file order (so the stream of batches does not depend on the worker count)"""
        from collections import deque
        from concurrent.futures import ThreadPoolExecutor
        try:
            files = read_file_list(self.file_list)
            lab_i, con_i, cat_i = self._columns(files)
            gb = self.b * self.world
            carry = None
            self._tls = threading.local()
            pending = deque()
            it = self._row_groups(files)
            self._out = deque()
            self._bind_device()
            with ThreadPoolExecutor(max_workers=self.num_workers, initializer=self._bind_device) as ex:
                self._ex = ex
                while not self._stop.is_set():
                    while len(pending) < self.num_workers + 1:
                        nxt = next(it, None)
                        if nxt is None:
                            break
                        pending.append(ex.submit(self._decode_row_group, nxt[0], nxt[1], lab_i, con_i, cat_i))
                    if not pending:
                        break
                    carry = self._emit(pending.popleft().result(), carry, gb)
                for f in pending:
                    f.cancel()
                if not self._stop.is_set():
                    if carry is not None and carry[3] > 0 and not self.drop_incomplete:
                        self._emit_batch(carry, carry[3])
                    self._drain(0)
                for f in self._out:
                    f.cancel()
                self._ex = None
            if self._stop.is_set():
                return
            self.q.put(None)
        except Exception as e:  # surface errors to the consumer
            self.q.put(e)

    @staticmethod
    def _slice_cat(cat, a, b):
        offs, vals, w = cat
        if offs is None:
            return (None, vals[a:b], None if w is None else w[a:b])
        o = offs[a:b + 1]
        return (o - o[0], vals[o[0]:o[-1]], None if w is None else w[o[0]:o[-1]])

    @staticmethod
    def _cat_concat(c1, c2):
        w = None if c1[2] is None else np.concatenate([c1[2], c2[2]])
        if c1[0] is None:
            return (None, np.concatenate([c1[1], c2[1]]), w)
        o = np.concatenate([c1[0], c2[0][1:] + c1[0][-1]])
        return (o, np.concatenate([c1[1], c2[1]]), w)

    def _emit(self, chunk, carry, gb):
        if carry is not None:
            lab = np.concatenate([carry[0], chunk[0]])
            den = np.concatenate([carry[1], chunk[1]])
            cats = [self._cat_concat(a, b) for a, b in zip(carry[2], chunk[2])]
            n = carry[3] + chunk[3]
            chunk = (lab, den, cats, n)
        lab, den, cats, n = chunk
        pos = 0
        while n - pos >= gb:
            self._emit_batch((lab[pos:pos + gb], den[pos:pos + gb],
                              [self._slice_cat(c, pos, pos + gb) for c in cats], gb), gb)
            pos += gb
        if pos == n:
            return None
        return (lab[pos:], den[pos:], [self._slice_cat(c, pos, n) for c in cats], n - pos)

    def _emit_batch(self, chunk, nvalid_global):
        ex = getattr(self, "_ex", None)
        if ex is None:
            self.q.put(self._assemble(chunk, nvalid_global))
            return
        # assembly is native (GIL released): batches are built on the worker pool, leave in submission order
        self._out.append(ex.submit(self._assemble, chunk, nvalid_global))
        self._drain(self.num_workers)

    def _drain(self, keep: int):
        while self._out and (len(self._out) > keep or self._out[0].done()):
            if self._stop.is_set():
                return
            self.q.put(self._out.popleft().result())

    def _assemble(self, chunk, nvalid_global):
        """this rank's slice of one global batch -> HostBatch (label, dense, feature-major padded key blocks,
        bag lengths).  Assembled with numpy into the final dtypes (torch CPU ops called from a side thread pay
        for their own thread-pool start-up: 2 ms per ``torch.zeros`` here), wrapped zero-copy."""
        lab, den, cats, n = chunk
        b, r = self.b, self.rank
        lo, hi = r * b, min((r + 1) * b, n)
        nloc = max(0, hi - lo)
        L = np.zeros((b, self.inp.label_dim), dtype="float32")
        D = np.zeros((b, self.inp.dense_dim), dtype="float32")
        if nloc > 0:
            L[:nloc] = lab[lo:hi]
            D[:nloc] = den[lo:hi]
        kdt = "int64" if self.key_dtype == torch.int64 else "int32"
        blocks = self.layout.blocks
        kelems = sum(b * S * H for (_, S, H, _) in blocks)
        nelems = sum(S * b for (_, S, H, _) in blocks)
        keys = np.full(kelems, -1, dtype=kdt)
        nnz = np.zeros(nelems, dtype="int32")
        # weights in the key layout: 1 for unweighted inputs, 0 at the padding of weighted ones
        wts = np.ones(kelems, dtype="float32") if any(self.weighted) else None
        si = ko = no = 0
        for (name, S, H, fixed), weighted in zip(blocks, self.weighted):
            blk = keys[ko:ko + b * S * H].reshape(b, S, H)
            nz = nnz[no:no + S * b].reshape(S, b)
            if weighted:
                wblk = wts[ko:ko + b * S * H].reshape(b, S, H)
                wblk[...] = 0
                for s in range(S):
                    if nloc > 0:
                        offs, _, wv = self._slice_cat(cats[si + s], lo, hi)
                        if offs is None:
                            wblk[:nloc, s, 0] = wv[:nloc]
                        else:
                            _csr_to_padded_f32(offs, wv, nloc, H, wblk, s)
            if H == 1 and all(cats[si + s][0] is None for s in range(S)):
                # one-hot block: one strided store per slot, offsets added in the key dtype
                _onehot_block([cats[si + s][1] for s in range(S)],
                              None if self.slot_offsets is None else self.slot_offsets[si:si + S],
                              lo, nloc, b, blk, nz)
                si += S
            else:
                tmp = blk if kdt == "int64" else np.full((b, S, H), -1, dtype="int64")
                for s in range(S):
                    offs, vals, _ = self._slice_cat(cats[si], lo, hi) if nloc > 0 else (None, np.zeros(0, "int64"), None)
                    off_add = 0 if self.slot_offsets is None else self.slot_offsets[si]
                    if offs is None:
                        tmp[:nloc, s, 0] = vals[:nloc] + off_add
                        nz[s, :nloc] = 1
                    else:
                        _csr_to_padded(offs, vals, nloc, H, int(off_add), tmp, s, nz)
                    si += 1
                if tmp is not blk:
                    blk[...] = tmp
            ko += b * S * H
            no += S * b
        hb = HostBatch(torch.from_numpy(L), torch.from_numpy(D), torch.from_numpy(keys),
                       torch.from_numpy(nnz) if blocks else None, nloc,
                       weights=None if wts is None else torch.from_numpy(wts)).pin()
        return (hb, nvalid_global)

    # -------------------------------------------------------------- consumer
    def start(self):
        if self.thread is None:
            self._stop.clear()
            self.thread = threading.Thread(target=self._produce, daemon=True)
            self.thread.start()
        self.started = True

    def set_source(self, source=None):
        self.stop()
        if source:
            self.file_list = source if isinstance(source, str) else source[0]
        self.q = queue.Queue(maxsize=4)
        self.start()

    def read_a_batch(self):
        if self.thread is None:
            self.start()
        item = self.q.get()
        if item is None:
            self.thread = None
            return None
        if isinstance(item, Exception):
            raise item
        hb, nvalid = item
        self.current_batchsize = nvalid
        return hb

    def stop(self):
        if self.thread is not None:
            self._stop.set()
            try:
                while True:
                    self.q.get_nowait()
            except queue.Empty:
                pass
            self.thread.join(timeout=2)
            self.thread = None
