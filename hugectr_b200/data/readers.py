"""Data readers: common interface + the synthetic in-memory source.

IDataReader parity (HugeCTR/include/data_reader.hpp:40-66): ``start``, ``set_source``,
``read_a_batch`` (-> HostBatch in pinned memory), ``current_batch_incomplete``,
``get_current_batchsize``.  File-backed readers (Parquet, RawAsync, Norm) live in
``parquet_reader.py`` / ``raw_reader.py`` / ``norm_reader.py``.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .batch import HostBatch, power_law_keys


class IDataReader:
    def __init__(self, batch_per_rank: int, rank: int, world: int, repeat: bool = True):
        self.b, self.rank, self.world, self.repeat = batch_per_rank, rank, world, repeat
        self.current_batchsize = batch_per_rank * world
        self.started = False

    def start(self):
        self.started = True

    def set_source(self, source):
        raise NotImplementedError

    def read_a_batch(self) -> Optional[HostBatch]:
        raise NotImplementedError

    def is_started(self) -> bool:
        return self.started

    def current_batch_incomplete(self) -> bool:
        return self.current_batchsize != self.b * self.world

    def get_current_batchsize(self) -> int:
        return self.current_batchsize

    def get_current_batchsize_per_device(self, local_id: int = 0) -> int:
        lo = self.rank * self.b
        return max(0, min(self.b, self.current_batchsize - lo))

    def stop(self):
        pass

    # ---- handle API of model.get_data_reader_train()/eval() (Core23DataReader32/64,
    # HugeCTR/include/pybind/data_reader_wrapper.hpp:50-72)
    def _bind(self, model, is_train: bool):
        self._model, self._is_train, self._eof = model, is_train, False

    def ready_to_collect(self):
        """the staging slot of the previous batch may be recycled (the copy-complete handshake of the
        ring readers does this implicitly on the next read)"""

    def read_a_batch_to_device(self) -> int:
        """next batch -> the model's input tensors; returns the global batch size read (0 at the end)"""
        hb = self.read_a_batch()
        if hb is None:
            self._eof = True
            return 0
        self._eof = False
        self._model._load_batch(hb, self._is_train)
        return int(self.current_batchsize)

    read_a_batch_to_device_delay_release = read_a_batch_to_device

    def is_eof(self) -> bool:
        return bool(getattr(self, "_eof", False))


class CachedEvalReader(IDataReader):
    """``DataReaderParams.cache_eval_data = N``: keeps the first N evaluation batches resident on the
    device and replays them for every later evaluation round (no file IO / H2D after the first round).
    Active when N covers a whole round (N >= max_eval_batches) -- the MLPerf configuration, where the
    round is the complete evaluation set; a smaller N only bounds the look-ahead, as in the reference
    (HugeCTR/src/pybind/add_input.cpp:152-158)."""

    def __init__(self, inner: IDataReader, capacity: int, device):
        super().__init__(inner.b, inner.rank, inner.world, inner.repeat)
        self.inner, self.capacity, self.device = inner, int(capacity), device
        self.cache, self.sizes, self.pos = [], [], 0

    def start(self):
        self.inner.start()
        self.started = True

    def is_started(self):
        return self.started

    def set_source(self, source=None):
        self.cache, self.sizes, self.pos = [], [], 0
        self.inner.set_source(source)

    def read_a_batch(self):
        if len(self.cache) >= self.capacity or (self.cache and getattr(self, "_inner_done", False)):
            hb = self.cache[self.pos % len(self.cache)]
            self.current_batchsize = self.sizes[self.pos % len(self.cache)]
            self.pos += 1
            return hb
        hb = self.inner.read_a_batch()
        if hb is None:
            self._inner_done = True
            return None if not self.cache else self.read_a_batch()
        if getattr(hb, "raw", None) is not None:
            # device-split reader: split the raw records into fresh device tensors and keep those
            sp = hb.splitter
            lab = torch.empty(sp.batch, sp.label_dim, device=self.device)
            den = torch.empty(sp.batch, max(sp.dense_dim, 1), device=self.device)[:, :sp.dense_dim].contiguous()
            keys = torch.empty(max(sp.total_keys, 1), dtype=sp.key_dtype, device=self.device)
            sp.run(hb.raw, hb.raw_skew, hb.num_valid, lab, den, keys)
            kept = HostBatch(lab, den, keys, None, hb.num_valid)
        else:
            mv = lambda t: None if t is None else t.to(self.device, copy=True)
            kept = HostBatch(mv(hb.label), mv(hb.dense), mv(hb.keys), mv(hb.nnz), hb.num_valid,
                             weights=mv(hb.weights))
        hb.mark_copied()
        self.cache.append(kept)
        self.current_batchsize = self.inner.current_batchsize
        self.sizes.append(self.current_batchsize)
        return kept

    def stop(self):
        self.inner.stop()


class SparseLayout:
    """Per sparse param: slot_num, max nnz per slot, fixed-length flag, per-slot vocab sizes."""

    def __init__(self, sparse_params, slot_size_array: Optional[List[int]] = None):
        self.params = list(sparse_params)
        self.blocks = []   # (name, slot_num, H, fixed)
        for p in self.params:
            self.blocks.append((p.top_name, p.slot_num, max(p.nnz_per_slot), p.is_fixed_length))
        self.weighted = [bool(getattr(p, "weighted", False)) for p in self.params]
        self.total_slots = sum(b[1] for b in self.blocks)
        self.slot_sizes = list(slot_size_array or [])

    def keys_per_sample(self) -> int:
        return sum(s * h for (_, s, h, _) in self.blocks)

    def key_block_offsets(self, b: int):
        offs, o = {}, 0
        for (n, s, h, _) in self.blocks:
            offs[n] = o
            o += b * s * h
        return offs, o

    def nnz_block_offsets(self, b: int):
        offs, o = {}, 0
        for (n, s, h, _) in self.blocks:
            offs[n] = o
            o += b * s
        return offs, o

    def has_variable(self) -> bool:
        return any(not f for (_, _, _, f) in self.blocks)

    def has_weights(self) -> bool:
        return any(self.weighted)


class SyntheticReader(IDataReader):
    """Pre-generates a pool of pinned batches (power-law or uniform keys) and cycles through it."""

    def __init__(self, batch_per_rank, rank, world, label_dim, dense_dim, layout: SparseLayout,
                 slot_vocab: List[int], alpha: float = 1.1, seed: int = 0, pool: int = 8,
                 key_dtype=torch.int32, power_law: bool = True, num_batches: int = -1):
        super().__init__(batch_per_rank, rank, world)
        self.pool = []
        self.layout = layout
        gen = torch.Generator()
        gen.manual_seed(seed * 1000003 + rank * 7919 + 17)
        b = batch_per_rank
        wgen = None
        for _ in range(pool):
            label = (torch.rand(b, label_dim, generator=gen) < 0.3).float()
            dense = torch.rand(b, dense_dim, generator=gen)
            blocks, nnzs = [], []
            si = 0
            for (name, S, H, fixed) in layout.blocks:
                cols = []
                for s in range(S):
                    vocab = slot_vocab[si] if si < len(slot_vocab) else 1000
                    si += 1
                    if power_law:
                        k = power_law_keys(b * H, vocab, alpha, gen, torch.int64)
                    else:
                        k = torch.randint(0, max(vocab, 1), (b * H,), generator=gen)
                    k = k.view(b, H)
                    if not fixed:
                        n = torch.randint(1, H + 1, (b,), generator=gen)
                        k = torch.where(torch.arange(H).view(1, -1) < n.view(-1, 1), k,
                                        torch.full_like(k, -1))
                        nnzs.append(n.int())
                    else:
                        nnzs.append(torch.full((b,), H, dtype=torch.int32))
                    cols.append(k)
                blocks.append(torch.stack(cols, 1).reshape(-1))   # [b, S, H]
            keys = torch.cat(blocks).to(key_dtype) if blocks else torch.zeros(0, dtype=key_dtype)
            nnz = torch.cat(nnzs) if (nnzs and layout.has_variable()) else None
            weights = None
            if layout.has_weights():
                # a generator of their own: the key, label and dense streams stay as without weights
                if wgen is None:
                    wgen = torch.Generator()
                    wgen.manual_seed(seed * 1000003 + rank * 7919 + 29)
                wb = []
                for (name, S, H, fixed), wt in zip(layout.blocks, layout.weighted):
                    wb.append(torch.rand(b * S * H, generator=wgen) + 0.5 if wt else torch.ones(b * S * H))
                weights = torch.cat(wb)
            self.pool.append(HostBatch(label, dense, keys, nnz, b, weights=weights).pin())
        self.i = 0
        self.num_batches = num_batches
        self.served = 0

    def set_source(self, source=None):
        self.i = 0
        self.served = 0

    def read_a_batch(self):
        if self.num_batches >= 0 and self.served >= self.num_batches:
            if not self.repeat:
                return None
            self.served = 0
        hb = self.pool[self.i % len(self.pool)]
        self.i += 1
        self.served += 1
        self.current_batchsize = self.b * self.world
        return hb
