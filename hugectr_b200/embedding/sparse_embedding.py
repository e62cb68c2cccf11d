"""Legacy SparseEmbedding runtimes: DistributedSlotSparseEmbeddingHash and
LocalizedSlotSparseEmbeddingHash (dynamic-vocabulary hash embeddings).

Reference semantics:
  Distributed  row-wise MP over all GPUs (owner = key % N), forward = hash get_insert -> pooled
               partial sums for the whole global batch -> reduce-scatter; backward = all-gather of
               top grads -> per-row update   (include/embeddings/distributed_slot_sparse_embedding_hash.hpp:41-440)
  Localized    slot s lives on GPU s % N, forward = local pooled lookup -> all-to-all -> reorder
               (include/embeddings/localized_slot_sparse_embedding_hash.hpp:217-345)
  max_vocabulary_size_per_gpu = workspace_MB * 2^20 / ((1 + n_opt_states) * 4 * vec)  (model.cpp:186-196)
  eval uses lookup-only (get_mark): unseen keys contribute zero vectors
  check_overflow: "Runtime vocabulary size ... exceeds max_vocabulary_size_per_gpu"

Implementation: keys are translated to dense rows by the GPU HashTable (ownership filter + bounded insert
in ONE kernel, overflow raised through a device flag), then the SAME owner-side pool / accumulate /
fused-update kernels as the EmbeddingCollection run on the row buffer.  Exchange:
  fused       (CUDA, world > 1, peer-mapped heap) every rank scatters its key block into all owners'
              inboxes and its top-gradients into their gradient inboxes with posted peer stores
              (csrc/emb_dispatch.cu); owners write their partial pooled vectors straight into the
              requesters' receive slabs.  Device barriers only: no NCCL, no host sync -- the whole step is
              captured in the model's CUDA graph like the EmbeddingCollection path.
  collective  (CPU / gloo, HCTR_DISABLE_P2P) all-gather of keys, all-to-all of pooled vectors, all-gather
              of gradients through torch.distributed.
"""
from __future__ import annotations

import math
import os
from typing import List

import numpy as np
import torch

from ..io import filesystem as FS

from ..enums import Embedding_t, Optimizer_t, Update_t
from ..ops.optim import opt_hp, opt_states
from . import ops as E
from .hashtable import HashTable


class SparseEmbeddingRuntime:
    def __init__(self, cfg, param, layout, batch_per_gpu, device, act_dtype, comm, opt, key_dtype,
                 scaler=1.0, seed=0, share_from=None):
        from ..solver import check_not_rowwise
        check_not_rowwise(opt, "a legacy sparse embedding (also with CreateETC / offloaded tables)")
        self.cfg, self.param, self.layout = cfg, param, layout
        self.name = cfg.sparse_embedding_name
        self.top_name = cfg.sparse_embedding_name
        self.b = batch_per_gpu
        self.device, self.act_dtype, self.comm = device, act_dtype, comm
        self.rank, self.world = comm.rank, comm.world_size
        self.opt = opt
        self.scaler = scaler
        self.key_dtype = key_dtype
        self.S = param.slot_num
        self.H = max(param.nnz_per_slot)
        self.vec = cfg.embedding_vec_size
        self.localized = cfg.embedding_type != Embedding_t.DistributedSlotSparseEmbeddingHash
        self.combiner = 1 if cfg.combiner == "mean" else 0
        self.is_train = share_from is None
        ns = opt.num_states
        if share_from is None:
            ws = cfg.workspace_size_per_gpu_in_mb
            if cfg.max_vocabulary_size_per_gpu > 0:
                self.max_rows = cfg.max_vocabulary_size_per_gpu
            elif ws > 0:
                self.max_rows = int(ws * 1024 * 1024 // ((1 + ns) * 4 * self.vec))
            else:
                self.max_rows = max(1024, sum(cfg.slot_size_array) // max(1, self.world) + 1024)
            self.table = torch.zeros(self.max_rows * self.vec, dtype=torch.float32, device=device)
            self._init_table(seed)
            self.s0, self.s1 = opt_states(opt, self.table.numel(), device=device)
            self.hash = HashTable(self.max_rows, device)
            # (one spare entry behind the table: the write target of batch entries this rank does not own)
            self.slot_of_row = torch.full((self.max_rows + 1,), -1, dtype=torch.int64, device=device) \
                if self.localized else None
        else:
            for k in ("max_rows", "table", "s0", "s1", "hash", "slot_of_row"):
                setattr(self, k, getattr(share_from, k))
        b, S, H, vec, W = self.b, self.S, self.H, self.vec, self.world
        self.top_shape = (b, S, vec)
        self.top_data = torch.zeros(b, S, vec, dtype=act_dtype, device=device)
        self.top_grad = torch.zeros(b, S, vec, dtype=act_dtype, device=device) if self.is_train else None
        self.keys_loc = torch.full((b * S * H,), -1, dtype=torch.int64, device=device)
        self.rows_all = torch.full((W, b * S * H), -1, dtype=torch.int64, device=device)
        nk, nv = b * S * H, b * S * vec
        self.fused = (device.type == "cuda" and W > 1 and comm.p2p_available
                      and os.environ.get("HCTR_LEGACY_FUSED", "1") == "1")
        if self.fused:
            sa = comm.symm_alloc
            self.keys_all = sa(W * nk, torch.int64).view(W, nk)
            self.keys_all.fill_(-1)
            self.recv = sa(W * nv, act_dtype).view(W, nv)            # slot o: partial sums from owner o
            self.peer_keys_all = comm.peer_ptrs(self.keys_all)
            esz = 2 if act_dtype == torch.bfloat16 else 4
            self.peer_recv_me = [p + self.rank * nv * esz for p in comm.peer_ptrs(self.recv)]
            self.partial = None
            me = self.rank
            self._key_routes = [E.Route(0, me * nk, 1, nk, nk, nk, g) for g in range(W)]
            self._key_routes_dev = E.routes_to_device(self._key_routes, device)
            if self.is_train:
                self.grads_all = sa(W * nv, act_dtype).view(W, nv)
                self.peer_grads_all = comm.peer_ptrs(self.grads_all)
                self._grad_routes = [E.Route(0, me * nv, 1, nv, nv, nv, g) for g in range(W)]
                self._grad_routes_dev = E.routes_to_device(self._grad_routes, device)
            else:
                self.grads_all = None
            self._out_sum = torch.zeros(nv, dtype=act_dtype, device=device)
        else:
            self.keys_all = torch.full((W, nk), -1, dtype=torch.int64, device=device)
            self.partial = torch.zeros(W, nv, dtype=act_dtype, device=device)
            self.recv = torch.zeros(W, nv, dtype=act_dtype, device=device)
            self.grads_all = torch.zeros(W, nv, dtype=act_dtype, device=device) if self.is_train else None
        # no per-step host work (device-side overflow flag): the step is graph capturable unless the
        # optimizer variant needs torch.unique (LazyGlobal Adam)
        self.graph_safe = (W == 1 or self.fused) and device.type == "cuda" and not (
            opt.update_type == Update_t.LazyGlobal and opt.optimizer_type == Optimizer_t.Adam)
        # one lookup per slot over the row buffer: keys [b, S, H] sample-major
        self.lookups: List[E.LookupDesc] = []
        for s in range(S):
            self.lookups.append(E.LookupDesc(
                table_row_off=0, key_off=s * H, out_off=s * vec, grad_off=s * vec, hotness=H,
                key_stride=S * H, num_shards=1, shard_idx=0, out_stride=S * vec, grad_stride=S * vec,
                combiner=0, ev_size=vec, rows=self.max_rows))
        po = 0
        for l in self.lookups:
            l.pair_off = po
            po += W * b * H
        self.lookups_dev = E.lookups_to_device(self.lookups, device)
        if self.is_train:
            self.indexed = device.type == "cuda" and E.vec4_aligned(self.lookups, vec) and \
                os.environ.get("HCTR_EMB_BWD", "indexed") == "indexed"
            self.ws = E.UniqueWorkspace(max(po, 1), vec, device, indexed=self.indexed)
        self.slot_offsets = None
        ssa = list(cfg.slot_size_array)
        self._nnz_cnt = torch.ones(b, S, dtype=torch.float32, device=device)

    def eval_clone(self, batch_per_gpu):
        return SparseEmbeddingRuntime(self.cfg, self.param, self.layout, batch_per_gpu, self.device,
                                      self.act_dtype, self.comm, self.opt, self.key_dtype, self.scaler,
                                      0, share_from=self)

    def _init_table(self, seed):
        """U(+-sqrt(1/slot_size)) per slot when slot_size_array is given, else a global bound
        (src/embeddings/init_embedding_functor.cu:34-55)."""
        ssa = self.cfg.slot_size_array
        vocab = max(1, sum(ssa) if ssa else self.max_rows * self.world)
        bound = math.sqrt(1.0 / max(1.0, vocab / max(1, len(ssa) or 1)))
        g = torch.Generator(device=self.device)
        g.manual_seed(seed * 7919 + self.rank + 13)
        self.table.uniform_(-bound, bound, generator=g)

    # ------------------------------------------------------------------ data in
    def set_keys(self, hb, key_offs, nnz_offs):
        o = key_offs[self.param.top_name]
        n = self.b * self.S * self.H
        self.keys_loc.copy_(hb.keys[o:o + n].to(torch.int64), non_blocking=True)

    def _owner_mask(self, keys_all):
        """which keys of the gathered batch does this rank own"""
        valid = keys_all >= 0
        if self.localized:
            slot = (torch.arange(keys_all.shape[1], device=keys_all.device) // self.H) % self.S
            own = (slot % self.world) == self.rank
            return valid & own.view(1, -1)
        return valid & ((keys_all % self.world) == self.rank)

    def check_overflow(self):
        if self.hash.overflowed():
            n = self.hash.size()
            raise RuntimeError(f"Runtime vocabulary size (>= {n}) exceeds max_vocabulary_size_per_gpu "
                               f"({self.max_rows}) of {self.name}, new feature insertion failed.")
        E.check_workspace_overflow(getattr(self, "ws", None), self.name)

    # ------------------------------------------------------------------ forward / backward
    def _translate(self, is_train: bool):
        """keys_all -> rows_all: rows of the keys this rank owns, -1 elsewhere (one kernel, no host sync)"""
        n = self.b * self.S * self.H
        if self.localized:
            self.hash.translate(self.keys_all, self.rows_all, is_train, n, key_mod=self.world, key_rem=self.rank,
                                slot_div=self.H, slot_num=self.S)
        else:
            self.hash.translate(self.keys_all, self.rows_all, is_train, n, key_mod=self.world, key_rem=self.rank)
        if self.localized and is_train and self.slot_of_row is not None:
            # remember the slot of every row (dumped as slot_id; the reference stores it per hash value)
            r = self.rows_all.reshape(-1)
            slot = (torch.arange(r.numel(), device=r.device) % n) // self.H % self.S
            # every occurrence of an owned row writes the same value (a Localized key lives in one slot); entries
            # that are not mine go to the spare entry, so no write races with a row's real slot
            self.slot_of_row.index_put_((torch.where(r >= 0, r, torch.full_like(r, self.max_rows)),), slot)

    def forward(self, is_train: bool):
        W, b, S, H, vec = self.world, self.b, self.S, self.H, self.vec
        if self.fused:
            # key all-gather by posted peer stores into every owner's inbox, one device barrier
            E.dispatch(self.keys_loc, self._key_routes, self._key_routes_dev, self.peer_keys_all)
            self.comm.barrier_device()
        else:
            self.comm.all_gather(self.keys_all, self.keys_loc)
        self._translate(is_train)
        if is_train and not self.graph_safe and os.environ.get("HUGECTR_DISABLE_OVERFLOW_CHECK", "0") != "1":
            self.check_overflow()
        if self.fused:
            # partial pooled vectors of MY rows go straight into slot [me] of every requester's slab
            E.forward(self.lookups, self.lookups_dev, self.table, vec, list(self.rows_all.unbind(0)),
                      self.peer_recv_me, b, self.rank, key_bytes=8, act_bf16=self.act_dtype == torch.bfloat16)
            self.comm.barrier_device()
            if self.recv.is_cuda and self.recv.dtype in (torch.float32, torch.bfloat16):
                from ..ops import layer_ops as LO
                LO.reduce_mid(self.recv, self._out_sum, 1, W, b * S * vec, 1.0, False)
                out = self._out_sum.view(b, S, vec)
            else:
                out = self.recv.float().sum(0).view(b, S, vec)
        else:
            self.partial.zero_()
            E.forward(self.lookups, self.lookups_dev, self.table, vec, list(self.rows_all.unbind(0)),
                      list(self.partial.unbind(0)), b, self.rank)
            self.comm.all_to_all(self.recv, self.partial)
            out = self.recv.float().sum(0).view(b, S, vec)
        if self.combiner == 1:
            cnt = (self.keys_loc.view(b, S, H) >= 0).sum(-1).clamp(min=1).float()
            self._nnz_cnt = cnt
            out = out.float() / cnt.unsqueeze(-1)
        self.top_data.copy_(out.to(self.top_data.dtype))

    def backward(self, lr_t, step_t):
        W, b, S, H, vec = self.world, self.b, self.S, self.H, self.vec
        g = self.top_grad
        if self.combiner == 1:
            g = (g.float() / self._nnz_cnt.unsqueeze(-1)).to(self.top_grad.dtype)
        if self.fused:
            # gradient all-gather by posted peer stores, one device barrier; no end-of-step barrier is
            # needed (the next step's key dispatch barrier orders the inbox reuse)
            gsrc = g.reshape(-1)
            if not gsrc.is_contiguous():
                gsrc = gsrc.contiguous()
            E.dispatch(gsrc, self._grad_routes, self._grad_routes_dev, self.peer_grads_all)
            self.comm.barrier_device()
        else:
            self.comm.all_gather(self.grads_all, g.reshape(-1))
        kb = list(self.rows_all.unbind(0))
        gb = list(self.grads_all.unbind(0))
        hp = opt_hp(self.opt, self.scaler)
        if self.opt.update_type == Update_t.LazyGlobal and self.opt.optimizer_type == Optimizer_t.Adam:
            return self._lazy_adam(lr_t, step_t)
        if self.indexed:
            abf = self.act_dtype == torch.bfloat16
            E.bwd_index(self.lookups, self.lookups_dev, self.table, vec, kb, b, self.ws, self.rank, key_bytes=8)
            E.bwd_reduce_update(self.opt.optimizer_type, self.lookups, self.lookups_dev, self.table,
                                self.s0, self.s1, vec, kb, gb, b, self.ws, hp, lr_t, step_t, 1.0, self.rank,
                                key_bytes=8, act_bf16=abf)
        else:
            E.backward_accum(self.lookups, self.lookups_dev, self.table, vec, kb, gb, b, self.ws, 1.0,
                             self.rank)
            E.update(self.opt.optimizer_type, self.table, self.s0, self.s1, vec, self.ws, hp, lr_t, step_t)
        if self.opt.update_type in (Update_t.Global, Update_t.LazyGlobal) and \
                self.opt.optimizer_type in (Optimizer_t.Adam, Optimizer_t.MomentumSGD, Optimizer_t.Nesterov):
            self._global_sweep(lr_t, step_t)

    def _lazy_adam(self, lr_t, step_t):
        """Update_t.LazyGlobal with Adam (sparse_optimizer.cu:523-561, opt_adam_kernel_lazy): only the
        touched rows are visited; a row first catches up on the weight movement of the steps it
        skipped (geometric sum of its decaying first moment), then its moments absorb the skipped
        decays and the new gradient -- whose own weight update is applied at the row's next visit.
        Needs the step of the last visit per row (the extra state of model.cpp:189-192)."""
        vec, o = self.vec, self.opt
        if not hasattr(self, "prev_time"):
            # initialised to 1 like the reference (sparse_optimizer.cu:137-139)
            self.prev_time = torch.ones(self.max_rows, dtype=torch.float32, device=self.device)
        r = self.rows_all.reshape(-1)
        own = r >= 0
        if not bool(own.any()):
            return
        # gradient of every (rank, sample, slot) bucket, repeated for its H keys
        W, b, S, H = self.world, self.b, self.S, self.H
        g = self.grads_all.view(W, b, S, 1, vec).float().expand(W, b, S, H, vec).reshape(-1, vec)
        rows, inv = torch.unique(r[own], return_inverse=True)
        gi = torch.zeros(rows.numel(), vec, device=self.device).index_add_(0, inv, g[own]) / self.scaler
        w = self.table.view(-1, vec)
        m, v = self.s0.view(-1, vec), self.s1.view(-1, vec)
        t = step_t.reshape(()).float()
        prev = self.prev_time[rows].unsqueeze(1)
        skipped = t - prev
        b1s = o.beta1 ** skipped
        alpha_common = lr_t.reshape(()).float() / (1.0 - o.beta1)
        alpha_t = alpha_common * torch.sqrt(1.0 - o.beta2 ** prev) / (1.0 - o.beta1 ** prev) * (1.0 - b1s)
        mi, vi = m[rows], v[rows]
        w[rows] = w[rows] - alpha_t * mi / (vi.sqrt() + o.epsilon)
        m[rows] = b1s * mi + (1.0 - o.beta1) * gi
        v[rows] = (o.beta2 ** skipped) * vi + (1.0 - o.beta2) * gi * gi
        self.prev_time[rows] = t

    def _global_sweep(self, lr_t, step_t):
        """Update_t.Global (sparse_optimizer.cu:241-292): the touched rows were updated by the fused
        kernel above; every OTHER allocated row gets the dense-optimizer step with a zero gradient
        (moments decay, the weight keeps moving along the decayed momentum), which makes the sparse
        update mathematically identical to the dense optimizer.  LazyGlobal (the reference's cheaper
        approximation of the same thing) takes this exact path too."""
        vec = self.vec
        if self.device.type == "cuda":
            n = self.max_rows                  # (allocated rows only, masked on the device: no host sync)
            alive = torch.arange(n, device=self.device) < self.hash.counter
        else:
            n = max(1, int(self.hash.size()))  # the host knows the size: sweep the allocated prefix only
            alive = torch.ones(n, dtype=torch.bool)
        # rows of this step: every write stores True (entries that are not mine go to a spare slot behind the
        # table) -- duplicates are harmless and no row's flag depends on the order of conflicting writes
        touched = torch.zeros(n + 1, dtype=torch.int32, device=self.device)
        r = self.rows_all.reshape(-1)
        touched.index_fill_(0, torch.where(r >= 0, r, torch.full_like(r, n)), 1)
        touched = (touched[:n] > 0) | ~alive    # never-allocated rows are left alone
        unt = (~touched).unsqueeze(1)
        w = self.table.view(-1, vec)[:n]
        s0 = self.s0.view(-1, vec)[:n]
        lr = lr_t.reshape(()).float()
        o = self.opt
        zero = torch.zeros((), device=self.device)
        if o.optimizer_type == Optimizer_t.Adam:
            t = step_t.reshape(()).float()
            alpha = lr * torch.sqrt(1.0 - o.beta2 ** t) / (1.0 - o.beta1 ** t)
            s1 = self.s1.view(-1, vec)[:n]
            m = torch.where(unt, s0 * o.beta1, s0)
            v = torch.where(unt, s1 * o.beta2, s1)
            w.sub_(torch.where(unt, alpha * m / (v.sqrt() + o.epsilon), zero))
            s0.copy_(m)
            s1.copy_(v)
        elif o.optimizer_type == Optimizer_t.MomentumSGD:
            m = torch.where(unt, s0 * o.momentum_factor, s0)
            w.add_(torch.where(unt, m, zero))
            s0.copy_(m)
        else:  # Nesterov: a' = mu a ; w += -mu a + (1 + mu) a'
            mu = o.momentum_factor
            an = s0 * mu
            w.add_(torch.where(unt, -mu * s0 + (1.0 + mu) * an, zero))
            s0.copy_(torch.where(unt, an, s0))

    # ------------------------------------------------------------------ checkpoint (SURVEY 3.6)
    def _gather_all(self):
        keys, rows = self.hash.dump()
        w = self.table.view(-1, self.vec)[rows.to(self.device)].cpu()
        slots = None
        if self.localized:
            # the slot recorded when the row was created (forward); rows that only exist through
            # load_parameters fall back to the slot_size_array ranges
            rec = self.slot_of_row[rows.to(self.device)].cpu()
            slots = torch.where(rec >= 0, rec, self._slot_ids(keys))
        return self.comm.all_gather_object((keys, w, slots))

    def dump_parameters(self, path: str):
        parts = self._gather_all()
        if self.comm.rank == 0:
            keys = torch.cat([p[0] for p in parts])
            w = torch.cat([p[1] for p in parts])
            FS.write_array(FS.path_join(path, "key"), keys.numpy().astype("<i8"))
            FS.write_array(FS.path_join(path, "emb_vector"), w.numpy().astype("<f4"))
            if self.localized:
                slots = torch.cat([p[2] for p in parts])
                FS.write_array(FS.path_join(path, "slot_id"), slots.numpy().astype("<u8"))
        self.comm.barrier()

    def _slot_ids(self, keys):
        ssa = self.cfg.slot_size_array
        if not ssa:
            return torch.zeros_like(keys)
        bounds = torch.tensor(np.cumsum([0] + list(ssa)), dtype=torch.int64)
        return (torch.searchsorted(bounds, keys, right=True) - 1).clamp(0, len(ssa) - 1)

    def load_parameters(self, path: str):
        keys = torch.from_numpy(FS.read_array(FS.path_join(path, "key"), "<i8").astype("int64"))
        w = torch.from_numpy(FS.read_array(FS.path_join(path, "emb_vector"), "<f4")).view(-1, self.vec)
        if self.localized and FS.path_exists(FS.path_join(path, "slot_id")):
            slot = torch.from_numpy(FS.read_array(FS.path_join(path, "slot_id"), "<u8").astype("int64"))
            m = (slot % self.world) == self.rank
        else:
            m = (keys % self.world) == self.rank
        k = keys[m]
        rows = self.hash.get_insert(k.to(self.device))
        self.check_overflow()
        self.table.view(-1, self.vec)[rows] = w[m].to(self.device)
        self._loaded_keys = keys                 # file order: optimizer states are matched by key
        if self.localized and self.slot_of_row is not None and FS.path_exists(FS.path_join(path, "slot_id")):
            self.slot_of_row[rows] = slot[m].to(self.device)

    def dump_opt_states(self, path: str):
        keys, rows = self.hash.dump()
        st = [s.view(-1, self.vec)[rows.to(self.device)].cpu() for s in (self.s0, self.s1) if s is not None]
        parts = self.comm.all_gather_object(st)
        if self.comm.rank == 0:
            FS.write_array(path, np.concatenate([torch.cat([p[i] for p in parts]).numpy().astype("<f4").reshape(-1)
                                                 for i in range(len(st))]) if st else np.zeros(0, "<f4"))
        self.comm.barrier()

    def load_opt_states(self, path: str):
        """States are stored in the order of the sparse model's ``key`` file (all ranks' rows concatenated).
        They are matched BY KEY: the hash table hands out rows in arbitrary order within a launch, so the
        row order of this process says nothing about the file order."""
        raw = FS.read_array(path, "<f4")
        states = [s for s in (self.s0, self.s1) if s is not None]
        if not states:
            return
        keys = getattr(self, "_loaded_keys", None)
        if keys is None:
            # no sparse model loaded in this process: the file order is the order a dump would write now
            kd, _ = self.hash.dump()
            keys = torch.cat([p for p in self.comm.all_gather_object(kd)])
        tot = keys.numel()
        if raw.size != len(states) * tot * self.vec:
            raise RuntimeError(f"optimizer state file {path} holds {raw.size} values, expected "
                               f"{len(states)} x {tot} x {self.vec} for the loaded sparse model")
        rows = self.hash.get(keys.to(self.device))           # -1: key lives on another rank
        mine = (rows >= 0).cpu()
        r = rows[mine.to(rows.device)]
        per = tot * self.vec
        for i, s in enumerate(states):
            blk = torch.from_numpy(raw[i * per:(i + 1) * per].copy()).view(tot, self.vec)
            s.view(-1, self.vec)[r] = blk[mine].to(self.device)
