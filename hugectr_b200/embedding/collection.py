"""EmbeddingCollection ("3G" embedding): configs, sharding resolution and the per-rank runtime.

API parity: HugeCTR/include/pybind/embedding_collection_wrapper.hpp:29-65,
HugeCTR/include/embeddings/embedding_collection.hpp:55-90 (shard_matrix / shard_strategy),
key->shard rule  owner = shard_gpus[key % num_shards], row = key // num_shards
(HugeCTR/embedding/data_distributor/key_filtering_operators.cu:88, operators/keys_to_indices.cu:39),
column-wise split (HugeCTR/src/embeddings/embedding_collection.cpp:25-150).

Runtime design (differs from the reference on purpose): one process per GPU; every rank keeps its
keys / EBC outputs / EBC top-grads in *slabs* with identical layout on all ranks.  In ``fused`` mode
the slabs live in a peer-mapped symmetric heap and the owner-side kernels read the requesters' keys
and write their outputs (and read their gradients) directly over NVLink, so no NCCL all-to-all runs
on the forward or backward path.  In ``collective`` mode (CPU/gloo tests and the NCCL baseline the
fused path is measured against) the same local kernels run on the key blocks each owner received and
the pooled vectors travel through variable-size all-to-alls.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from ..enums import CommunicationStrategy, Optimizer_t
from ..ops.optim import opt_hp, opt_states
from ..solver import OptParamsPy
from . import ops as E


def _stable_seed(*parts) -> int:
    import zlib
    return zlib.crc32(repr(parts).encode()) & 0x7FFFFFFF


# ------------------------------------------------------------------------- configs
WEIGHT_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


@dataclass
class InitParams:
    """embedding_storage/common.hpp:43-77: Uniform(up_bound) or Sinusoidal(max_sequence_len, ev)."""
    initializer_type: str = "Default"
    up_bound: float = -1.0
    max_sequence_len: int = 0
    ev_size: int = 0


class EmbeddingTableConfig:
    def __init__(self, name: str, max_vocabulary_size: int, ev_size: int,
                 opt_params_or_empty: Optional[OptParamsPy] = None,
                 init_param_or_empty: Optional[InitParams] = None, **kw):
        self.name = str(name)
        self.max_vocabulary_size = int(max_vocabulary_size)
        self.ev_size = int(ev_size)
        self.opt_params = kw.get("opt_params", opt_params_or_empty)
        self.init_param = kw.get("init_param", init_param_or_empty)
        # max_vocabulary_size < 0: dynamic table (embedding_storage/common.hpp:78) -- arbitrary 64-bit
        # keys, rows handed out on first sight by a per-shard hash table; ``init_capacity`` rows per
        # shard are reserved at first and doubled when a shard runs out (EmbeddingCollection.grow_dynamic)
        self.dynamic = self.max_vocabulary_size < 0
        self.init_capacity = int(kw.get("init_capacity", 1 << 20))
        # rows per shard a dynamic table may grow to (0 = no limit but memory): see EmbeddingCollection.grow_dynamic
        self.max_capacity = int(kw.get("max_capacity", 0))
        # storage of the weights of a model-parallel table: "fp32" or "bf16" (half the bytes; every
        # optimizer store rounds stochastically, see csrc/embedding.cuh).  Data-parallel tables stay fp32.
        self.weight_dtype = str(kw.get("weight_dtype", "fp32"))
        if self.weight_dtype not in WEIGHT_DTYPES:
            raise ValueError(f"table {self.name}: weight_dtype must be one of {sorted(WEIGHT_DTYPES)}, "
                             f"not {self.weight_dtype!r}")
        # "lru" | "lfu": a dynamic table of a fixed max_capacity rows per shard that evicts cold keys
        # instead of growing (see docs/embedding.md); None keeps the growing table
        self.evict_strategy = kw.get("evict_strategy", None)
        if self.evict_strategy is not None:
            from .hashtable import EVICT_STRATEGIES
            if self.evict_strategy not in EVICT_STRATEGIES:
                raise ValueError(f"table {self.name}: evict_strategy must be one of {EVICT_STRATEGIES} or None, "
                                 f"not {self.evict_strategy!r}")
            if not self.dynamic:
                raise ValueError(f"table {self.name}: evict_strategy needs a dynamic table (max_vocabulary_size=-1)")
            if self.max_capacity <= 0:
                raise ValueError(f"table {self.name}: evict_strategy needs max_capacity > 0 (rows per shard)")


class EmbeddingCollectionConfig:
    def __init__(self, use_exclusive_keys: bool = False,
                 comm_strategy: CommunicationStrategy = CommunicationStrategy.Uniform):
        self.use_exclusive_keys = use_exclusive_keys
        self.comm_strategy = comm_strategy
        self.lookups: List[dict] = []       # one entry per embedding_lookup call
        self.shard_matrix: Optional[List[List[int]]] = None
        self.shard_strategy: Optional[list] = None
        self.compression_strategy: dict = {}

    def embedding_lookup(self, table_config, bottom_name, top_name: str, combiner):
        if isinstance(table_config, (list, tuple)):
            assert len(table_config) == len(bottom_name) == len(combiner)
            self.lookups.append({"tables": list(table_config), "bottoms": list(bottom_name),
                                 "top": top_name, "combiners": list(combiner), "batch_major": True})
        else:
            self.lookups.append({"tables": [table_config], "bottoms": [bottom_name],
                                 "top": top_name, "combiners": [combiner], "batch_major": False})

    def shard(self, shard_matrix, shard_strategy, compression_strategy=None):
        self.shard_matrix = [list(r) for r in shard_matrix]
        self.shard_strategy = list(shard_strategy)
        self.compression_strategy = dict(compression_strategy or {})

    def tables(self) -> List[EmbeddingTableConfig]:
        seen, res = set(), []
        for lk in self.lookups:
            for t in lk["tables"]:
                if t.name not in seen:
                    seen.add(t.name)
                    res.append(t)
        return res


# ------------------------------------------------------------------------- placement
@dataclass
class TablePlacement:
    kind: str                  # "mp" | "dp"
    shard_gpus: List[int]      # GPUs holding a row shard (mp) ; all GPUs (dp)
    col_factor: int = 1        # column-wise split factor


def resolve_placement(cfg: EmbeddingCollectionConfig, num_gpus: int) -> Dict[str, TablePlacement]:
    tables = cfg.tables()
    names = [t.name for t in tables]
    place: Dict[str, TablePlacement] = {}
    if cfg.shard_matrix is None:
        # default plan: every table model-parallel, table-wise round robin (sample round_robin plan)
        for i, n in enumerate(names):
            place[n] = TablePlacement("mp", [i % num_gpus])
        return place
    sm = cfg.shard_matrix
    if len(sm) != num_gpus:
        # a plan written for another GPU count (a graph JSON of an 8-GPU training run opened by a single-GPU
        # inference session, or a job restarted on a different machine): keep which tables are data parallel, place
        # the model-parallel ones table-wise round robin.  Checkpoints load under any sharding, so nothing is lost.
        from ..utils import logger
        logger.warning(f"sharding plan has {len(sm)} GPU rows, the job runs {num_gpus}: re-planned "
                       "(data-parallel tables kept, model-parallel tables table-wise round robin)")
        dp = set()
        for kind, items in (cfg.shard_strategy or []):
            if kind == "dp":
                dp |= {str(it[0] if isinstance(it, (tuple, list)) else it) for it in items}
        for i, n in enumerate(names):
            place[n] = TablePlacement("dp", list(range(num_gpus))) if n in dp else TablePlacement("mp", [i % num_gpus])
        return place
    if any(isinstance(x, str) for row in sm for x in row):
        # the reference's form (embedding_collection.hpp:55-90, samples/dlrm/sharding/generate_plan.py):
        # row g lists the NAMES of the tables GPU g holds -> 0/1 matrix over the table order
        unknown = {x for row in sm for x in row} - set(names)
        if unknown:
            raise ValueError(f"shard_matrix names unknown tables: {sorted(unknown)}")
        sm = [[1 if n in set(map(str, row)) else 0 for n in names] for row in sm]
    for n in names:
        place[n] = None
    for kind, items in cfg.shard_strategy:
        for it in items:
            if isinstance(it, (tuple, list)):
                tn, factor = str(it[0]), int(it[1])
            else:
                tn, factor = str(it), 1
            ti = names.index(tn)
            gpus = [g for g in range(num_gpus) if sm[g][ti]]
            if kind == "dp":
                place[tn] = TablePlacement("dp", list(range(num_gpus)))
            else:
                assert gpus, f"table {tn} is not placed on any GPU"
                assert len(gpus) % factor == 0, "column-wise factor must divide the shard count"
                place[tn] = TablePlacement("mp", gpus, factor)
    for n in names:
        if place[n] is None:
            ti = names.index(n)
            gpus = [g for g in range(num_gpus) if sm[g][ti]]
            place[n] = TablePlacement("mp", gpus or [ti % num_gpus])
    return place


def _uniform_fill(view, bound, gen):
    """U(-bound, bound) into ``view``: drawn in fp32, a bf16 arena gets them rounded to nearest"""
    if view.dtype == torch.float32:
        view.uniform_(-bound, bound, generator=gen)
    else:
        view.copy_(torch.empty(view.shape, dtype=torch.float32, device=view.device).uniform_(-bound, bound, generator=gen))


def shard_rows(vocab: int, k: int, s: int) -> int:
    """number of keys in [0, vocab) with key % k == s"""
    return (vocab - s + k - 1) // k if vocab > s else 0


# ------------------------------------------------------------------------- runtime
class _Group:
    """Local tables of one (kind, ev pitch, weight dtype) group: one arena + optimizer state.
    Row-wise AdaGrad tables form groups of their own, keyed also by their epsilon and initial value,
    whose state ``s0`` holds one fp32 accumulator per arena row."""

    def __init__(self, kind, pitch, wdtype="fp32", rowwise=False):
        self.kind, self.pitch, self.wdtype = kind, pitch, wdtype
        self.rowwise = rowwise
        self.rows = 0
        self.table_slices = []   # (table name, col part, row_off, rows, num_shards, shard_idx, col0)
        self.lookups: List[E.LookupDesc] = []
        self.opt: Optional[OptParamsPy] = None

    @property
    def state_pitch(self) -> int:
        """state values per arena row: the pitch, or 1 for row-wise AdaGrad"""
        return 1 if self.rowwise else self.pitch


@dataclass
class _KeyChannel:
    """One key-side buffer (the keys, or the fp32 weights of weighted lookups) and its exchange: the
    owners read row r of ``all`` as rank r's copy of ``slab``."""
    slab: torch.Tensor
    all: Optional[torch.Tensor] = None         # [world, n]
    peers: Optional[list] = None               # peer-memory path: every rank's ``all`` (the inboxes)
    routes: Optional[list] = None              # peer-memory path: this rank's dispatch plan
    routes_dev: Optional[torch.Tensor] = None
    nnz_all: Optional[torch.Tensor] = None     # keys on the peer-memory path: [world, nnz_slab_elems]
    nnz_peers: Optional[list] = None           # split lengths, written by the key dispatch
    recv: Optional[torch.Tensor] = None        # packed collective exchange: blocks from every rank


@dataclass
class _SourceBufs:
    """What a group's kernels read and write, one entry per source rank whose batch they serve (this
    rank alone for data-parallel groups and single-GPU jobs)."""
    keys: list
    out: list
    grads: Optional[list]
    nnz: Optional[list]
    weights: Optional[list]


def fused_backward_ok(grp: _Group) -> bool:
    """Whether a model-parallel group may use the fused index + reduce/update backward: it locates
    gradient rows in 4-element units, so every lookup's gradient columns must be 4-aligned (a top
    that concatenates an ev-6 table in front of another table, or that follows a width-6 top at an
    odd batch, is not); other groups take the accumulate + update path."""
    return E.vec4_aligned(grp.lookups, grp.pitch) and \
        os.environ.get("HCTR_EMB_BWD", "indexed") == "indexed"


class EmbeddingCollection:
    def __init__(self, cfg: EmbeddingCollectionConfig, batch_per_gpu: int, hotness: Dict[str, int],
                 device, act_dtype, comm, default_opt: OptParamsPy, key_dtype=torch.int32,
                 scaler: float = 1.0, state_dtype=torch.float32, seed: int = 0,
                 fused: Optional[bool] = None, is_train: bool = True, weighted=()):
        """``weighted``: names of the sparse inputs whose keys carry an fp32 weight each (see
        docs/embedding.md): every lookup of such an input pools ``sum_h w_h * T[key_h]`` (mean: divided
        by ``sum_h w_h``, or by 1 when that is 0)."""
        self.cfg, self.b, self.device, self.act_dtype = cfg, batch_per_gpu, device, act_dtype
        self.weighted_inputs = frozenset(weighted)
        # who am I / whom do I talk to: through the backend-neutral interface (core.py; reference core.hpp)
        from ..core import as_core
        self.core = as_core(comm)
        self.comm = comm = self.core.get_comm()
        self.rank, self.world = self.core.get_global_gpu_id(), self.core.get_global_gpu_count()
        self.key_dtype = key_dtype
        self.scaler = scaler
        self.state_dtype = state_dtype
        self.default_opt = default_opt
        self.tables = cfg.tables()
        self.tmap = {t.name: t for t in self.tables}
        self.placement = resolve_placement(cfg, self.world)
        for t in self.tables:
            pl = self.placement[t.name]
            if t.evict_strategy is not None and (pl.kind != "mp" or pl.col_factor > 1):
                raise ValueError(f"table {t.name}: an evicting table is model parallel, table-wise or row-wise "
                                 f"(placement {pl.kind!r}, column factor {pl.col_factor})")
        self.native = device.type == "cuda"
        self.has_dynamic = any(t.dynamic for t in self.tables)
        self.fused = (self.native and self.world > 1 and comm.p2p_available) if fused is None else fused
        # requester-side split of row-sharded bags (see _build_layout): part of the fused key dispatch
        self.shard_split = self.world > 1 and bool(self.fused)
        # dynamic tables translate keys with a device hash table and flag overflow on the device: the
        # step has no host sync (graph capturable); check_overflow() reads the flags on demand
        self.dynamic_graph_safe = True
        # node-aware two-stage exchange (collective path only; inside one NVSwitch box the fused
        # peer-memory kernels are used instead)
        self.hier = (not self.fused and self.world > 1
                     and cfg.comm_strategy == CommunicationStrategy.Hierarchical
                     and getattr(comm, "num_nodes", 1) > 1)
        self.is_train = is_train
        self.hotness = dict(hotness)
        self.seed = seed
        # seed of the stochastic rounding of bf16 weights (with the device step counter and the arena
        # index: a run is reproducible for a fixed sharding plan)
        self.sr_seed = int(seed) & 0xFFFFFFFF
        self._unique_tables = self._resolve_unique_tables()
        self._check_weighted()
        self._kb = 8 if key_dtype == torch.int64 else 4
        self._abf = act_dtype == torch.bfloat16
        # clock of the evicting tables: ticked once per training step inside the step (not Model.step_t,
        # which a learning-rate scheduler reset zeroes and Adam's bias correction reads)
        self.evict_clock = torch.zeros(1, dtype=torch.int64, device=device)
        self._build_layout(hotness)
        self._build_storage(seed)
        self._alloc_buffers()

    def _resolve_unique_tables(self):
        """Tables whose lookups use CompressionStrategy.Unique (embedding/unique_exchange.py): named (or
        indexed) in ``cfg.compression_strategy``, model parallel, static, not column-split -- and only on the
        collective path: the peer-memory path moves pooled vectors with posted stores and keeps them."""
        from ..enums import CompressionStrategy
        req = None
        for k, v in (self.cfg.compression_strategy or {}).items():
            if k == CompressionStrategy.Unique or str(k).endswith("Unique"):
                req = v
        if not req or self.world == 1:
            return set()
        names = [t.name for t in self.tables]
        want = {names[x] if isinstance(x, int) else str(x) for x in req}
        unknown = want - set(names)
        if unknown:
            raise ValueError(f"compression_strategy names unknown tables: {sorted(unknown)}")
        from ..utils import logger
        if self.fused or self.hier:
            logger.info("CompressionStrategy.Unique: %s exchange keeps pooled-vector transfers for tables %s"
                        % ("peer-memory" if self.fused else "hierarchical", sorted(want)))
            return set()
        ok = set()
        for n in want:
            pl, t = self.placement[n], self.tmap[n]
            if pl.kind == "mp" and pl.col_factor == 1 and not t.dynamic:
                ok.add(n)
            else:
                logger.info(f"CompressionStrategy.Unique: table {n} ({pl.kind}, column factor {pl.col_factor}, "
                            f"dynamic={t.dynamic}) stays on the Reduction exchange")
        return ok

    def _check_weighted(self):
        """Weighted inputs pool weighted sums or means; the lookups that cannot honour weights reject them."""
        from ..enums import CompressionStrategy
        unique = set()
        for k, v in (self.cfg.compression_strategy or {}).items():
            if k == CompressionStrategy.Unique or str(k).endswith("Unique"):
                names = [t.name for t in self.tables]
                unique |= {names[x] if isinstance(x, int) else str(x) for x in v}
        for lk in self.cfg.lookups:
            for t, bot, comb in zip(lk["tables"], lk["bottoms"], lk["combiners"]):
                if bot not in self.weighted_inputs:
                    continue
                if comb not in ("sum", "mean", "average"):
                    raise ValueError(f"weighted input {bot}: lookup {lk['top']} of table {t.name} uses the {comb!r} "
                                     "combiner; weighted inputs pool with sum or mean")
                if t.name in unique:
                    raise ValueError(f"weighted input {bot}: table {t.name} is listed under CompressionStrategy.Unique, "
                                     "which does not carry weights")

    def eval_clone(self, batch_per_gpu: int) -> "EmbeddingCollection":
        """Second plan (different batch, no grads) over the SAME tables -- the eval graph."""
        import copy
        c = copy.copy(self)
        c.b = batch_per_gpu
        c.is_train = False
        c._shared = self
        self._clones = getattr(self, "_clones", []) + [c]
        c._build_layout(self.hotness)
        c._build_storage(self.seed, share_from=self)
        c._alloc_buffers()
        return c

    # ---- layout of key / output / grad slabs (identical on every rank)
    def _build_layout(self, hotness):
        b = self.b
        self.glookups = []          # global lookup list
        self.tops = []              # (top name, width, batch_major, [global lookup ids])
        koff = 0
        ooff = 0
        for lk in self.cfg.lookups:
            ids, col = [], 0
            width = 0
            for t, bot, comb in zip(lk["tables"], lk["bottoms"], lk["combiners"]):
                H = int(hotness[bot])
                w = t.ev_size * (H if comb == "concat" else 1)
                width += w
            for t, bot, comb in zip(lk["tables"], lk["bottoms"], lk["combiners"]):
                H = int(hotness[bot])
                gl = {"table": t.name, "bottom": bot, "combiner": comb, "hotness": H,
                      "key_off": koff, "top": len(self.tops), "col": col, "ev": t.ev_size,
                      "out_off": ooff + col, "out_stride": width,
                      "weighted": bot in getattr(self, "weighted_inputs", ())}
                koff += b * H
                col += t.ev_size * (H if comb == "concat" else 1)
                ids.append(len(self.glookups))
                self.glookups.append(gl)
            self.tops.append({"name": lk["top"], "width": width, "batch_major": lk["batch_major"],
                              "lookups": ids, "off": ooff})
            ooff += b * width
        self.user_key_elems = koff
        self.key_slab_elems = koff
        # fp32 per-key weights in the layout of the user region of the key slab (weighted inputs only)
        self.has_weights = any(gl["weighted"] for gl in self.glookups)
        self.nnz_slab_elems = 0
        self.top_slab_elems = ooff
        # partial blocks for row-sharded lookups (k > 1 on the mp side)
        poff = ooff
        for gl in self.glookups:
            pl = self.placement[gl["table"]]
            k = len(pl.shard_gpus) // pl.col_factor if pl.kind == "mp" else 1
            gl["k"] = k
            if gl["table"] in getattr(self, "_unique_tables", ()):
                # distinct keys travel once, rows come back once per distinct key (unique_exchange.py):
                # no owner-side lookup descriptors, no per-shard partial blocks
                gl["unique"], gl["unique_owners"] = True, list(pl.shard_gpus)
                continue
            # (not for evicting tables: their owners translate the raw keys of the whole bag; not for
            # weighted lookups: their owners read each key's weight at the key's own position)
            if getattr(self, "shard_split", False) and pl.kind == "mp" and k > 1 and pl.col_factor == 1 \
                    and gl["combiner"] == "sum" and self.tmap[gl["table"]].evict_strategy is None \
                    and not gl["weighted"]:
                # Requester-side split: every rank rewrites its bag of a row-sharded table into k
                # compacted per-shard lists of LOCAL ROW INDICES (key // k) plus their lengths, stored
                # behind the user keys in the (symmetric) key slab.  A shard owner then reads only
                # its 1/k of the bag instead of scanning all of it and filtering `key % k`.
                gl["split_off"] = self.key_slab_elems
                gl["split_nnz_off"] = self.nnz_slab_elems
                self.key_slab_elems += k * b * gl["hotness"]
                self.nnz_slab_elems += k * b
            if pl.kind == "mp" and k > 1:
                gl["partial_off"] = poff
                gl["partial_w"] = k * gl["ev"] * (gl["hotness"] if gl["combiner"] == "concat" else 1)
                poff += b * gl["partial_w"]
        self.out_slab_elems = poff
        # Default (HCTR_CONCAT_ALIAS=0 disables): spare room behind the slabs so that a downstream Concat
        # layer can have a batch-major top written straight into ITS output buffer (alias_top): the
        # kernels already take a row stride / offset per lookup, so the strided copy disappears.
        import os as _os
        self.alias_reserve = 1024 if _os.environ.get("HCTR_CONCAT_ALIAS", "1") == "1" else 0
        self.alias_out_off, self.alias_grad_off = {}, {}
        goff = self.top_slab_elems
        if self.alias_reserve:
            for tp in self.tops:
                if tp["batch_major"]:
                    self.alias_out_off[tp["name"]] = self.out_slab_elems
                    self.alias_grad_off[tp["name"]] = goff
                    self.out_slab_elems += b * (tp["width"] + self.alias_reserve)
                    goff += b * (tp["width"] + self.alias_reserve)
        self.grad_slab_elems = goff

    # ---- local storage + owner-side lookup descriptors
    def _build_storage(self, seed, share_from=None):
        groups: Dict[Tuple[str, int, str], _Group] = {}
        b = self.b
        wdtype = {t.name: getattr(t, "weight_dtype", "fp32") for t in self.tables}
        dp_bf16 = [n for n, w in wdtype.items() if w != "fp32" and self.placement[n].kind == "dp"]
        if dp_bf16 and share_from is None:
            from ..utils import logger
            logger.info(f"weight_dtype: data-parallel tables {sorted(dp_bf16)} keep fp32 weights (their gradients "
                        "take the dense all-reduce and the dense optimizer)")
        for t in self.tables:
            pl = self.placement[t.name]
            cf = pl.col_factor
            ev_part = t.ev_size // cf
            assert ev_part * cf == t.ev_size, "ev_size must be divisible by the column factor"
            if self.device.type == "cuda":
                E.check_ev_size(ev_part, f"table {t.name}: embedding vector")
            if pl.kind == "dp":
                parts = [(0, 1, 0)]
            else:
                parts = []
                kk = len(pl.shard_gpus) // cf
                for idx, g in enumerate(pl.shard_gpus):
                    if g == self.rank:
                        parts.append((idx // kk, kk, idx % kk))   # (col part, num row shards, shard)
            o = t.opt_params or self.default_opt
            rowwise = o is not None and o.optimizer_type == Optimizer_t.RowWiseAdaGrad
            for (cpart, k, s) in parts:
                wdt = wdtype[t.name] if pl.kind == "mp" else "fp32"
                key = (pl.kind, ev_part, wdt)
                if rowwise:
                    # never shares an arena (and its first table's optimizer) with another optimizer
                    key += ("rowwise", float(o.epsilon), float(o.initial_accu_value))
                grp = groups.setdefault(key, _Group(pl.kind, ev_part, wdt, rowwise))
                if t.evict_strategy is not None:
                    rows = (t.max_capacity + 31) // 32 * 32       # whole 32-way sets, allocated once
                else:
                    rows = t.init_capacity if t.dynamic else shard_rows(t.max_vocabulary_size, k, s)
                grp.table_slices.append({"table": t.name, "cpart": cpart, "row_off": grp.rows,
                                         "rows": rows, "k": k, "s": s, "col0": cpart * ev_part,
                                         "ev": ev_part, "dynamic": t.dynamic, "evict": t.evict_strategy})
                grp.rows += rows
                if grp.opt is None:
                    grp.opt = o
        # lookups per group
        for gi, gl in enumerate(self.glookups):
            t = self.tmap[gl["table"]]
            pl = self.placement[t.name]
            for grp in groups.values():
                for sl in grp.table_slices:
                    if sl["table"] != t.name:
                        continue
                    if gl.get("unique"):
                        gl["unique_local"] = (grp, sl)
                        continue
                    H = gl["hotness"]
                    concat = gl["combiner"] == "concat"
                    nsub = H if concat else 1
                    for sub in range(nsub):
                        if pl.kind == "mp" and sl["k"] > 1:
                            base = gl["partial_off"]
                            ostride = gl["partial_w"]
                            ocol = sl["s"] * gl["ev"] * nsub + sub * gl["ev"] + sl["col0"]
                        else:
                            base = gl["out_off"]
                            ostride = gl["out_stride"]
                            ocol = sub * gl["ev"] + sl["col0"]
                        split = ("split_off" in gl and pl.kind == "mp" and sl["k"] > 1) or sl["dynamic"]
                        grp.lookup_gl = getattr(grp, "lookup_gl", [])
                        grp.lookup_gl.append((gi, pl.kind == "mp" and sl["k"] > 1))
                        grp.lookup_slices = getattr(grp, "lookup_slices", [])
                        grp.lookup_slices.append(sl)
                        grp.lookups.append(E.LookupDesc(
                            table_row_off=sl["row_off"],
                            key_off=(gl["split_off"] + sl["s"] * b * H)
                            if (split and not sl["dynamic"]) else gl["key_off"] + sub,
                            out_off=base + ocol, grad_off=gl["out_off"] + sub * gl["ev"] + sl["col0"],
                            hotness=1 if concat else H, key_stride=H,
                            num_shards=1 if split else sl["k"], shard_idx=0 if split else sl["s"],
                            out_stride=ostride, grad_stride=gl["out_stride"],
                            combiner=1 if gl["combiner"] in ("mean", "average") else 0,
                            ev_size=sl["ev"], rows=sl["rows"],
                            nnz_off=(gl["split_nnz_off"] + sl["s"] * b)
                            if (split and not sl["dynamic"]) else -1,
                            weighted=int(gl["weighted"])))
        self.groups = list(groups.values())
        dev = self.device
        gen = torch.Generator(device="cpu")
        if share_from is not None:
            for grp, src in zip(self.groups, share_from.groups):
                assert (grp.kind, grp.pitch, grp.wdtype, grp.rowwise, len(grp.table_slices)) == \
                    (src.kind, src.pitch, src.wdtype, src.rowwise, len(src.table_slices))
                grp.opt = src.opt
                grp.ws = None
            self._resync_storage(share_from)     # arrays + row windows (dynamic shards may have grown since)
            return
        for grp in self.groups:
            n = max(grp.rows, 1) * grp.pitch
            grp.table = torch.empty(n, dtype=WEIGHT_DTYPES[grp.wdtype], device=dev)
            self._init_group(grp, gen, seed)
            sdt = self.state_dtype if grp.kind == "mp" else torch.float32
            grp.s0, grp.s1 = opt_states(grp.opt, n, sdt, dev) if self.is_train else (None, None)
            if grp.rowwise and self.is_train:
                # one fp32 accumulator per row, whatever the state dtype (an only-growing bf16 value
                # would drop small increments)
                grp.s0 = torch.full((max(grp.rows, 1),), float(grp.opt.initial_accu_value),
                                    dtype=torch.float32, device=dev)
            R = self.world if grp.kind == "mp" else 1
            po = 0
            for l in grp.lookups:
                l.pair_off = po
                po += R * self.b * l.hotness
            grp.lookups_dev = E.lookups_to_device(grp.lookups, dev)
            for sl in grp.table_slices:
                if sl["evict"]:
                    self._dyn_hash(sl["table"], sl)
            pairs = po
            if self.is_train:
                if grp.kind == "mp":
                    grp.indexed = dev.type == "cuda" and fused_backward_ok(grp)
                    grp.ws = E.UniqueWorkspace(max(pairs, 1), grp.pitch, dev, indexed=grp.indexed,
                                               need_scale=any(l.combiner == 1 or l.weighted for l in grp.lookups))
                else:
                    n_pad = (n + 4 * self.world - 1) // (4 * self.world) * (4 * self.world)
                    if self.fused and self.world > 1 and not getattr(self.comm, "emulated", False):
                        from ..parallel.p2p import P2PAllReduce
                        grp.dense_wgrad_full = self.comm.symm_alloc(n_pad, torch.float32)
                        grp.p2p_ar = P2PAllReduce(self.comm, grp.dense_wgrad_full, blocks=32)
                    else:
                        grp.dense_wgrad_full = torch.zeros(n_pad, dtype=torch.float32, device=dev)
                        grp.p2p_ar = None
                    grp.dense_wgrad = grp.dense_wgrad_full[:n]
                    grp.ws = None

    def _init_group(self, grp, gen, seed):
        """default U(+-sqrt(1/max_vocabulary_size)) (ragged_static_embedding.cu:501-530)."""
        for sl in grp.table_slices:
            t = self.tmap[sl["table"]]
            bound = math.sqrt(1.0 / max(t.max_vocabulary_size if not t.dynamic else t.init_capacity, 1))
            ip = t.init_param
            if ip is not None and ip.up_bound > 0:
                bound = ip.up_bound
            view = grp.table[sl["row_off"] * grp.pitch:(sl["row_off"] + sl["rows"]) * grp.pitch]
            if view.numel() == 0:
                continue
            if grp.kind == "dp" or self.device.type == "cpu":
                # identical on every replica: generate by global row on host
                gen.manual_seed(_stable_seed(seed, sl["table"], sl["cpart"]))
                full_rows = t.max_vocabulary_size
                if not t.dynamic and full_rows * grp.pitch <= (1 << 26):
                    full = (torch.rand(full_rows, grp.pitch, generator=gen) * 2 - 1) * bound
                    view.copy_(full[sl["s"]::sl["k"]].reshape(-1).to(view.device))   # bf16: to nearest
                    continue
            g2 = torch.Generator(device=self.device)
            g2.manual_seed(_stable_seed(seed, sl["table"], sl["cpart"], sl["s"]))
            _uniform_fill(view, bound, g2)

    def _alloc_buffers(self):
        dev, b, W = self.device, self.b, self.world
        z = lambda n, dt: torch.zeros(max(int(n), 1), dtype=dt, device=dev)
        self.key_slab = z(self.key_slab_elems, self.key_dtype)
        self.weight_slab = z(self.user_key_elems, torch.float32) if self.has_weights else None
        # the key-side channels: the keys (whose peer-memory dispatch also writes the split lengths), then
        # the weights of weighted lookups, which follow their keys' blocks
        self.key_chans = [_KeyChannel(self.key_slab)]
        if self.has_weights:
            self.key_chans.append(_KeyChannel(self.weight_slab))
        self.grads_all = None
        if self.fused:
            # Inboxes in the peer-mapped heap, one slot per source rank, same layout as a key / grad
            # slab: requesters scatter their key blocks and gradient rows into them with posted peer
            # stores (csrc/emb_dispatch.cu); owners write pooled vectors into the requesters' out slabs.
            # Every owner-side kernel then reads LOCAL memory only.
            sa = self.comm.symm_alloc
            for ch in self.key_chans:
                n = ch.slab.numel()
                ch.all = sa(W * n, ch.slab.dtype).view(W, n)
                ch.peers = self.comm.peer_ptrs(ch.all)
            if self.nnz_slab_elems:
                ns, kc = self.nnz_slab_elems, self.key_chans[0]
                kc.nnz_all = sa(W * ns, torch.int32).view(W, ns)
                kc.nnz_peers = self.comm.peer_ptrs(kc.nnz_all)
            self.out_slab = sa(max(self.out_slab_elems, 1), self.act_dtype)
            self.peer_out = self.comm.peer_ptrs(self.out_slab)
            self.grad_slab = z(self.grad_slab_elems, self.act_dtype) if self.is_train else None
            if self.is_train:
                gs = max(self.grad_slab_elems, 1)
                self.grads_all = sa(W * gs, self.act_dtype).view(W, gs)
                self.peer_grads_all = self.comm.peer_ptrs(self.grads_all)
            for ch, routes in zip(self.key_chans, self._build_key_routes(self.rank)):
                ch.routes, ch.routes_dev = routes, E.routes_to_device(routes, dev)
            # bytes this rank stores into peers per step (roofline accounting)
            self.dispatch_key_bytes = sum(r.rows * r.row_elems * ch.slab.element_size()
                                          for ch in self.key_chans for r in ch.routes if r.dst_rank != self.rank)
            self._grad_routes = None
        else:
            self.out_slab = z(self.out_slab_elems, self.act_dtype)
            self.grad_slab = z(self.grad_slab_elems, self.act_dtype) if self.is_train else None
            if W > 1:
                for ch in self.key_chans:
                    ch.all = torch.zeros(W, ch.slab.numel(), dtype=ch.slab.dtype, device=dev)
                self.send_out = torch.zeros(W, max(self.out_slab_elems, 1), dtype=self.act_dtype, device=dev)
                if self.is_train:
                    self.grads_all = torch.zeros(W, max(self.grad_slab_elems, 1), dtype=self.act_dtype,
                                                 device=dev)
                if not self.hier:
                    self._build_packed_exchange()
        rows = lambda t: None if t is None else list(t.unbind(0))
        for grp in self.groups:
            if W == 1 or grp.kind == "dp":
                grp.src = _SourceBufs([self.key_slab], [self.out_slab],
                                      None if self.grad_slab is None else [self.grad_slab], None,
                                      None if self.weight_slab is None else [self.weight_slab])
            else:
                kc = self.key_chans[0]
                grp.src = _SourceBufs(rows(kc.all), self.peer_out if self.fused else rows(self.send_out),
                                      rows(self.grads_all), rows(kc.nnz_all),
                                      rows(self.key_chans[1].all) if self.has_weights else None)
        # evicting tables: the ways admitted by one step (at most one per key position), re-initialised
        # after the table's last insert
        self._evict_adm = {}
        if self.is_train:
            for name, gls in self._evicting_lookups().items():
                if self._evict_local(name) is not None:
                    n = sum(W * b * gl["hotness"] for gl in gls)
                    self._evict_adm[name] = (torch.zeros(n, dtype=torch.int64, device=dev),
                                             torch.zeros(1, dtype=torch.int32, device=dev))
        uq = [gi for gi, gl in enumerate(self.glookups) if gl.get("unique")]
        self._uniq = None
        if uq:
            from .unique_exchange import UniqueExchange
            self._uniq = UniqueExchange(self, uq)
        # named views
        self.key_views, self.weight_views = {}, {}
        for gl in self.glookups:
            self.key_views[gl["bottom"]] = self.key_slab[gl["key_off"]:gl["key_off"] + b * gl["hotness"]] \
                .view(b, gl["hotness"])
            if gl["weighted"]:
                self.weight_views[gl["bottom"]] = self.weight_slab[gl["key_off"]:gl["key_off"] + b * gl["hotness"]] \
                    .view(b, gl["hotness"])
        self.top_data, self.top_grad = {}, {}
        for tp in self.tops:
            w = tp["width"]
            shp = (b, w) if tp["batch_major"] else (b, 1, w)
            self.top_data[tp["name"]] = self.out_slab[tp["off"]:tp["off"] + b * w].view(shp)
            if self.is_train:
                self.top_grad[tp["name"]] = self.grad_slab[tp["off"]:tp["off"] + b * w].view(shp)

    def _mp_owners(self, gl):
        """[(rank, column part, row shards k, row shard s)] of the table behind a lookup (mp only)"""
        pl = self.placement[gl["table"]]
        if pl.kind != "mp":
            return []
        kk = len(pl.shard_gpus) // pl.col_factor
        return [(g, idx // kk, kk, idx % kk) for idx, g in enumerate(pl.shard_gpus)]

    def _build_key_routes(self, me):
        """Forward dispatch plan of rank ``me``'s batch, one route list per key-side channel: per
        model-parallel lookup one route per owner -- the whole block of keys (and of their weights), or
        (row-sharded, peer-memory path) the owner's compacted shard list + lengths."""
        b = self.b
        ks, ns, wn = max(self.key_slab_elems, 1), self.nnz_slab_elems, max(self.user_key_elems, 1)
        keys, weights = [], []
        for gl in self.glookups:
            H, n, off = gl["hotness"], b * gl["hotness"], gl["key_off"]
            if "split_off" in gl:
                for (g, _, kk, s_) in self._mp_owners(gl):
                    keys.append(E.Route(src_off=off, dst_off=me * ks + gl["split_off"] + s_ * b * H, rows=b,
                                        row_elems=H, src_stride=H, dst_stride=H, dst_rank=g, kind=1, k=kk,
                                        shard=s_, nnz_off=me * ns + gl["split_nnz_off"] + s_ * b))
                continue
            for g in sorted({o[0] for o in self._mp_owners(gl)}):
                keys.append(E.Route(src_off=off, dst_off=me * ks + off, rows=1, row_elems=n, src_stride=n,
                                    dst_stride=n, dst_rank=g))
                if gl["weighted"]:
                    weights.append(E.Route(src_off=off, dst_off=me * wn + off, rows=1, row_elems=n,
                                           src_stride=n, dst_stride=n, dst_rank=g))
        return [keys, weights] if self.has_weights else [keys]

    def _build_grad_routes(self):
        """Backward push plan: the gradient columns of every model-parallel lookup go to each rank that
        owns (a shard of) its table.  Built at the first backward, after any alias_top() re-homing."""
        b, me = self.b, self.rank
        gs = max(self.grad_slab_elems, 1)
        routes = []
        for gl in self.glookups:
            tp = self.tops[gl["top"]]
            w = gl["ev"] * (gl["hotness"] if gl["combiner"] == "concat" else 1)
            al = tp.get("alias")
            if al:
                base, stride = al["goff"] + al["col"] + (gl["out_off"] - tp["off"]), al["stride"]
            else:
                base, stride = gl["out_off"], gl["out_stride"]
            for g in sorted({o[0] for o in self._mp_owners(gl)}):
                routes.append(E.Route(src_off=base, dst_off=me * gs + base, rows=b, row_elems=w,
                                      src_stride=stride, dst_stride=stride, dst_rank=g))
        self._grad_routes = routes
        self._grad_routes_dev = E.routes_to_device(routes, self.device)
        esz = 2 if self._abf else 4
        self.push_grad_bytes = sum(r.rows * r.row_elems * esz for r in routes if r.dst_rank != me)

    def alias_top(self, name: str, total_width: int, col_off: int):
        """Re-home the batch-major top ``name`` inside a [b, total_width] buffer carved from the slabs
        (columns [col_off, col_off + width)): lookups write / read it with row stride total_width.
        Returns (data [b, total_width], grad [b, total_width] or None), or None when not possible."""
        if not getattr(self, "alias_reserve", 0) or name not in self.alias_out_off:
            return None
        if self.world > 1 and not self.fused:
            return None                       # the collective exchanges are planned over the slab layout
        tp = [t for t in self.tops if t["name"] == name][0]
        w, b = tp["width"], self.b
        esz = 2 if self.act_dtype == torch.bfloat16 else 4
        if tp.get("alias") or total_width > w + self.alias_reserve or col_off + w > total_width \
                or (col_off * esz) % 16 or (total_width * esz) % 16:
            return None
        oo, go = self.alias_out_off[name], self.alias_grad_off[name]
        ti = self.tops.index(tp)
        for grp in self.groups:
            for lk, (gi, partial) in zip(grp.lookups, grp.lookup_gl):
                gl = self.glookups[gi]
                if gl["top"] != ti:
                    continue
                if not partial:
                    lk.out_off = oo + col_off + (lk.out_off - tp["off"])
                    lk.out_stride = total_width
                lk.grad_off = go + col_off + (lk.grad_off - tp["off"])
                lk.grad_stride = total_width
            grp.lookups_dev = E.lookups_to_device(grp.lookups, self.device)
        tp["alias"] = {"off": oo, "goff": go, "stride": total_width, "col": col_off}
        full = self.out_slab[oo:oo + b * total_width].view(b, total_width)
        self.top_data[name] = full[:, col_off:col_off + w]
        gfull = None
        if self.is_train:
            gfull = self.grad_slab[go:go + b * total_width].view(b, total_width)
            self.top_grad[name] = gfull[:, col_off:col_off + w]
        return full, gfull

    # ------------------------------------------------------------------ API
    def top_shapes(self):
        return {tp["name"]: ((self.b, tp["width"]) if tp["batch_major"] else (self.b, 1, tp["width"]))
                for tp in self.tops}

    def _build_packed_exchange(self):
        """Flat collective (NCCL / gloo) path: every element of a requester's output slab is produced by
        exactly one owner, and an owner needs only the key blocks and gradient columns of its own
        lookups.  So nothing travels as a whole slab (``world`` times the useful bytes): every requester
        sends owner o the key (and weight) blocks o serves, o sends requester r the ``n_o`` output
        elements it owns, r returns the ``n_o`` matching gradient elements.  The region lists are
        exchanged once here."""
        mine = [(int(d.out_off), int(d.out_stride), int(d.grad_off), int(d.grad_stride), int(d.ev_size))
                for grp in self.groups if grp.kind == "mp" for d in grp.lookups]
        # key blocks [key_off, key_off + b * hotness) of the lookups this rank serves
        kmine = sorted({(int(self.glookups[gi]["key_off"]), int(self.b * self.glookups[gi]["hotness"]))
                        for grp in self.groups if grp.kind == "mp" for (gi, _) in getattr(grp, "lookup_gl", [])})
        both = self.comm.all_gather_object((mine, kmine))
        regions, kregions = [x[0] for x in both], [x[1] for x in both]
        dev, b = self.device, self.b
        rows = torch.arange(b, dtype=torch.int64).view(b, 1)

        def flat(off, stride, ev):
            return (off + rows * stride + torch.arange(ev, dtype=torch.int64).view(1, ev)).reshape(-1)
        oidx, gidx = [], []
        for regs in regions:
            oidx.append(torch.cat([flat(o, s, e) for (o, s, _, _, e) in regs]) if regs
                        else torch.zeros(0, dtype=torch.int64))
            gidx.append(torch.cat([flat(g, gs, e) for (_, _, g, gs, e) in regs]) if regs
                        else torch.zeros(0, dtype=torch.int64))
        n = [int(x.numel()) for x in oidx]
        kidx = [torch.cat([torch.arange(o, o + ln, dtype=torch.int64) for (o, ln) in regs]) if regs
                else torch.zeros(0, dtype=torch.int64) for regs in kregions]
        kn = [int(x.numel()) for x in kidx]
        for ch in self.key_chans:
            ch.recv = torch.zeros(max(self.world * kn[self.rank], 1), dtype=ch.slab.dtype, device=dev)
        self.packed = {
            "kn": kn, "kn_me": kn[self.rank], "key_me": kidx[self.rank].to(dev), "key_all": torch.cat(kidx).to(dev),
            "n": n, "n_me": n[self.rank],
            "out_me": oidx[self.rank].to(dev), "out_all": torch.cat(oidx).to(dev),
            "grad_me": gidx[self.rank].to(dev), "grad_all": torch.cat(gidx).to(dev),
            "fwd_recv": torch.zeros(max(sum(n), 1), dtype=self.act_dtype, device=dev),
            "bwd_recv": torch.zeros(max(self.world * n[self.rank], 1), dtype=self.act_dtype, device=dev),
        }

    def set_keys(self, feature_major_keys: torch.Tensor):
        """Copy a whole feature-major key batch into the key slab (H2D lands here directly)."""
        self.key_slab[:feature_major_keys.numel()].copy_(feature_major_keys.reshape(-1), non_blocking=True)

    def set_weights(self, feature_major_weights: torch.Tensor):
        """Copy the fp32 per-key weights of a batch, in the layout of ``set_keys``, into the weight slab."""
        self.weight_slab[:feature_major_weights.numel()].copy_(feature_major_weights.reshape(-1), non_blocking=True)

    def forward(self, is_train: bool = True):
        self.forward_begin()
        self.forward_compute()
        self.forward_end()

    def forward_begin(self):
        """every rank's keys are in place (fused mode: device-side barrier; collective: all-to-all)"""
        if self.world > 1:
            if self.fused:
                # forward all-to-all of keys: posted peer stores into the owners' inboxes, then ONE
                # device barrier (also orders the previous step's readers of these inboxes)
                for ch in self.key_chans:
                    E.dispatch(ch.slab, ch.routes, ch.routes_dev, ch.peers, ch.nnz_peers, blocks_x=48)
                self.comm.barrier_device()
            elif os.environ.get("SKIP_DATA_DISTRIBUTOR", "0") not in ("0", ""):
                pass          # ablation (model_pipeline.cpp:118): owners keep the keys of an earlier step
            elif self.hier:
                for ch in self.key_chans:
                    self.comm.hier_all_gather(ch.all, ch.slab)
            else:
                pk, W = self.packed, self.world   # every owner receives only the blocks of the lookups it serves
                for ch in self.key_chans:
                    recv = ch.recv[:W * pk["kn_me"]]
                    self.comm.all_to_all_v(recv, ch.slab.index_select(0, pk["key_all"]), [pk["kn_me"]] * W, pk["kn"])
                    if pk["kn_me"]:
                        ch.all.index_copy_(1, pk["key_me"], recv.view(W, pk["kn_me"]))
        if self.has_dynamic:
            self._translate_dynamic_keys()

    def _dyn_hash(self, name, sl):
        """per (table, local shard) key -> row hash table, shared between the train and eval plans"""
        owner = getattr(self, "_shared", self)
        if not hasattr(owner, "_dyn_tables"):
            owner._dyn_tables = {}
        key = (name, sl["cpart"], sl["s"])
        if key not in owner._dyn_tables:
            if sl.get("evict"):
                from .hashtable import SetAssocTable
                owner._dyn_tables[key] = SetAssocTable(sl["rows"], sl["evict"], owner.evict_clock, self.device)
            else:
                from .hashtable import HashTable
                owner._dyn_tables[key] = HashTable(sl["rows"], self.device)
        return owner._dyn_tables[key]

    def _evicting_lookups(self):
        """{evicting table name: [its global lookups]}"""
        res = {}
        for gl in self.glookups:
            if self.tmap[gl["table"]].evict_strategy is not None:
                res.setdefault(gl["table"], []).append(gl)
        return res

    def _evict_local(self, name):
        """(group, slice) of this rank's shard of evicting table ``name``, or None"""
        for grp in self.groups:
            for sl in grp.table_slices:
                if sl["table"] == name:
                    return grp, sl
        return None

    def _evict_reinit(self, grp, sl, ht, adm):
        """fresh weights and initial optimizer state for the ways ``adm`` admitted"""
        t = self.tmap[sl["table"]]
        bound = math.sqrt(1.0 / max(t.init_capacity, 1))
        if t.init_param is not None and t.init_param.up_bound > 0:
            bound = t.init_param.up_bound
        o = grp.opt
        s0_init = o.initial_accu_value if (o is not None and o.optimizer_type in
                                           (Optimizer_t.AdaGrad, Optimizer_t.RowWiseAdaGrad)) else 0.0
        ht.reinit(adm, adm[0].numel(), grp.table, grp.s0, grp.s1, sl["row_off"], grp.pitch, grp.state_pitch,
                  s0_init, bound, self.evict_init_key(t.name), sl["col0"])

    def evict_init_key(self, name: str) -> int:
        """key of the stateless initializer of table ``name``'s admitted rows (ops.evict_init_rows)"""
        return E.evict_init_key(self.seed, _stable_seed("evict_init", name))

    def _translate_evicting(self, buf):
        """Evicting tables (see csrc/evict_table.cu): a training lookup ticks the clock, touches every key
        region of a table, then inserts into every region (rows in place over the keys), then re-initialises
        the admitted rows; an evaluation lookup only reads.  No host synchronisation."""
        b = self.b
        owner = getattr(self, "_shared", self)
        if self.is_train:
            owner.evict_clock.add_(1)
        for name, gls in self._evicting_lookups().items():
            regs = [(gl["key_off"], b * gl["hotness"]) for gl in gls]
            loc = self._evict_local(name)
            if loc is None:
                for off, n in regs:
                    buf[:, off:off + n].fill_(-1)
                continue
            grp, sl = loc
            ht = self._dyn_hash(name, sl)
            if not self.is_train:
                for off, n in regs:
                    ht.get(buf, off, n, sl["k"], sl["s"])
                continue
            for off, n in regs:
                ht.touch(buf, off, n, sl["k"], sl["s"])
            adm = self._evict_adm[name]
            adm[1].zero_()
            for off, n in regs:
                ht.insert(buf, off, n, sl["k"], sl["s"], adm=adm)
            self._evict_reinit(grp, sl, ht, adm)

    def eviction_stats(self):
        """{(table, shard): {live, admitted, evicted, dropped}} of the evicting tables held here: cumulative
        device counters, read with one host synchronisation (call it outside the step)"""
        from .hashtable import SetAssocTable
        owner = getattr(self, "_shared", self)
        items = [(k, ht) for k, ht in getattr(owner, "_dyn_tables", {}).items() if isinstance(ht, SetAssocTable)]
        if not items:
            return {}
        vals = torch.stack([torch.cat([ht.live().view(1), ht.stats]) for _, ht in items]).cpu().tolist()
        return {(name, s_): dict(zip(("live", "admitted", "evicted", "dropped"), (int(x) for x in v)))
                for ((name, _, s_), _), v in zip(items, vals)}

    def _translate_dynamic_keys(self):
        """Dynamic tables: overwrite the (gathered) keys of their lookups with local row indices -- new
        keys get the next free row while training, unknown keys read as empty (-1) in evaluation; keys
        owned by another shard become -1.  The lookup kernels then run exactly as for static tables."""
        b = self.b
        buf = self.key_slab.view(1, -1) if self.world == 1 else self.key_chans[0].all
        for gl in self.glookups:
            t = self.tmap[gl["table"]]
            if not t.dynamic or t.evict_strategy is not None:
                continue
            region = buf[:, gl["key_off"]:gl["key_off"] + b * gl["hotness"]]
            keys = region.to(torch.int64)
            out = torch.full_like(keys, -1)
            for grp in self.groups:
                for sl in grp.table_slices:
                    if sl["table"] != t.name or sl["cpart"] != 0:
                        continue
                    own = (keys >= 0) & ((keys % sl["k"]) == sl["s"])
                    ht = self._dyn_hash(t.name, sl)
                    k = torch.where(own, keys, torch.full_like(keys, -1)).reshape(-1)
                    # bounded insert: a key that finds no free row reads as empty (-1) and raises the
                    # table's sticky device flag -- no host sync here, see check_overflow()
                    rows = (ht.get_insert(k) if self.is_train else ht.get(k)).reshape(keys.shape)
                    out = torch.where(own & (rows >= 0), rows.to(torch.int64), out)
            region.copy_(out.to(region.dtype))
        if any(t.evict_strategy is not None for t in self.tables):
            self._translate_evicting(buf)

    def check_overflow(self):
        """Raise if a dynamic table ran out of rows (reads device flags: a host sync -- called by
        ``Model`` at display / evaluation / checkpoint time, never inside the captured step)."""
        owner = getattr(self, "_shared", self)
        for (name, cpart, s_), ht in getattr(owner, "_dyn_tables", {}).items():
            if self.tmap[name].evict_strategy is None and ht.overflowed():
                raise RuntimeError(f"dynamic embedding table {name}: more than init_capacity="
                                   f"{ht.max_rows} distinct keys on one shard (shard {s_})")
        for grp in self.groups:
            E.check_workspace_overflow(getattr(grp, "ws", None), f"{grp.kind} group ev={grp.pitch}")

    def grow_dynamic(self, factor: float = 2.0):
        """DynamicEmbeddingTable semantics (embedding_storage/dynamic_embedding.cu: the vocabulary is not bounded):
        every shard whose hash table ran out of rows gets ``factor`` times the rows -- the group's weight and
        optimizer-state arrays are re-laid out around the enlarged slice, the key -> row map is rebuilt with the same
        rows, new rows start from the initializer.  Keys that found no row since the overflow read as empty and their
        updates were dropped; they are admitted from the next step on.  Returns the grown (table, shard, old rows,
        new rows) list; the caller re-captures its CUDA graphs (table pointers are baked into them).  Reads device
        flags (host sync): call it where ``check_overflow`` is called.  Raises when ``max_capacity`` is reached."""
        owner = getattr(self, "_shared", self)
        grown = []
        for (name, cpart, s_), ht in list(getattr(owner, "_dyn_tables", {}).items()):
            if self.tmap[name].evict_strategy is not None or not ht.overflowed():
                continue
            old = ht.max_rows
            new = owner._grow_to(name, cpart, s_, int(old * factor) + 1)
            grown.append((name, s_, old, new))
        return grown

    def _grow_to(self, name, cpart, s_, want_rows: int) -> int:
        """(owner plan) enlarge shard ``s_`` of dynamic table ``name`` to ``want_rows`` rows (capped by the
        table's ``max_capacity``): storage, key -> row map with the same rows, every plan that shares the storage"""
        t = self.tmap[name]
        ht = self._dyn_tables[(name, cpart, s_)]
        grp, sl = [(g, x) for g in self.groups for x in g.table_slices
                   if x["table"] == name and x["cpart"] == cpart and x["s"] == s_][0]
        old = sl["rows"]
        new = min(want_rows, t.max_capacity) if t.max_capacity > 0 else want_rows
        if new <= old:
            raise RuntimeError(f"dynamic embedding table {name}: shard {s_} is full at max_capacity={old} rows")
        self._grow_slice(grp, sl, new)
        keys, rows = ht.dump()
        from .hashtable import HashTable
        nh = HashTable(new, self.device)
        if keys.numel():
            nh.set(keys, rows)
        self._dyn_tables[(name, cpart, s_)] = nh
        for c in [self] + list(getattr(self, "_clones", [])):
            c._resync_storage(self)
        return new

    def _grow_slice(self, grp, sl, new_rows: int):
        """re-layout ``grp``'s flat arrays with ``sl`` enlarged to ``new_rows`` (slices behind it shift)"""
        dev = self.device
        delta = new_rows - sl["rows"]

        def relayout(a, fill, pitch=grp.pitch):
            if a is None:
                return None
            cut = (sl["row_off"] + sl["rows"]) * pitch           # first element behind the slice
            out = torch.empty(a.numel() + delta * pitch, dtype=a.dtype, device=dev)
            out[:cut].copy_(a[:cut])
            out[cut + delta * pitch:].copy_(a[cut:])
            fill(out[cut:cut + delta * pitch])
            return out
        t = self.tmap[sl["table"]]
        bound = math.sqrt(1.0 / max(t.init_capacity, 1))
        if t.init_param is not None and t.init_param.up_bound > 0:
            bound = t.init_param.up_bound
        gen = torch.Generator(device=dev)
        gen.manual_seed(_stable_seed(self.seed, sl["table"], sl["cpart"], sl["s"], new_rows))
        table = relayout(grp.table, lambda v: _uniform_fill(v, bound, gen))
        accu = grp.opt.initial_accu_value if (grp.opt is not None and grp.opt.optimizer_type in
                                              (Optimizer_t.AdaGrad, Optimizer_t.RowWiseAdaGrad)) else 0.0
        s0 = relayout(grp.s0, lambda v: v.fill_(accu), grp.state_pitch)
        s1 = relayout(grp.s1, lambda v: v.zero_())
        grp.table, grp.s0, grp.s1 = table, s0, s1
        old_end = sl["row_off"] + sl["rows"]
        for other in grp.table_slices:
            if other is not sl and other["row_off"] >= old_end:
                other["row_off"] += delta
        sl["rows"] = new_rows
        grp.rows += delta

    def _resync_storage(self, owner):
        """after a growth: this plan's groups point at the owner's arrays and carry the new row windows"""
        for grp, src in zip(self.groups, owner.groups):
            grp.table, grp.s0, grp.s1, grp.rows = src.table, src.s0, src.s1, src.rows
            for sl, so in zip(grp.table_slices, src.table_slices):
                sl["row_off"], sl["rows"] = so["row_off"], so["rows"]
            for d, sl in zip(grp.lookups, getattr(grp, "lookup_slices", [])):
                d.table_row_off, d.rows = sl["row_off"], sl["rows"]
            grp.lookups_dev = E.lookups_to_device(grp.lookups, self.device)

    def _lookup(self, grp):
        s = grp.src
        E.forward(grp.lookups, grp.lookups_dev, grp.table, grp.pitch, s.keys, s.out, self.b, self.rank,
                  nnz_bufs=s.nnz, key_bytes=self._kb, act_bf16=self._abf, weight_bufs=s.weights)

    def forward_compute(self):
        collective = self.world > 1 and not self.fused
        if collective:
            self.send_out.zero_()
        for grp in self.groups:
            # (collective path: data-parallel lookups run in forward_end, after the exchange wrote the out slab)
            if grp.lookups and not (collective and grp.kind == "dp"):
                self._lookup(grp)

    def forward_end(self):
        if self.world > 1:
            if self.fused:
                self.comm.barrier_device()       # every owner finished writing my outputs
            elif os.environ.get("SKIP_ALL2ALL", "0") not in ("0", ""):
                pass          # ablation (communication.cpp:52-148): no vector exchange
            else:
                if self.hier:
                    self.out_slab.copy_(self.comm.hier_all_to_all_sum(self.send_out))
                else:
                    pk = self.packed
                    send = self.send_out.index_select(1, pk["out_me"]).reshape(-1)        # [world * n_me]
                    recv = pk["fwd_recv"][:sum(pk["n"])]
                    self.comm.all_to_all_v(recv, send, pk["n"], [pk["n_me"]] * self.world)
                    self.out_slab.index_copy_(0, pk["out_all"], recv)
                for grp in self.groups:
                    if grp.kind == "dp":
                        self._lookup(grp)
        if getattr(self, "_uniq", None) is not None:
            self._uniq.forward()
        self._reduce_partials()
        self._rescale_mean(forward=True)

    def _rescale_mean(self, forward: bool):
        """Mean-combined bags may be shorter than the maximum hotness (padding keys are -1): the lookup
        kernels divide by the maximum hotness, the requester -- who owns the keys -- rescales its
        pooled vectors (forward) / their gradients (backward) by hotness / (number of valid keys), i.e.
        the mean is over the actual bag like the reference's bucket ranges.  A weighted bag takes
        hotness / (sum of the valid keys' weights), with 1 for a sum of exactly 0; all-ones weights sum to
        the count exactly, so they rescale as the unweighted bag does."""
        for gi, gl in enumerate(self.glookups):
            if gl["combiner"] not in ("mean", "average") or (gl["hotness"] <= 1 and not gl["weighted"]):
                continue
            tp = self.tops[gl["top"]]
            if forward:
                keys = self.key_views[gl["bottom"]]
                if gl["weighted"]:
                    w = torch.where(keys >= 0, self.weight_views[gl["bottom"]], torch.zeros((), device=keys.device))
                    sw = w.sum(1)
                    cnt = torch.where(sw == 0, torch.ones_like(sw), sw)
                else:
                    cnt = (keys >= 0).sum(1).clamp(min=1).to(torch.float32)
                self._mean_factor = getattr(self, "_mean_factor", {})
                self._mean_factor[gi] = (float(gl["hotness"]) / cnt).unsqueeze(1)
                t2d = self.top_data[tp["name"]].reshape(self.b, -1) if not tp.get("alias") \
                    else self.top_data[tp["name"]]
            else:
                if gi not in getattr(self, "_mean_factor", {}):
                    continue
                t2d = self.top_grad[tp["name"]].reshape(self.b, -1) if not tp.get("alias") \
                    else self.top_grad[tp["name"]]
            col = t2d[:, gl["col"]:gl["col"] + gl["ev"]]
            col.copy_((col.float() * self._mean_factor[gi]).to(col.dtype))

    def _reduce_partials(self):
        b = self.b
        for gl in self.glookups:
            if gl.get("k", 1) > 1 and "partial_off" in gl:
                w = gl["partial_w"] // gl["k"]
                part = self.out_slab[gl["partial_off"]:gl["partial_off"] + b * gl["partial_w"]] \
                    .view(b, gl["k"], w)
                tp = self.tops[gl["top"]]
                if tp.get("alias"):
                    full = self.top_data[tp["name"]]
                else:
                    full = self.out_slab[tp["off"]:tp["off"] + b * tp["width"]].view(b, tp["width"])
                from ..ops import dense as D
                D.partial_sum(part, full, gl["col"], gl["k"], w)

    def backward_index(self):
        """gradient-independent part of the backward (unique rows + bucket lists); may run on a
        side stream concurrently with the dense network once the keys are in place."""
        for grp in self.groups:
            if grp.kind == "mp" and getattr(grp, "indexed", False) and grp.lookups:
                E.bwd_index(grp.lookups, grp.lookups_dev, grp.table, grp.pitch, grp.src.keys, self.b, grp.ws,
                            self.rank, nnz_bufs=grp.src.nnz, key_bytes=self._kb, weight_bufs=grp.src.weights)
        self._index_done = True

    def backward(self, lr_t, step_t, dp_stream=None):
        """Consumes top grads (grad slab), updates local tables. grads are already / global batch.

        Data-parallel groups only need the local gradients: their accumulate -> all-reduce ->
        optimizer chain runs on ``dp_stream`` (when given) next to the model-parallel chain, and in the
        same position on every rank (the all-reduce is a rendezvous)."""
        if not getattr(self, "_index_done", False):
            self.backward_index()
        self._index_done = False
        self._rescale_mean(forward=False)
        dp_groups = [g for g in self.groups if g.kind == "dp"]
        mp_groups = [g for g in self.groups if g.kind != "dp"]
        side = dp_stream is not None and self.device.type == "cuda" and bool(dp_groups)
        if side:
            cur = torch.cuda.current_stream()
            dp_stream.wait_stream(cur)
            with torch.cuda.stream(dp_stream):
                for grp in dp_groups:
                    self._accum_update(grp, lr_t, step_t)
        if self.world > 1:
            if self.fused:
                # backward all-to-all of gradients: every rank pushes the gradient columns of each
                # lookup to the owner's inbox (posted peer stores), one barrier, then the owners'
                # reduce + optimizer kernels read local memory only
                if self._grad_routes is None:
                    self._build_grad_routes()
                E.dispatch(self.grad_slab, self._grad_routes, self._grad_routes_dev, self.peer_grads_all,
                           blocks_x=24)
                self.comm.barrier_device()
            elif os.environ.get("SKIP_ALL2ALL", "0") not in ("0", ""):
                pass
            elif self.hier:
                self.comm.hier_all_gather(self.grads_all, self.grad_slab)
            else:
                pk = self.packed
                send = self.grad_slab.index_select(0, pk["grad_all"])                    # chunks per owner
                recv = pk["bwd_recv"][:self.world * pk["n_me"]]
                self.comm.all_to_all_v(recv, send, [pk["n_me"]] * self.world, pk["n"])
                if pk["n_me"]:
                    self.grads_all.index_copy_(1, pk["grad_me"], recv.view(self.world, pk["n_me"]))
        for grp in mp_groups:
            self._accum_update(grp, lr_t, step_t)
        if getattr(self, "_uniq", None) is not None:
            self._uniq.backward(lr_t, step_t)
        if side:
            torch.cuda.current_stream().wait_stream(dp_stream)
        else:
            for grp in dp_groups:
                self._accum_update(grp, lr_t, step_t)
        sched = os.environ.get("HCTR_STEP_SCHEDULE", "")
        end_default = "0" if (sched == "aggressive" or (sched != "safe" and self.world <= 4)) else "1"
        if self.world > 1 and self.fused and os.environ.get("HCTR_EMB_END_BARRIER", end_default) == "1":
            # (<= 4 ranks skip it: a rank can only overwrite an owner's inbox after that owner passed the NEXT
            # step's dispatch barrier, i.e. after its reduce of this step was queued on the same stream ahead
            # of it; kept for larger jobs, see Model._aggressive_schedule)
            self.comm.barrier_device()

    def _hp(self, o: OptParamsPy):
        return opt_hp(o, self.scaler, self.sr_seed)

    def _accum_update(self, grp, lr_t, step_t):
        o, s = grp.opt, grp.src
        if not grp.lookups:
            return            # (every lookup of this group travels through the Unique exchange)
        if grp.kind == "mp" and getattr(grp, "indexed", False):
            E.bwd_reduce_update(o.optimizer_type, grp.lookups, grp.lookups_dev, grp.table, grp.s0,
                                grp.s1, grp.pitch, s.keys, s.grads, self.b, grp.ws, self._hp(o),
                                lr_t, step_t, 1.0, self.rank, nnz_bufs=s.nnz, key_bytes=self._kb,
                                act_bf16=self._abf)
        elif grp.kind == "mp":
            E.backward_accum(grp.lookups, grp.lookups_dev, grp.table, grp.pitch, s.keys, s.grads,
                             self.b, grp.ws, 1.0, self.rank, nnz_bufs=s.nnz, key_bytes=self._kb,
                             act_bf16=self._abf, weight_bufs=s.weights)
            E.update(o.optimizer_type, grp.table, grp.s0, grp.s1, grp.pitch, grp.ws, self._hp(o),
                     lr_t, step_t)
        else:
            from ..ops import dense as D
            E.backward_accum(grp.lookups, grp.lookups_dev, grp.table, grp.pitch, s.keys, s.grads,
                             self.b, None, 1.0, self.rank, dense_wgrad=grp.dense_wgrad,
                             weight_bufs=s.weights)
            if self.world > 1:
                if grp.p2p_ar is not None:
                    grp.p2p_ar.run()
                else:
                    self.comm.all_reduce(grp.dense_wgrad)
            if grp.rowwise:
                E.dp_rowwise_update(grp.table, grp.s0, grp.dense_wgrad, grp.pitch, self._hp(o), lr_t)
                return
            D.dense_opt_step(o.optimizer_type, grp.table, grp.dense_wgrad, None, grp.s0, grp.s1, lr_t,
                             step_t, self._hp(o), zero_grad=True)

    # ------------------------------------------------------------------ checkpoint helpers
    def local_table_items(self):
        """yield (table name, column part, global keys tensor, weights [rows, ev], group, slice); the
        weights are fp32 (a view of an fp32 arena, an exact fp32 copy of a bf16 one)"""
        for grp in self.groups:
            for sl in grp.table_slices:
                w = grp.table[sl["row_off"] * grp.pitch:(sl["row_off"] + sl["rows"]) * grp.pitch] \
                    .view(sl["rows"], grp.pitch).float()
                keys = torch.arange(sl["rows"], dtype=torch.int64) * sl["k"] + sl["s"]
                yield sl["table"], sl, keys, w, grp

    def load_table_rows(self, name: str, keys: torch.Tensor, values: torch.Tensor, state=None):
        """Scatter (key, row-vector) pairs of table ``name`` into the local shards (re-sharding on
        load: only keys with key % num_shards == shard_id are kept, parameter_IO.cpp:262-350).
        ``state``: optional list of per-state [n, ev] tensors (optimizer states).  A bf16 arena stores
        the values rounded to nearest."""
        keys = keys.to(torch.int64).cpu()
        for grp in self.groups:
            for sl in grp.table_slices:
                if sl["table"] != name:
                    continue
                if sl.get("evict"):
                    m = (keys % sl["k"] == sl["s"]) & (keys >= 0)
                    if not bool(m.any()):
                        continue
                    rows = sl["row_off"] + self._evict_admit(grp, sl, keys[m])
                elif sl.get("dynamic"):
                    m = (keys % sl["k"] == sl["s"]) & (keys >= 0)
                    if not bool(m.any()):
                        continue
                    ht = self._dyn_hash(name, dict(sl, cpart=0))
                    kk = keys[m].to(self.device)
                    fresh = int((ht.get(kk) < 0).sum()) if ht.size() else int(kk.numel())
                    if ht.size() + fresh > ht.max_rows:
                        # a checkpoint with more keys than the shard currently holds: grow first (a failed insert
                        # would hand back row -1)
                        owner = getattr(self, "_shared", self)
                        owner._grow_to(name, 0, sl["s"], max(2 * ht.max_rows, ht.size() + fresh))
                        ht = self._dyn_hash(name, dict(sl, cpart=0))
                    rows = sl["row_off"] + ht.get_insert(kk).to(grp.table.device).long()
                else:
                    m = (keys % sl["k"] == sl["s"]) & (keys // sl["k"] < sl["rows"]) & (keys >= 0)
                    if not bool(m.any()):
                        continue
                    rows = (sl["row_off"] + keys[m] // sl["k"]).to(grp.table.device)
                c0, ev = sl["col0"], sl["ev"]
                grp.table.view(-1, grp.pitch)[rows] = values[m][:, c0:c0 + ev].to(grp.table.device,
                                                                                 torch.float32).to(grp.table.dtype)
                if state is not None:
                    for st, dst in zip(state, (grp.s0, grp.s1)):
                        if dst is not None and st is not None:
                            v = st[m][:, c0:c0 + ev]
                            if grp.rowwise:
                                # a row's accumulator: the mean of the state over the slice's columns
                                # (exact for a row-wise file, the natural conversion of an AdaGrad one)
                                v = v.double().mean(1, keepdim=True).float()
                            dst.view(-1, grp.state_pitch)[rows] = v.to(dst.device, dst.dtype)

    def _evict_admit(self, grp, sl, keys):
        """(checkpoint load) local rows of ``keys`` in an evicting shard: present keys keep theirs, the
        others take empty ways with the clock as stamp and a count of 1, and start from fresh weights and
        state (overwritten by the caller).  Never evicts: raises when a key finds no free way."""
        ht = self._dyn_hash(sl["table"], sl)
        dev = self.device
        kk = keys.to(dev, torch.int64).view(1, -1).clone()
        n = kk.shape[1]
        adm = (torch.zeros(n, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
        ht.insert(kk, 0, n, adm=adm, evict=False, stats=torch.zeros(3, dtype=torch.int64, device=dev))
        slots = kk.view(-1)
        dropped = int((slots < 0).sum())
        if dropped:
            raise RuntimeError(f"evicting embedding table {sl['table']}: shard {sl['s']} cannot hold the loaded keys: "
                               f"{dropped} of {n} found no free way (capacity {ht.capacity}, "
                               f"{int(ht.live())} live keys)")
        self._evict_reinit(grp, sl, ht, adm)
        return slots.to(grp.table.device)

    def table_parts(self, name: str):
        """Metadata of the local shards of table ``name`` in ``dump_table_local`` order (no data is
        moved): rows, row shard (s of k), column window, group kind, dynamic flag, state count."""
        res = []
        for grp in self.groups:
            for sl in grp.table_slices:
                if sl["table"] != name:
                    continue
                rows = sl["rows"]
                if sl.get("dynamic"):
                    rows = int(self._dyn_hash(name, dict(sl, cpart=0)).dump()[0].numel())
                res.append(dict(rows=int(rows), s=int(sl["s"]), k=int(sl["k"]), col0=int(sl["col0"]),
                                width=int(sl["ev"]), kind=grp.kind, dynamic=bool(sl.get("dynamic")),
                                nstate=sum(t is not None for t in (grp.s0, grp.s1))))
        return res

    def dump_table_local(self, name: str, only=None):
        """-> list of (keys int64 [n], values fp32 [n, ev_part], col0, states list) local shards (a bf16
        arena's values widen to fp32 exactly).
        ``only``: optional set of part indices to materialise (others are returned as None)."""
        res = []
        for grp in self.groups:
            for sl in grp.table_slices:
                if sl["table"] != name:
                    continue
                if only is not None and len(res) not in only:
                    res.append(None)
                    continue
                lo, hi = sl["row_off"], sl["row_off"] + sl["rows"]
                w = grp.table.view(-1, grp.pitch)[lo:hi].detach().float().cpu()
                keys = torch.arange(sl["rows"], dtype=torch.int64) * sl["k"] + sl["s"]
                sts = [None if t is None else t.view(-1, grp.state_pitch)[lo:hi].detach().float().cpu()
                       .expand(hi - lo, grp.pitch).contiguous() for t in (grp.s0, grp.s1)]
                if sl.get("dynamic"):
                    dk, dr = self._dyn_hash(name, dict(sl, cpart=0)).dump()
                    order = torch.argsort(dk)
                    keys, dr = dk[order].to(torch.int64), dr[order].to(torch.int64)
                    w = w[dr]
                    sts = [None if t is None else t[dr] for t in sts]
                res.append((keys, w, sl["col0"], sts, grp.kind))
        return res

    def memory_bytes(self) -> int:
        tot = 0
        for grp in self.groups:
            for t in (grp.table, grp.s0, grp.s1):
                if t is not None:
                    tot += t.numel() * t.element_size()
        return tot
