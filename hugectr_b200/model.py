"""hugectr.Model: graph construction by tensor names, compile, fit/train/eval, checkpoints.

Reference: HugeCTR/src/pybind/model.cpp (1508 lines), model_compile.cpp, model_pipeline.cpp,
HugeCTR/include/pybind/model_wrapper.hpp:133-221.  Execution model here: one process per GPU; a
training iteration = [H2D of the batch] + ONE statically scheduled step (embedding forward ->
dense fprop -> dense bprop -> dense wgrad all-reduce -> fused dense optimizer -> fused embedding
backward/update) that is captured into a CUDA graph on the first iterations (solver.use_cuda_graph).
"""
from __future__ import annotations

import json
import math
import os
import time
from typing import Dict, List, Optional

import torch

from . import metrics as M
from .data.batch import HostBatch
from .data.readers import SparseLayout
from .embedding.collection import EmbeddingCollection, EmbeddingCollectionConfig
from .enums import MetricsRawType, MetricsType, Tensor_t
from .layers import BuildCtx, ParamArena, TensorBag
from .lr_scheduler import LearningRateScheduler
from .network import Network, insert_fanout_slices
from .ops import dense as D
from .ops.optim import opt_hp, opt_states
from .parallel.comm import Comm
from .solver import (DataReaderParams, DenseLayer, Input, OptParamsPy, Solver, SparseEmbedding,
                     check_not_rowwise)
from .utils import logger


def _ones(shape, gen):
    """initial position weights: 1.0, the unweighted pooling (draws nothing from the arena's generator)"""
    return torch.ones(shape)


class TrainingCallback:
    """Overridable hooks (training_callback_wrapper.hpp:62-86)."""

    def on_training_start(self): pass
    def on_training_end(self, current_iter: int): pass
    def on_eval_start(self, current_iter: int): return False
    def on_eval_end(self, current_iter: int, eval_results: dict): return False


class Model:
    def __init__(self, solver: Solver, reader_params: DataReaderParams,
                 opt_params: Optional[OptParamsPy] = None, etc=None, comm: Optional[Comm] = None):
        self.solver = solver
        self.etc = etc                 # hugectr.CreateETC(...): host parameter server + gpu_cache per embedding
        self.reader_params = reader_params
        check_not_rowwise(opt_params, "the model optimizer (dense layers have no embedding rows)")
        self.opt_params = opt_params or OptParamsPy()
        self.comm = comm or Comm.init_from_env()
        self.device = self.comm.device
        if solver.batchsize % max(1, solver.num_gpus) != 0:
            raise ValueError("batchsize must be divisible by the total number of GPUs")  # model.cpp:357
        if self.comm.world_size not in (1, solver.num_gpus):
            logger.warning(f"vvgpu lists {solver.num_gpus} GPUs but the job runs {self.comm.world_size} ranks")
        self.world = self.comm.world_size
        if self.world > 1 and len(solver.vvgpu) > 1 and hasattr(self.comm, "set_topology"):
            self.comm.set_topology(len(solver.vvgpu[0]))       # several nodes: vvgpu = one list per node
        self.input: Optional[Input] = None
        self.sparse_embeddings: List[SparseEmbedding] = []
        self.ebc_configs: List[EmbeddingCollectionConfig] = []
        self.dense_layers: List[DenseLayer] = []
        self.graph_order: List[object] = []
        self.compiled = False
        self.lr_sched = LearningRateScheduler(solver.lr, solver.warmup_steps, solver.decay_start,
                                              solver.decay_steps, solver.decay_power, solver.end_lr)
        self.callbacks = list(solver.training_callbacks)
        self.embedding_frozen: Dict[str, bool] = {}
        self.dense_frozen = False
        self._graph = None
        self._graph_warm = 0
        self._iter = 0
        self.mixed = bool(solver.use_mixed_precision)
        self.act_dtype = torch.bfloat16 if self.mixed else torch.float32
        if solver.enable_tf32_compute and not self.mixed:
            # fp32 models: GEMMs of the fp32 path (library matmul) may use TF32 tensor cores, as the
            # reference's enable_tf32_compute does for cuBLAS (fully_connected_layer.cu compute types)
            torch.backends.cuda.matmul.allow_tf32 = True
            torch.backends.cudnn.allow_tf32 = True
        self.key_dtype = torch.int64 if solver.i64_input_key else torch.int32
        self.launches_per_step = 0
        # set before compile() by an inference session: the embedding collections are built for serving (no
        # optimizer state, workspace or gradient buffers), with fp8 tables when fp8_quant is set
        self.serving = False
        self.fp8_quant = False

    # ------------------------------------------------------------------ graph construction
    def add(self, obj):
        if self.compiled:
            raise RuntimeError("model.add() after compile()")
        if isinstance(obj, Input):
            self.input = obj
        elif isinstance(obj, SparseEmbedding):
            self.sparse_embeddings.append(obj)
        elif isinstance(obj, EmbeddingCollectionConfig):
            self.ebc_configs.append(obj)
        elif isinstance(obj, DenseLayer):
            self.dense_layers.append(obj)
        else:
            raise TypeError(f"cannot add {type(obj)} to a Model")
        self.graph_order.append(obj)

    # ------------------------------------------------------------------ compile
    def compile(self, loss_names: Optional[List[str]] = None,
                loss_weights: Optional[List[float]] = None):
        assert self.input is not None, "model.add(Input) first"
        s = self.solver
        if not s.use_algorithm_search:
            # reference: cublasLt algorithm search off -> default heuristic; here: no tile autotuning
            os.environ["HCTR_GEMM_AUTOTUNE"] = "0"
        self.b_train = s.batchsize // self.world
        self.b_eval = s.batchsize_eval // self.world
        inp = self.input
        self.layout = SparseLayout(inp.data_reader_sparse_param_array,
                                   self.reader_params.slot_size_array)
        self.arena = ParamArena()
        self._build_embeddings()
        self.net_train = self._build_network(True)
        self.arena.begin_replay()
        self.net_eval = self._build_network(False)
        self.arena.end_replay()
        # the weights of the position-weighted inputs: dense parameters behind the network's own, so that a model
        # without such inputs keeps its arena, dense files and optimizer state as they were
        self.position_weights = {p.top_name: self.arena.add(f"{p.top_name}.position_weight",
                                                            (p.slot_num, max(p.nnz_per_slot)), _ones)
                                 for p in inp.data_reader_sparse_param_array if getattr(p, "position_weighted", False)}
        from .enums import AllReduceAlgo
        p2p_ar = (self.world > 1 and self.device.type == "cuda"
                  and s.all_reduce_algo in (AllReduceAlgo.OneShot, AllReduceAlgo.TwoShot)
                  and self.comm.p2p_available)
        self.arena.finalize(self.device, self.mixed, pad_to=max(64, 4 * self.world),
                            wgrad_alloc=self.comm.symm_alloc if p2p_ar else None)
        self.net_train.finalize()
        self.net_eval.finalize()
        if self.position_weights:
            pw = {n: (p.w, p.g) for n, p in self.position_weights.items()}
            for e in self.ebcs_train + self.ebcs_eval:
                e.bind_position_weights({n: pw[n] for n in e.pw_inputs})
        self.arena.init_params(s.seed)
        self._setup_losses(loss_names, loss_weights)
        self._create_dense_optimizer()
        self._create_metrics()
        self._create_readers()
        from .parallel.allreduce import ExchangeWgrad
        self.exchange_wgrad = ExchangeWgrad(self.comm, self.arena.wgrad, s.all_reduce_algo)
        self.compiled = True
        if s.perf_logging:
            logger.perf_log("init_stop")

    def _src_tensors(self, b: int, is_train: bool):
        inp = self.input
        dev = self.device
        t = {}
        lab = TensorBag(inp.label_name, (b, inp.label_dim), torch.float32)
        lab.data = torch.zeros(b, inp.label_dim, device=dev)
        lab.needs_grad = False
        t[inp.label_name] = lab
        if len(inp.label_names) > 1:      # multi-label: per-label views (model_compile.cpp:88-95)
            off = 0
            for n, d in zip(inp.label_names, inp.label_dims):
                lb = TensorBag(n, (b, d), torch.float32)
                lb.data = lab.data[:, off:off + d]
                lb.needs_grad = False
                t[n] = lb
                off += d
        den = TensorBag(inp.dense_name, (b, inp.dense_dim), torch.float32)
        den.data = torch.zeros(b, max(inp.dense_dim, 0), device=dev)
        den.needs_grad = False
        t[inp.dense_name] = den
        return t

    def _apply_device_layout(self, cfg):
        """``DeviceLayout.NodeFirst`` (device_map.hpp:76-115): row ``local * num_nodes + node`` of a
        shard matrix describes GPU ``local`` of node ``node``.  Ranks here are node-major
        (``node * gpus_per_node + local``), so the rows are permuted once into rank order."""
        s = self.solver
        if getattr(s.device_layout, "name", s.device_layout) != "NodeFirst" or len(s.vvgpu) < 2 \
                or cfg.shard_matrix is None or getattr(cfg, "_layout_applied", False):
            return cfg
        from .parallel.comm import DeviceMap
        dm = DeviceMap(s.vvgpu, "NodeFirst")
        gpn = len(s.vvgpu[0])
        rows = [cfg.shard_matrix[dm.get_global_id(r % gpn, r // gpn)] for r in range(len(cfg.shard_matrix))]
        import copy
        out = copy.copy(cfg)
        out.shard_matrix, out._layout_applied = rows, True
        return out

    def _check_weighted_inputs(self):
        """Weighted sparse inputs need a reader that delivers weights and embeddings that pool them."""
        from .enums import DataReaderType_t
        weighted = [p.top_name for p in self.input.data_reader_sparse_param_array if getattr(p, "weighted", False)]
        if not weighted:
            return
        t = self.reader_params.data_reader_type
        if t in (DataReaderType_t.Norm, DataReaderType_t.Raw, DataReaderType_t.RawAsync):
            raise ValueError(f"weighted input {weighted[0]}: the {t.name} data format has no weights")
        for se in self.sparse_embeddings:
            if se.bottom_name in weighted:
                raise ValueError(f"weighted input {se.bottom_name}: the legacy SparseEmbedding "
                                 f"{getattr(se, 'sparse_embedding_name', '')} cannot pool weights "
                                 "(use an EmbeddingCollection lookup)")

    def _check_position_weighted_inputs(self):
        """Position-weighted inputs are pooled by embedding-collection lookups only."""
        pw = {p.top_name for p in self.input.data_reader_sparse_param_array if getattr(p, "position_weighted", False)}
        for se in self.sparse_embeddings:
            if se.bottom_name in pw:
                raise ValueError(f"position-weighted input {se.bottom_name}: the legacy SparseEmbedding "
                                 f"{getattr(se, 'sparse_embedding_name', '')} cannot pool weights "
                                 "(use an EmbeddingCollection lookup)")

    def _build_embeddings(self):
        s = self.solver
        self._check_weighted_inputs()
        self._check_position_weighted_inputs()
        hot = {p.top_name: max(p.nnz_per_slot) for p in self.input.data_reader_sparse_param_array}
        weighted = {p.top_name for p in self.input.data_reader_sparse_param_array if getattr(p, "weighted", False)}
        pw = {p.top_name for p in self.input.data_reader_sparse_param_array if getattr(p, "position_weighted", False)}
        self.ebcs_train, self.ebcs_eval = [], []
        state_dtype = torch.float32
        if os.environ.get("HCTR_EMB_STATE_BF16", "0") == "1":
            state_dtype = torch.bfloat16
        for cfg in self.ebc_configs:
            for lk in cfg.lookups:
                for bname in lk["bottoms"]:
                    prm = [p for p in self.input.data_reader_sparse_param_array if p.top_name == bname]
                    if not prm:
                        raise KeyError(f"embedding_lookup bottom '{bname}' is not a sparse input")
                    if prm[0].slot_num != 1:
                        raise ValueError("EmbeddingCollection requires slot_num == 1 per sparse param")
            cfg = self._apply_device_layout(cfg)
            # a serving model has one collection at the eval batch: it serves the eval graph and is the one
            # embedding_load / embedding_dump reach through ebcs_train
            kw = dict(is_train=False, fp8_quant=self.fp8_quant) if self.serving else {}
            e = EmbeddingCollection(cfg, self.b_eval if self.serving else self.b_train, hot, self.device,
                                    self.act_dtype, self.comm, self.opt_params, self.key_dtype,
                                    scaler=s.scaler if self.mixed else 1.0, state_dtype=state_dtype,
                                    seed=s.seed,
                                    fused=None if s.fused_embedding_comm else False, weighted=weighted,
                                    position_weighted=pw, **kw)
            self.ebcs_train.append(e)
            self.ebcs_eval.append(e if self.serving else e.eval_clone(self.b_eval))
        self.legacy_train, self.legacy_eval = [], []
        if self.sparse_embeddings:
            from .embedding.sparse_embedding import SparseEmbeddingRuntime
            for se in self.sparse_embeddings:
                prm = [p for p in self.input.data_reader_sparse_param_array
                       if p.top_name == se.bottom_name][0]
                idx = len(self.legacy_train)
                kw = dict(scaler=s.scaler if self.mixed else 1.0, seed=s.seed)
                cls = SparseEmbeddingRuntime
                if self.etc is not None and idx < len(self.etc.ps_types):
                    from .embedding.offloaded import CachedSparseEmbeddingRuntime as cls   # noqa: N813
                    kw.update(ps_type=self.etc.ps_types[idx], host_capacity=self.etc.host_capacity_rows,
                              local_path=(self.etc.local_paths[idx] if idx < len(self.etc.local_paths) else None))
                rt = cls(se, prm, self.layout, self.b_train, self.device, self.act_dtype, self.comm,
                         se.optimizer or self.opt_params, self.key_dtype, **kw)
                if cls is not SparseEmbeddingRuntime and idx < len(self.etc.sparse_models) \
                        and self.etc.sparse_models[idx] and os.path.isdir(self.etc.sparse_models[idx]):
                    rt.load_parameters(self.etc.sparse_models[idx])
                self.legacy_train.append(rt)
                self.legacy_eval.append(rt.eval_clone(self.b_eval))

    def _build_network(self, is_train: bool) -> Network:
        b = self.b_train if is_train else self.b_eval
        ctx = BuildCtx(self.arena, self.device, self.act_dtype, b, is_train, self.solver, self.mixed)
        src = self._src_tensors(b, is_train)
        emb_tops = []
        for e in (self.ebcs_train if is_train else self.ebcs_eval):
            for name, shp in e.top_shapes().items():
                tb = TensorBag(name, shp, self.act_dtype)
                if is_train and not e.is_train:
                    # the training graph of a serving model is never run: stand-in tops
                    tb.data = torch.zeros(shp, dtype=self.act_dtype, device=self.device)
                    tb.grad = torch.zeros_like(tb.data)
                else:
                    tb.data = e.top_data[name]
                    tb.grad = e.top_grad[name] if is_train else None
                    tb.ebc, tb.ebc_top = e, name          # lets a Concat alias the top into its output
                src[name] = tb
                emb_tops.append(name)
        for rt in (self.legacy_train if is_train else self.legacy_eval):
            tb = TensorBag(rt.top_name, rt.top_shape, self.act_dtype)
            tb.data = rt.top_data
            tb.grad = rt.top_grad if is_train else None
            src[rt.top_name] = tb
            emb_tops.append(rt.top_name)
        net = Network(ctx, src, emb_tops)
        cfgs = insert_fanout_slices(self.dense_layers, list(src.keys()))
        for c in cfgs:
            net.add_layer(c)
        if is_train:
            self._resolved_layers = cfgs
        return net

    def _setup_losses(self, loss_names, loss_weights):
        for net in (self.net_train, self.net_eval):
            if not net.loss_layers:
                raise RuntimeError("the model has no loss layer")
            if loss_names:
                wmap = dict(zip(loss_names, loss_weights))
                for ll in net.loss_layers:
                    ll.loss_weight = float(wmap.get(ll.cfg.top_names[0], 1.0))
            elif len(self.input.label_names) > 1:
                lw = dict(zip(self.input.label_names, self.input.label_weights))
                for ll in net.loss_layers:
                    ll.loss_weight = float(lw.get(ll.cfg.bottom_names[1], 1.0))

    def _create_dense_optimizer(self):
        o = self.opt_params
        dev = self.device
        self.opt_s0, self.opt_s1 = opt_states(o, self.arena.weights.numel(), device=dev)
        self.lr_t = torch.full((1,), float(self.solver.lr), device=dev)
        self.step_t = torch.zeros(1, dtype=torch.int32, device=dev)
        self.dense_hp = opt_hp(o, self.solver.scaler if self.mixed else 1.0)

    def _create_metrics(self):
        ncls = self.input.label_dim
        self.metrics = [(k, thr, M.create_metric(k, self.comm, ncls))
                        for k, thr in self.solver.metrics_spec.items()]

    def _create_readers(self):
        from .data import create_reader
        self.reader_train = create_reader(self, True)
        self.reader_eval = create_reader(self, False)
        n_cache = int(getattr(self.reader_params, "cache_eval_data", 0) or 0)
        if n_cache > 0 and n_cache >= self.solver.max_eval_batches:
            from .data.readers import CachedEvalReader
            self.reader_eval = CachedEvalReader(self.reader_eval, n_cache, self.device)
        self.reader_train._bind(self, True)
        self.reader_eval._bind(self, False)

    # ------------------------------------------------------------------ summary / json
    def summary(self):
        if self.comm.rank != 0:
            return
        line = "=" * 95
        print(line)
        print("%-28s%-32s%-35s" % ("Label", "Dense", "Sparse"))
        inp = self.input
        print("%-28s%-32s%-35s" % (inp.label_name, inp.dense_name,
                                  ",".join(p.top_name for p in inp.data_reader_sparse_param_array)[:34]))
        print("%-28s%-32s" % (f"(None, {inp.label_dim})", f"(None, {inp.dense_dim})"))
        print("-" * 95)
        print("%-36s%-30s%-30s%-20s" % ("Layer Type", "Input Name", "Output Name", "Output Shape"))
        print("-" * 95)
        for se in self.sparse_embeddings:
            print("%-36s%-30s%-30s" % (se.embedding_type.name, se.bottom_name, se.sparse_embedding_name))
        for e in getattr(self, "ebcs_train", []):
            for tp in e.tops:
                shp = f"(None, {tp['width']})" if tp["batch_major"] else f"(None, 1, {tp['width']})"
                print("%-36s%-30s%-30s%-20s" % ("EmbeddingCollection", "", tp["name"], shp))
        if self.compiled:
            for (t, i, o, shp) in self.net_train.summary_rows():
                print("%-36s%-30s%-30s%-20s" % (t, i[:29], o[:29], shp))
        else:
            for c in self.dense_layers:
                print("%-36s%-30s%-30s" % (c.layer_type.name, ",".join(c.bottom_names)[:29],
                                           ",".join(c.top_names)[:29]))
        print(line)

    def graph_to_json(self, graph_config_file: str):
        from .graph_json import model_to_json
        if self.comm.rank == 0:
            os.makedirs(os.path.dirname(graph_config_file) or ".", exist_ok=True)
            with open(graph_config_file, "w") as f:
                json.dump(model_to_json(self), f, indent=2)

    def construct_from_json(self, graph_config_file: str, include_dense_network: bool = True):
        from .graph_json import add_from_json
        with open(graph_config_file) as f:
            add_from_json(self, json.load(f), include_dense_network)

    # ------------------------------------------------------------------ data
    def _load_batch(self, hb: HostBatch, is_train: bool):
        net = self.net_train if is_train else self.net_eval
        inp = self.input
        nb = True
        if getattr(hb, "raw", None) is not None:
            # device-split reader: ONE H2D of the raw records, the split kernel writes label / dense and
            # the feature-major keys straight into the input tensors / the key slab
            ebcs = self.ebcs_train if is_train else self.ebcs_eval
            legs = self.legacy_train if is_train else self.legacy_eval
            if len(ebcs) == 1 and not legs and ebcs[0].key_slab.dtype == hb.splitter.key_dtype:
                hb.splitter.run(hb.raw, hb.raw_skew, hb.num_valid, net.tensors[inp.label_name].data,
                                net.tensors[inp.dense_name].data if inp.dense_dim > 0 else None, ebcs[0].key_slab)
                hb.mark_copied()
                return
            hb = self._materialize_raw(hb)
        net.tensors[inp.label_name].data.copy_(hb.label, non_blocking=nb)
        if inp.dense_dim > 0:
            net.tensors[inp.dense_name].data.copy_(hb.dense, non_blocking=nb)
        ebcs = self.ebcs_train if is_train else self.ebcs_eval
        legs = self.legacy_train if is_train else self.legacy_eval
        if len(ebcs) == 1 and not legs:
            ebcs[0].set_keys(hb.keys)
            if ebcs[0].has_data_weights:
                ebcs[0].set_weights(hb.weights)
        else:
            b = self.b_train if is_train else self.b_eval
            offs, _ = self.layout.key_block_offsets(b)
            for e in ebcs:
                for gl in e.glookups:
                    o = offs[gl["bottom"]]
                    e.key_views[gl["bottom"]].copy_(
                        hb.keys[o:o + b * gl["hotness"]].view(b, gl["hotness"]), non_blocking=nb)
                    if gl["weighted"] and not gl["pw"]:
                        e.weight_views[gl["bottom"]].copy_(
                            hb.weights[o:o + b * gl["hotness"]].view(b, gl["hotness"]), non_blocking=nb)
            for rt in legs:
                rt.set_keys(hb, offs, self.layout.nnz_block_offsets(b)[0])
        hb.mark_copied()

    def _materialize_raw(self, hb: HostBatch) -> HostBatch:
        """raw batch -> device label / dense / keys tensors (models with several collections or legacy
        embeddings copy from these)"""
        sp = hb.splitter
        dev = self.device
        if not hasattr(self, "_raw_tmp"):
            self._raw_tmp = (torch.empty(sp.batch, sp.label_dim, device=dev),
                             torch.empty(sp.batch, max(sp.dense_dim, 1), device=dev)[:, :sp.dense_dim].contiguous(),
                             torch.empty(max(sp.total_keys, 1), dtype=sp.key_dtype, device=dev))
        lab, den, keys = self._raw_tmp
        sp.run(hb.raw, hb.raw_skew, hb.num_valid, lab, den, keys)
        hb.mark_copied()
        return HostBatch(lab, den, keys, None, hb.num_valid)

    def start_data_reading(self):
        self.reader_train.start()
        self.reader_eval.start()

    def set_source(self, source=None, eval_source=None):
        if source is not None:
            self.reader_train.set_source(source)
        if eval_source is not None:
            self.reader_eval.set_source(eval_source)

    def get_data_reader_train(self):
        return self.reader_train

    def get_data_reader_eval(self):
        return self.reader_eval

    def get_learning_rate_scheduler(self):
        return self.lr_sched

    # ------------------------------------------------------------------ one training step
    def _step_body(self):
        s = self.solver
        D.lr_step(self.step_t, self.lr_t, s.lr, s.end_lr, s.decay_power, s.warmup_steps,
                  s.decay_start, s.decay_steps)
        net = self.net_train
        # ablation switches of the reference pipeline (model_pipeline.cpp:118-286, benchmarks/
        # embedding_collection/README.md): attribute step time by leaving a stage out
        skip = getattr(self, "_skip", None)
        if skip is None:
            env = lambda k: os.environ.get(k, "0") not in ("0", "")
            skip = self._skip = {"emb": env("SKIP_EMBEDDING"), "bottom": env("SKIP_BOTTOM_MLP"),
                                 "top": env("SKIP_TOP_MLP"), "ar": env("SKIP_ALLREDUCE")}
            if any(skip.values()):
                logger.warning(f"ablation switches active, the model does not train correctly: {skip}")
        if any(skip.values()):
            return self._step_body_ablation(skip)
        bucketed = (self.device.type == "cuda" and not self.dense_frozen
                    and os.environ.get("HCTR_DISABLE_AR_OVERLAP", "0") == "0")
        if bucketed:
            self.exchange_wgrad.begin_step(after_bucket=self._dense_opt_range)
            net.wgrad_hook = self.exchange_wgrad.layer_done
        else:
            net.wgrad_hook = None
        overlap = (self.device.type == "cuda" and not self.legacy_train and self.ebcs_train
                   and os.environ.get("HCTR_DISABLE_OVERLAP", "0") == "0"
                   and (s.train_intra_iteration_overlap or True))
        frozen_emb = self.embedding_frozen.get("*", False)
        if overlap:
            # intra-iteration overlap (reference model_pipeline.cpp:299-345): embedding forward and
            # the backward index build run on side streams next to the bottom MLP; the embedding
            # reduce+update runs next to bottom-MLP bprop / all-reduce / dense optimizer.
            main = torch.cuda.current_stream()
            if not hasattr(self, "_s_emb"):
                # the embedding forward gates the top MLP: high priority.  The backward index build
                # is only needed at the end of the step: same (lowest) priority as everything else,
                # so forward CTAs are scheduled ahead of its still-pending blocks.
                self._s_emb = torch.cuda.Stream(priority=int(os.environ.get("HCTR_PRIO_EMB", "-1")))
                self._s_idx = torch.cuda.Stream(priority=int(os.environ.get("HCTR_PRIO_IDX", "0")))
                # The bottom-MLP backward (a chain of small kernels) and the last all-reduce bucket end the
                # step: above the embedding update's priority, so their blocks take the first SM slots that
                # free up instead of queueing behind a GPU-filling update kernel (measured: the chain took
                # ~180 us beside the update at priority 0, ~80 us of work)
                self._s_bot = torch.cuda.Stream(priority=int(os.environ.get("HCTR_PRIO_BOTTOM", "-3")))
            s_emb, s_idx = self._s_emb, self._s_idx
            for e in self.ebcs_train:
                e.forward_begin()
            s_emb.wait_stream(main)
            s_idx.wait_stream(main)
            # HCTR_BOTTOM_FIRST=1 enqueues the (tiny) bottom MLP before the embedding kernels (the block
            # scheduler may still run the embedding forward first)
            bottom_first = os.environ.get("HCTR_BOTTOM_FIRST", "0") == "1"
            if bottom_first:
                net.fprop(True, "bottom")
            with torch.cuda.stream(s_emb):
                for e in self.ebcs_train:
                    e.forward_compute()
            if not frozen_emb:
                with torch.cuda.stream(s_idx):
                    for e in self.ebcs_train:
                        e.backward_index()
            if not bottom_first:
                net.fprop(True, "bottom")
            main.wait_stream(s_emb)
            for e in self.ebcs_train:
                e.forward_end()
            net.fprop(True, "top")
            net.bprop("top")
            main.wait_stream(s_idx)
            if not frozen_emb:
                s_emb.wait_stream(main)
                with torch.cuda.stream(s_emb):
                    for e in self.ebcs_train:
                        e.backward(self.lr_t, self.step_t, dp_stream=s_idx)
            if self._aggressive_schedule():
                self._s_bot.wait_stream(main)
                with torch.cuda.stream(self._s_bot):
                    net.bprop("bottom")
                main.wait_stream(self._s_bot)
            else:
                net.bprop("bottom")
        else:
            for e in self.ebcs_train:
                e.forward(True)
            for rt in self.legacy_train:
                rt.forward(True)
            net.fprop(True)
            net.bprop()
            if self.position_weights and not frozen_emb:
                # the embedding backward produces the gradient of the position weights: ahead of the dense step
                for e in self.ebcs_train:
                    e.backward(self.lr_t, self.step_t)
        for e in self.ebcs_train:
            e.wait_position_weight_grad()
        if not self.dense_frozen:
            if bucketed:
                self.exchange_wgrad.finish_step()      # all-reduce + optimizer, bucket by bucket
            else:
                self.exchange_wgrad.allreduce()
                self._dense_opt_range(0, self.arena.weights.numel())
        else:
            self.arena.wgrad.zero_()
        if overlap:
            torch.cuda.current_stream().wait_stream(self._s_emb)
        else:
            for e in self.ebcs_train:
                if not frozen_emb and not self.position_weights:
                    e.backward(self.lr_t, self.step_t)
            for rt in self.legacy_train:
                if not self.embedding_frozen.get(rt.name, frozen_emb):
                    rt.backward(self.lr_t, self.step_t)

    def _step_body_ablation(self, skip):
        """Sequential step with stages left out (SKIP_EMBEDDING / SKIP_BOTTOM_MLP / SKIP_TOP_MLP /
        SKIP_ALLREDUCE).  Timing attribution only: skipped stages leave stale activations behind."""
        net = self.net_train
        net.wgrad_hook = None
        frozen_emb = self.embedding_frozen.get("*", False)
        if not skip["emb"]:
            for e in self.ebcs_train:
                e.forward(True)
            for rt in self.legacy_train:
                rt.forward(True)
        if not skip["bottom"]:
            net.fprop(True, "bottom")
        if not skip["top"]:
            net.fprop(True, "top")
            net.bprop("top")
        if not skip["bottom"]:
            net.bprop("bottom")
        if not self.dense_frozen:
            if not skip["ar"]:
                self.exchange_wgrad.allreduce()
            self._dense_opt_range(0, self.arena.weights.numel())
        else:
            self.arena.wgrad.zero_()
        if not skip["emb"] and not frozen_emb:
            for e in self.ebcs_train:
                e.backward(self.lr_t, self.step_t)
            for rt in self.legacy_train:
                if not self.embedding_frozen.get(rt.name, frozen_emb):
                    rt.backward(self.lr_t, self.step_t)

    def _dense_opt_range(self, lo: int, hi: int):
        """fused dense optimizer over arena elements [lo, hi) (also zeroes that wgrad range)"""
        a = self.arena
        sl = lambda t: None if t is None else t[lo:hi]
        D.dense_opt_step(self.opt_params.optimizer_type, a.weights[lo:hi],
                         a.wgrad[lo:hi], sl(a.weights16), sl(self.opt_s0), sl(self.opt_s1),
                         self.lr_t, self.step_t, self.dense_hp, zero_grad=True)

    def _run_step(self):
        use_graph = (self.solver.use_cuda_graph and self.device.type == "cuda"
                     and os.environ.get("HCTR_DISABLE_CUDA_GRAPH", "0") == "0"
                     and not getattr(self.comm, "emulated", False)     # (rank threads share one device)
                     and self._graph_safe())
        if not use_graph:
            c0 = D.launch_count
            self._step_body()
            self.launches_per_step = D.launch_count - c0
            return
        if self._graph is None:
            if self._graph_warm < 2:           # eager warm-up iterations (lazy inits, autotune)
                c0 = D.launch_count
                self._step_body()
                self.launches_per_step = D.launch_count - c0
                self._graph_warm += 1
                return
            torch.cuda.synchronize()
            self.comm.barrier()
            g = torch.cuda.CUDAGraph()
            prio = int(os.environ.get("HCTR_PRIO_MAIN", "0"))
            cap_stream = torch.cuda.Stream(priority=prio) if prio != 0 else None
            with torch.cuda.graph(g, stream=cap_stream):
                self._step_body()
            self._graph = g
            self.comm.barrier()                # pipeline.cpp:111-125 barrier after first capture
            # capture does not execute: run the captured step now
        self._graph.replay()

    def _aggressive_schedule(self) -> bool:
        """Step-tail scheduling.  "aggressive": bottom-network backward and the
        all-reduce buckets on streams above the embedding update's priority, no end-of-step device barrier
        (the next step's dispatch barrier orders the inbox reuse).  More than 4 ranks run the round-1 schedule
        (bottom backward on the main stream, default-priority communication streams, end-of-step barrier):
        an 8-GPU run of the aggressive schedule stopped making progress after the warm-up in the only 8-GPU
        slot this round had, and could not be re-run.  HCTR_STEP_SCHEDULE=aggressive|safe overrides."""
        mode = os.environ.get("HCTR_STEP_SCHEDULE", "")
        if mode in ("aggressive", "safe"):
            return mode == "aggressive"
        return self.world <= 4

    def _graph_safe(self) -> bool:
        """The step can be captured when nothing in it needs the host: legacy embeddings whose hash
        insert is checked on the host and collections with dynamic tables on the translate-on-host
        path (their overflow check reads a device counter) run eagerly."""
        if any(not getattr(rt, "graph_safe", False) for rt in self.legacy_train):
            return False
        if any(getattr(e, "has_dynamic", False) and not getattr(e, "dynamic_graph_safe", False)
               for e in self.ebcs_train):
            return False
        if any(getattr(e, "_uniq", None) is not None for e in self.ebcs_train):
            return False          # Unique-compression exchange sizes its all-to-all on the host
        return True

    def close(self):
        """Release what outlives a Python reference drop: the captured graph (it pins NCCL kernels and
        peer mappings), side streams, reader worker threads.  The model is unusable afterwards."""
        self._graph = None
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)
        for r in (getattr(self, "reader_train", None), getattr(self, "reader_eval", None)):
            try:
                if r is not None:
                    r.stop()
            except Exception:
                pass
        for n in ("_s_emb", "_s_idx", "_copy_stream", "_stg", "_staged", "exchange_wgrad"):
            if hasattr(self, n):
                setattr(self, n, None)
        self.compiled = False

    def train(self) -> bool:
        """One iteration on the next batch; with ``HCTR_STEP_TIMEOUT`` set a watchdog dumps all Python
        stacks (and optionally aborts the rank) when the call does not return in time."""
        wd = getattr(self, "_watchdog", False)
        if wd is False:
            from .utils.watchdog import StepWatchdog
            wd = self._watchdog = StepWatchdog.from_env()
        if wd is None:
            return self._train_step()
        with wd:
            return self._train_step()

    def _train_step(self) -> bool:
        """One iteration on the next batch (Model::train, model.cpp:1048-1138).

        With train_inter_iteration_overlap on a GPU the H2D copy of batch i+1 runs on a copy stream
        while step i executes (double-buffered staging; reference model_pipeline.cpp:370-418)."""
        if not self.reader_train.is_started():
            self.reader_train.start()
        if getattr(self, "_h2d_done", False) and os.environ.get("SKIP_H2D", "0") not in ("0", ""):
            self._run_step()                   # ablation (model.cpp:1067): keep re-using the resident batch
            self._iter += 1
            self.lr_sched.step = self._iter
            return True
        self._h2d_done = True
        prefetch = (self.device.type == "cuda" and self.solver.train_inter_iteration_overlap
                    and len(self.ebcs_train) == 1 and not self.legacy_train
                    and os.environ.get("HCTR_DISABLE_PREFETCH", "0") == "0")
        if not prefetch:
            hb = self.reader_train.read_a_batch()
            if hb is None:
                return False
            if self.reader_train.current_batch_incomplete() and self.solver.drop_incomplete_batch:
                return True
            self._load_batch(hb, True)
        else:
            if getattr(self, "_staged", None) is None:
                hb = self.reader_train.read_a_batch()
                if hb is None:
                    return False
                self._stage_batch(hb)
            if self._staged == "eof":
                self._staged = None
                return False
            self._commit_staged()
        self._run_step()
        self._iter += 1
        self.lr_sched.step = self._iter
        if prefetch:
            nxt = self.reader_train.read_a_batch()
            if nxt is None:
                self._staged = "eof"
            elif self.reader_train.current_batch_incomplete() and self.solver.drop_incomplete_batch:
                self._staged = None
            else:
                self._stage_batch(nxt)
        return True

    def _stage_batch(self, hb: HostBatch):
        """H2D of a batch into staging buffers on the copy stream."""
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream()
            dev = self.device
            self._stg = {"label": torch.empty_like(self.net_train.tensors[self.input.label_name].data),
                         "dense": torch.empty_like(self.net_train.tensors[self.input.dense_name].data),
                         "keys": torch.empty_like(self.ebcs_train[0].key_slab)}
            if self.ebcs_train[0].has_data_weights:
                self._stg["weights"] = torch.empty_like(self.ebcs_train[0].weight_slab)
            self._stg_free = torch.cuda.Event()
            self._stg_free.record()
        cs = self._copy_stream
        cs.wait_event(self._stg_free)           # previous D2D commit has consumed the staging area
        if getattr(hb, "raw", None) is not None and self._stg["keys"].dtype == hb.splitter.key_dtype:
            with torch.cuda.stream(cs):
                hb.splitter.run(hb.raw, hb.raw_skew, hb.num_valid, self._stg["label"],
                                self._stg["dense"] if self.input.dense_dim > 0 else None, self._stg["keys"])
                hb.mark_copied()
            self._staged = hb
            return
        if getattr(hb, "raw", None) is not None:
            hb = self._materialize_raw(hb)
        with torch.cuda.stream(cs):
            self._stg["label"].copy_(hb.label, non_blocking=True)
            if self.input.dense_dim > 0:
                self._stg["dense"].copy_(hb.dense, non_blocking=True)
            self._stg["keys"][:hb.keys.numel()].copy_(hb.keys, non_blocking=True)
            if "weights" in self._stg:
                self._stg["weights"][:hb.weights.numel()].copy_(hb.weights, non_blocking=True)
            hb.mark_copied()
        self._staged = hb

    def _commit_staged(self):
        main = torch.cuda.current_stream()
        main.wait_stream(self._copy_stream)
        net = self.net_train
        net.tensors[self.input.label_name].data.copy_(self._stg["label"], non_blocking=True)
        if self.input.dense_dim > 0:
            net.tensors[self.input.dense_name].data.copy_(self._stg["dense"], non_blocking=True)
        self.ebcs_train[0].key_slab.copy_(self._stg["keys"], non_blocking=True)
        if "weights" in self._stg:
            self.ebcs_train[0].weight_slab.copy_(self._stg["weights"], non_blocking=True)
        self._stg_free.record(main)
        self._staged = None

    def train_on_host_batch(self, hb: HostBatch):
        self._load_batch(hb, True)
        self._run_step()
        self._iter += 1

    def eval(self) -> bool:
        if not self.reader_eval.is_started():
            self.reader_eval.start()
        hb = self.reader_eval.read_a_batch()
        if hb is None:
            return False
        self._load_batch(hb, False)
        self._eval_pipeline().run_graph() if self._eval_graph_ok() else self._eval_pipeline().run()
        raw = self._raw_metrics()
        self._eval_pending = getattr(self, "_eval_pending", 0) + 1
        for (_, _, m) in self.metrics:
            m.set_current_batch_size(self.reader_eval.get_current_batchsize())
            m.local_reduce(raw)
        return True

    def _eval_graph_ok(self) -> bool:
        return (self.solver.use_cuda_graph and self.device.type == "cuda" and self._graph_safe()
                and os.environ.get("HCTR_DISABLE_CUDA_GRAPH", "0") == "0"
                and os.environ.get("HCTR_EVAL_GRAPH", "1") == "1"
                and not getattr(self.comm, "emulated", False))

    def _eval_pipeline(self):
        """The evaluation step as a ``Pipeline`` (pipeline.py, the reference's scheduler of
        HugeCTR/include/pipeline.hpp:28-108 / model_pipeline.cpp:420-520): embedding forward on its own
        stream beside the embedding-independent bottom layers, the top network behind both; with
        ``use_cuda_graph`` the whole pipeline is captured once and replayed (GraphScheduleable)."""
        if getattr(self, "_eval_pipe", None) is None:
            from .pipeline import Pipeline, StreamContextScheduleable

            def emb():
                for e in self.ebcs_eval:
                    e.forward(False)
                for rt in self.legacy_eval:
                    rt.forward(False)
            s_emb = StreamContextScheduleable(emb, "embedding_forward").set_stream("eval_emb")
            s_bot = StreamContextScheduleable(lambda: self.net_eval.fprop(False, "bottom"), "bottom_network")
            s_top = StreamContextScheduleable(lambda: self.net_eval.fprop(False, "top"), "top_network") \
                .wait_event([s_emb, s_bot])
            self._eval_pipe = Pipeline("evaluate", self.device, [s_emb, s_bot, s_top])
        return self._eval_pipe

    def _raw_metrics(self):
        net = self.net_eval
        ll = net.loss_layers
        if len(ll) == 1:
            pred = ll[0].pred
        else:
            pred = torch.cat([l.pred.reshape(l.pred.shape[0], -1) for l in ll], 1)
        label = net.tensors[self.input.label_name].data
        nvalid = self.reader_eval.get_current_batchsize_per_device()
        return {MetricsRawType.Loss: net.loss_value(), MetricsRawType.Pred: pred[:nvalid],
                MetricsRawType.Label: label[:nvalid]}

    def get_eval_metrics(self):
        """(name, value) of every metric over the evaluation batches since the previous call (collective on several
        ranks).  Called again without new ``eval()`` batches -- e.g. after ``fit`` -- it returns the values of the
        last evaluation instead of finalising empty accumulators."""
        if getattr(self, "_eval_pending", 0) == 0 and getattr(self, "_last_eval_metrics", None) is not None:
            return list(self._last_eval_metrics)
        res = [(k.name, m.finalize_metric()) for (k, _, m) in self.metrics]
        self._last_eval_metrics, self._eval_pending = res, 0
        return res

    def get_current_loss(self) -> float:
        v = self.net_train.loss_value().detach().float().clone()
        if self.world > 1:
            self.comm.all_reduce(v)
            v = v / self.world
        return float(v.item())

    def set_learning_rate(self, lr: float):
        self.solver.lr = lr
        self.lr_sched.base_lr = lr
        self._graph = None

    def reset_learning_rate_scheduler(self, base_lr, warmup_steps=1, decay_start=0, decay_steps=1,
                                      decay_power=2.0, end_lr=0.0):
        s = self.solver
        s.lr, s.warmup_steps, s.decay_start = base_lr, warmup_steps, decay_start
        s.decay_steps, s.decay_power, s.end_lr = decay_steps, decay_power, end_lr
        self.lr_sched = LearningRateScheduler(base_lr, warmup_steps, decay_start, decay_steps,
                                              decay_power, end_lr)
        if self.compiled:
            self.step_t.zero_()
        self._graph = None

    # ------------------------------------------------------------------ freeze
    def freeze_embedding(self, name: Optional[str] = None):
        self.embedding_frozen[name or "*"] = True
        self._graph = None

    def unfreeze_embedding(self, name: Optional[str] = None):
        self.embedding_frozen[name or "*"] = False
        self._graph = None

    def freeze_dense(self):
        self.dense_frozen = True
        self._graph = None

    def unfreeze_dense(self):
        self.dense_frozen = False
        self._graph = None

    # ------------------------------------------------------------------ fit
    def fit(self, num_epochs: int = 0, max_iter: int = 2000, display: int = 200,
            eval_interval: int = 1000, snapshot: int = 10000, snapshot_prefix: str = "",
            delta_interval: int = 0, delta_prefix: str = ""):
        """``delta_interval`` = N > 0: every N iterations write ``embedding_dump_delta(f"{delta_prefix}{iter}")``
        of the rows changed since the previous one (the first since the clocks at the start of fit)."""
        s = self.solver
        if not self.compiled:
            raise RuntimeError("call compile() before fit()")
        rank0 = self.comm.rank == 0
        if s.perf_logging:
            logger.perf_log("run_start")
        for cb in self.callbacks:
            cb.on_training_start()
        self.start_data_reading()
        epoch_mode = num_epochs > 0
        if epoch_mode:
            self.reader_train.repeat = False
            self.reader_eval.repeat = False
            logger.info(f"Use epoch mode with number of epochs: {num_epochs}")
        else:
            logger.info(f"Use non-epoch mode with number of iterations: {max_iter}")
        logger.info(f"Training batchsize: {s.batchsize}, evaluation batchsize: {s.batchsize_eval}")
        logger.info(f"Evaluation interval: {eval_interval}, snapshot interval: {snapshot}")
        logger.info(f"Dense network trainable: {not self.dense_frozen}")
        logger.info(f"Use mixed precision: {self.mixed}, scaler: {s.scaler}, use cuda graph: {s.use_cuda_graph}")
        logger.info(f"lr: {s.lr}, warmup_steps: {s.warmup_steps}, end_lr: {s.end_lr}")
        logger.info(f"decay_start: {s.decay_start}, decay_steps: {s.decay_steps}, decay_power: {s.decay_power}")
        t_start = time.time()
        t_disp = time.time()
        it = 0
        epoch = 0
        stop = False
        total_iters = max_iter if not epoch_mode else 1 << 62
        delta_since = self.embedding_clocks() if delta_interval > 0 else None
        while it < total_iters and not stop:
            ok = self.train()
            if not ok:                                  # end of an epoch
                epoch += 1
                if not epoch_mode or epoch >= num_epochs:
                    break
                self.reader_train.set_source(None)
                continue
            it += 1
            if display > 0 and it % display == 0:
                self._dynamic_tables_checkpoint()
                loss = self.get_current_loss()
                if math.isnan(loss):
                    raise RuntimeError("Train Runtime error: Loss cannot converge")  # model.cpp:889
                now = time.time()
                logger.info("Iter: %d Time(%d iters): %.2fs Loss: %f lr:%f" %
                            (it, display, now - t_disp, loss, float(self.lr_t.item())))
                t_disp = now
            if eval_interval > 0 and it % eval_interval == 0:
                stop = self._evaluate(it, t_start) or stop
            if snapshot > 0 and it % snapshot == 0 and it != max_iter:
                self.save_params_to_files(snapshot_prefix, it)
            if delta_interval > 0 and it % delta_interval == 0:
                delta_since = self.embedding_dump_delta(f"{delta_prefix}{it}", delta_since)
        for cb in self.callbacks:
            cb.on_training_end(it)
        if rank0:
            logger.info("Finish %d iterations with batchsize: %d in %.2fs." %
                        (it, s.batchsize, time.time() - t_start))
        return it

    def _evaluate(self, it: int, t_start: float) -> bool:
        s = self.solver
        for cb in self.callbacks:
            cb.on_eval_start(it)
        if s.perf_logging:
            logger.perf_log("eval_start", it)
        t0 = time.time()
        self.reader_eval.set_source(None) if not self.reader_eval.repeat else None
        for _ in range(s.max_eval_batches):
            if not self.eval():
                break
        res = self.get_eval_metrics()
        stop = False
        results = {}
        for (name, val), (kind, thr, _) in zip(res, self.metrics):
            results[name] = val
            logger.info("Evaluation, %s: %f" % (name, val))
            if kind == MetricsType.AUC and thr < 1.0 and val >= thr:   # model.cpp:956-981
                dt = time.time() - t_start
                logger.info("Hit target accuracy AUC %f at %d / %d iterations with batchsize %d in %.2fs. "
                            "Average speed %f records/s." % (val, it, it, s.batchsize, dt,
                                                             it * s.batchsize / max(dt, 1e-9)))
                stop = True
        logger.info("Eval Time for %d iters: %.2fs" % (s.max_eval_batches, time.time() - t0))
        if s.perf_logging:
            logger.perf_log("eval_accuracy", results.get("AUC"), iter=it)
            logger.perf_log("eval_stop", it)
        for cb in self.callbacks:
            if cb.on_eval_end(it, results):
                stop = True
        return stop

    # ------------------------------------------------------------------ checkpoints
    def _dynamic_tables_checkpoint(self):
        """Dynamic tables that ran out of rows grow (``HCTR_DYNAMIC_GROW=0``: raise instead, the round-1
        behaviour).  Collective: every rank learns whether ANY shard grew, because the step graph holds table
        pointers and its re-capture is a rendezvous."""
        ebcs = [e for e in getattr(self, "ebcs_train", []) if getattr(e, "has_dynamic", False)]
        if not ebcs:
            return
        # evicting tables never grow: their counters are logged, the step graph stays (the admission counters of
        # admitting tables are logged as well)
        seen = self.__dict__.setdefault("_evict_dropped", {})
        for ei, e in enumerate(ebcs):
            for (name, shard), st in e.eviction_stats().items():
                logger.info(f"evicting embedding table {name} shard {shard}: live {st['live']} admitted "
                            f"{st['admitted']} evicted {st['evicted']} dropped {st['dropped']}")
                prev = seen.get((ei, name, shard), 0)
                if st["dropped"] > prev:
                    logger.warning(f"evicting embedding table {name} shard {shard}: {st['dropped'] - prev} keys "
                                   "dropped since the last report (every way of their set held a key of the "
                                   "running step); they read as empty rows and got no update")
                seen[(ei, name, shard)] = st["dropped"]
            for (name, shard), st in e.admission_stats().items():
                logger.info(f"admitting embedding table {name} shard {shard}: counted {st['counted']} "
                            f"rejected {st['rejected']}")
        if os.environ.get("HCTR_DYNAMIC_GROW", "1") == "0":
            for e in ebcs:
                e.check_overflow()
            return
        grown = []
        for e in ebcs:
            grown += e.grow_dynamic()
        if self.world > 1:
            grown_any = any(self.comm.all_gather_object(bool(grown)))
        else:
            grown_any = bool(grown)
        for (name, shard, old, new) in grown:
            logger.warning(f"dynamic embedding table {name} shard {shard}: {old} -> {new} rows "
                           f"(keys seen while it was full were read as empty)")
        if grown_any:
            self._graph = None
            self._graph_warm = 0
            self._eval_pipe = None

    def save_params_to_files(self, prefix: str, iter: int = 0):
        self._dynamic_tables_checkpoint()
        from .io.checkpoint import save_model
        save_model(self, prefix, iter)

    def resume(self, prefix: str, iter: Optional[int] = None) -> int:
        """Continue a run from the snapshot ``save_params_to_files(prefix, iter)`` / ``fit(snapshot=...)``
        wrote (latest one when ``iter`` is None): weights, every optimizer state and the training
        counters.  Returns the iteration to continue from (call after ``compile()``)."""
        from .io.checkpoint import resume
        return resume(self, prefix, iter)

    def download_params_to_files(self, prefix: str, iter: int = 0):
        self.save_params_to_files(prefix, iter)

    def load_dense_weights(self, path: str):
        from .io.checkpoint import load_dense_weights
        load_dense_weights(self, path)
        self._graph = None

    def load_dense_optimizer_states(self, path: str):
        from .io.checkpoint import load_dense_opt_states
        load_dense_opt_states(self, path)

    def load_sparse_weights(self, paths):
        from .io.checkpoint import load_sparse_weights
        load_sparse_weights(self, paths)

    def load_sparse_optimizer_states(self, paths):
        from .io.checkpoint import load_sparse_opt_states
        load_sparse_opt_states(self, paths)

    def embedding_dump(self, path: str, table_names=None):
        from .io.checkpoint import embedding_dump
        embedding_dump(self, path, table_names)

    def embedding_load(self, path: str, table_names=None):
        from .io.checkpoint import embedding_load
        embedding_load(self, path, table_names)

    def embedding_clocks(self) -> Dict[int, int]:
        """{collection id: clock} of the embedding collections, read with one host synchronisation: each clock
        ticks once per training step of a collection with a tracked (or evicting, or admitting) table.  Record
        them beside a full ``embedding_dump`` as the base of a chain of ``embedding_dump_delta``."""
        ebcs = getattr(self, "ebcs_train", [])
        if not ebcs:
            return {}
        return {i: int(c) for i, c in enumerate(torch.cat([e.evict_clock for e in ebcs]).cpu().tolist())}

    def embedding_dump_delta(self, path: str, since: Optional[Dict[int, int]] = None,
                             table_names=None) -> Dict[int, int]:
        """Write the rows of the tables with ``track_updates`` that changed after the clocks ``since``
        {collection id: clock} (None: 0) with their current fp32 values, in the ``embedding_dump`` layout plus
        ``delta.json``; returns the clocks at the dump, the ``since`` of the next delta (docs/embedding.md).
        Every rank takes part.  ``InferenceModel.update_embedding`` applies such a folder."""
        from .io.checkpoint import embedding_dump_delta
        return embedding_dump_delta(self, path, since, table_names)

    # ------------------------------------------------------------------ debugging
    def check_out_tensor(self, name: str, which: Tensor_t = Tensor_t.Train):
        net = self.net_train if which == Tensor_t.Train else self.net_eval
        if name not in net.tensors:
            raise KeyError(f"no tensor named {name}")
        t = net.tensors[name].data.detach().float().cpu()
        if self.world > 1:
            parts = self.comm.all_gather_object(t)
            t = torch.cat(parts, 0)
        return t.numpy()
