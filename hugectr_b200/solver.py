"""Plain parameter structs of the Python API.

Parity with the reference pybind wrappers:
  CreateSolver      HugeCTR/include/pybind/solver_wrapper.hpp:27-153
  CreateOptimizer   HugeCTR/include/pybind/optimizer_wrapper.hpp:25-57
  DataReaderParams / Input / SparseEmbedding / DenseLayer   HugeCTR/include/pybind/model_wrapper.hpp:27-131
  DataReaderSparseParam / AsyncParam   HugeCTR/include/pybind/common_wrapper.hpp:133-150
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Union

from .enums import (Activation_t, Alignment_t, AllReduceAlgo, Check_t, DataReaderType_t,
                    DeviceLayout, Embedding_t, FcPosition_t, Initializer_t, Layer_t, LrPolicy_t,
                    MetricsType, OPT_STATES_PER_WEIGHT, Optimizer_t, Regularizer_t, Update_t)


# --------------------------------------------------------------------------- solver
@dataclass
class Solver:
    model_name: str = ""
    seed: int = 0
    lr_policy: LrPolicy_t = LrPolicy_t.fixed
    lr: float = 0.001
    warmup_steps: int = 1
    decay_start: int = 0
    decay_steps: int = 1
    decay_power: float = 2.0
    end_lr: float = 0.0
    max_eval_batches: int = 100
    batchsize_eval: int = 2048
    batchsize: int = 2048
    vvgpu: List[List[int]] = field(default_factory=lambda: [[0]])
    repeat_dataset: bool = True
    use_mixed_precision: bool = False
    enable_tf32_compute: bool = False
    scaler: float = 1.0
    metrics_spec: Dict[MetricsType, float] = field(default_factory=lambda: {MetricsType.AUC: 1.0})
    i64_input_key: bool = False
    use_algorithm_search: bool = True
    use_cuda_graph: bool = True
    gen_loss_summary: bool = True
    train_intra_iteration_overlap: bool = False
    train_inter_iteration_overlap: bool = False
    eval_intra_iteration_overlap: bool = False
    eval_inter_iteration_overlap: bool = False
    device_layout: DeviceLayout = DeviceLayout.LocalFirst
    use_embedding_collection: bool = False
    all_reduce_algo: AllReduceAlgo = AllReduceAlgo.NCCL
    grouped_all_reduce: bool = False
    num_iterations_statistics: int = 20
    perf_logging: bool = False
    drop_incomplete_batch: bool = True
    kafka_brockers: str = ""
    training_callbacks: list = field(default_factory=list)
    # extensions of this framework (ignored by reference scripts)
    use_fp8_mlp: bool = False
    fused_embedding_comm: bool = True

    @property
    def num_gpus(self) -> int:
        return sum(len(v) for v in self.vvgpu)

    @property
    def num_nodes(self) -> int:
        return len(self.vvgpu)


def CreateSolver(model_name: str = "", seed: int = 0, lr_policy=LrPolicy_t.fixed, lr: float = 0.001,
                 warmup_steps: int = 1, decay_start: int = 0, decay_steps: int = 1,
                 decay_power: float = 2.0, end_lr: float = 0.0, max_eval_batches: int = 100,
                 batchsize_eval: int = 2048, batchsize: int = 2048, vvgpu=None,
                 repeat_dataset: bool = True, use_mixed_precision: bool = False,
                 enable_tf32_compute: bool = False, scaler: float = 1.0, metrics_spec=None,
                 i64_input_key: bool = False, use_algorithm_search: bool = True,
                 use_cuda_graph: bool = True, gen_loss_summary: bool = True,
                 train_intra_iteration_overlap: bool = False,
                 train_inter_iteration_overlap: bool = False,
                 eval_intra_iteration_overlap: bool = False,
                 eval_inter_iteration_overlap: bool = False,
                 device_layout=DeviceLayout.LocalFirst, use_embedding_collection: bool = False,
                 all_reduce_algo=AllReduceAlgo.NCCL, grouped_all_reduce: bool = False,
                 num_iterations_statistics: int = 20, perf_logging: bool = False,
                 drop_incomplete_batch: bool = True, kafka_brockers: str = "",
                 training_callbacks=None, use_fp8_mlp: bool = False,
                 fused_embedding_comm: bool = True) -> Solver:
    if use_mixed_precision and enable_tf32_compute:
        # solver_wrapper.hpp:40-43
        raise RuntimeError("use_mixed_precision and enable_tf32_compute cannot be true at the same time")
    if use_mixed_precision and scaler not in (1.0, 128.0, 256.0, 512.0, 1024.0) and scaler <= 0:
        raise RuntimeError("scaler must be positive")
    if use_fp8_mlp and not use_mixed_precision:
        raise RuntimeError("use_fp8_mlp needs use_mixed_precision=True (bf16 activations, fp8 forward GEMMs)")
    return Solver(
        model_name=model_name, seed=seed, lr_policy=lr_policy, lr=lr, warmup_steps=warmup_steps,
        decay_start=decay_start, decay_steps=decay_steps, decay_power=decay_power, end_lr=end_lr,
        max_eval_batches=max_eval_batches, batchsize_eval=batchsize_eval, batchsize=batchsize,
        vvgpu=[list(v) for v in (vvgpu if vvgpu is not None else [[0]])],
        repeat_dataset=repeat_dataset, use_mixed_precision=use_mixed_precision,
        enable_tf32_compute=enable_tf32_compute, scaler=scaler,
        metrics_spec=dict(metrics_spec) if metrics_spec is not None else {MetricsType.AUC: 1.0},
        i64_input_key=i64_input_key, use_algorithm_search=use_algorithm_search,
        use_cuda_graph=use_cuda_graph, gen_loss_summary=gen_loss_summary,
        train_intra_iteration_overlap=train_intra_iteration_overlap,
        train_inter_iteration_overlap=train_inter_iteration_overlap,
        eval_intra_iteration_overlap=eval_intra_iteration_overlap,
        eval_inter_iteration_overlap=eval_inter_iteration_overlap, device_layout=device_layout,
        use_embedding_collection=use_embedding_collection, all_reduce_algo=all_reduce_algo,
        grouped_all_reduce=grouped_all_reduce, num_iterations_statistics=num_iterations_statistics,
        perf_logging=perf_logging, drop_incomplete_batch=drop_incomplete_batch,
        kafka_brockers=kafka_brockers, training_callbacks=list(training_callbacks or []),
        use_fp8_mlp=use_fp8_mlp, fused_embedding_comm=fused_embedding_comm)


# --------------------------------------------------------------------------- optimizer
@dataclass
class OptParamsPy:
    optimizer_type: Optimizer_t = Optimizer_t.Adam
    update_type: Update_t = Update_t.Global
    beta: float = 0.0           # ftrl
    lambda1: float = 0.0        # ftrl
    lambda2: float = 0.0        # ftrl
    beta1: float = 0.9          # adam / partial row-wise adam
    beta2: float = 0.999        # adam / partial row-wise adam
    epsilon: float = 1e-7       # adam / adagrad / row-wise adagrad / partial row-wise adam
    initial_accu_value: float = 0.0  # adagrad / row-wise adagrad
    momentum_factor: float = 0.0     # momentum sgd / nesterov
    atomic_update: bool = True       # sgd
    initialized: bool = True

    @property
    def num_states(self) -> int:
        n = OPT_STATES_PER_WEIGHT[self.optimizer_type]
        if self.optimizer_type == Optimizer_t.Adam and self.update_type == Update_t.LazyGlobal:
            n += 1  # prev_time copy (model.cpp:189-192)
        return n

    def to_json(self) -> dict:
        t = self.optimizer_type
        d = {"type": t.name, "update_type": self.update_type.name}
        if t in (Optimizer_t.Adam, Optimizer_t.PartialRowWiseAdam):
            d["adam_hparam"] = {"beta1": self.beta1, "beta2": self.beta2, "epsilon": self.epsilon}
        elif t in (Optimizer_t.AdaGrad, Optimizer_t.RowWiseAdaGrad):
            d["adagrad_hparam"] = {"initial_accu_value": self.initial_accu_value,
                                   "epsilon": self.epsilon}
        elif t == Optimizer_t.Ftrl:
            d["ftrl_hparam"] = {"beta": self.beta, "lambda1": self.lambda1, "lambda2": self.lambda2}
        elif t == Optimizer_t.MomentumSGD:
            d["momentum_sgd_hparam"] = {"momentum_factor": self.momentum_factor}
        elif t == Optimizer_t.Nesterov:
            d["nesterov_hparam"] = {"momentum_factor": self.momentum_factor}
        elif t == Optimizer_t.SGD:
            d["sgd_hparam"] = {"atomic_update": self.atomic_update}
        elif t == Optimizer_t.RMSProp:
            d["rmsprop_hparam"] = {"beta": self.beta2, "epsilon": self.epsilon}
        return d

    @staticmethod
    def from_json(d: dict) -> "OptParamsPy":
        t = Optimizer_t[d["type"]]
        o = OptParamsPy(optimizer_type=t, update_type=Update_t[d.get("update_type", "Global")])
        for key in ("adam_hparam", "adagrad_hparam", "ftrl_hparam", "momentum_sgd_hparam",
                    "nesterov_hparam", "sgd_hparam", "rmsprop_hparam"):
            for k, v in d.get(key, {}).items():
                if hasattr(o, k):
                    setattr(o, k, v)
        return o


def check_not_rowwise(opt: Optional[OptParamsPy], where: str) -> None:
    """Row-wise AdaGrad and partial row-wise Adam keep one state value per embedding row: only
    embedding-collection tables have them.  Raises ValueError for any other user of an optimizer
    (``where``)."""
    t = getattr(opt, "optimizer_type", opt)
    if t in (Optimizer_t.RowWiseAdaGrad, Optimizer_t.PartialRowWiseAdam):
        raise ValueError(f"Optimizer_t.{t.name} is not supported for {where}; it applies to "
                         "embedding-collection tables only: pass it per table with "
                         "EmbeddingTableConfig(opt_params=...)")


def CreateOptimizer(optimizer_type=Optimizer_t.Adam, update_type=Update_t.Global, beta: float = 0.0,
                    lambda1: float = 0.0, lambda2: float = 0.0, beta1: float = 0.9,
                    beta2: float = 0.999, epsilon: float = 1e-7, initial_accu_value: float = 0.0,
                    momentum_factor: float = 0.0, atomic_update: bool = True) -> OptParamsPy:
    return OptParamsPy(optimizer_type, update_type, beta, lambda1, lambda2, beta1, beta2, epsilon,
                       initial_accu_value, momentum_factor, atomic_update, True)


# --------------------------------------------------------------------------- data reader params
class DataReaderSparseParam:
    def __init__(self, top_name: str, nnz_per_slot: Union[int, Sequence[int]],
                 is_fixed_length: bool, slot_num: int, weighted: bool = False, position_weighted: bool = False):
        """``weighted``: the reader delivers an fp32 weight with every key of this input, and every
        embedding lookup of it pools weighted (see docs/embedding.md).
        ``position_weighted``: key h of slot f of every sample weighs ``P[f, h]``, a trainable fp32 parameter
        ``[slot_num, max(nnz_per_slot)]`` of the dense network that starts at 1.0 (see docs/embedding.md)."""
        self.top_name = top_name
        self.weighted = bool(weighted)
        if not isinstance(position_weighted, bool):
            raise ValueError(f"input {top_name}: position_weighted must be a bool, not {position_weighted!r}")
        if position_weighted and self.weighted:
            raise ValueError(f"input {top_name}: weighted and position_weighted exclude each other (the weights "
                             "come either from the reader or from the model)")
        self.position_weighted = position_weighted
        if isinstance(nnz_per_slot, int):
            self.nnz_per_slot = [nnz_per_slot] * slot_num
        else:
            self.nnz_per_slot = list(nnz_per_slot)
            if len(self.nnz_per_slot) != slot_num:
                raise ValueError("nnz_per_slot length must equal slot_num")
        self.is_fixed_length = bool(is_fixed_length)
        self.slot_num = int(slot_num)
        self.max_feature_num = sum(self.nnz_per_slot)
        self.max_nnz = max(self.nnz_per_slot) if self.nnz_per_slot else 0

    def to_json(self):
        return {"top": self.top_name, "type": "DistributedSlot",
                "nnz_per_slot": self.nnz_per_slot if len(set(self.nnz_per_slot)) > 1
                else self.nnz_per_slot[0],
                "is_fixed_length": self.is_fixed_length, "slot_num": self.slot_num,
                **({"weighted": True} if self.weighted else {}),
                **({"position_weighted": True} if self.position_weighted else {})}


@dataclass
class AsyncParam:
    num_threads: int = 16
    num_batches_per_thread: int = 4
    max_num_requests_per_thread: int = 0
    io_depth: int = 0
    io_alignment: int = 0
    shuffle: bool = False
    aligned_type: Alignment_t = Alignment_t.Non
    multi_hot_reader: bool = True
    is_dense_float: bool = True


@dataclass
class DataSourceParams:
    """hugectr.data.DataSourceParams (data_source_wrapper.hpp:27-35)."""
    source: "object" = None   # FileSystemType_t
    server: str = "localhost"
    port: int = 9000

    def __post_init__(self):
        from .enums import FileSystemType_t
        if self.source is None:
            self.source = FileSystemType_t.Local


class DataReaderParams:
    def __init__(self, data_reader_type: DataReaderType_t, source, keyset=None, eval_source="",
                 check_type=Check_t.Non, cache_eval_data: int = 0, num_samples: int = 0,
                 eval_num_samples: int = 0, float_label_dense: bool = False,
                 read_file_sequentially: bool = False, num_workers: int = 12,
                 slot_size_array=None, data_source_params=None, async_param=None):
        self.data_reader_type = data_reader_type
        self.source = [source] if isinstance(source, str) else list(source)
        if keyset is None:
            keyset = []
        self.keyset = [keyset] if isinstance(keyset, str) else list(keyset)
        self.eval_source = eval_source
        self.check_type = check_type
        self.cache_eval_data = cache_eval_data
        self.num_samples = num_samples
        self.eval_num_samples = eval_num_samples
        self.float_label_dense = float_label_dense
        self.read_file_sequentially = read_file_sequentially
        self.num_workers = num_workers
        self.slot_size_array = list(slot_size_array or [])
        self.data_source_params = data_source_params or DataSourceParams()
        self.async_param = async_param or AsyncParam(16, 4, 512000, 4, 512, False,
                                                     Alignment_t.Non, False, False)


# --------------------------------------------------------------------------- graph nodes
class Input:
    """Three overloads: single label, multi label, multi label + weights (model_wrapper.hpp:57-72)."""

    def __init__(self, label_dim=None, label_name=None, dense_dim: int = 0, dense_name: str = "dense",
                 data_reader_sparse_param_array=None, label_dims=None, label_names=None,
                 label_weights=None):
        if label_dims is None:
            if isinstance(label_dim, (list, tuple)):
                label_dims, label_names = list(label_dim), list(label_name)
            else:
                label_dims, label_names = [int(label_dim)], [label_name]
        self.label_dims = list(label_dims)
        self.label_names = list(label_names)
        self.label_weights = list(label_weights) if label_weights is not None else [1.0] * len(self.label_dims)
        self.dense_dim = int(dense_dim)
        self.dense_name = dense_name
        self.data_reader_sparse_param_array = list(data_reader_sparse_param_array or [])

    @property
    def label_dim(self):
        return sum(self.label_dims)

    @property
    def label_name(self):
        return self.label_names[0] if len(self.label_names) == 1 else "combined_multi_label"


class SparseEmbedding:
    def __init__(self, embedding_type: Embedding_t, workspace_size_per_gpu_in_mb: int = 0,
                 embedding_vec_size: int = 0, combiner: str = "sum", sparse_embedding_name: str = "",
                 bottom_name: str = "", slot_size_array=None, optimizer: Optional[OptParamsPy] = None,
                 max_vocabulary_size_per_gpu: int = 0):
        if combiner not in ("sum", "mean"):
            raise ValueError("combiner must be 'sum' or 'mean'")
        check_not_rowwise(optimizer, "a legacy SparseEmbedding")
        self.embedding_type = embedding_type
        self.workspace_size_per_gpu_in_mb = int(workspace_size_per_gpu_in_mb)
        self.embedding_vec_size = int(embedding_vec_size)
        self.combiner = combiner
        self.sparse_embedding_name = sparse_embedding_name
        self.bottom_name = bottom_name
        self.slot_size_array = list(slot_size_array or [])
        self.optimizer = optimizer
        self.max_vocabulary_size_per_gpu = int(max_vocabulary_size_per_gpu)


class HMemCacheConfig:
    """hugectr.CreateHMemCache(num_blocks, target_hit_rate, max_num_evict) of the 22.x releases: sizing hints of
    the host-memory cache; the host parameter server here keeps the whole table, the hints are recorded."""

    def __init__(self, num_blocks: int = 1, target_hit_rate: float = 0.5, max_num_evict: int = 0):
        self.num_blocks, self.target_hit_rate, self.max_num_evict = num_blocks, target_hit_rate, max_num_evict


def CreateHMemCache(num_blocks: int = 1, target_hit_rate: float = 0.5, max_num_evict: int = 0) -> HMemCacheConfig:
    return HMemCacheConfig(num_blocks, target_hit_rate, max_num_evict)


class EmbeddingTrainingCacheParams:
    """``hugectr.CreateETC(ps_types, sparse_models, local_paths, hmem_cache_configs)`` (embedding training cache,
    HugeCTR/include/embedding_training_cache/*.hpp): one entry per SparseEmbedding, in model.add order.
    ``TrainPSType_t.Cached``: table on the host parameter server, hot rows in the HBM gpu_cache;
    ``TrainPSType_t.Staged``: host table, every step stages its rows.  ``sparse_models[i]``: directory the
    table is initialised from / saved to ("" = fresh)."""

    def __init__(self, ps_types, sparse_models, local_paths=None, hmem_cache_configs=None, host_capacity_rows=0):
        self.ps_types = list(ps_types)
        self.sparse_models = list(sparse_models)
        self.local_paths = list(local_paths or [])
        self.hmem_cache_configs = list(hmem_cache_configs or [])
        self.host_capacity_rows = int(host_capacity_rows)
        if len(self.sparse_models) not in (0, len(self.ps_types)):
            raise ValueError("CreateETC: one sparse model path per ps_type")


def CreateETC(ps_types, sparse_models=(), local_paths=None, hmem_cache_configs=None, host_capacity_rows=0):
    return EmbeddingTrainingCacheParams(ps_types, sparse_models, local_paths, hmem_cache_configs, host_capacity_rows)


@dataclass
class DenseLayerComputeConfig:
    async_wgrad: bool = False
    fuse_wb: bool = False


class DenseLayer:
    """46 kwargs, same names and defaults as model_wrapper.hpp:86-131."""

    def __init__(self, layer_type: Layer_t, bottom_names: Sequence[str], top_names: Sequence[str],
                 factor: float = 1.0, eps: float = 1e-5,
                 gamma_init_type=Initializer_t.Default, beta_init_type=Initializer_t.Default,
                 dropout_rate: float = 0.5, elu_alpha: float = 1.0, num_output: int = 1,
                 weight_init_type=Initializer_t.Default, bias_init_type=Initializer_t.Default,
                 num_layers: int = 0, leading_dim: int = 0, time_step: int = 0, batchsize: int = 1,
                 SeqLength: int = 1, vector_size: int = 1, selected: bool = False,
                 selected_slots=None, ranges=None, indices=None, weight_dims=None,
                 projection_dim: int = 0, out_dim: int = 0, axis: int = 1,
                 max_sequence_len_from: int = 1, max_sequence_len_to: int = 1,
                 num_attention_heads: int = 1, transpose_b: bool = False, target_weight_vec=None,
                 use_regularizer: bool = False, regularizer_type=Regularizer_t.L1,
                 lambda_: float = 0.0, pos_type=FcPosition_t.Non, act_type=Activation_t.Relu,
                 num_outputs=None, use_bias: bool = True, activations=None, biases=None,
                 compute_config: Optional[DenseLayerComputeConfig] = None, shape=None, dim: int = 0,
                 index=None, **kw):
        if "lambda" in kw:  # python keyword in the reference API
            lambda_ = kw.pop("lambda")
        if kw:
            raise TypeError("unexpected DenseLayer kwargs: %s" % sorted(kw))
        self.layer_type = layer_type
        self.bottom_names = list(bottom_names)
        self.top_names = list(top_names)
        self.factor = factor
        self.eps = eps
        self.gamma_init_type = gamma_init_type
        self.beta_init_type = beta_init_type
        self.dropout_rate = dropout_rate
        self.elu_alpha = elu_alpha
        self.num_output = num_output
        self.weight_init_type = weight_init_type
        self.bias_init_type = bias_init_type
        self.num_layers = num_layers
        self.leading_dim = leading_dim
        self.time_step = time_step
        self.batchsize = batchsize
        self.SeqLength = SeqLength
        self.vector_size = vector_size
        self.selected = selected
        self.selected_slots = list(selected_slots or [])
        self.ranges = [tuple(r) for r in (ranges or [])]
        self.indices = list(indices or [])
        self.weight_dims = list(weight_dims or [])
        self.projection_dim = projection_dim
        self.out_dim = out_dim
        self.axis = axis
        self.max_sequence_len_from = max_sequence_len_from
        self.max_sequence_len_to = max_sequence_len_to
        self.num_attention_heads = num_attention_heads
        self.transpose_b = transpose_b
        self.target_weight_vec = list(target_weight_vec or [])
        self.use_regularizer = use_regularizer
        self.regularizer_type = regularizer_type
        self.lambda_ = lambda_
        self.pos_type = pos_type
        self.act_type = act_type
        self.num_outputs = list(num_outputs or [])
        self.use_bias = use_bias
        self.activations = list(activations or [])
        self.biases = list(biases or [])
        self.compute_config = compute_config or DenseLayerComputeConfig()
        self.shape = list(shape or [])
        self.dim = dim
        self.index = list(index or [])
