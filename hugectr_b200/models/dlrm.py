"""DLRM (MLPerf v1) and DLRM-DCNv2 (MLPerf v3.1) through the public API.

Reference model definitions: samples/dlrm/train.py:31-85,330-500 (DCNv2: bottom MLP 512-256-128,
Concat, MultiCross(projection_dim 512, num_layers 3), top MLP 1024-1024-512-256-1, BCE, AdaGrad) and
test/embedding_collection_test/dgx_a100_one_hot.py (DLRM: Interaction, SGD).
"""
from __future__ import annotations

from typing import List, Optional

import hugectr_b200 as hugectr

CRITEO_TB_TABLE_SIZES = [40000000, 39060, 17295, 7424, 20265, 3, 7122, 1543, 63, 40000000, 3067956,
                         405282, 10, 2209, 11938, 155, 4, 976, 14, 40000000, 40000000, 40000000,
                         590152, 12973, 108, 36]
CRITEO_TB_MULTI_HOT = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3,
                       1, 1]
NUM_DENSE = 13


def _default_ar():
    """MLPerf DLRM config uses the custom one-shot all-reduce (train.py --all_reduce_algo OneShot)"""
    import os
    return (hugectr.AllReduceAlgo.NCCL if os.environ.get("HCTR_ALLREDUCE", "p2p") == "nccl"
            else hugectr.AllReduceAlgo.OneShot)


def _solver(batchsize, num_gpus, lr, mixed, scaler, **kw):
    gpn = kw.pop("gpus_per_node", 0)      # > 0: several nodes -> one vvgpu list per node
    vvgpu = [list(range(num_gpus))] if not gpn or gpn >= num_gpus else \
        [list(range(gpn)) for _ in range(num_gpus // gpn)]
    return hugectr.CreateSolver(
        model_name=kw.pop("model_name", "dlrm"), seed=kw.pop("seed", 0), max_eval_batches=kw.pop("max_eval_batches", 10),
        batchsize_eval=kw.pop("batchsize_eval", batchsize), batchsize=batchsize,
        vvgpu=vvgpu, repeat_dataset=kw.pop("repeat_dataset", True), lr=lr, warmup_steps=kw.pop("warmup_steps", 1),
        use_mixed_precision=mixed, scaler=scaler, use_cuda_graph=kw.pop("use_cuda_graph", True),
        train_intra_iteration_overlap=True, train_inter_iteration_overlap=True,
        use_embedding_collection=True, grouped_all_reduce=True, gen_loss_summary=True,
        all_reduce_algo=kw.pop("all_reduce_algo", _default_ar()), **kw)


def build_dlrm_dcnv2(batchsize: int = 55296, num_gpus: int = 8, table_sizes: Optional[List[int]] = None,
                     multi_hot: Optional[List[int]] = None, ev_size: int = 128, lr: float = 0.004,
                     mixed: bool = True, scaler: float = 1.0, source=None, shard_plan=None,
                     optimizer: str = "adagrad", bottom=(512, 256, 128),
                     top=(1024, 1024, 512, 256, 1), cross_layers: int = 3, projection_dim: int = 512,
                     comm=None, comm_strategy=None, compression_strategy=None,
                     embedding_optimizer: str = "adagrad", weight_dtype: str = "fp32",
                     **solver_kw) -> "hugectr.Model":
    """``embedding_optimizer``: "adagrad" (the model optimizer for every table), "rowwise_adagrad"
    (every table gets row-wise AdaGrad with the model optimizer's epsilon and initial value, one fp32
    accumulator per row) or "partial_rowwise_adam" (every table gets partial row-wise Adam with
    ``CreateOptimizer``'s Adam defaults: a per-weight first moment, one fp32 second moment per row); the
    dense layers keep the model optimizer.  ``weight_dtype``: "fp32" or "bf16" storage of the tables'
    weights."""
    choices = ("adagrad", "rowwise_adagrad", "partial_rowwise_adam")
    if embedding_optimizer not in choices:
        raise ValueError(f"embedding_optimizer must be one of {choices}, not {embedding_optimizer!r}")
    table_sizes = list(table_sizes or CRITEO_TB_TABLE_SIZES)
    multi_hot = list(multi_hot or CRITEO_TB_MULTI_HOT)
    n = len(table_sizes)
    solver = _solver(batchsize, num_gpus, lr, mixed, scaler, model_name="dlrm_dcnv2", **solver_kw)
    if optimizer == "adagrad":
        opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad, hugectr.Update_t.Global,
                                      initial_accu_value=0.0, epsilon=1e-8)
    else:
        opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD, hugectr.Update_t.Local,
                                      atomic_update=True)
    reader = hugectr.DataReaderParams(
        data_reader_type=hugectr.DataReaderType_t.RawAsync, source=source or ["synthetic:1.1"],
        eval_source=(source[0] if source else "synthetic:1.1"), check_type=hugectr.Check_t.Non,
        slot_size_array=table_sizes,
        async_param=hugectr.AsyncParam(1, 16, shuffle=False, multi_hot_reader=True,
                                       is_dense_float=True))
    model = hugectr.Model(solver, reader, opt, comm=comm)
    model.add(hugectr.Input(
        label_dim=1, label_name="label", dense_dim=NUM_DENSE, dense_name="dense",
        data_reader_sparse_param_array=[
            hugectr.DataReaderSparseParam(f"data{i}", multi_hot[i], True, 1) for i in range(n)]))
    evs = [int(ev_size)] * n if isinstance(ev_size, int) else [int(e) for e in ev_size]   # per-table widths
    table_opt = None
    if embedding_optimizer == "rowwise_adagrad":
        table_opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.RowWiseAdaGrad, hugectr.Update_t.Global,
                                            initial_accu_value=opt.initial_accu_value, epsilon=opt.epsilon)
    elif embedding_optimizer == "partial_rowwise_adam":
        table_opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.PartialRowWiseAdam, hugectr.Update_t.Global)
    tables = [hugectr.EmbeddingTableConfig(name=str(i), max_vocabulary_size=table_sizes[i],
                                           ev_size=evs[i], opt_params=table_opt, weight_dtype=weight_dtype)
              for i in range(n)]
    ebc = hugectr.EmbeddingCollectionConfig(
        use_exclusive_keys=True, comm_strategy=comm_strategy or hugectr.CommunicationStrategy.Uniform)
    ebc.embedding_lookup(table_config=tables, bottom_name=[f"data{i}" for i in range(n)],
                         top_name="sparse_embedding", combiner=["sum"] * n)
    if shard_plan is None:
        from hugectr_b200.tools.planner import generate_plan
        shard_plan = generate_plan(table_sizes, multi_hot, num_gpus, ev_size=max(evs))
    ebc.shard(shard_matrix=shard_plan[0], shard_strategy=shard_plan[1], compression_strategy=compression_strategy)
    model.add(ebc)
    cc = hugectr.DenseLayerComputeConfig(async_wgrad=True, fuse_wb=False)
    model.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["dense"], ["mlp1"], num_outputs=list(bottom),
                                 act_type=hugectr.Activation_t.Relu, compute_config=cc))
    model.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["sparse_embedding", "mlp1"], ["concat1"]))
    model.add(hugectr.DenseLayer(hugectr.Layer_t.MultiCross, ["concat1"], ["interaction1"],
                                 projection_dim=projection_dim, num_layers=cross_layers,
                                 compute_config=cc))
    acts = [hugectr.Activation_t.Relu] * (len(top) - 1) + [hugectr.Activation_t.Non]
    model.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["interaction1"], ["mlp2"],
                                 num_outputs=list(top), activations=acts, compute_config=cc))
    model.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["mlp2", "label"], ["loss"]))
    return model


def build_dlrm(batchsize: int = 55296, num_gpus: int = 8, table_sizes=None, ev_size: int = 128,
               lr: float = 24.0, mixed: bool = True, scaler: float = 1.0, source=None,
               shard_plan=None, comm=None, compression_strategy=None, **solver_kw):
    """MLPerf-v1 DLRM: one-hot lookups, concat combiner, dot Interaction, SGD."""
    table_sizes = list(table_sizes or CRITEO_TB_TABLE_SIZES)
    n = len(table_sizes)
    solver = _solver(batchsize, num_gpus, lr, mixed, scaler, model_name="dlrm", **solver_kw)
    opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD, hugectr.Update_t.Local, atomic_update=True)
    reader = hugectr.DataReaderParams(
        data_reader_type=hugectr.DataReaderType_t.RawAsync, source=source or ["synthetic:1.1"],
        eval_source=(source[0] if source else "synthetic:1.1"), check_type=hugectr.Check_t.Non,
        slot_size_array=table_sizes)
    model = hugectr.Model(solver, reader, opt, comm=comm)
    model.add(hugectr.Input(
        label_dim=1, label_name="label", dense_dim=NUM_DENSE, dense_name="dense",
        data_reader_sparse_param_array=[
            hugectr.DataReaderSparseParam(f"data{i}", 1, True, 1) for i in range(n)]))
    tables = [hugectr.EmbeddingTableConfig(str(i), table_sizes[i], ev_size) for i in range(n)]
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup(tables, [f"data{i}" for i in range(n)], "sparse_embedding", ["concat"] * n)
    if shard_plan is None:
        from hugectr_b200.tools.planner import generate_plan
        shard_plan = generate_plan(table_sizes, [1] * n, num_gpus, ev_size=ev_size)
    ebc.shard(shard_plan[0], shard_plan[1], compression_strategy=compression_strategy)
    model.add(ebc)
    model.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["dense"], ["mlp1"], num_outputs=[512, 256, ev_size],
                                 act_type=hugectr.Activation_t.Relu))
    model.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["sparse_embedding"], ["emb3d"],
                                 shape=[-1, n, ev_size]))
    model.add(hugectr.DenseLayer(hugectr.Layer_t.Interaction, ["mlp1", "emb3d"], ["interaction1"]))
    acts = [hugectr.Activation_t.Relu] * 4 + [hugectr.Activation_t.Non]
    model.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["interaction1"], ["mlp2"],
                                 num_outputs=[1024, 1024, 512, 256, 1], activations=acts))
    model.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["mlp2", "label"], ["loss"]))
    return model
