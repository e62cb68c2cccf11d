"""embedding_workspace_calculator: workspace_size_per_gpu_in_mb for legacy SparseEmbedding.

max_vocabulary_size_per_gpu = workspace_MB * 2^20 / ((1 + n_opt_states) * 4 * vec)  (model.cpp:186-196)
-> the inverse, as computed by the reference tool
(tools/embedding_workspace_calculator/cal_vocabulary_size_per_gpu_and_workspace_size_per_gpu.py);
``load_factor`` < 1 adds head room on top of it.  The three ``cal_*`` functions carry the tool's names.
"""
from __future__ import annotations

import math

from ..enums import Embedding_t, Optimizer_t, Update_t
from ..solver import OptParamsPy


def calculate(slot_size_array, vec_size: int, optimizer: Optimizer_t = Optimizer_t.Adam,
              update_type: Update_t = Update_t.Global, num_gpus: int = 1,
              embedding_type: Embedding_t = Embedding_t.DistributedSlotSparseEmbeddingHash,
              load_factor: float = 1.0) -> int:
    ns = OptParamsPy(optimizer, update_type).num_states
    if embedding_type == Embedding_t.DistributedSlotSparseEmbeddingHash:
        rows = math.ceil(sum(slot_size_array) / num_gpus)
    else:
        per = [0] * num_gpus
        for i, s in enumerate(slot_size_array):
            per[i % num_gpus] += s
        rows = max(per)
    rows = math.ceil(rows / load_factor)
    return math.ceil(rows * (1 + ns) * 4 * vec_size / (1 << 20))


_OPT = {"adam": Optimizer_t.Adam, "adagrad": Optimizer_t.AdaGrad, "momentumsgd": Optimizer_t.MomentumSGD,
        "nesterov": Optimizer_t.Nesterov, "sgd": Optimizer_t.SGD}
_UPD = {"local": Update_t.Local, "global": Update_t.Global, "lazy_global": Update_t.LazyGlobal}


def cal_vocabulary_size_per_gpu_for_distributed_slot(total_vocabulary_size, num_gpus):
    return math.ceil(total_vocabulary_size / num_gpus)


def cal_vocabulary_size_per_gpu_for_localized_slot(slot_size_array, num_gpus):
    per = [0] * num_gpus
    for i, s in enumerate(slot_size_array):
        per[i % num_gpus] += s
    return math.ceil(max(per))


def cal_workspace_size_per_gpu_from_vocabulary_size_per_gpu(vocabulary_size_per_gpu, emb_vec_size, num_gpus,
                                                            optimizer, optimizer_update_type):
    assert optimizer_update_type in _UPD
    ns = OptParamsPy(_OPT[optimizer], _UPD[optimizer_update_type]).num_states
    return math.ceil(vocabulary_size_per_gpu * emb_vec_size * 4 * (1 + ns) / (1024 * 1024))
