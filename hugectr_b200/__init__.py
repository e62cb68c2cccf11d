"""hugectr_b200 -- a Hopper (sm_90a, H100) native CTR training framework with HugeCTR's API.

``import hugectr`` resolves to this package (see the top-level ``hugectr`` shim): CreateSolver,
DataReaderParams, CreateOptimizer, Model, Input, SparseEmbedding, DenseLayer,
EmbeddingTableConfig, EmbeddingCollectionConfig, tools.DataGenerator, data.DataSourceParams,
TrainingCallback (HugeCTR/src/pybind/module_main.cpp:36-48).
"""
from .enums import *  # noqa: F401,F403
import os as _os

# The step runs up to ten concurrent branches (main, embedding forward / backward, index build, heavy rows,
# bottom-network backward, bucketed all-reduce, per-bucket optimizer, data-parallel tables, H2D prefetch) and
# several of them contain kernels that spin on flags written by OTHER GPUs.  With the default of 8 hardware
# work queues two branches can share a queue: a spinning kernel then blocks an unrelated branch that a peer
# is waiting for -- a cross-GPU deadlock.  Must be set before the CUDA context exists.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from .enums import (Activation_t, Alignment_t, AllReduceAlgo, Check_t, CommunicationStrategy,
                    CompressionStrategy, DataReaderType_t, DeviceLayout, Distribution_t,
                    Embedding_t, Error_t, FcPosition_t, FileSystemType_t, Initializer_t, Layer_t,
                    LrPolicy_t, MetricsRawType, MetricsType, Optimizer_t, PowerLaw_t,
                    Regularizer_t, SourceType_t, Tensor_t, TrainPSType_t, Update_t)
from .solver import (AsyncParam, CreateETC, CreateHMemCache, CreateOptimizer, CreateSolver, DataReaderParams,
                     DataReaderSparseParam, DataSourceParams, DenseLayer, DenseLayerComputeConfig,
                     EmbeddingTrainingCacheParams, HMemCacheConfig, Input, OptParamsPy, Solver, SparseEmbedding)
from .embedding.collection import (EmbeddingCollectionConfig, EmbeddingTableConfig, InitParams)
from .lr_scheduler import LearningRateScheduler
from .model import Model, TrainingCallback

__version__ = "25.03.b200.1"


def __getattr__(name):
    # lazy sub-namespaces: hugectr.tools / hugectr.data / hugectr.sok / hugectr.inference
    import importlib
    if name in ("tools", "data", "sok", "onnx", "cache", "io", "parallel", "utils", "models", "inference", "core23"):
        return importlib.import_module(f"{__name__}.{name}")
    if name in ("Core23DataReader32", "Core23DataReader64", "DataReader32", "DataReader64"):
        from .data.readers import IDataReader     # reader handle classes (data_reader_wrapper.hpp:50-72)
        return IDataReader
    if name == "Optimizer":
        from .solver import OptParamsPy           # the docs call CreateOptimizer's result hugectr.Optimizer
        return OptParamsPy
    raise AttributeError(name)
