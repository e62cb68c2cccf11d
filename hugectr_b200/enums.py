"""Enumerations of the public API (parity with HugeCTR/include/pybind/common_wrapper.hpp:31-218)."""
from enum import Enum, IntEnum


class Error_t(IntEnum):
    Success = 0
    FileCannotOpen = 1
    BrokenFile = 2
    OutOfMemory = 3
    OutOfBound = 4
    WrongInput = 5
    IllegalCall = 6
    NotInitialized = 7
    UnSupportedFormat = 8
    InvalidEnv = 9
    MpiError = 10
    CublasError = 11
    CudnnError = 12
    CudaDriverError = 13
    CudaRuntimeError = 14
    NcclError = 15
    DataCheckError = 16
    UnspecificError = 17
    EndOfFile = 18


class Check_t(Enum):
    Sum = 0
    Non = 1


class DataReaderType_t(Enum):
    Norm = 0
    Raw = 1
    Parquet = 2
    RawAsync = 3


class FileSystemType_t(Enum):
    Local = 0
    HDFS = 1
    S3 = 2
    GCS = 3
    Other = 4


DataSourceType_t = FileSystemType_t   # name used by releases before 23.04 (notebooks/training_with_remote_filesystem)


class SourceType_t(Enum):
    FileList = 0
    Mmap = 1
    Parquet = 2


class TrainPSType_t(Enum):
    Staged = 0
    Cached = 1


class Embedding_t(Enum):
    DistributedSlotSparseEmbeddingHash = 0
    LocalizedSlotSparseEmbeddingHash = 1
    # kept for config compatibility (deprecated upstream, mapped onto Localized here)
    LocalizedSlotSparseEmbeddingOneHot = 2
    HybridSparseEmbedding = 3


class Initializer_t(Enum):
    Default = 0
    Uniform = 1
    XavierNorm = 2
    XavierUniform = 3
    Zero = 4
    Sinusoidal = 5


class Layer_t(Enum):
    BatchNorm = 0
    LayerNorm = 1
    BinaryCrossEntropyLoss = 2
    Reshape = 3
    Select = 4
    Concat = 5
    CrossEntropyLoss = 6
    Dropout = 7
    ElementwiseMultiply = 8
    ELU = 9
    InnerProduct = 10
    MLP = 11
    Interaction = 12
    MultiCrossEntropyLoss = 13
    ReLU = 14
    ReLUHalf = 15
    Sigmoid = 16
    Slice = 17
    WeightMultiply = 18
    FmOrder2 = 19
    Add = 20
    ReduceSum = 21
    Softmax = 22
    Gather = 23
    PReLU_Dice = 24
    GRU = 25
    MatrixMultiply = 26
    MultiHeadAttention = 27
    Scale = 28
    FusedReshapeConcat = 29
    FusedReshapeConcatGeneral = 30
    Sub = 31
    ReduceMean = 32
    MultiCross = 33
    Cast = 34
    SequenceMask = 35
    # extras kept from older releases / used internally
    FusedInnerProduct = 36
    MaskedSoftmax = 37
    Concat3D = 38
    DotProduct = 39


class Alignment_t(Enum):
    Auto = 0
    Non = 1


class LrPolicy_t(Enum):
    fixed = 0


class Optimizer_t(Enum):
    Ftrl = 0
    Adam = 1
    RMSProp = 2
    AdaGrad = 3
    MomentumSGD = 4
    Nesterov = 5
    SGD = 6
    # embedding-collection tables only: one fp32 accumulator per row (docs/embedding.md)
    RowWiseAdaGrad = 7
    # embedding-collection tables only: per-weight first moment, one fp32 second moment per row
    # (docs/embedding.md)
    PartialRowWiseAdam = 8


class Update_t(Enum):
    Local = 0
    Global = 1
    LazyGlobal = 2


class Activation_t(Enum):
    Relu = 0
    Non = 1


class FcPosition_t(Enum):
    Non = 0
    Head = 1
    Body = 2
    Tail = 3
    Isolated = 4


class Regularizer_t(Enum):
    L1 = 0
    L2 = 1
    Non = 2


class MetricsRawType(Enum):
    Loss = 0
    Pred = 1
    Label = 2


class MetricsType(Enum):
    AUC = 0
    AverageLoss = 1
    HitRate = 2
    NDCG = 3
    SMAPE = 4


class DeviceLayout(Enum):
    LocalFirst = 0
    NodeFirst = 1


class AllReduceAlgo(Enum):
    OneShot = 0
    NCCL = 1
    # extension: two-shot reduce-scatter/all-gather over peer memory (large buffers)
    TwoShot = 2


class Distribution_t(Enum):
    Uniform = 0
    PowerLaw = 1


class PowerLaw_t(Enum):
    Long = 0
    Medium = 1
    Short = 2
    Specific = 3


class Tensor_t(Enum):
    Train = 0
    Evaluate = 1


class CommunicationStrategy(Enum):
    Uniform = 0
    Hierarchical = 1


class CompressionStrategy(Enum):
    Reduction = 0
    Unique = 1


class EmbeddingLayout(Enum):
    FeatureMajor = 0
    BatchMajor = 1


# number of optimizer state values per weight (include/optimizer.hpp:37-110)
OPT_STATES_PER_WEIGHT = {
    Optimizer_t.Ftrl: 2,
    Optimizer_t.Adam: 2,
    Optimizer_t.RMSProp: 1,
    Optimizer_t.AdaGrad: 1,
    Optimizer_t.MomentumSGD: 1,
    Optimizer_t.Nesterov: 1,
    Optimizer_t.SGD: 0,
    Optimizer_t.RowWiseAdaGrad: 0,   # one value per row, not per weight
    Optimizer_t.PartialRowWiseAdam: 1,   # the first moment; the second is one value per row
}
