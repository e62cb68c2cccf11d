"""Backend-neutral resource interface of the embedding stack.

Reference: ``core::CoreResourceManager`` / ``core::GPUResourceBase`` (HugeCTR/core/core.hpp:28-75) with the HugeCTR
backend in core/hctr_impl/hctr_backend.hpp:41-83 -- the seam that lets the embedding collection and SOK run on
"whatever owns the GPU": HugeCTR's resource manager there, a TensorFlow runtime in SOK.

Here the embedding collection (embedding/collection.py) and SOK (sok/__init__.py) ask this interface for who
they are and whom they talk to; two back-ends implement it:

* ``TorchCoreResourceManager`` over ``parallel.comm.Comm`` -- one process per GPU, torch.distributed (NCCL /
  gloo) plus the CUDA-IPC symmetric heap;
* the same class over ``parallel.emu.EmuComm`` -- N ranks as threads of one process on one device (tests, the
  one-GPU proof of the peer kernels).

``KernelParams`` mirrors core23::KernelParams (SM count, warp size, max threads per block / SM) and is what
launch-size decisions should read instead of a literal SM count (132 on an H100 SXM).
"""
from __future__ import annotations

import abc
from dataclasses import dataclass
from typing import Dict, Optional

import torch


@dataclass(frozen=True)
class KernelParams:
    num_sms: int = 132
    warp_size: int = 32
    max_threads_per_block: int = 1024
    max_threads_per_sm: int = 2048
    smem_per_block_optin: int = 227 * 1024

    @staticmethod
    def init(device: Optional[torch.device] = None) -> "KernelParams":
        if device is not None and device.type == "cuda" and torch.cuda.is_available():
            p = torch.cuda.get_device_properties(device)
            return KernelParams(num_sms=p.multi_processor_count, warp_size=getattr(p, "warp_size", 32),
                                max_threads_per_sm=getattr(p, "max_threads_per_multi_processor", 2048),
                                smem_per_block_optin=getattr(p, "shared_memory_per_block_optin", 227 * 1024))
        return KernelParams()


class GPUResourceBase(abc.ABC):
    """named streams of one GPU (core.hpp:28-35); ``get_stream`` is the CURRENT one"""

    @abc.abstractmethod
    def set_stream(self, name: str) -> None: ...

    @abc.abstractmethod
    def get_current_stream_name(self) -> str: ...

    @abc.abstractmethod
    def get_stream(self): ...


class CoreResourceManager(abc.ABC):
    """core.hpp:37-72; ``get_comm`` stands where ``get_nccl`` does (the communicator object of the back-end)"""

    def __init__(self, kernel_params: Optional[KernelParams] = None):
        self.kernel_params_ = kernel_params or KernelParams()

    @abc.abstractmethod
    def get_local_gpu(self) -> GPUResourceBase: ...

    @abc.abstractmethod
    def get_comm(self): ...

    @abc.abstractmethod
    def get_local_gpu_id(self) -> int: ...

    @abc.abstractmethod
    def get_global_gpu_id(self) -> int: ...

    @abc.abstractmethod
    def get_device_id(self) -> int: ...

    @abc.abstractmethod
    def get_local_gpu_count(self) -> int: ...

    @abc.abstractmethod
    def get_global_gpu_count(self) -> int: ...

    @abc.abstractmethod
    def get_gpu_global_id_from_local_id(self, local_id: int) -> int: ...

    @abc.abstractmethod
    def get_gpu_local_id_from_global_id(self, global_id: int) -> int: ...

    def get_kernel_param(self) -> KernelParams:
        return self.kernel_params_

    get_nccl = property(lambda self: self.get_comm)       # the reference's spelling


class TorchGPUResource(GPUResourceBase):
    """streams by name on one device; "default" is whatever stream is current when the resource is made.
    Stream priorities follow the step scheduler's convention (lower number = scheduled first)."""

    def __init__(self, device: torch.device):
        self.device = device
        self._streams: Dict[str, object] = {}
        self._name = "default"

    def _make(self, name: str):
        if self.device.type != "cuda":
            return None
        prio = {"emb": -1, "comm": -3, "bottom": -3}.get(name, 0)
        return torch.cuda.Stream(self.device, priority=prio)

    def set_stream(self, name: str) -> None:
        if name != "default" and name not in self._streams:
            self._streams[name] = self._make(name)
        self._name = name

    def get_current_stream_name(self) -> str:
        return self._name

    def get_stream(self):
        if self.device.type != "cuda":
            return None
        if self._name == "default":
            return torch.cuda.current_stream(self.device)
        return self._streams[self._name]


class TorchCoreResourceManager(CoreResourceManager):
    """the interface over a ``Comm`` / ``EmuComm`` (anything with rank, world_size, device and, after
    ``set_topology``, local_size / num_nodes)"""

    def __init__(self, comm):
        super().__init__(KernelParams.init(getattr(comm, "device", None)))
        self.comm = comm
        self._gpu = TorchGPUResource(comm.device)

    def _local_size(self) -> int:
        return int(getattr(self.comm, "local_size", None) or self.comm.world_size)

    def get_local_gpu(self) -> GPUResourceBase:
        return self._gpu

    def get_comm(self):
        return self.comm

    def get_local_gpu_id(self) -> int:
        return self.comm.rank % self._local_size()

    def get_global_gpu_id(self) -> int:
        return self.comm.rank

    def get_device_id(self) -> int:
        d = self.comm.device
        return int(d.index or 0) if d.type == "cuda" else -1

    def get_local_gpu_count(self) -> int:
        return self._local_size()

    def get_global_gpu_count(self) -> int:
        return self.comm.world_size

    def get_gpu_global_id_from_local_id(self, local_id: int) -> int:
        node = self.comm.rank // self._local_size()
        return node * self._local_size() + int(local_id)

    def get_gpu_local_id_from_global_id(self, global_id: int) -> int:
        return int(global_id) % self._local_size()


def as_core(obj) -> CoreResourceManager:
    """a CoreResourceManager for ``obj``: itself, or the (cached) view of a communicator"""
    if isinstance(obj, CoreResourceManager):
        return obj
    core = getattr(obj, "_core", None)
    if core is None:
        core = TorchCoreResourceManager(obj)
        try:
            obj._core = core
        except Exception:
            pass
    return core
