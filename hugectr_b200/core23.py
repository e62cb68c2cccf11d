"""core23-style tensor / buffer runtime on top of torch (component C1 of the survey; reference
HugeCTR/core23/{tensor.hpp:33, tensor_params.hpp, buffer.hpp:30, buffer_channel.hpp:29, buffer_params.hpp,
details/unitary_buffer.cpp, tensor_container.hpp, allocator_params.hpp}).

What the reference's runtime provides and the training path relies on is kept as behaviour:

* **lazy tensors**: a ``Tensor`` is declared with shape / dtype / ``TensorParams`` and only gets memory at its
  first ``data()`` (or at an explicit ``AllocateBuffers``);
* **buffer channels**: tensors declared with the same ``(device, channel)`` -- and a ``unitary`` buffer --
  are carved from ONE contiguous allocation in declaration order, 256-byte aligned, so that a whole
  parameter set can be addressed as one flat array (``Buffer.decay()``): this is what makes the in-place
  gradient all-reduce and the fused optimizer single launches (``layers.base.ParamArena`` is the
  specialised form used by the networks);
* **allocators**: device (torch caching allocator), pinned host, managed / plain host;
* **TensorContainer**: an N-d collection of same-dtype tensors of one channel with ``flatten()`` -> the flat
  view over all of them (the reference's WeightTensors / WgradTensors);
* ``Tensor.bind`` wraps foreign memory (any torch tensor) without owning it.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from enum import Enum
from typing import Dict, List, Optional, Sequence, Tuple

import torch

ALIGN = 256


class DeviceType(Enum):
    CPU = "cpu"
    GPU = "cuda"
    UNIFIED = "managed"      # served from pinned host memory here (the GPU reads it over PCIe)


@dataclass(frozen=True)
class Device:
    type: DeviceType = DeviceType.CPU
    index: int = 0

    @staticmethod
    def current() -> "Device":
        return Device(DeviceType.GPU, torch.cuda.current_device()) if torch.cuda.is_available() else Device()

    def torch(self) -> torch.device:
        return torch.device("cuda", self.index) if self.type == DeviceType.GPU else torch.device("cpu")


class AllocatorType(Enum):
    Default = 0        # torch caching allocator (device) / malloc (host)
    PinnedHost = 1
    Managed = 2
    NewDelete = 3


class BufferChannel:
    """named group of tensors that share one buffer per device ("Blobs", "Weight", "WeightHalf", "Wgrad",
    "WgradHalf", "OptState", "EVAL_*": include/network_buffer_channels.hpp)"""
    _auto = 0

    def __init__(self, name: Optional[str] = None):
        if name is None:
            BufferChannel._auto += 1
            name = f"__anonymous_{BufferChannel._auto}"
        self.name = name

    def __eq__(self, o):
        return isinstance(o, BufferChannel) and o.name == self.name

    def __hash__(self):
        return hash(self.name)

    def __repr__(self):
        return f"BufferChannel({self.name})"


def GetRandomBufferChannel() -> BufferChannel:
    return BufferChannel()


@dataclass
class BufferParams:
    channel: BufferChannel = field(default_factory=lambda: BufferChannel("Blobs"))
    unitary: bool = True                 # one contiguous allocation (else: one allocation per tensor)
    allocator: AllocatorType = AllocatorType.Default


@dataclass
class TensorParams:
    shape: Tuple[int, ...] = ()
    data_type: torch.dtype = torch.float32
    device: Device = field(default_factory=Device.current)
    buffer_params: BufferParams = field(default_factory=BufferParams)
    alignment: int = ALIGN

    def with_(self, **kw) -> "TensorParams":
        d = dict(shape=self.shape, data_type=self.data_type, device=self.device,
                 buffer_params=self.buffer_params, alignment=self.alignment)
        d.update(kw)
        return TensorParams(**d)


class Buffer:
    """all tensors of one (device, channel): reserve-then-allocate"""

    def __init__(self, device: Device, params: BufferParams):
        self.device, self.params = device, params
        self.clients: List["Tensor"] = []
        self.offsets: List[int] = []
        self.nbytes = 0
        self.storage: Optional[torch.Tensor] = None     # uint8 [nbytes]
        self.frozen = False

    def subscribe(self, t: "Tensor"):
        if self.frozen:
            raise RuntimeError(f"buffer of {self.params.channel} is already allocated: declare tensors first")
        a = max(1, t.params.alignment)
        self.nbytes = (self.nbytes + a - 1) // a * a
        self.clients.append(t)
        self.offsets.append(self.nbytes)
        self.nbytes += t.num_bytes()

    def allocate(self):
        if self.frozen:
            return
        dev, kind = self.device.torch(), self.params.allocator
        n = max(self.nbytes, 1)
        if self.params.unitary:
            st = torch.zeros(n, dtype=torch.uint8, device=dev)
            if dev.type == "cpu" and (kind in (AllocatorType.PinnedHost, AllocatorType.Managed)
                                      or self.device.type == DeviceType.UNIFIED) and torch.cuda.is_available():
                st = st.pin_memory()
            self.storage = st
            for t, off in zip(self.clients, self.offsets):
                t._data = st[off:off + t.num_bytes()].view(t.params.data_type).view(t.params.shape)
        else:
            for t in self.clients:
                t._data = torch.zeros(t.params.shape, dtype=t.params.data_type, device=dev)
        self.frozen = True

    def decay(self, dtype: torch.dtype = torch.uint8) -> torch.Tensor:
        """the whole buffer as one flat array (unitary buffers only)"""
        self.allocate()
        if self.storage is None:
            raise RuntimeError("decay() needs a unitary buffer")
        n = self.storage.numel() // torch.empty(0, dtype=dtype).element_size()
        return self.storage[:n * torch.empty(0, dtype=dtype).element_size()].view(dtype)


_buffers: Dict[Tuple[Device, BufferChannel], Buffer] = {}


def GetBuffer(params: BufferParams, device: Device) -> Buffer:
    key = (device, params.channel)
    if key not in _buffers or (_buffers[key].frozen and not _buffers[key].clients):
        _buffers[key] = Buffer(device, params)
    return _buffers[key]


def AllocateBuffers(device: Optional[Device] = None) -> bool:
    """allocate every declared-but-unallocated buffer (of one device)"""
    for key, buf in list(_buffers.items()):
        if device is None or key[0] == device:
            buf.allocate()
    return True


def ForgetChannel(device: Device, channel: BufferChannel):
    """drop a (single-use) channel from the registry; its tensors keep the storage alive"""
    _buffers.pop((device, channel), None)


def ReleaseBuffers():
    """forget all channels (tests / model teardown); tensors keep their memory alive"""
    _buffers.clear()


class Tensor:
    def __init__(self, shape_or_params=None, data_type: Optional[torch.dtype] = None,
                 params: Optional[TensorParams] = None):
        if isinstance(shape_or_params, TensorParams):
            params = shape_or_params
        else:
            params = (params or TensorParams()).with_(shape=tuple(shape_or_params or ()),
                                                      data_type=data_type or (params or TensorParams()).data_type)
        self.params = params
        self._data: Optional[torch.Tensor] = None
        self._owner = True
        self._buffer = None
        if params.shape:
            buf = GetBuffer(params.buffer_params, params.device)
            if buf.frozen:       # the channel was already allocated: a new generation of the channel starts
                buf = _buffers[(params.device, params.buffer_params.channel)] = Buffer(params.device, params.buffer_params)
            buf.subscribe(self)
            self._buffer = buf

    @staticmethod
    def bind(data: torch.Tensor, shape=None, data_type=None, device: Optional[Device] = None) -> "Tensor":
        t = Tensor.__new__(Tensor)
        d = data if shape is None else data.view(*shape)
        dev = device or (Device(DeviceType.GPU, d.device.index or 0) if d.is_cuda else Device())
        t.params = TensorParams(tuple(d.shape), d.dtype, dev)
        t._data, t._owner, t._buffer = d, False, None
        return t

    # ---- metadata
    def shape(self): return self.params.shape
    def dims(self): return len(self.params.shape)
    def size(self, dim): return self.params.shape[dim]
    def data_type(self): return self.params.data_type
    def device(self): return self.params.device
    def my_params(self): return self.params
    def own_data(self): return self._owner
    def empty(self): return self._data is None and not self.params.shape

    def num_elements(self) -> int:
        n = 1
        for s in self.params.shape:
            n *= int(s)
        return n if self.params.shape else 0

    def num_bytes(self) -> int:
        return self.num_elements() * torch.empty(0, dtype=self.params.data_type).element_size()

    # ---- data
    def data(self) -> torch.Tensor:
        if self._data is None:
            if self._buffer is None:
                raise RuntimeError("empty tensor")
            self._buffer.allocate()
        return self._data

    def reshape(self, new_shape) -> "Tensor":
        n = 1
        for s in new_shape:
            n *= int(s)
        if n != self.num_elements():
            raise ValueError("reshape changes the number of elements")
        t = Tensor.__new__(Tensor)
        t.params, t._owner, t._buffer = self.params.with_(shape=tuple(new_shape)), False, None
        t._data = self.data().view(*new_shape)
        return t

    def view(self, *shape) -> torch.Tensor:
        return self.data().view(*shape) if shape else self.data()


class TensorContainer:
    """N-d collection of tensors of one dtype / channel with a flat view over all of them"""

    def __init__(self, tensors: Sequence[Tensor], shape: Optional[Sequence[int]] = None):
        self.tensors = list(tensors)
        self.shape = tuple(shape) if shape is not None else (len(self.tensors),)
        if self.tensors:
            p0 = self.tensors[0].params
            for t in self.tensors:
                if t.params.data_type != p0.data_type or t.params.buffer_params.channel != p0.buffer_params.channel:
                    raise ValueError("a TensorContainer holds tensors of one dtype and one buffer channel")

    def __len__(self): return len(self.tensors)
    def __getitem__(self, i): return self.tensors[i]
    def __iter__(self): return iter(self.tensors)

    def flatten(self) -> torch.Tensor:
        """1-d view from the first element of the first tensor to the last element of the last one
        (includes alignment padding, which stays zero), without copying"""
        if not self.tensors:
            return torch.zeros(0)
        first, last = self.tensors[0].data(), self.tensors[-1].data()
        buf = self.tensors[0]._buffer
        if buf is None or buf.storage is None or any(t._buffer is not buf for t in self.tensors):
            raise RuntimeError("flatten() needs tensors of one unitary buffer")
        esz = first.element_size()
        lo = first.data_ptr() - buf.storage.data_ptr()
        hi = last.data_ptr() - buf.storage.data_ptr() + last.numel() * esz
        return buf.storage[lo:hi].view(first.dtype)


# ---- low-level primitives / tensor operations (core23/low_level_primitives.cu, tensor_operations.hpp)
def zeros_sync(t: Tensor): t.data().zero_()
def zeros_async(t: Tensor, stream=None): t.data().zero_()
def fill_sync(t: Tensor, value): t.data().fill_(value)
def copy_sync(dst: Tensor, src: Tensor): dst.data().copy_(src.data())
def copy_async(dst: Tensor, src: Tensor, stream=None): dst.data().copy_(src.data(), non_blocking=True)
def convert_async(dst: Tensor, src: Tensor, stream=None): dst.data().copy_(src.data().to(dst.data_type()), non_blocking=True)


def uniform_async(t: Tensor, a: float, b: float, generator: Optional[torch.Generator] = None):
    t.data().uniform_(a, b, generator=generator)


def normal_async(t: Tensor, mean: float, stddev: float, generator: Optional[torch.Generator] = None):
    t.data().normal_(mean, stddev, generator=generator)
