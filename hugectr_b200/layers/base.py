"""Layer / tensor / parameter-arena runtime.

Design (GPU-native, not a port of core23):
  * tensors are torch tensors with static shapes, pre-allocated at compile() so one training step
    is CUDA-graph capturable;
  * all trainable dense parameters live in ONE flat fp32 master buffer (+ flat fp32 wgrad, flat
    bf16 compute shadow, flat optimizer state) -- that is what makes the single fused optimizer
    launch, the bucketed in-place all-reduce and the raw checkpoint dump possible (the role of
    core23 "Weight"/"Wgrad" UnitaryBuffers, HugeCTR/include/network_buffer_channels.hpp and
    HugeCTR/src/pybind/model_compile.cpp:887-900);
  * every layer implements explicit fprop/bprop (reference Layer::fprop/bprop,
    HugeCTR/include/layer.hpp:31-92); hot layers call the sm_90a kernels, the long tail derives
    bprop from torch autograd (``TorchLayer``).
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence

import torch

from ..enums import Initializer_t


class TensorBag:
    """Named activation: ``data`` (+ ``grad`` in the training graph)."""

    def __init__(self, name: str, shape: Sequence[int], dtype: torch.dtype):
        self.name = name
        self.shape = tuple(int(s) for s in shape)
        self.dtype = dtype
        self.data: Optional[torch.Tensor] = None
        self.grad: Optional[torch.Tensor] = None
        self.needs_grad = True
        self.producer = None

    def allocate(self, device, with_grad: bool):
        if self.data is None:
            self.data = torch.zeros(self.shape, dtype=self.dtype, device=device)
        if with_grad and self.needs_grad and self.grad is None and self.dtype.is_floating_point:
            self.grad = torch.zeros(self.shape, dtype=self.dtype, device=device)

    def view2d(self, which="data"):
        t = self.data if which == "data" else self.grad
        return None if t is None else t.reshape(t.shape[0], -1)

    def __repr__(self):
        return f"TensorBag({self.name}, {self.shape}, {self.dtype})"


class Param:
    def __init__(self, name, shape, offset, numel, padded_numel, init):
        self.name = name
        self.shape = tuple(shape)
        self.offset = offset
        self.numel = numel
        self.padded_numel = padded_numel
        self.init = init
        self.w = self.g = self.w16 = None  # views, set by ParamArena.finalize()

    def compute(self, mixed: bool):
        """Tensor the kernels read: bf16 shadow in mixed precision, else fp32 master."""
        return self.w16 if (mixed and self.w16 is not None) else self.w


class ParamArena:
    ALIGN = 64  # elements; keeps every parameter 256-byte aligned in fp32 and 128 B in bf16

    def __init__(self):
        self.params: List[Param] = []
        self._size = 0
        self._replay = None
        self.weights = self.wgrad = self.weights16 = None
        self.finalized = False

    # ---- construction
    def add(self, name: str, shape, init: Callable[[tuple], torch.Tensor], pad_rows: int = 0) -> Param:
        if self._replay is not None:  # building the eval graph: hand out the same parameters
            p = self._replay.pop(0)
            assert tuple(shape) == p.shape, (name, shape, p.shape)
            return p
        numel = int(math.prod(shape))
        padded = numel + pad_rows * int(shape[-1])
        p = Param(name, shape, self._size, numel, padded, init)
        self._size += (padded + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.params.append(p)
        return p

    def begin_replay(self):
        self._replay = list(self.params)

    def end_replay(self):
        self._replay = None

    @property
    def num_params(self) -> int:
        return sum(p.numel for p in self.params)

    @property
    def flat_size(self) -> int:
        return self._size

    def finalize(self, device, mixed: bool, pad_to: int = 1, wgrad_alloc=None):
        """``wgrad_alloc(numel, dtype)``: optional allocator for the gradient buffer (the symmetric
        peer-mapped heap when the P2P all-reduce is used)."""
        n = max(self._size, 1)
        n = (n + pad_to - 1) // pad_to * pad_to  # model_compile.cpp:853-869 pads wgrad to 16*N bytes
        # The flat arrays are core23 unitary buffers, one per channel like the reference's network buffer
        # channels (include/network_buffer_channels.hpp: "Weight", "WeightHalf", "Wgrad"): a lazily allocated
        # core23.Tensor is declared per channel, AllocateBuffers() materialises them, decay() gives the flat
        # view the fused optimizer / in-place all-reduce / raw checkpoint dump work on.  The peer-mapped wgrad
        # of the P2P all-reduce is external memory bound into a core23.Tensor.
        from .. import core23
        cdev = core23.Device(core23.DeviceType.GPU, device.index or 0) if device.type == "cuda" else core23.Device()
        tag = f"#{id(self):x}"

        def chan(name, dtype):
            tp = core23.TensorParams(shape=(n,), data_type=dtype, device=cdev,
                                     buffer_params=core23.BufferParams(channel=core23.BufferChannel(name + tag)))
            return core23.Tensor(tp)
        self.c23_weights = chan("Weight", torch.float32)
        self.c23_weights16 = chan("WeightHalf", torch.bfloat16) if mixed else None
        self.c23_wgrad = (core23.Tensor.bind(wgrad_alloc(n, torch.float32)) if wgrad_alloc is not None
                          else chan("Wgrad", torch.float32))
        # data() allocates the tensor's own buffer (AllocateBuffers() would walk every channel of the process,
        # including those other rank threads are declaring); the per-arena channels are single use
        self.weights = self.c23_weights.data()
        self.wgrad = self.c23_wgrad.data()
        self.weights16 = self.c23_weights16.data() if mixed else None
        for nm in ("Weight", "WeightHalf", "Wgrad"):
            core23.ForgetChannel(cdev, core23.BufferChannel(nm + tag))
        for p in self.params:
            p.w = self.weights[p.offset:p.offset + p.numel].view(p.shape)
            p.g = self.wgrad[p.offset:p.offset + p.numel].view(p.shape)
            if mixed:
                rows_p = p.padded_numel // p.shape[-1] if len(p.shape) > 1 else p.padded_numel
                if len(p.shape) == 2:
                    p.w16 = self.weights16[p.offset:p.offset + p.padded_numel].view(rows_p, p.shape[-1])
                    p.g_padded = self.wgrad[p.offset:p.offset + p.padded_numel].view(rows_p, p.shape[-1])
                else:
                    p.w16 = self.weights16[p.offset:p.offset + p.numel].view(p.shape)
                    p.g_padded = p.g
            else:
                p.g_padded = p.g
        self.finalized = True

    def init_params(self, seed: int):
        """Host-side generation with one seed for every replica (core23_network.cpp:209-214)."""
        gen = torch.Generator(device="cpu")
        gen.manual_seed(int(seed))
        for p in self.params:
            v = p.init(p.shape, gen).to(torch.float32)
            p.w.copy_(v.to(p.w.device))
        self.sync_shadow()

    def sync_shadow(self):
        if self.weights16 is not None:
            self.weights16.copy_(self.weights.to(torch.bfloat16))

    # ---- checkpoint helpers: unpadded fp32 in creation order (Appendix 3.6 format)
    def dump_flat(self) -> torch.Tensor:
        if not self.params:
            return torch.zeros(0)
        return torch.cat([p.w.reshape(-1).detach().cpu() for p in self.params])

    def load_flat(self, flat: torch.Tensor):
        off = 0
        for p in self.params:
            p.w.copy_(flat[off:off + p.numel].view(p.shape).to(p.w.device))
            off += p.numel
        self.sync_shadow()

    def dump_state(self, state: Optional[torch.Tensor]) -> torch.Tensor:
        if state is None or not self.params:
            return torch.zeros(0)
        return torch.cat([state[p.offset:p.offset + p.numel].detach().cpu() for p in self.params])

    def load_state(self, state: torch.Tensor, flat: torch.Tensor):
        off = 0
        for p in self.params:
            state[p.offset:p.offset + p.numel].copy_(flat[off:off + p.numel].to(state.device))
            off += p.numel


# ------------------------------------------------------------------ initialisers (Appendix A.4)
def _uniform(shape, gen, bound):
    return (torch.rand(shape, generator=gen) * 2.0 - 1.0) * bound


def make_init(kind: Initializer_t, fan_in: int, fan_out: int, default: str):
    """default: 'mlp' U(+-sqrt(1/fan_in)); 'fc_w' U(+-1/(fan_in+fan_out)) ... see Appendix A.4"""
    def init(shape, gen):
        k = kind
        if k == Initializer_t.Zero:
            return torch.zeros(shape)
        if k == Initializer_t.Default:
            if default == "mlp":
                return _uniform(shape, gen, math.sqrt(1.0 / max(fan_in, 1)))
            if default == "fc_w":
                return _uniform(shape, gen, 1.0 / max(fan_in + fan_out, 1))
            if default == "fc_b":
                return _uniform(shape, gen, 1.0 / max(fan_out, 1))
            if default == "xavier":
                k = Initializer_t.XavierUniform
            elif default == "zero":
                return torch.zeros(shape)
            elif default == "one":
                return torch.ones(shape)
        if k == Initializer_t.Uniform:
            return _uniform(shape, gen, 1.0 / max(fan_in + fan_out, 1))
        if k == Initializer_t.XavierUniform:  # variance scaling(1, fan_avg, uniform)
            limit = math.sqrt(3.0 / ((fan_in + fan_out) / 2.0))
            return _uniform(shape, gen, limit)
        if k == Initializer_t.XavierNorm:
            std = math.sqrt(1.0 / ((fan_in + fan_out) / 2.0))
            return torch.randn(shape, generator=gen) * std
        return torch.zeros(shape)
    return init


class BuildCtx:
    """What a layer sees while it is being constructed."""

    def __init__(self, arena: ParamArena, device, act_dtype, batch: int, is_train: bool, solver,
                 mixed: bool):
        self.arena = arena
        self.device = device
        self.act_dtype = act_dtype
        self.batch = batch
        self.is_train = is_train
        self.solver = solver
        self.mixed = mixed
        self.layer_index = 0

    @property
    def native(self) -> bool:
        return self.device.type == "cuda"


class Layer:
    """Base class; subclasses create ``self.outputs`` in __init__ (shape inference)."""
    trainable = False
    is_loss = False

    def __init__(self, cfg, inputs: List[TensorBag], ctx: BuildCtx):
        self.cfg = cfg
        self.inputs = inputs
        self.ctx = ctx
        self.outputs: List[TensorBag] = []
        self.params: List[Param] = []
        self.name = "%s%d" % (type(self).__name__, ctx.layer_index)
        self.regularizer = None

    # helpers
    def _out(self, idx, shape, dtype=None) -> TensorBag:
        name = self.cfg.top_names[idx]
        t = TensorBag(name, shape, dtype or self.ctx.act_dtype)
        t.producer = self
        self.outputs.append(t)
        return t

    def _param(self, tag, shape, init, pad_rows=0) -> Param:
        p = self.ctx.arena.add(f"{self.name}.{tag}", shape, init, pad_rows)
        self.params.append(p)
        return p

    def allocate(self):
        for o in self.outputs:
            o.allocate(self.ctx.device, self.ctx.is_train)

    def fprop(self, is_train: bool):
        raise NotImplementedError

    def bprop(self):
        raise NotImplementedError

    # layers that only re-view memory override this to alias instead of allocate
    def post_allocate(self):
        pass


class TorchLayer(Layer):
    """Layer whose math is a pure torch function; backward comes from autograd.

    Keeps API coverage broad (36 layer types) without hand-writing the long tail; none of these are
    on the hot path of the headline models.
    """

    def forward(self, *xs):  # pragma: no cover - abstract
        raise NotImplementedError

    def _weights(self, requires_grad):
        ws = []
        for p in self.params:
            w = p.w.detach()
            if requires_grad:
                w = w.clone().requires_grad_(True) if False else w.requires_grad_(False)
            ws.append(w)
        return ws

    def fprop(self, is_train: bool):
        self.training = is_train
        if is_train:
            xs = []
            for t in self.inputs:
                x = t.data.detach()
                if x.dtype.is_floating_point:
                    x = x.float() if x.dtype != torch.float32 and not x.is_cuda else x
                    x = x.requires_grad_(t.grad is not None)
                xs.append(x)
            self._ws = [p.w.detach().clone().requires_grad_(True) for p in self.params]
            with torch.enable_grad():
                ys = self.forward(*xs)
            if not isinstance(ys, (tuple, list)):
                ys = (ys,)
            self._xs, self._ys = xs, ys
        else:
            self._ws = [p.w for p in self.params]
            with torch.no_grad():
                ys = self.forward(*[t.data for t in self.inputs])
            if not isinstance(ys, (tuple, list)):
                ys = (ys,)
        for o, y in zip(self.outputs, ys):
            o.data.copy_(y.detach().reshape(o.data.shape).to(o.data.dtype))

    def bprop(self):
        outs, gouts = [], []
        for o, y in zip(self.outputs, self._ys):
            if y.requires_grad and o.grad is not None:
                outs.append(y)
                gouts.append(o.grad.reshape(y.shape).to(y.dtype))
        targets = [x for x, t in zip(self._xs, self.inputs)
                   if x.dtype.is_floating_point and x.requires_grad]
        tbags = [t for x, t in zip(self._xs, self.inputs)
                 if x.dtype.is_floating_point and x.requires_grad]
        allt = targets + self._ws
        if not outs or not allt:
            return
        grads = torch.autograd.grad(outs, allt, gouts, allow_unused=True)
        for t, g in zip(tbags, grads[:len(tbags)]):
            if g is None:
                t.grad.zero_()
            else:
                t.grad.copy_(g.reshape(t.grad.shape).to(t.grad.dtype))
        for p, g in zip(self.params, grads[len(tbags):]):
            if g is not None:
                p.g.add_(g.reshape(p.g.shape).to(p.g.dtype))
        self._xs = self._ys = self._ws = None
