"""The remaining dense layer inventory (SURVEY 2.2): shape ops, elementwise, reductions,
normalisation, attention, GRU.  Views are zero-copy where the reference copies; elementwise hot
ones (ReLU/Sigmoid/Concat) call the sm_90a kernels, the rest derive backward from autograd.
File references are given per class.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from ..ops import dense as D
from ..ops import layer_ops as LO
from .base import Layer, TorchLayer, make_init


class NativeTail(TorchLayer):
    """Long-tail layer with hand-written sm_90a forward / backward kernels (csrc/layers.cu).  On CUDA the
    native path runs (no at:: kernels, no autograd tape, graph capturable); on CPU -- and for inputs the
    kernels do not take (non-contiguous, integer) -- the PyTorch formulation of ``TorchLayer`` runs, which
    is also the oracle of the numerics tests."""

    def _native(self) -> bool:
        if not self.ctx.native:
            return False
        ts = [t.data for t in self.inputs] + [o.data for o in self.outputs]
        return LO.ok(*ts)

    def fprop(self, is_train: bool):
        self.training = is_train
        self._ran_native = self._native()
        if self._ran_native:
            self.n_fprop(is_train)
        else:
            super().fprop(is_train)

    def bprop(self):
        if getattr(self, "_ran_native", False):
            self.n_bprop()
        else:
            super().bprop()

    def _f32(self, name, n, fill=0.0):
        """cached fp32 scratch vector"""
        t = getattr(self, name, None)
        if t is None or t.numel() != n:
            t = torch.full((n,), float(fill), dtype=torch.float32, device=self.ctx.device)
            setattr(self, name, t)
        return t


# ------------------------------------------------------------------------- activations
class ReLULayer(Layer):
    """HugeCTR/src/layers/relu_layer.cu:35"""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def fprop(self, is_train):
        D.elementwise(D.EW_RELU, self.inputs[0].data, None, self.outputs[0].data)

    def bprop(self):
        if self.inputs[0].grad is not None:
            D.elementwise(D.EW_RELU_BWD, self.outputs[0].grad, self.outputs[0].data,
                          self.inputs[0].grad)


class SigmoidLayer(Layer):
    """HugeCTR/src/layers/sigmoid_layer.cu"""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def fprop(self, is_train):
        D.elementwise(D.EW_SIGMOID, self.inputs[0].data, None, self.outputs[0].data)

    def bprop(self):
        if self.inputs[0].grad is not None:
            D.elementwise(D.EW_SIGMOID_BWD, self.outputs[0].grad, self.outputs[0].data,
                          self.inputs[0].grad)


class ELULayer(NativeTail):
    """HugeCTR/src/layers/elu_layer.cu"""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, x):
        return F.elu(x, alpha=self.cfg.elu_alpha)

    def n_fprop(self, is_train):
        D.elementwise(D.EW_ELU, self.inputs[0].data, None, self.outputs[0].data, alpha=self.cfg.elu_alpha)

    def n_bprop(self):
        if self.inputs[0].grad is not None:
            D.elementwise(D.EW_ELU_BWD, self.outputs[0].grad, self.outputs[0].data, self.inputs[0].grad,
                          alpha=self.cfg.elu_alpha)


class PReLUDiceLayer(NativeTail):
    """HugeCTR/src/layers/prelu_dice_layer.cu:45-86 (batch statistics per feature)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, x):
        x2 = x.reshape(-1, x.shape[-1]).float()
        ex = x2.mean(0, keepdim=True)
        var = (x2 * x2).mean(0, keepdim=True) - ex * ex
        ps = torch.sigmoid((x2 - ex) / torch.sqrt(var + self.cfg.eps))
        y = ps * x2 + (1 - ps) * self.cfg.elu_alpha * x2
        return y.reshape(x.shape).to(x.dtype)

    def n_fprop(self, is_train):
        x = self.inputs[0].data
        n = x.shape[-1]
        rows = x.numel() // n
        st = self._f32("_stats", 2 * n)
        st.zero_()
        self._mean, self._rstd = self._f32("_m", n), self._f32("_r", n)
        LO.colreduce2(x, None, None, None, st[:n], st[n:], 0)
        LO.bn_finalize(st[:n], st[n:], self._mean, self._rstd, None, None, None, rows, self.cfg.eps, 0.0)
        LO.colwise(x, None, self._mean, self._rstd, None, None, self.outputs[0].data, 2, self.cfg.elu_alpha)

    def n_bprop(self):
        if self.inputs[0].grad is None:
            return
        x, dy = self.inputs[0].data, self.outputs[0].grad
        n = x.shape[-1]
        st = self._f32("_stats", 2 * n)
        st.zero_()
        LO.colreduce2(x, dy, self._mean, self._rstd, st[:n], st[n:], 3, self.cfg.elu_alpha)
        LO.colwise(x, dy, self._mean, self._rstd, st[:n], st[n:], self.inputs[0].grad, 3, self.cfg.elu_alpha)


class DropoutLayer(Layer):
    """HugeCTR/src/layers/dropout_layer.cu:91-104 (inverted dropout, identity in eval)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self.rate = float(cfg.dropout_rate)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def allocate(self):
        super().allocate()
        if self.ctx.is_train:
            self.mask = torch.ones(self.inputs[0].shape, dtype=self.inputs[0].dtype,
                                   device=self.ctx.device)

    def fprop(self, is_train):
        x = self.inputs[0].data
        if is_train and self.rate > 0:
            keep = 1.0 - self.rate
            self.mask.bernoulli_(keep).mul_(1.0 / keep)
            torch.mul(x, self.mask, out=self.outputs[0].data)
        else:
            self.outputs[0].data.copy_(x)

    def bprop(self):
        if self.inputs[0].grad is not None:
            if self.rate > 0:
                torch.mul(self.outputs[0].grad, self.mask, out=self.inputs[0].grad)
            else:
                self.inputs[0].grad.copy_(self.outputs[0].grad)


class CastLayer(Layer):
    """HugeCTR/src/layers/cast_layer.cu:26-40 (fp32 <-> compute dtype)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        src = inputs[0].dtype
        dst = ctx.act_dtype if src == torch.float32 else torch.float32
        self._out(0, inputs[0].shape, dst)

    def fprop(self, is_train):
        self.outputs[0].data.copy_(self.inputs[0].data)

    def bprop(self):
        if self.inputs[0].grad is not None:
            self.inputs[0].grad.copy_(self.outputs[0].grad)


# ------------------------------------------------------------------------- shape ops
class ReshapeLayer(Layer):
    """reshape_layer.cu / reshape_layer_v2.cu: leading_dim, (time_step, leading_dim), selected
    slots, or explicit ``shape``.  Zero-copy view unless slots are selected."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        x = inputs[0]
        n = math.prod(x.shape)
        self.sel = list(cfg.selected_slots) if cfg.selected else None
        if cfg.shape:
            shp = list(cfg.shape)
            if -1 in shp:
                known = -math.prod(shp)
                shp[shp.index(-1)] = n // known
            out = tuple(shp)
        elif self.sel is not None:
            assert len(x.shape) == 3
            out = (x.shape[0], len(self.sel) * x.shape[2])
        elif cfg.time_step > 0:
            out = (n // (cfg.time_step * cfg.leading_dim), cfg.time_step, cfg.leading_dim)
        else:
            ld = cfg.leading_dim if cfg.leading_dim > 0 else math.prod(x.shape[1:])
            out = (n // ld, ld)
        assert math.prod(out) == (n if self.sel is None else out[0] * out[1]), "Reshape size mismatch"
        self._out(0, out, x.dtype)

    def allocate(self):
        if self.sel is not None:
            return super().allocate()
        o, x = self.outputs[0], self.inputs[0]
        o.data = x.data.view(o.shape)
        if self.ctx.is_train:
            o.grad = x.grad.view(o.shape) if x.grad is not None else None
            if o.grad is None and o.dtype.is_floating_point and x.needs_grad is False:
                o.needs_grad = False

    def fprop(self, is_train):
        if self.sel is not None:
            x = self.inputs[0].data
            self.outputs[0].data.copy_(x[:, self.sel, :].reshape(self.outputs[0].shape))

    def bprop(self):
        if self.sel is not None and self.inputs[0].grad is not None:
            g = self.inputs[0].grad
            g.zero_()
            g[:, self.sel, :] = self.outputs[0].grad.view(g.shape[0], len(self.sel), g.shape[2])


class ConcatLayer(Layer):
    """concat_layer.cu / concat_3d_layer.cu: concatenate along ``axis`` (default 1)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        ax = cfg.axis if cfg.axis >= 0 else len(inputs[0].shape) + cfg.axis
        self.axis = ax
        shp = list(inputs[0].shape)
        shp[ax] = sum(t.shape[ax] for t in inputs)
        for t in inputs:
            assert len(t.shape) == len(shp), "Concat rank mismatch"
        self._out(0, shp, inputs[0].dtype)

    def _views(self, which):
        big = getattr(self.outputs[0], which)
        outer = math.prod(self.outputs[0].shape[:self.axis])
        big2 = big.reshape(outer, -1)
        off = 0
        res = []
        for t in self.inputs:
            w = math.prod(t.shape[self.axis:])
            res.append((t, big2[:, off:off + w], outer, w))
            off += w
        return res

    def allocate(self):
        """Default (HCTR_CONCAT_ALIAS=0 disables): when exactly one input is a batch-major embedding
        collection top, the output buffer is carved from the collection's slabs and that top is
        produced (and its gradient consumed) in place -- no strided copy in either direction."""
        import os
        self._aliased = None
        o = self.outputs[0]
        if os.environ.get("HCTR_CONCAT_ALIAS", "1") == "1" and self.axis == 1 and len(o.shape) == 2:
            cands = [i for i, t in enumerate(self.inputs)
                     if getattr(t, "ebc", None) is not None and len(t.shape) == 2 and t.dtype == o.dtype]
            if len(cands) == 1:
                i = cands[0]
                t = self.inputs[i]
                col = sum(x.shape[1] for x in self.inputs[:i])
                res = t.ebc.alias_top(t.ebc_top, o.shape[1], col)
                if res is not None:
                    o.data = res[0]
                    if self.ctx.is_train:
                        o.grad = res[1]
                    t.data = t.ebc.top_data[t.ebc_top]
                    t.grad = t.ebc.top_grad[t.ebc_top] if self.ctx.is_train else None
                    self._aliased = i
        super().allocate()

    def fprop(self, is_train):
        for i, (t, dst, outer, w) in enumerate(self._views("data")):
            if i != getattr(self, "_aliased", None):
                D.copy2d(t.data.reshape(outer, w), dst)

    def bprop(self):
        for i, (t, src, outer, w) in enumerate(self._views("grad")):
            if t.grad is not None and i != getattr(self, "_aliased", None):
                D.copy2d(src, t.grad.reshape(outer, w))


class SliceLayer(Layer):
    """slice_layer.cu: multiple [start,end) column ranges; also the fan-out copy layer inserted by
    the graph builder (model_compile.cpp:624-684).  Backward sums overlapping ranges."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        x = inputs[0]
        self.ranges = [tuple(r) for r in cfg.ranges]
        assert len(self.ranges) == len(cfg.top_names), "Slice: one range per top"
        for i, (a, b_) in enumerate(self.ranges):
            assert 0 <= a < b_ <= x.shape[-1], "Slice range out of bound"
            self._out(i, tuple(x.shape[:-1]) + (b_ - a,), x.dtype)
        self.full_copy = all(r == (0, x.shape[-1]) for r in self.ranges)

    def allocate(self):
        x = self.inputs[0]
        if self.full_copy:
            # pure fan-out: forward aliases the input, backward accumulates
            for o in self.outputs:
                o.data = x.data
                if self.ctx.is_train and o.dtype.is_floating_point and x.grad is not None:
                    o.grad = torch.zeros(o.shape, dtype=o.dtype, device=self.ctx.device)
                elif x.grad is None:
                    o.needs_grad = False
        else:
            super().allocate()

    def fprop(self, is_train):
        if self.full_copy:
            return
        x2 = self.inputs[0].view2d()
        for o, (a, b_) in zip(self.outputs, self.ranges):
            D.copy2d(x2[:, a:b_], o.view2d())

    def bprop(self):
        g = self.inputs[0].grad
        if g is None:
            return
        g2 = g.reshape(g.shape[0], -1) if g.dim() != 2 else g
        if self.full_copy:
            first = True
            for o in self.outputs:
                if o.grad is None:
                    continue
                if first:
                    g.copy_(o.grad)
                    first = False
                else:
                    g.add_(o.grad)
            if first:
                g.zero_()
            return
        g.zero_()
        for o, (a, b_) in zip(self.outputs, self.ranges):
            if o.grad is not None:
                D.copy2d(o.view2d("grad"), g2[:, a:b_], accumulate=True)


class SelectLayer(NativeTail):
    """select_layer.cu: index_select on ``dim``."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        shp = list(inputs[0].shape)
        shp[cfg.dim] = len(cfg.index)
        self._out(0, shp, inputs[0].dtype)

    def forward(self, x):
        idx = torch.tensor(self.cfg.index, device=x.device, dtype=torch.long)
        return torch.index_select(x, self.cfg.dim, idx)

    def _geom(self):
        shp = self.inputs[0].shape
        dim = self.cfg.dim if self.cfg.dim >= 0 else len(shp) + self.cfg.dim
        return math.prod(shp[:dim]), shp[dim], math.prod(shp[dim + 1:])

    def n_fprop(self, is_train):
        outer, R, inner = self._geom()
        K = len(self.cfg.index)
        x, y = self.inputs[0].data, self.outputs[0].data
        for k, j in enumerate(self.cfg.index):        # one strided block copy per selected index
            LO.copy4d(x, y, [outer, inner], [R * inner, 1], [K * inner, 1], src_off=j * inner, dst_off=k * inner)

    def n_bprop(self):
        g = self.inputs[0].grad
        if g is None:
            return
        outer, R, inner = self._geom()
        K = len(self.cfg.index)
        g.zero_()
        for k, j in enumerate(self.cfg.index):
            LO.copy4d(self.outputs[0].grad, g, [outer, inner], [K * inner, 1], [R * inner, 1], accumulate=True,
                      src_off=k * inner, dst_off=j * inner)


class GatherLayer(NativeTail):
    """gather_layer.cu: gathers rows ``indices`` -> (num_indices, num_elems)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        x = inputs[0]
        self._out(0, (len(cfg.indices),) + tuple(x.shape[1:]), x.dtype)

    def forward(self, x):
        idx = torch.tensor(self.cfg.indices, device=x.device, dtype=torch.long)
        return torch.index_select(x, 0, idx)

    def n_fprop(self, is_train):
        x, y = self.inputs[0].data, self.outputs[0].data
        inner = math.prod(x.shape[1:])
        for k, j in enumerate(self.cfg.indices):
            LO.copy4d(x, y, [inner], [1], [1], src_off=j * inner, dst_off=k * inner)

    def n_bprop(self):
        g = self.inputs[0].grad
        if g is None:
            return
        inner = math.prod(g.shape[1:])
        g.zero_()
        for k, j in enumerate(self.cfg.indices):
            LO.copy4d(self.outputs[0].grad, g, [inner], [1], [1], accumulate=True, src_off=k * inner,
                      dst_off=j * inner)


class ScaleLayer(NativeTail):
    """scale_layer.cu:32-78: axis 0 repeats every element ``factor`` times along the row, axis 1
    repeats every row ``factor`` times."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        b, n = inputs[0].shape
        f = int(cfg.factor)
        self._out(0, (b, n * f) if cfg.axis == 0 else (b * f, n), inputs[0].dtype)

    def forward(self, x):
        f = int(self.cfg.factor)
        return x.repeat_interleave(f, dim=1) if self.cfg.axis == 0 else x.repeat_interleave(f, dim=0)

    def n_fprop(self, is_train):
        x, y = self.inputs[0].data, self.outputs[0].data
        b, n = x.shape
        f = int(self.cfg.factor)
        if self.cfg.axis == 0:      # y[b, j * f + r] = x[b, j]
            LO.copy4d(x, y, [b, n, f], [n, 1, 0], [n * f, f, 1])
        else:                       # y[b * f + r, j] = x[b, j]
            LO.copy4d(x, y, [b, f, n], [n, 0, 1], [f * n, n, 1])

    def n_bprop(self):
        g = self.inputs[0].grad
        if g is None:
            return
        b, n = g.shape
        f = int(self.cfg.factor)
        if self.cfg.axis == 0:
            LO.reduce_mid(self.outputs[0].grad, g, b * n, f, 1, 1.0, False)
        else:
            LO.reduce_mid(self.outputs[0].grad, g, b, f, n, 1.0, False)


class FusedReshapeConcatLayer(NativeTail):
    """fused_reshape_concat_layer.cu: inputs [b, F+1, e_i] -> item_his [b*F, sum e], item [b, sum e]."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        b, f1 = inputs[0].shape[0], inputs[0].shape[1]
        e = sum(t.shape[2] for t in inputs)
        self._out(0, (b * (f1 - 1), e), inputs[0].dtype)
        self._out(1, (b, e), inputs[0].dtype)

    def forward(self, *xs):
        x = torch.cat(xs, dim=2)
        b, f1, e = x.shape
        return x[:, :f1 - 1, :].reshape(b * (f1 - 1), e), x[:, f1 - 1, :]

    def _walk(self, fn):
        b, f1 = self.inputs[0].shape[0], self.inputs[0].shape[1]
        E = sum(t.shape[2] for t in self.inputs)
        col = 0
        for t in self.inputs:
            e = t.shape[2]
            fn(t, b, f1, e, E, col)
            col += e

    def n_fprop(self, is_train):
        his, item = self.outputs[0].data, self.outputs[1].data

        def go(t, b, f1, e, E, col):
            LO.copy4d(t.data, his, [b, f1 - 1, e], [f1 * e, e, 1], [(f1 - 1) * E, E, 1], dst_off=col)
            LO.copy4d(t.data, item, [b, e], [f1 * e, 1], [E, 1], src_off=(f1 - 1) * e, dst_off=col)
        self._walk(go)

    def n_bprop(self):
        ghis, gitem = self.outputs[0].grad, self.outputs[1].grad

        def go(t, b, f1, e, E, col):
            if t.grad is None:
                return
            if ghis is not None:
                LO.copy4d(ghis, t.grad, [b, f1 - 1, e], [(f1 - 1) * E, E, 1], [f1 * e, e, 1], src_off=col)
            else:
                t.grad.zero_()
            if gitem is not None:
                LO.copy4d(gitem, t.grad, [b, e], [E, 1], [f1 * e, 1], src_off=col, dst_off=(f1 - 1) * e)
            else:
                t.grad.view(b, f1, e)[:, f1 - 1, :].zero_()
        self._walk(go)


class FusedReshapeConcatGeneralLayer(NativeTail):
    """fused_reshape_concat_general_layer.cu: inputs [b, F, e_i] -> [b*F, sum e]."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        b, f = inputs[0].shape[0], inputs[0].shape[1]
        self._out(0, (b * f, sum(t.shape[2] for t in inputs)), inputs[0].dtype)

    def forward(self, *xs):
        x = torch.cat(xs, dim=2)
        return x.reshape(-1, x.shape[2])

    def n_fprop(self, is_train):
        E = sum(t.shape[2] for t in self.inputs)
        col = 0
        for t in self.inputs:
            b, f, e = t.shape
            LO.copy4d(t.data, self.outputs[0].data, [b * f, e], [e, 1], [E, 1], dst_off=col)
            col += e

    def n_bprop(self):
        E = sum(t.shape[2] for t in self.inputs)
        col = 0
        for t in self.inputs:
            b, f, e = t.shape
            if t.grad is not None:
                LO.copy4d(self.outputs[0].grad, t.grad, [b * f, e], [E, 1], [e, 1], src_off=col)
            col += e


# ------------------------------------------------------------------------- arithmetic / reductions
class AddLayer(NativeTail):
    """add_layer.cu:28-77 (N inputs)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, *xs):
        y = xs[0]
        for x in xs[1:]:
            y = y + x
        return y

    def n_fprop(self, is_train):
        o = self.outputs[0].data
        xs = [t.data for t in self.inputs]
        if len(xs) == 1:
            D.elementwise(D.EW_COPY, xs[0], None, o)
            return
        D.elementwise(D.EW_ADD, xs[0], xs[1], o)
        for x in xs[2:]:
            D.elementwise(D.EW_ADD_INPLACE, x, None, o)

    def n_bprop(self):
        for t in self.inputs:
            if t.grad is not None:
                D.elementwise(D.EW_COPY, self.outputs[0].grad, None, t.grad)


class SubLayer(NativeTail):
    """sub_layer.cu"""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, x, y):
        return x - y

    def n_fprop(self, is_train):
        D.elementwise(D.EW_SUB, self.inputs[0].data, self.inputs[1].data, self.outputs[0].data)

    def n_bprop(self):
        dy = self.outputs[0].grad
        if self.inputs[0].grad is not None:
            D.elementwise(D.EW_COPY, dy, None, self.inputs[0].grad)
        if self.inputs[1].grad is not None:
            D.elementwise(D.EW_SCALE, dy, None, self.inputs[1].grad, alpha=-1.0)


class ElementwiseMultiplyLayer(NativeTail):
    """elementwise_multiply_layer.cu (N inputs)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, *xs):
        y = xs[0]
        for x in xs[1:]:
            y = y * x
        return y

    def n_fprop(self, is_train):
        o = self.outputs[0].data
        xs = [t.data for t in self.inputs]
        if len(xs) == 1:
            D.elementwise(D.EW_COPY, xs[0], None, o)
            return
        D.elementwise(D.EW_MUL, xs[0], xs[1], o)
        for x in xs[2:]:
            D.elementwise(D.EW_MUL, o, x, o)

    def n_bprop(self):
        dy = self.outputs[0].grad
        xs = [t.data for t in self.inputs]
        for i, t in enumerate(self.inputs):
            if t.grad is None:
                continue
            others = [x for j, x in enumerate(xs) if j != i]
            if not others:
                D.elementwise(D.EW_COPY, dy, None, t.grad)
                continue
            D.elementwise(D.EW_MUL, dy, others[0], t.grad)
            for x in others[1:]:
                D.elementwise(D.EW_MUL, t.grad, x, t.grad)


class WeightMultiplyLayer(NativeTail):
    """weight_multiply_layer.cu:32-82: out[b, s*v + j] = in[b, s] * W[s, j]."""
    trainable = True

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        b, s = inputs[0].shape
        ws, wv = cfg.weight_dims
        assert ws == s, "WeightMultiply: weight_dims[0] must equal the slot dim"
        self._param("W", (ws, wv), make_init(cfg.weight_init_type, ws, wv, "xavier"))
        self._out(0, (b, ws * wv), inputs[0].dtype)

    def forward(self, x):
        w = self._ws[0].to(x.dtype)
        return (x.unsqueeze(2) * w.unsqueeze(0)).reshape(x.shape[0], -1)

    def n_fprop(self, is_train):
        b, S = self.inputs[0].shape
        V = self.cfg.weight_dims[1]
        LO.weight_mul_fwd(self.inputs[0].data, self.params[0].w, self.outputs[0].data, b, S, V)

    def n_bprop(self):
        b, S = self.inputs[0].shape
        V = self.cfg.weight_dims[1]
        LO.weight_mul_bwd(self.outputs[0].grad, self.inputs[0].data, self.params[0].w, self.inputs[0].grad,
                          self.params[0].g, b, S, V)


class FmOrder2Layer(NativeTail):
    """fm_order2_layer.cu:24-91: 0.5 * ((sum_s v)^2 - sum_s v^2) per embedding element."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        b, n = inputs[0].shape
        assert cfg.out_dim > 0 and n % cfg.out_dim == 0
        self._out(0, (b, cfg.out_dim), inputs[0].dtype)

    def forward(self, x):
        v = x.reshape(x.shape[0], -1, self.cfg.out_dim).float()
        s = v.sum(1)
        return (0.5 * (s * s - (v * v).sum(1))).to(x.dtype)

    def n_fprop(self, is_train):
        b, n = self.inputs[0].shape
        Dm = self.cfg.out_dim
        LO.fm_order2(self.inputs[0].data, None, self.outputs[0].data, b, n // Dm, Dm, False)

    def n_bprop(self):
        if self.inputs[0].grad is None:
            return
        b, n = self.inputs[0].shape
        Dm = self.cfg.out_dim
        LO.fm_order2(self.inputs[0].data, self.outputs[0].grad, self.inputs[0].grad, b, n // Dm, Dm, True)


class ReduceSumLayer(NativeTail):
    """reduce_sum_layer.cu: keepdim sum over ``axis``."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        shp = list(inputs[0].shape)
        shp[cfg.axis] = 1
        self._out(0, shp, inputs[0].dtype)

    def forward(self, x):
        return x.float().sum(self.cfg.axis, keepdim=True).to(x.dtype)

    _mean = False

    def _geom(self):
        shp = self.inputs[0].shape
        ax = self.cfg.axis if self.cfg.axis >= 0 else len(shp) + self.cfg.axis
        return math.prod(shp[:ax]), shp[ax], math.prod(shp[ax + 1:])

    def n_fprop(self, is_train):
        outer, R, inner = self._geom()
        LO.reduce_mid(self.inputs[0].data, self.outputs[0].data, outer, R, inner, (1.0 / R) if self._mean else 1.0,
                      False)

    def n_bprop(self):
        if self.inputs[0].grad is None:
            return
        outer, R, inner = self._geom()
        LO.reduce_mid(self.outputs[0].grad, self.inputs[0].grad, outer, R, inner,
                      (1.0 / R) if self._mean else 1.0, True)


class ReduceMeanLayer(NativeTail):
    """reduce_mean_layer.cu"""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        shp = list(inputs[0].shape)
        shp[cfg.axis] = 1
        self._out(0, shp, inputs[0].dtype)

    def forward(self, x):
        return x.float().mean(self.cfg.axis, keepdim=True).to(x.dtype)

    _mean = True
    _geom = ReduceSumLayer._geom
    n_fprop = ReduceSumLayer.n_fprop
    n_bprop = ReduceSumLayer.n_bprop


class MatrixMultiplyLayer(NativeTail):
    """matrix_multiply_layer.cu:135-180: 2Dx2D, 3Dx3D (batched), 2Dx3D -> 3D."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        a, b_ = inputs[0].shape, inputs[1].shape
        if len(a) == 2 and len(b_) == 2:
            out = (a[0], b_[1])
        elif len(a) == 3 and len(b_) == 3:
            out = (a[0], a[1], b_[2])
        elif len(a) == 2 and len(b_) == 3:
            out = (a[0], b_[1], b_[2])
        else:
            raise ValueError("MatrixMultiply: unsupported ranks")
        self._out(0, out, inputs[0].dtype)

    def forward(self, a, b_):
        if a.dim() == 2 and b_.dim() == 3:
            return (a @ b_.reshape(b_.shape[0], -1)).reshape(a.shape[0], b_.shape[1], b_.shape[2])
        return torch.matmul(a, b_)

    def _geom(self):
        a, b_ = self.inputs[0].shape, self.inputs[1].shape
        if len(a) == 3:                       # batched [Z, M, K] x [Z, K, N]
            Z, M, K, N = a[0], a[1], a[2], b_[2]
            return Z, M, N, K, (M * K, 0, K, 1), (K * N, 0, N, 1), (M * N, 0, N, 1)
        M, K = a
        N = math.prod(b_[1:])                 # 2D x 2D, or 2D x 3D with the trailing dims flattened
        return 1, M, N, K, (0, 0, K, 1), (0, 0, N, 1), (0, 0, N, 1)

    def n_fprop(self, is_train):
        Z, M, N, K, sa, sb, sc = self._geom()
        LO.bmm(self.inputs[0].data, self.inputs[1].data, self.outputs[0].data, M, N, K, Z, 1, sa, sb, sc)

    def n_bprop(self):
        Z, M, N, K, sa, sb, sc = self._geom()
        dy = self.outputs[0].grad
        A, B = self.inputs
        if A.grad is not None:     # dA[m, k] = sum_n dY[m, n] B[k, n]
            LO.bmm(dy, B.data, A.grad, M, K, N, Z, 1, sc, (sb[0], 0, sb[3], sb[2]), sa)
        if B.grad is not None:     # dB[k, n] = sum_m A[m, k] dY[m, n]
            LO.bmm(A.data, dy, B.grad, K, N, M, Z, 1, (sa[0], 0, sa[3], sa[2]), sc, sb)


# ------------------------------------------------------------------------- softmax / attention
class SoftmaxLayer(NativeTail):
    """softmax_layer.cu:53-173 / masked_softmax_layer.cu:33-140 (mask==0 -> -10000 before softmax)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, x, mask=None):
        v = x.float()
        if mask is not None:
            v = v * getattr(self.cfg, "factor", 1.0) if False else v
            v = torch.where(mask.float() > 0, v, torch.full_like(v, -10000.0))
        return torch.softmax(v, dim=-1).to(x.dtype)

    def _mask(self):
        if len(self.inputs) < 2:
            return None
        m = self.inputs[1].data
        return m if m.numel() == self.inputs[0].data.numel() else m.expand_as(self.inputs[0].data).contiguous()

    def n_fprop(self, is_train):
        self._m = self._mask()
        LO.softmax_fwd(self.inputs[0].data, self._m, self.outputs[0].data)

    def n_bprop(self):
        if self.inputs[0].grad is not None:
            LO.softmax_bwd(self.outputs[0].grad, self.outputs[0].data, self._m, self.inputs[0].grad)


class SequenceMaskLayer(Layer):
    """sequence_mask_layer.cu:28-76: (len_from[b], len_to[b]) -> [b,1,Lf,Lt] 0/1 mask."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        b = inputs[0].shape[0]
        self.lf, self.lt = int(cfg.max_sequence_len_from), int(cfg.max_sequence_len_to)
        o = self._out(0, (b, 1, self.lf, self.lt), ctx.act_dtype)
        o.needs_grad = False

    def fprop(self, is_train):
        lf = self.inputs[0].data.reshape(-1)[:self.outputs[0].shape[0]].float()
        lt = self.inputs[1].data.reshape(-1)[:self.outputs[0].shape[0]].float()
        dev = lf.device
        mf = torch.arange(self.lf, device=dev).view(1, -1, 1) < lf.view(-1, 1, 1)
        mt = torch.arange(self.lt, device=dev).view(1, 1, -1) < lt.view(-1, 1, 1)
        self.outputs[0].data.copy_((mf & mt).unsqueeze(1).to(self.outputs[0].dtype))

    def bprop(self):
        pass


class MultiHeadAttentionLayer(NativeTail):
    """multi_head_attention_layer.cu:33-519: O = softmax(QK^T/sqrt(dh) masked) V, heads split on
    the hidden dim.  Projections are separate FC layers in the reference."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        q = inputs[0]
        self.h = int(cfg.num_attention_heads)
        assert q.shape[-1] % self.h == 0
        self._out(0, q.shape, q.dtype)

    def forward(self, q, k, v, mask=None):
        b, sf, hd = q.shape
        st = k.shape[1]
        dh = hd // self.h
        qh = q.reshape(b, sf, self.h, dh).transpose(1, 2).float()
        kh = k.reshape(b, st, self.h, dh).transpose(1, 2).float()
        vh = v.reshape(b, st, self.h, dh).transpose(1, 2).float()
        s = torch.matmul(qh, kh.transpose(-1, -2)) / math.sqrt(dh)
        if mask is not None:
            s = torch.where(mask.float() > 0, s, torch.full_like(s, -10000.0))
        p = torch.softmax(s, dim=-1)
        o = torch.matmul(p, vh).transpose(1, 2).reshape(b, sf, hd)
        return o.to(q.dtype)

    # Native path: the reference's structure (2 strided-batched GEMMs forward, 4 backward,
    # multi_head_attention_layer.cu:324-481) without its transposes -- heads are addressed by strides.
    def _geom(self):
        b, sf, hd = self.inputs[0].shape
        st = self.inputs[1].shape[1]
        dh = hd // self.h
        qs = (sf * hd, dh, hd, 1)             # [b, h](row = position, col = feature)
        ks = (st * hd, dh, hd, 1)
        ps = (self.h * sf * st, sf * st, st, 1)
        return b, sf, st, hd, dh, qs, ks, ps

    def n_fprop(self, is_train):
        b, sf, st, hd, dh, qs, ks, ps = self._geom()
        q, k, v = (t.data for t in self.inputs[:3])
        dev, dt = q.device, q.dtype
        if getattr(self, "_p", None) is None or self._p.shape != (b, self.h, sf, st):
            self._s = torch.empty(b, self.h, sf, st, dtype=dt, device=dev)
            self._p = torch.empty_like(self._s)
        # S = Q K^T / sqrt(dh): B operand = K read as (k = feature, n = position)
        LO.bmm(q, k, self._s, sf, st, dh, b, self.h, qs, (ks[0], ks[1], 1, hd), ps, alpha=1.0 / math.sqrt(dh))
        m = None
        if len(self.inputs) > 3:
            m = self.inputs[3].data
            m = m.expand(b, self.h, sf, st).contiguous() if m.numel() != self._s.numel() else m
        self._m = m
        LO.softmax_fwd(self._s, m, self._p)
        LO.bmm(self._p, v, self.outputs[0].data, sf, dh, st, b, self.h, ps, ks, qs)

    def n_bprop(self):
        b, sf, st, hd, dh, qs, ks, ps = self._geom()
        q, k, v = self.inputs[:3]
        do = self.outputs[0].grad
        ds = self._s                            # reuse: dP then dS
        # dP = dO V^T
        LO.bmm(do, v.data, ds, sf, st, dh, b, self.h, qs, (ks[0], ks[1], 1, hd), ps)
        if v.grad is not None:                  # dV = P^T dO
            LO.bmm(self._p, do, v.grad, st, dh, sf, b, self.h, (ps[0], ps[1], 1, st), qs, ks)
        LO.softmax_bwd(ds, self._p, self._m, ds)
        sc = 1.0 / math.sqrt(dh)
        if q.grad is not None:                  # dQ = dS K / sqrt(dh)
            LO.bmm(ds, k.data, q.grad, sf, dh, st, b, self.h, ps, ks, qs, alpha=sc)
        if k.grad is not None:                  # dK = dS^T Q / sqrt(dh)
            LO.bmm(ds, q.data, k.grad, st, dh, sf, b, self.h, (ps[0], ps[1], 1, st), qs, ks, alpha=sc)


# ------------------------------------------------------------------------- normalisation / recurrent
class BatchNormLayer(NativeTail):
    """batch_norm_layer.cu:155-185 (cuDNN in the reference): gamma, beta trainable; running
    mean/var are non-trainable parameters saved to <dense>.ntp.json."""
    trainable = True

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        n = inputs[0].shape[-1]
        self._param("gamma", (1, n), make_init(cfg.gamma_init_type, n, n, "one"))
        self._param("beta", (1, n), make_init(cfg.beta_init_type, n, n, "zero"))
        self.momentum = float(cfg.factor)
        self.eps = float(cfg.eps)
        self._out(0, inputs[0].shape, inputs[0].dtype)
        key = "_bn_state_%s" % self.name
        st = getattr(ctx.arena, key, None)
        if st is None:
            st = {"mean": torch.zeros(n), "var": torch.ones(n)}
            setattr(ctx.arena, key, st)
        self.state = st

    def allocate(self):
        super().allocate()
        for k in ("mean", "var"):
            self.state[k] = self.state[k].to(self.ctx.device)

    def forward(self, x):
        g, b_ = self._ws[0].reshape(-1), self._ws[1].reshape(-1)
        xf = x.reshape(-1, x.shape[-1]).float()
        if self.training:
            mean = xf.mean(0)
            var = xf.var(0, unbiased=False)
            with torch.no_grad():
                m = self.momentum
                self.state["mean"].mul_(m).add_((1 - m) * mean.detach())
                self.state["var"].mul_(m).add_((1 - m) * var.detach())
        else:
            mean, var = self.state["mean"], self.state["var"]
        y = (xf - mean) / torch.sqrt(var + self.eps) * g + b_
        return y.reshape(x.shape).to(x.dtype)

    def n_fprop(self, is_train):
        x = self.inputs[0].data
        n = x.shape[-1]
        rows = x.numel() // n
        g, b_ = self.params[0].w.reshape(-1), self.params[1].w.reshape(-1)
        self._mean, self._rstd = self._f32("_m", n), self._f32("_r", n)
        if is_train:
            st = self._f32("_stats", 2 * n)
            st.zero_()
            LO.colreduce2(x, None, None, None, st[:n], st[n:], 0)
            LO.bn_finalize(st[:n], st[n:], self._mean, self._rstd, None, self.state["mean"], self.state["var"],
                           rows, self.eps, self.momentum)
        else:   # running statistics: mean as is, rstd from the running variance (sum = mean*1, sumsq = var + mean^2)
            st = self._f32("_stats", 2 * n)
            st[:n].copy_(self.state["mean"])
            st[n:].copy_(self.state["var"] + self.state["mean"] * self.state["mean"])
            LO.bn_finalize(st[:n], st[n:], self._mean, self._rstd, None, None, None, 1, self.eps, 0.0)
        LO.colwise(x, None, self._mean, self._rstd, g, b_, self.outputs[0].data, 0)

    def n_bprop(self):
        x, dy = self.inputs[0].data, self.outputs[0].grad
        n = x.shape[-1]
        st = self._f32("_stats", 2 * n)
        st.zero_()
        LO.colreduce2(x, dy, self._mean, self._rstd, st[:n], st[n:], 1)       # dbeta, dgamma
        if self.inputs[0].grad is not None:
            LO.bn_bwd_dx(x, dy, self._mean, self._rstd, self.params[0].w.reshape(-1), st[:n], st[n:],
                         self.inputs[0].grad)
        D.elementwise(D.EW_ADD_INPLACE, st[n:], None, self.params[0].g.reshape(-1))
        D.elementwise(D.EW_ADD_INPLACE, st[:n], None, self.params[1].g.reshape(-1))


class LayerNormLayer(NativeTail):
    """layer_norm_layer.cu:43-239"""
    trainable = True

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        n = inputs[0].shape[-1]
        self._param("gamma", (1, n), make_init(cfg.gamma_init_type, n, n, "one"))
        self._param("beta", (1, n), make_init(cfg.beta_init_type, n, n, "zero"))
        self._out(0, inputs[0].shape, inputs[0].dtype)

    def forward(self, x):
        n = x.shape[-1]
        return F.layer_norm(x.float(), (n,), self._ws[0].reshape(-1), self._ws[1].reshape(-1),
                            self.cfg.eps).to(x.dtype)

    def n_fprop(self, is_train):
        x = self.inputs[0].data
        rows = x.numel() // x.shape[-1]
        self._mean, self._rstd = self._f32("_m", rows), self._f32("_r", rows)
        LO.layernorm_fwd(x, self.params[0].w.reshape(-1), self.params[1].w.reshape(-1), self.outputs[0].data,
                         self._mean, self._rstd, self.cfg.eps)

    def n_bprop(self):
        LO.layernorm_bwd(self.outputs[0].grad, self.inputs[0].data, self.params[0].w.reshape(-1), self._mean,
                         self._rstd, self.inputs[0].grad, self.params[0].g.reshape(-1),
                         self.params[1].g.reshape(-1))


class GRULayer(NativeTail):
    """gru_layer.cu:265 (cuDNN GRU in the reference): input (1, b*S*v) -> output (1, b*S*h)."""
    trainable = True

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        self.b, self.S, self.v, self.hid = cfg.batchsize, cfg.SeqLength, cfg.vector_size, cfg.num_output
        h, v = self.hid, self.v
        self._param("W_ih", (3 * h, v), make_init(cfg.weight_init_type, v, h, "xavier"))
        self._param("W_hh", (3 * h, h), make_init(cfg.weight_init_type, h, h, "xavier"))
        self._param("b_ih", (1, 3 * h), make_init(cfg.bias_init_type, h, h, "zero"))
        self._param("b_hh", (1, 3 * h), make_init(cfg.bias_init_type, h, h, "zero"))
        self._out(0, (1, self.b * self.S * h), inputs[0].dtype)

    def forward(self, x):
        wih, whh, bih, bhh = self._ws
        xs = x.reshape(self.b, self.S, self.v).float()
        h = torch.zeros(self.b, self.hid, device=x.device)
        outs = []
        for t in range(self.S):
            gi = xs[:, t] @ wih.t() + bih.reshape(-1)
            gh = h @ whh.t() + bhh.reshape(-1)
            ir, iz, inn = gi.chunk(3, 1)
            hr, hz, hn = gh.chunk(3, 1)
            r = torch.sigmoid(ir + hr)
            z = torch.sigmoid(iz + hz)
            n = torch.tanh(inn + r * hn)
            h = (1 - z) * n + z * h
            outs.append(h)
        return torch.stack(outs, 1).reshape(1, -1).to(x.dtype)

    # Native path (the reference calls cuDNN): input projections of all steps in ONE matmul, then per step a
    # recurrent matmul + fused gate kernel; backward through time with the mirrored kernels.  fp32 state.
    def _native(self):
        return super()._native() and self.inputs[0].data.dtype == torch.float32

    def n_fprop(self, is_train):
        b, S, v, h = self.b, self.S, self.v, self.hid
        dev = self.ctx.device
        wih, whh, bih, bhh = (p.w for p in self.params)
        x = self.inputs[0].data.reshape(b * S, v)
        f32 = dict(dtype=torch.float32, device=dev)
        if getattr(self, "_gi", None) is None:
            self._gi = torch.empty(b * S, 3 * h, **f32)          # x W_ih^T + b_ih for every step
            self._gh = torch.empty(S, b, 3 * h, **f32)
            self._save = torch.empty(S, b, 3 * h, **f32)
            self._hs = torch.zeros(S + 1, b, h, **f32)           # h_0 = 0
        gi3 = self._gi.view(b, S, 3 * h)
        # gi[b*S, 3h] = x[b*S, v] . W_ih[3h, v]^T  (+ bias broadcast: accumulate on a bias-filled buffer)
        LO.copy4d(bih.reshape(-1), self._gi, [b * S, 3 * h], [0, 1], [3 * h, 1])
        LO.bmm(x, wih, self._gi, b * S, 3 * h, v, 1, 1, (0, 0, v, 1), (0, 0, 1, v), (0, 0, 3 * h, 1),
               accumulate=True)
        out = self.outputs[0].data.view(b, S, h)
        for t in range(S):
            LO.copy4d(bhh.reshape(-1), self._gh[t], [b, 3 * h], [0, 1], [3 * h, 1])
            LO.bmm(self._hs[t], whh, self._gh[t], b, 3 * h, h, 1, 1, (0, 0, h, 1), (0, 0, 1, h), (0, 0, 3 * h, 1),
                   accumulate=True)
            # the step's input projections sit at row stride S in gi: gather them next to gh
            LO.copy4d(self._gi, self._save[t], [b, 3 * h], [S * 3 * h, 1], [3 * h, 1], src_off=t * 3 * h)
            LO.gru_gate_fwd(self._save[t], self._gh[t], self._hs[t], self._hs[t + 1], self._save[t], b, h)
            LO.copy4d(self._hs[t + 1], self.outputs[0].data, [b, h], [h, 1], [S * h, 1], dst_off=t * h)

    def n_bprop(self):
        b, S, v, h = self.b, self.S, self.v, self.hid
        dev = self.ctx.device
        wih, whh, bih, bhh = self.params
        f32 = dict(dtype=torch.float32, device=dev)
        if getattr(self, "_dgi", None) is None:
            self._dgi = torch.empty(b, S, 3 * h, **f32)
            self._dgh = torch.empty(b, 3 * h, **f32)
            self._dgi_t = torch.empty(b, 3 * h, **f32)
            self._dh = torch.empty(b, h, **f32)
            self._dhp = torch.empty(b, h, **f32)
        dy = self.outputs[0].grad
        self._dh.zero_()
        for t in range(S - 1, -1, -1):
            # dh_t = dY[:, t] + carry
            LO.copy4d(dy, self._dh, [b, h], [S * h, 1], [h, 1], accumulate=True, src_off=t * h)
            LO.gru_gate_bwd(self._dh, self._save[t], self._gh[t], self._hs[t], self._dgi_t, self._dgh, self._dhp, b, h)
            LO.copy4d(self._dgi_t, self._dgi, [b, 3 * h], [3 * h, 1], [S * 3 * h, 1], dst_off=t * 3 * h)
            # dW_hh[3h, h] += dgh^T h_{t-1} ; db_hh += colsum(dgh) ; carry = dhprev + dgh W_hh
            LO.bmm(self._dgh, self._hs[t], whh.g, 3 * h, h, b, 1, 1, (0, 0, 1, 3 * h), (0, 0, h, 1), (0, 0, h, 1),
                   accumulate=True)
            D.colsum_accum(self._dgh, bhh.g.reshape(-1))
            LO.bmm(self._dgh, whh.w, self._dhp, b, h, 3 * h, 1, 1, (0, 0, 3 * h, 1), (0, 0, h, 1), (0, 0, h, 1),
                   accumulate=True)
            self._dh, self._dhp = self._dhp, self._dh
        dgi = self._dgi.view(b * S, 3 * h)
        x = self.inputs[0].data.reshape(b * S, v)
        LO.bmm(dgi, x, wih.g, 3 * h, v, b * S, 1, 1, (0, 0, 1, 3 * h), (0, 0, v, 1), (0, 0, v, 1), accumulate=True)
        D.colsum_accum(dgi, bih.g.reshape(-1))
        if self.inputs[0].grad is not None:
            LO.bmm(dgi, wih.w, self.inputs[0].grad, b * S, v, 3 * h, 1, 1, (0, 0, 3 * h, 1), (0, 0, v, 1),
                   (0, 0, v, 1))
