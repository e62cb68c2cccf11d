"""MLP / InnerProduct / FusedInnerProduct on the wgmma GEMM with fused epilogues.

Reference behaviour: HugeCTR/src/layers/mlp_layer.cu:25-298 (N x cuBLASLt matmul with bias+ReLU
epilogue, DRELU_BGRAD dgrad, beta=1 wgrad on an overlap stream, skip_head_dgrad),
HugeCTR/src/layers/fully_connected_layer.cu:87-173 (kernel [in,out] row-major, bias [1,out]).
Weight order inside the flat arena / checkpoint: W0,b0,W1,b1,...
"""
from __future__ import annotations

from typing import List

import torch

from ..core import KernelParams
from ..enums import Activation_t
from ..ops import dense as D
from ..ops import gemm as G
from .base import Layer, make_init


def _ceil8(n):
    return (n + 7) // 8 * 8


class MLPLayer(Layer):
    trainable = True

    def __init__(self, cfg, inputs, ctx, num_outputs=None, activations=None, biases=None,
                 default_init=("mlp", "mlp")):
        super().__init__(cfg, inputs, ctx)
        x = inputs[0]
        self.lead = tuple(x.shape[:-1])
        self.rows = 1
        for d in self.lead:
            self.rows *= d
        self.dims_out = list(num_outputs if num_outputs is not None else cfg.num_outputs)
        n = len(self.dims_out)
        acts = list(activations if activations is not None else cfg.activations)
        if not acts:
            acts = [cfg.act_type] * n
        self.relu = [a == Activation_t.Relu for a in acts]
        bs = list(biases if biases is not None else cfg.biases)
        if not bs:
            bs = [cfg.use_bias] * n
        self.use_bias = bs
        self.async_wgrad = bool(getattr(cfg.compute_config, "async_wgrad", False))
        self.mixed = ctx.mixed
        self.W, self.B = [], []
        k = x.shape[-1]
        self.k_in = k
        self.k_pad = _ceil8(k) if ctx.mixed else k
        kin = k
        for i, nout in enumerate(self.dims_out):
            wi = make_init(cfg.weight_init_type, kin, nout, default_init[0])
            bi = make_init(cfg.bias_init_type, kin, nout, default_init[1])
            pad = (self.k_pad - k) if i == 0 else 0
            self.W.append(self._param(f"W{i}", (kin, nout), wi, pad_rows=pad))
            if bs[i]:
                self.B.append(self._param(f"b{i}", (1, nout), bi))
            else:
                self.B.append(None)
            kin = nout
        self._out(0, self.lead + (self.dims_out[-1],))
        self._side = None
        # Solver.use_fp8_mlp: forward GEMMs in block-scaled fp8 (OCP MX: e4m3 values, one UE8M0 scale per 32
        # K elements, applied per 32-wide K slice of the fp8 wgmma); backward stays bf16 on the
        # bf16 activations.  Layers whose K is not a multiple of 128 (or N == 1) keep the bf16 GEMM.
        self.fp8 = bool(getattr(ctx.solver, "use_fp8_mlp", False)) and ctx.mixed and ctx.native

    # ------------------------------------------------------------------ buffers
    def allocate(self):
        super().allocate()
        dev, dt, b = self.ctx.device, self.ctx.act_dtype, self.rows
        x = self.inputs[0]
        # input staging (cast / pad) only when needed
        self.x_stage = None
        if x.dtype != dt or self.k_pad != self.k_in:
            self.x_stage = torch.zeros(b, self.k_pad, dtype=dt, device=dev)
        self.acts: List[torch.Tensor] = []
        for i, n in enumerate(self.dims_out):
            if i == len(self.dims_out) - 1:
                self.acts.append(self.outputs[0].data.view(b, n))
            else:
                self.acts.append(torch.zeros(b, n, dtype=dt, device=dev))
        if self.ctx.is_train:
            self.dacts = []
            for i, n in enumerate(self.dims_out):
                if i == len(self.dims_out) - 1 and not self.relu[i]:
                    self.dacts.append(None)  # use outputs[0].grad directly
                else:
                    self.dacts.append(torch.zeros(b, n, dtype=dt, device=dev))

    def _x(self):
        x = self.inputs[0].data.reshape(self.rows, self.k_in)
        if self.x_stage is None:
            return x
        if x.dtype == torch.float32 and self.x_stage.dtype == torch.bfloat16:
            D.cast_pad(x, self.x_stage)
        else:
            self.x_stage.zero_()
            self.x_stage[:, :self.k_in].copy_(x.to(self.x_stage.dtype))
        return self.x_stage

    # ------------------------------------------------------------------ forward
    def fprop(self, is_train: bool):
        h = self._x()
        self._x_in = h
        for i, nout in enumerate(self.dims_out):
            W = self.W[i].compute(self.mixed)
            bias = None if self.B[i] is None else self.B[i].w.reshape(-1)
            out = self.acts[i]
            if nout == 1 and W.shape[0] >= 8:
                D.fc1_fwd(h, self.W[i].w.reshape(-1), bias, out, relu=self.relu[i])
            elif self.fp8 and h.shape[1] % 128 == 0 and h.dtype == torch.bfloat16 and out.stride(1) == 1:
                self._fprop_fp8(i, h, W, bias, out)
            else:
                G.gemm_bf16(h, W, out, b_mn=True, bias=bias,
                            flags=G.EPI_RELU if self.relu[i] else 0)
            h = out

    def _fprop_fp8(self, i, h, W, bias, out):
        """out = act(deq(Q(h)) @ deq(Q(W)) + bias): activations and weights are quantised to MX fp8 (the
        weights from their transposed view, so both operands are K-major)"""
        from ..ops import mxfp8 as MX
        K, N = h.shape[1], W.shape[1]
        bufs = getattr(self, "_fp8_bufs", None)
        if bufs is None:
            bufs = self._fp8_bufs = {}
        if i not in bufs:
            bufs[i] = (MX.mx_buffers(h.shape[0], K, h.device), MX.mx_buffers(N, K, h.device))
        (aq, sfa), (bq, sfb) = bufs[i]
        MX.mx_quantize(h, aq, sfa)
        MX.mx_quantize(W[:K], bq, sfb, transposed=True)          # W is [K, N] row-major: quantise W^T
        MX.gemm_mxfp8(aq, sfa, bq, sfb, h.shape[0], N, K, out=out, bias=bias,
                      flags=G.EPI_RELU if self.relu[i] else 0)

    # ------------------------------------------------------------------ backward
    def bprop(self):
        n = len(self.dims_out)
        dy = self.outputs[0].grad.view(self.rows, self.dims_out[-1])
        want_dx = self.inputs[0].grad is not None
        bgrad_done = set()   # layers whose bias gradient came out of the upstream dgrad epilogue
        for i in range(n - 1, -1, -1):
            x_i = self._x_in if i == 0 else self.acts[i - 1]
            if i == n - 1:
                if self.relu[i]:
                    # last-layer dReLU (reference reverse_relu_kernel, fused_fc_layer_functors.cu:79)
                    D.elementwise(D.EW_RELU_BWD, dy, self.acts[i], self.dacts[i])
                    dz = self.dacts[i]
                else:
                    dz = dy
            else:
                dz = self.dacts[i]  # produced (already dReLU-masked) by layer i+1's dgrad epilogue
            W = self.W[i]
            nout = self.dims_out[i]
            need_dx = (i > 0) or want_dx
            if nout == 1 and W.shape[0] >= 8:
                dxo = None
                if need_dx:
                    dxo = self.dacts[i - 1] if i > 0 else self._dx_stage()
                D.fc1_bwd(x_i, W.w.reshape(-1), dz, dxo, W.g.reshape(-1),
                          None if self.B[i] is None else self.B[i].g.reshape(-1),
                          mask_relu=(i > 0 and self.relu[i - 1]))
                continue
            if self.B[i] is not None and i not in bgrad_done:
                D.colsum_accum(dz, self.B[i].g.reshape(-1))
            # wgrad: dW[k, n] += x^T dz   (both operands MN-major, fp32 atomic split-K, beta = 1)
            self._wgrad(x_i, dz, W)
            if need_dx:
                if i > 0:
                    # the dgrad epilogue also accumulates the bias gradient of layer i-1 (column sums
                    # of its dY) when it can; gemm_bf16 falls back to a separate reduction otherwise
                    bg = None
                    if self.B[i - 1] is not None and not (self.dims_out[i - 1] == 1 and self.W[i - 1].shape[0] >= 8):
                        bg = self.B[i - 1].g.reshape(-1)
                    G.gemm_bf16(dz, W.compute(self.mixed)[:W.shape[0]], self.dacts[i - 1],
                                mask=self.acts[i - 1] if self.relu[i - 1] else None,
                                flags=G.EPI_MASK if self.relu[i - 1] else 0, colsum=bg)
                    if bg is not None:
                        bgrad_done.add(i - 1)
                else:
                    G.gemm_bf16(dz, W.compute(self.mixed), self._dx_stage())
        if want_dx:
            g = self.inputs[0].grad.view(self.rows, self.k_in)
            st = self._dx_stage()
            if st.data_ptr() != g.data_ptr():
                g.copy_(st[:, :self.k_in].to(g.dtype))

    def _dx_stage(self):
        g = self.inputs[0].grad
        if self.x_stage is None:
            return g.view(self.rows, self.k_in)
        if not hasattr(self, "_dxs"):
            self._dxs = torch.zeros_like(self.x_stage)
        return self._dxs

    def _wgrad(self, x, dz, W):
        gW = W.g_padded if x.shape[1] == W.g_padded.shape[0] else W.g
        K = x.shape[0]
        tiles = ((gW.shape[0] + 127) // 128) * ((gW.shape[1] + 127) // 128)
        splits = 1
        sms = KernelParams.init(x.device).num_sms
        if tiles < sms:
            splits = max(1, min(8, sms // max(tiles, 1), K // 512))
        G.gemm_bf16(x, dz, gW, a_mn=True, b_mn=True, flags=G.EPI_ATOMIC, splits=splits)


class InnerProductLayer(MLPLayer):
    """FullyConnected: one GEMM + bias, no activation (fully_connected_layer.cu:128-173)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx, num_outputs=[cfg.num_output],
                         activations=[Activation_t.Non], biases=[True],
                         default_init=("fc_w", "fc_b"))


class FusedInnerProductLayer(MLPLayer):
    """FusedReluBiasFullyConnected of older releases == 1-layer MLP with ReLU (release_notes.md:1021)."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx, num_outputs=[cfg.num_output],
                         activations=[Activation_t.Relu], biases=[True],
                         default_init=("fc_w", "fc_b"))
