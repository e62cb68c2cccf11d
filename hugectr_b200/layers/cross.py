"""MultiCross (DCN v1 and low-rank DCN v2) and the DLRM dot Interaction layer.

DCN v2 low-rank: x_{l+1} = x_0 * (x_l U_l V_l + b_l) + x_l   as two wgmma GEMMs per layer with the
elementwise part fused into the second GEMM's epilogue (csrc/gemm_tc.cu EPI_CROSS); backward =
4 GEMMs per layer + one fused elementwise kernel.  Reference: HugeCTR/src/layers/multi_cross_layer.cu
(v1 :582-600/:698-731, v2 fwd :625-672, bwd :733-812, weights U[w,p],V[p,w],b per layer :857-886).
Interaction: HugeCTR/src/layers/interaction_layer.cu (output [B, D + n(n-1)/2 + 1], :637).
"""
from __future__ import annotations

import torch

from ..ops import dense as D
from ..ops import gemm as G
from ..ops import interaction as I
from .base import Layer, make_init


class MultiCrossLayer(Layer):
    trainable = True

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        x = inputs[0]
        b, w = x.shape
        self.w = w
        self.L = int(cfg.num_layers)
        self.p = int(cfg.projection_dim)
        self.mixed = ctx.mixed
        self.v2 = self.p > 0
        self.U, self.V, self.Bv, self.Wv = [], [], [], []
        for l in range(self.L):
            if self.v2:
                self.U.append(self._param(f"U{l}", (w, self.p),
                                          make_init(cfg.weight_init_type, w, self.p, "xavier")))
                self.V.append(self._param(f"V{l}", (self.p, w),
                                          make_init(cfg.weight_init_type, self.p, w, "xavier")))
                self.Bv.append(self._param(f"b{l}", (1, w), make_init(cfg.bias_init_type, w, w, "zero")))
            else:
                self.Wv.append(self._param(f"w{l}", (1, w), make_init(cfg.weight_init_type, w, 1, "xavier")))
                self.Bv.append(self._param(f"b{l}", (1, w), make_init(cfg.bias_init_type, w, 1, "zero")))
        self._out(0, (b, w))

    def allocate(self):
        super().allocate()
        dev, dt = self.ctx.device, self.ctx.act_dtype
        b = self.inputs[0].shape[0]
        L = self.L
        self.X = [self.inputs[0]] + [None] * L  # X[l] tensors (data)
        self.xs = [None] * (L + 1)
        for l in range(1, L):
            self.xs[l] = torch.zeros(b, self.w, dtype=dt, device=dev)
        if self.v2:
            self.H = [torch.zeros(b, self.p, dtype=dt, device=dev) for _ in range(L)]
            keep_t = self.ctx.is_train
            self.T = [torch.zeros(b, self.w, dtype=dt, device=dev) if keep_t else None
                      for _ in range(L)]
            if self.ctx.is_train:
                self.dT = torch.zeros(b, self.w, dtype=dt, device=dev)
                self.dH = torch.zeros(b, self.p, dtype=dt, device=dev)
                self.dXg = torch.zeros(b, self.w, dtype=dt, device=dev)
                self.dX = [torch.zeros(b, self.w, dtype=dt, device=dev) for _ in range(2)]
                # running sum of dy_l * T_l in the activation dtype (fp32 math in registers); the
                # last layer folds the residual dy in, so the final dgrad epilogue adds one tensor
                self.dx0 = torch.zeros(b, self.w, dtype=dt, device=dev)
        else:
            if self.ctx.is_train:
                self.dots = [torch.zeros(b, 1, dtype=torch.float32, device=dev) for _ in range(L)]

    def _xl(self, l):
        if l == 0:
            return self.inputs[0].data
        if l == self.L:
            return self.outputs[0].data
        return self.xs[l]

    # ------------------------------------------------------------------ forward
    def fprop(self, is_train: bool):
        x0 = self.inputs[0].data
        if not self.v2:
            return self._fprop_v1(is_train)
        for l in range(self.L):
            xl = self._xl(l)
            G.gemm_bf16(xl, self.U[l].compute(self.mixed), self.H[l], b_mn=True)
            G.gemm_bf16(self.H[l], self.V[l].compute(self.mixed), self._xl(l + 1), b_mn=True,
                        bias=self.Bv[l].w.reshape(-1), x0=x0, xl=xl, aux=self.T[l],
                        flags=G.EPI_CROSS)

    def _fprop_v1(self, is_train):
        x0 = self.inputs[0].data.float()
        x = x0
        for l in range(self.L):
            dot = x @ self.Wv[l].w.reshape(-1, 1)           # [b,1]
            if is_train and self.ctx.is_train:
                self.dots[l].copy_(dot)
            xn = x0 * dot + self.Bv[l].w.reshape(1, -1) + x
            if l + 1 < self.L:
                self.xs[l + 1].copy_(xn.to(self.xs[l + 1].dtype))
            else:
                self.outputs[0].data.copy_(xn.to(self.outputs[0].data.dtype))
            x = xn

    # ------------------------------------------------------------------ backward
    def bprop(self):
        if not self.v2:
            return self._bprop_v1()
        x0 = self.inputs[0].data
        dy = self.outputs[0].grad
        L = self.L
        for l in range(L - 1, -1, -1):
            xl = self._xl(l)
            first = (l == L - 1)
            D.cross_bwd_ew(dy, x0, self.T[l], self.dT, self.dx0, first, self.Bv[l].g.reshape(-1),
                           last=(l == 0))
            # dV += H^T dT
            G.gemm_bf16(self.H[l], self.dT, self.V[l].g, a_mn=True, b_mn=True,
                        flags=G.EPI_ATOMIC, splits=2)
            # dH = dT V^T      (B operand [N=p, K=w] K-major == V row-major)
            G.gemm_bf16(self.dT, self.V[l].compute(self.mixed), self.dH)
            # dU += x_l^T dH
            G.gemm_bf16(xl, self.dH, self.U[l].g, a_mn=True, b_mn=True, flags=G.EPI_ATOMIC,
                        splits=2)
            # dx_l = dH U^T + dy (+ dx0 on the first layer): the residual adds ride in the GEMM
            # epilogue (B operand [N=w, K=p] K-major == U row-major)
            if l == 0:
                out = self.inputs[0].grad
                if out is not None:
                    G.gemm_bf16(self.dH, self.U[l].compute(self.mixed), out, xl=self.dx0,
                                flags=G.EPI_ADD)
            else:
                out = self.dX[l & 1]
                G.gemm_bf16(self.dH, self.U[l].compute(self.mixed), out, xl=dy, flags=G.EPI_ADD)
                dy = out

    def _bprop_v1(self):
        x0 = self.inputs[0].data.float()
        dy = self.outputs[0].grad.float()
        dx0 = torch.zeros_like(x0)
        for l in range(self.L - 1, -1, -1):
            xl = self._xl(l).float()
            dot = self.dots[l]
            self.Bv[l].g.add_(dy.sum(0, keepdim=True))
            dx0 += dy * dot
            ddot = (dy * x0).sum(1, keepdim=True)           # [b,1]
            self.Wv[l].g.add_((ddot * xl).sum(0, keepdim=True))
            dy = dy + ddot * self.Wv[l].w.reshape(1, -1)
        if self.inputs[0].grad is not None:
            self.inputs[0].grad.copy_((dy + dx0).to(self.inputs[0].grad.dtype))


class InteractionLayer(Layer):
    """DLRM dot interaction: out = [mlp, lower_tri(X X^T), 0] with X = [mlp; emb_0..emb_{n-2}]."""

    def __init__(self, cfg, inputs, ctx):
        super().__init__(cfg, inputs, ctx)
        mlp, emb = inputs
        b, d = mlp.shape
        assert len(emb.shape) == 3 and emb.shape[2] == d, "Interaction: emb must be [b, slots, D]"
        self.n = emb.shape[1] + 1
        self.d = d
        self.out_w = d + self.n * (self.n - 1) // 2 + 1
        self._out(0, (b, self.out_w))

    def fprop(self, is_train: bool):
        I.interaction_fwd(self.inputs[0].data, self.inputs[1].data, self.outputs[0].data)

    def bprop(self):
        I.interaction_bwd(self.inputs[0].data, self.inputs[1].data, self.outputs[0].grad,
                          self.inputs[0].grad, self.inputs[1].grad)
