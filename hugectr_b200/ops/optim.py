"""The optimizers' facts in one place, for the dense optimizer (ops/dense.py) and the embedding updates
(embedding/ops.py): kernel codes and the hyper-parameter struct of csrc/optim.cuh, the hyper-parameter
dict of an ``OptParamsPy``, the per-weight state arrays, and the host rule (the CPU path and the test
oracle of every kernel)."""
from __future__ import annotations

import ctypes as C

import torch

from ..enums import OPT_STATES_PER_WEIGHT, Optimizer_t

# SparseOpt in csrc/optim.cuh; the dense optimizer takes the first seven
OPT_CODE = {Optimizer_t.SGD: 0, Optimizer_t.AdaGrad: 1, Optimizer_t.Adam: 2, Optimizer_t.Ftrl: 3,
            Optimizer_t.MomentumSGD: 4, Optimizer_t.Nesterov: 5, Optimizer_t.RMSProp: 6,
            Optimizer_t.RowWiseAdaGrad: 7, Optimizer_t.PartialRowWiseAdam: 8}


class COptHyper(C.Structure):
    _fields_ = [("lr_ptr", C.c_void_p), ("lr_scale", C.c_float), ("scaler", C.c_float),
                ("beta1", C.c_float), ("beta2", C.c_float), ("epsilon", C.c_float),
                ("lambda1", C.c_float), ("lambda2", C.c_float), ("ftrl_beta", C.c_float),
                ("momentum", C.c_float), ("initial_accu", C.c_float), ("step_ptr", C.c_void_p),
                ("sr_seed", C.c_uint), ("pad_", C.c_uint)]


def opt_hp(o, scaler: float = 1.0, sr_seed: int = 0) -> dict:
    """Hyper-parameters of the optimizer ``o`` (an ``OptParamsPy``) for gradients that arrive multiplied
    by the loss ``scaler``; ``sr_seed`` seeds the stochastic rounding of bf16 embedding weights."""
    return {"scaler": scaler, "beta1": o.beta1, "beta2": o.beta2, "epsilon": o.epsilon,
            "lambda1": o.lambda1, "lambda2": o.lambda2, "ftrl_beta": o.beta,
            "momentum": o.momentum_factor, "initial_accu_value": o.initial_accu_value,
            "sr_seed": sr_seed}


def sr_seed(hp: dict) -> int:
    """32-bit seed of the stochastic rounding of bf16 weights (``hp["sr_seed"]``, default 0)"""
    return int(hp.get("sr_seed", 0)) & 0xFFFFFFFF


def opt_hyper(hp: dict, lr_t, step_t) -> COptHyper:
    """Kernel hyper-parameters: the device learning rate ``lr_t`` and step counter ``step_t`` (None: the
    kernels take step 1) with the optimizer's values from ``hp``."""
    return COptHyper(lr_t.data_ptr(), 1.0, hp.get("scaler", 1.0), hp.get("beta1", 0.9),
                     hp.get("beta2", 0.999), hp.get("epsilon", 1e-7), hp.get("lambda1", 0.0),
                     hp.get("lambda2", 0.0), hp.get("ftrl_beta", 0.0), hp.get("momentum", 0.0),
                     hp.get("initial_accu_value", 0.0), None if step_t is None else step_t.data_ptr(),
                     sr_seed(hp), 0)


def opt_states(o, n: int, dtype=torch.float32, device=None):
    """(s0, s1) of ``n`` weights under the optimizer ``o`` (an ``OptParamsPy``):
    ``OPT_STATES_PER_WEIGHT`` arrays, None for the others; AdaGrad's s0 starts at its
    ``initial_accu_value``, every other state at zero."""
    ns = OPT_STATES_PER_WEIGHT[o.optimizer_type]
    s0 = torch.zeros(n, dtype=dtype, device=device) if ns >= 1 else None
    s1 = torch.zeros(n, dtype=dtype, device=device) if ns >= 2 else None
    if s0 is not None and o.optimizer_type == Optimizer_t.AdaGrad and o.initial_accu_value != 0.0:
        s0.fill_(o.initial_accu_value)
    return s0, s1


def opt_reference(opt: Optimizer_t, w, s0, s1, g, hp, lr, step):
    """fp32 PyTorch form of the update rules of csrc/optim.cuh, in place on ``w`` and the states
    (same shapes as ``g``; RowWiseAdaGrad: ``g`` [n, ev] and s0 [n], one accumulator per row;
    PartialRowWiseAdam: ``g`` and s0 = m [n, ev], s1 = v [n], one second moment per row)."""
    g = g / hp.get("scaler", 1.0)
    eps = hp.get("epsilon", 1e-7)
    if opt == Optimizer_t.RowWiseAdaGrad:
        # s += mean_c g^2 ; w -= (lr / (sqrt(s) + eps)) g  -- the factor first, as the kernels do
        s0 += (g * g).sum(1) / g.shape[1]
        w -= (lr / (s0.sqrt() + eps)).unsqueeze(1) * g
    elif opt == Optimizer_t.PartialRowWiseAdam:
        # m = b1 m + (1-b1) g ; v = b2 v + (1-b2) mean_c g^2 ; w -= (alpha / (sqrt(v) + eps)) m
        b1, b2 = hp.get("beta1", 0.9), hp.get("beta2", 0.999)
        s0.mul_(b1).add_((1 - b1) * g)
        s1.mul_(b2).add_((1 - b2) * ((g * g).sum(1) / g.shape[1]))
        alpha = lr * (1 - b2 ** step) ** 0.5 / (1 - b1 ** step)
        w -= (alpha / (s1.sqrt() + eps)).unsqueeze(1) * s0
    elif opt == Optimizer_t.SGD:
        w -= lr * g
    elif opt == Optimizer_t.AdaGrad:
        s0 += g * g
        w -= lr * g / (s0.sqrt() + eps)
    elif opt == Optimizer_t.Adam:
        b1, b2 = hp.get("beta1", 0.9), hp.get("beta2", 0.999)
        s0.mul_(b1).add_((1 - b1) * g)
        s1.mul_(b2).add_((1 - b2) * g * g)
        alpha = lr * (1 - b2 ** step) ** 0.5 / (1 - b1 ** step)
        w -= alpha * s0 / (s1.sqrt() + eps)
    elif opt == Optimizer_t.Ftrl:
        fb, l1, l2 = hp.get("ftrl_beta", 0.0), hp.get("lambda1", 0.0), hp.get("lambda2", 0.0)
        n_new = s1 + g * g
        s0 += g + ((s1 + fb).sqrt() - (n_new + fb).sqrt()) * w / lr
        s1.copy_(n_new)
        p = torch.where(s0 > 0, l1 - s0, -l1 - s0)
        q = (n_new + fb).sqrt() / lr + l2
        w.copy_(torch.where(s0.abs() > l1, p / q, torch.zeros_like(w)))
    elif opt == Optimizer_t.MomentumSGD:
        s0.mul_(hp.get("momentum", 0.0)).sub_(lr * g)
        w += s0
    elif opt == Optimizer_t.Nesterov:
        mu = hp.get("momentum", 0.0)
        an = mu * s0 - lr * g
        w += -mu * s0 + (1 + mu) * an
        s0.copy_(an)
    elif opt == Optimizer_t.RMSProp:
        b2 = hp.get("beta2", 0.999)
        s0.mul_(b2).add_((1 - b2) * g * g)
        w -= lr * g / (s0.sqrt() + eps)
