"""fp64 restatements of the reference's three solvers: Adam (the same formula as the oracle's adam_step, oracle/crnn_oracle.py,
restated per element with the error scale of an f32 evaluation), Momentum and RMSProp.

The reference picks its optimizer from cfg.TRAIN.SOLVER (lib/lstm/train.py:74-76): 'Adam' -> AdamOptimizer(lr), 'RMS' ->
RMSPropOptimizer(lr), anything else -> MomentumOptimizer(lr, cfg.TRAIN.MOMENTUM).  TensorFlow 1.0.1 semantics, restated from
its training_ops kernels and optimizer sources [upstream-memory -- transcribed, not fetched: there is no network]:
  * MomentumOptimizer (use_nesterov=False; one slot "momentum", zeros): accum = accum*momentum + g; var -= lr*accum.
  * RMSPropOptimizer (decay 0.9, momentum 0.0, epsilon 1e-10, centered=False; slots "rms" initialised to ONES and "momentum"
    zeros): ms += (g*g - ms)*(1 - decay); mom = mom*momentum + lr*g/sqrt(ms + epsilon); var -= mom.
Both are pinned to TF's own test vectors by tests/test_solvers_cpu.py (momentum_test.py::testBasic, rmsprop_test.py).

Every function works on OrderedDicts of fp64 torch tensors keyed by TF variable name (the oracle's convention).
Test infrastructure only (imported by tests/)."""
import math
from collections import OrderedDict

import numpy as np
import torch

from oracle import crnn_oracle as O

SOLVERS = ("Adam", "Momentum", "RMS")
RMS_DECAY, RMS_MOMENTUM, RMS_EPSILON = 0.9, 0.0, 1e-10
ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-8


def momentum_step(params, grads, accum, lr, momentum=0.9):
    """TF ApplyMomentum: accum = accum*momentum + g; var -= lr*accum."""
    for k in params:
        accum[k] = accum[k] * momentum + grads[k]
        params[k] = params[k] - lr * accum[k]
    return params, accum


def rmsprop_step(params, grads, ms, mom, lr, decay=RMS_DECAY, momentum=RMS_MOMENTUM, epsilon=RMS_EPSILON):
    """TF ApplyRMSProp: ms += (g^2 - ms)*(1 - decay); mom = mom*momentum + lr*g/sqrt(ms + eps); var -= mom."""
    for k in params:
        ms[k] = ms[k] + (grads[k] * grads[k] - ms[k]) * (1.0 - decay)
        mom[k] = mom[k] * momentum + lr * grads[k] / torch.sqrt(ms[k] + epsilon)
        params[k] = params[k] - mom[k]
    return params, ms, mom


def adam_lr_t(lr, step, b1=ADAM_B1, b2=ADAM_B2, f32=True):
    """TF Adam's bias-corrected step size lr*sqrt(1 - b2^t)/(1 - b1^t).  f32=True: as crnn_clip_adam_step hands it to the kernel
    (the f32 lr widened, the correction in double on the host, the product cast to f32)."""
    lr = float(np.float32(lr)) if f32 else float(lr)
    v = lr * math.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)
    return float(np.float32(v)) if f32 else v


def adam_update(p, g, m, v, lr_t, b1=ADAM_B1, b2=ADAM_B2, eps=ADAM_EPS, g_mag=None):
    """One TF ApplyAdam on fp64 arrays (numpy or torch) with the step size lr_t already bias-corrected: m = b1*m + (1 - b1)*g;
    v = b2*v + (1 - b2)*g^2; p -= lr_t*m/(sqrt(v) + eps).  Returns {"params" | "adam_m" | "adam_v": (value, magnitude)}: the
    magnitude is the sum of the terms' magnitudes that make up each value (g_mag: that of g, default |g|), the scale of an f32
    evaluation's rounding error.  v has no cancellation, so p's magnitude carries m's through the quotient."""
    sqrt = torch.sqrt if isinstance(p, torch.Tensor) else np.sqrt
    g_mag = abs(g) if g_mag is None else g_mag
    m1 = b1 * m + (1.0 - b1) * g
    v1 = b2 * v + (1.0 - b2) * g * g
    den = sqrt(v1) + eps
    m_mag = abs(b1 * m) + (1.0 - b1) * g_mag
    return {"adam_m": (m1, m_mag), "adam_v": (v1, abs(b2 * v) + (1.0 - b2) * g_mag * g_mag),
            "params": (p - lr_t * m1 / den, abs(p) + lr_t * m_mag / den)}


def adam_step(params, grads, m, v, step, lr, b1=ADAM_B1, b2=ADAM_B2, eps=ADAM_EPS):
    """adam_update over OrderedDicts keyed by TF variable name, the step size from adam_lr_t in full double (the oracle's
    adam_step, restated): returns (params, m, v)."""
    lr_t = adam_lr_t(lr, step, b1, b2, f32=False)
    for k in params:
        r = adam_update(params[k], grads[k], m[k], v[k], lr_t, b1, b2, eps)
        params[k], m[k], v[k] = r["params"][0], r["adam_m"][0], r["adam_v"][0]
    return params, m, v


def init_slots(solver, params):
    """TF's initial slot values: Adam m = v = 0, Momentum accum = 0, RMSProp ms = 1 and mom = 0."""
    z = lambda: OrderedDict((k, torch.zeros_like(t)) for k, t in params.items())
    if solver == "Adam":
        return {"m": z(), "v": z()}
    if solver == "Momentum":
        return {"accum": z()}
    return {"ms": OrderedDict((k, torch.ones_like(t)) for k, t in params.items()), "mom": z()}


def apply(solver, params, clipped, slots, step, lr, momentum=0.9):
    """One update of `solver` on already clipped gradients; returns (params, slots)."""
    if solver == "Adam":
        params, m, v = O.adam_step(params, clipped, slots["m"], slots["v"], step, lr)
        return params, {"m": m, "v": v}
    if solver == "Momentum":
        params, accum = momentum_step(params, clipped, slots["accum"], lr, momentum)
        return params, {"accum": accum}
    params, ms, mom = rmsprop_step(params, clipped, slots["ms"], slots["mom"], lr)
    return params, {"ms": ms, "mom": mom}


def train_step(params_np, batch, slots=None, step=1, lr=1e-4, wd=1e-5, clip=10.0, solver="Adam", momentum=0.9):
    """One full solver iteration (train.py:129-130) with the chosen optimizer: the oracle's fp64 autograd gradient, global-norm
    clip, then the update.  Returns the oracle's train_step dict with `params` / `slots` of the chosen solver."""
    if solver not in SOLVERS:
        raise ValueError(solver)
    out = O.train_step(params_np, batch, step=step, lr=lr, wd=wd, clip=clip)      # loss, gradients, norm (and an Adam step, unused)
    p = OrderedDict((k, torch.as_tensor(v, dtype=torch.float64).clone()) for k, v in params_np.items())
    if slots is None:
        slots = init_slots(solver, p)
    clipped, _ = O.clip_by_global_norm(out["grads"], clip)
    out["params"], out["slots"] = apply(solver, p, clipped, slots, step, lr, momentum)
    return out
