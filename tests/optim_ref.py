"""A float64 restatement of the optimizer step b2second.optim runs on the GPU (clip -> decay -> Adam -> schedule), of
the one-cycle / exponential / manual schedules in closed form, the literal torch sequence of the reference's training
loop, and seeded parameter sets.  Plain numpy / torch on the CPU; shared by test_optim.py, test_gpu_optim.py and
tools/optim_step_times.py."""
import numpy as np
import torch
from torch import nn

from b2second import optim

ONE_CYCLE = optim.OptimSettings(decoupled=True, weight_decay=optim._f32(0.01), beta1=0.9, beta2=0.99,
                                schedule="one_cycle", lr_max=optim._f32(2.25e-3),
                                moms=(optim._f32(0.95), optim._f32(0.85)), div_factor=10.0, pct_start=optim._f32(0.4))
STAIRCASE = optim.OptimSettings(decoupled=False, weight_decay=optim._f32(1e-4), beta1=0.9, beta2=0.999,
                                schedule="exponential_decay", initial_learning_rate=optim._f32(2e-4),
                                decay_length=optim._f32(0.1), decay_factor=optim._f32(0.8), staircase=True)
SETTINGS = {"one_cycle": ONE_CYCLE, "staircase": STAIRCASE}


# ---- schedules, vectorised closed forms ------------------------------------------------------------------------
def ref_schedule(s, total_step):
    """-> (lr, beta1) float64 arrays [total_step]"""
    step = np.arange(total_step, dtype=np.float64)
    mom = np.full(total_step, s.beta1)
    if s.schedule == "one_cycle":
        a1 = int(s.pct_start * total_step)
        up = step < a1
        pct = np.where(up, step / a1, (step - a1) / (total_step - a1))
        c = (np.cos(np.pi * pct) + 1) / 2                            # 1 at the phase's start, 0 at its end
        low = s.lr_max / s.div_factor
        lr = np.where(up, s.lr_max + (low - s.lr_max) * c, low / 1e4 + (s.lr_max - low / 1e4) * c)
        mom = np.where(up, s.moms[1] + (s.moms[0] - s.moms[1]) * c, s.moms[0] + (s.moms[1] - s.moms[0]) * c)
    elif s.schedule == "exponential_decay" and s.staircase:
        lr = s.initial_learning_rate * s.decay_factor ** np.floor(step / int(s.decay_length * total_step))
    elif s.schedule == "exponential_decay":
        lr = s.decay_factor ** (step / total_step / s.decay_length)
    else:
        edges = np.array([int(b * total_step) for b in s.boundaries])
        lr = np.asarray(s.rates)[np.searchsorted(edges, step, side="right")]
    return lr, mom


# ---- one step in float64 ---------------------------------------------------------------------------------------
def ref_step(s, p, g, m, v, lr, beta1, t):
    """in place on the float64 arrays of the lists p, m, v; g entries may be None.  -> (norm before clipping, per
    parameter None (no gradient) or a dict of the step's float64 intermediates, which ``step_bounds`` reads)"""
    total = np.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in g if x is not None))
    coef = min(1.0, s.clip_norm / (total + 1e-6))
    info = []
    for i in range(len(p)):
        if s.decoupled:
            p[i] *= 1 - s.weight_decay * lr
        if g[i] is None:
            info.append(None)
            continue
        gi = g[i].astype(np.float64) * coef
        mag = np.abs(gi)                                             # the magnitudes that entered the gradient
        if not s.decoupled:
            mag = mag + s.weight_decay * np.abs(p[i])
            gi = gi + s.weight_decay * p[i]
        m0, v0 = m[i].copy(), v[i].copy()
        m[i] += (gi - m[i]) * (1 - beta1)
        v[i][...] = s.beta2 * v[i] + (1 - s.beta2) * gi * gi
        step_size = lr / (1 - beta1 ** t)
        bc2_sqrt = np.sqrt(1 - s.beta2 ** t)
        denom = np.sqrt(v[i]) / bc2_sqrt + s.eps
        upd = step_size * m[i] / denom
        p[i] -= upd
        info.append({"mag": mag, "m0": m0, "v0": v0, "denom": denom, "upd": upd, "step_size": step_size,
                     "bc2_sqrt": bc2_sqrt, "beta1": beta1})
    return total, info


EPS32 = float(np.finfo(np.float32).eps)                              # 2^-23: two units of float32 roundoff


def step_bounds(s, info, p64, m64, v64, dm0=0.0, dv0=0.0, dp0=0.0):
    """what one float32 step of csrc/optim.cu may differ by from ``ref_step`` on the same inputs, per element, given
    the differences dm0, dv0, dp0 the state already carried.  With u = EPS32 / 2 and G = |clipped g| (+ wd |p| in the
    L2 form), fresh rounding contributes
      m:  the clip product (coef itself carries 1.5 u), the subtraction, the product by float32(1 - beta1), the sum
          -> at most 3 EPS32 (|m0| + G)
      v:  no cancellation: the clip product squared, three products, float32(beta2), the sum
          -> at most 7 EPS32 (beta2 v0 + (1 - beta2) G^2)
      p:  the decay product and the final subtraction -> 1.5 EPS32 |p|, plus the update's own error: 4 EPS32 |update|
          for sqrt, the two divisions, the sum, the product and the two float32 scalars, and dm / denom and |m| d(denom) / denom^2 carried
          through, with d(denom) = dv / (2 sqrt(v) bc2_sqrt)
    and carried differences pass through at most undiminished (beta1, beta2 < 1).  -> (dm, dv, dp)"""
    mag = info["mag"] + (0.0 if s.decoupled else s.weight_decay * dp0)
    dm = dm0 + 3 * EPS32 * (np.abs(info["m0"]) + mag) + (0.0 if s.decoupled else s.weight_decay * dp0)
    dv = dv0 + 7 * EPS32 * (s.beta2 * info["v0"] + (1 - s.beta2) * mag * mag) + \
        (0.0 if s.decoupled else 2 * (1 - s.beta2) * mag * s.weight_decay * dp0)
    root = np.sqrt(v64)
    ddenom = np.where(root > 0, dv / np.maximum(2 * root * info["bc2_sqrt"], 1e-300), np.sqrt(dv) / info["bc2_sqrt"])
    ddenom = np.minimum(ddenom, np.sqrt(dv) / info["bc2_sqrt"]) + 2 * EPS32 * info["denom"]
    dupd = 4 * EPS32 * np.abs(info["upd"]) + info["step_size"] * (
        dm / info["denom"] + np.abs(m64) * ddenom / (info["denom"] * np.maximum(info["denom"] - ddenom, 1e-300)))
    dp = dp0 * (1 + EPS32) + 1.5 * EPS32 * np.abs(p64) + dupd
    return dm, dv, dp


def f32_step(s, p, g, m, v, lr, beta1, t):
    """the float32 operation order of csrc/optim.cu's adam_element in numpy (each numpy float32 operation rounds once,
    as the kernel's round-to-nearest intrinsics do); in place on float32 arrays.  -> the float32 norm"""
    f = np.float32
    total = f(np.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in g if x is not None)))
    coef = f(s.clip_norm) / (total + f(1e-6))
    coef = f(1) if coef > 1 else coef
    decay, w1 = f(1 - s.weight_decay * lr), f(1 - beta1)
    step_size, bc2_sqrt = f(lr / (1 - beta1 ** t)), f((1 - s.beta2 ** t) ** 0.5)
    for i in range(len(p)):
        if s.decoupled:
            p[i] *= decay
        if g[i] is None:
            continue
        gi = g[i] * coef
        if not s.decoupled:
            gi = gi + f(s.weight_decay) * p[i]
        m[i] += (gi - m[i]) * w1
        v[i][...] = f(s.beta2) * v[i] + (f(1 - s.beta2) * gi) * gi
        p[i] -= step_size * (m[i] / (np.sqrt(v[i]) / bc2_sqrt + f(s.eps)))
    return total


# ---- the reference's sequence, literally, with torch -----------------------------------------------------------
def torch_adam(s, groups, **kw):
    """torch.optim.Adam as optimizer_builder.build makes it: two groups, lr set later by the schedule"""
    return torch.optim.Adam([{"params": g, "lr": 0} for g in groups], betas=(s.beta1, s.beta2), eps=s.eps,
                            weight_decay=0 if s.decoupled else s.weight_decay, **kw)


def torch_step(s, adam, lr, beta1, set_to_none=False):
    """train.py:299,323-325 with OptimWrapper.step spelled out; -> the norm clip_grad_norm_ returns"""
    params = [p for g in adam.param_groups for p in g["params"]]
    for g in adam.param_groups:
        g["lr"], g["betas"] = lr, (beta1, s.beta2)
    total = torch.nn.utils.clip_grad_norm_(params, s.clip_norm)
    if s.decoupled:
        for p in params:
            p.data.mul_(1 - s.weight_decay * lr)
    adam.step()
    adam.zero_grad(set_to_none=set_to_none)
    return total


# ---- parameter sets --------------------------------------------------------------------------------------------
SHAPES = [(1,), (3,), (5,), (64,), (4095,), (4097,), (3, 3, 3, 16, 32), (8195,), (64,), (64,), (2, 4096)]


class ParamSet(nn.Module):
    """parameters of the given shapes as one leaf module (the non-BN group) and, optionally, one BatchNorm1d"""

    def __init__(self, shapes, bn_channels=0):
        super().__init__()
        self.w = nn.ParameterList([nn.Parameter(torch.zeros(sh)) for sh in shapes])
        if bn_channels:
            self.bn = nn.BatchNorm1d(bn_channels)


def make_case(name, seed=0, steps=1):
    """-> dict: module (float32, CPU), grads [steps][param] float32 arrays or None, in optim.parameter_groups order.
    names: "above" / "below" (gradient norm about 4x over / well under the clip norm), "none_grad" (parameter 2 has no
    gradient), "frozen" (parameter 3 does not require grad), "zero" (all-zero gradients)."""
    rng = np.random.default_rng(seed)
    net = ParamSet(SHAPES, bn_channels=48)
    if name == "frozen":
        net.w[3].requires_grad_(False)
    params = [p for g in optim.parameter_groups(net) for p in g]
    with torch.no_grad():
        for p in params:
            p.copy_(torch.from_numpy(rng.standard_normal(tuple(p.shape)).astype(np.float32) * 0.1))
    n = sum(p.numel() for p in params)
    scale = {"below": 2.0, "zero": 0.0}.get(name, 40.0) / np.sqrt(n)
    grads = []
    for _ in range(steps):
        gs = [(rng.standard_normal(tuple(p.shape)) * scale * rng.uniform(0.2, 1.8)).astype(np.float32) for p in params]
        if name == "none_grad":
            gs[2] = None
        grads.append(gs)
    return {"module": net, "params": params, "grads": grads}


def set_grads(params, grads, device=None):
    """copy one step's gradients in place (or None) the way backward() fills persistent ``.grad`` buffers"""
    for p, g in zip(params, grads):
        if g is None:
            p.grad = None
        elif p.grad is None:
            p.grad = torch.from_numpy(g).to(p.device, p.dtype)
        else:
            p.grad.copy_(torch.from_numpy(g))
