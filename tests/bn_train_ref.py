"""TEST INFRASTRUCTURE: float64 reference of a train-mode BatchNorm + ReLU pair (b2s_bn_relu_train_forward /
b2s_bn_relu_train_backward, b2second.bn_train) with per-element bounds of the kernels' fp32 steps.  Works on torch
tensors on any device (the GPU tests run it in float64 on the GPU); tests/test_bn_train.py checks its formulas against
torch autograd in float64.

Every tensor is taken as rows [M, C] (``rows``).  The kernels' arithmetic (csrc/bn_train.cu):
  mean, var (biased), s = 1 / sqrt(var + eps) in float64 -- taken as exact here (their float64 error is far below the
  fp32 steps; SLACK covers it);
  forward  y = relu(v),  v = fl32(fl32(x - mu32) * a32 + beta) (one fma),  mu32 = fl32(mean), a32 = fl32(gamma s).
    With d = x - mean and u = 2^-24, each of mu32, a32 is within u of its value, fl32(x - mu32) within u |x - mu32|,
    and the fma within u |v|, so
      |v - (gamma s d + beta)| <= |a32| (u |mean| + u |x - mu32|) + |d| u |gamma s| + u (|a32| |x - mu32| + |beta|)
    (to first order; FACTOR covers the second-order terms), and relu does not increase it.  This form subtracts the
    fp32 mean before scaling, so nothing cancels when |mean| >> std: the bound scales with |x - mean| and u |mean| |a|,
    where x * scale + shift would carry u |x| |a| on both terms.
  running buffers  rm = fl(fl(m * fl(mean)) + fl(fl(1 - m) * rm)) and the same with fl(var M / (M - 1)): four fp32
    roundings of terms bounded by |m| |mean| and |rm| (|m| |var_u|, |rv|).
  backward  g = dY where !(y <= 0) (the kernels' mask is the forward's own v, so the reference takes it from the
    kernels' y), dbeta = sum g, dgamma = sum g xhat, xhat = (x - mean) s, dX = gamma s (g - dbeta / M - xhat dgamma / M),
    all in float64; the fp32 outputs carry one rounding, u |value|, plus float64 summation slack.
"""
import torch

U = 2.0 ** -24
FACTOR = 1.0 + 1e-6                 # second-order terms of the first-order bounds above
SLACK = 1e-10                       # float64 summation order and the kernels' float64 mean / s, relative


def rows(t):
    """[M, C] / channels_last or NCHW [B, C, H, W] / [B, C, L] -> float64 rows [M, C] (a copy)"""
    t = t.detach().double()
    if t.dim() == 2:
        return t.contiguous()
    C = t.shape[1]
    return t.movedim(1, -1).reshape(-1, C).contiguous()


def unrows(r, like):
    """rows [M, C] back to the shape of ``like`` (a copy, contiguous NCHW order of dims)"""
    if like.dim() == 2:
        return r
    B, C = like.shape[:2]
    return r.reshape(B, *like.shape[2:], C).movedim(-1, 1)


def forward(x, gamma, beta, rm, rv, momentum, eps):
    """x rows [M, C] float64; momentum and eps as the code under test has them (the kernels take them as fp32) -> dict:
    mean, var (biased), s, v (gamma s (x - mean) + beta), y, running_mean, running_var (exact, float64) and the
    per-element / per-channel bounds of the kernels' fp32 results"""
    M = x.shape[0]
    g, b = gamma.double(), beta.double()
    mean = x.mean(0)
    d = x - mean
    var = (d * d).mean(0)
    s = 1.0 / torch.sqrt(var + eps)
    gs = g * s
    v = d * gs + b
    y = torch.clamp_min(v, 0.0)
    mu32 = mean.float().double()
    a32 = gs.float().double()
    xm = (x - mu32).abs()
    y_bound = (a32.abs() * (U * mean.abs() + U * xm) + d.abs() * U * gs.abs() + U * (a32.abs() * xm + b.abs()))
    y_bound = y_bound * FACTOR + SLACK * (gs.abs() * d.abs() + b.abs())
    vu = var * (M / (M - 1.0))
    m = float(momentum)
    rm_new = m * mean + (1.0 - m) * rm.double()
    rv_new = m * vu + (1.0 - m) * rv.double()
    rm_bound = 4 * U * (abs(m) * mean.abs() + rm.double().abs()) * FACTOR
    rv_bound = 4 * U * (abs(m) * vu.abs() + rv.double().abs()) * FACTOR
    return dict(mean=mean, var=var, s=s, v=v, y=y, y_bound=y_bound, running_mean=rm_new, running_var=rv_new,
                running_mean_bound=rm_bound, running_var_bound=rv_bound)


def backward(x, dy, y_mask_from, gamma, fw):
    """x, dy rows [M, C] float64; ``y_mask_from`` rows [M, C]: the y whose !(y <= 0) is the ReLU mask (the kernels' own
    y on the GPU, the exact y on the CPU); fw: forward()'s dict -> dict: dx, dgamma, dbeta and their bounds"""
    M = x.shape[0]
    g = torch.where(y_mask_from <= 0, torch.zeros_like(dy), dy)
    xh = (x - fw["mean"]) * fw["s"]
    db = g.sum(0)
    dg = (g * xh).sum(0)
    gs = gamma.double() * fw["s"]
    dx = gs * (g - db / M - xh * dg / M)
    ag, agx = g.abs().sum(0), (g * xh).abs().sum(0)
    return dict(dx=dx, dgamma=dg, dbeta=db,
                dx_bound=U * dx.abs() * FACTOR + SLACK * gs.abs() * (g.abs() + ag / M + xh.abs() * agx / M),
                dgamma_bound=U * dg.abs() * FACTOR + SLACK * agx, dbeta_bound=U * db.abs() * FACTOR + SLACK * ag)


def ratio(got, want, bound):
    """max |got - want| / bound (0 where they are equal; inf where a bound of 0 is exceeded)"""
    err = (got.double() - want).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(r.max()) if r.numel() else 0.0
