"""TEST INFRASTRUCTURE: float64 reference of the PointPillars feature net in training (b2s_pfn_train_forward /
b2s_pfn_train_backward, b2second.pfn_train) with per-element bounds of the kernels' fp32 steps.  CPU-importable; the GPU
tests call it on CUDA tensors.

closed_form() is the arithmetic contract of csrc/pfn_train.cu in float64 on exact decorated inputs: BatchNorm1d's batch
statistics from the mean mu and covariance C of the decorated inputs d over all M = N * T slots (padded slots are zero
rows), the output max_p relu(BN(w . d_p)), the running-buffer update, and the weight gradient in closed form
    dW_c = gamma_c s_c (G - A mu - B s_c C w_c)
over the argmax slots.  tests/test_pfn_train.py checks it against torch autograd in float64.

reference() adds the bounds.  The decoration's fp32 error per real slot and Linear column (err) follows
tests/fp32_ref.pfn_ref term by term (the mean, the centre, the offsets, the radius).  The kernels take the fp32 d into
float64 moments, so the statistics carry err alone:
    dmu_k  <= mean_p err_pk,   dmean_c <= sum_k |w_ck| dmu_k,
    dvar_c <= mean_p (2 |y_p - mean_c| e_pc + e_pc^2),  e_pc = sum_k |w_ck| (err_pk + dmu_k),
    ds_c   <= s'^3 / 2 * dvar_c  with s' = 1 / sqrt(var_c - dvar_c + eps)  (the largest slope on the interval),
and the fp32 BN factors scale = fp32(gamma s), shift = fp32(beta - mean gamma s) one rounding each on top.  A slot's
fp32 y is one fmaf chain of D terms: gamma_D (S1 + E) + E with S1 = sum |d w|, E = sum err |w| (fp32_ref's chain
bound); BN is one fmaf: |scale| ey + |y| dscale + dshift + u |yhat| (+ the cross term).  ReLU and the max are
1-Lipschitz, so out[n, c] is bounded by the largest bound of the slots that can hold the maximum.  The output's aggregate
(out_aggregate, for fp32_ref.error_stats) takes unit = |scale| S1 and rest = every term of the bound but the chain's
gamma_D (S1 + E), so the RHO check sees the chain's precision.

Argmax near-ties (the certificate idea of tests/detect_ref.py): a slot whose float64 value lies within the sum of the
two bounds of the maximum may be the kernel's argmax, and when the maximum lies within its bound of 0 the ReLU may have
cut the gradient.  The reference keeps its own argmax and adds, per (n, c), the largest difference between the
contribution (delta, delta xhat, delta d) of any admissible choice and its own to the spreads of A, B and G.  The
gradient bounds then propagate the spreads, the slots' err and ey, dmu, dC, ds through
    dW_c = gamma_c s_c (G - A mu - B s_c C w_c)
first order with absolute values, plus one fp32 rounding and a 2^-40 relative allowance for the float64 sums.
"""
import collections

import torch

import fp32_ref as R
from fp32_ref import ETA, U, gamma

FAULTS = ("mean_nm1", "count_sum", "biased_var", "pad_drop", "second")
Bounded = collections.namedtuple("Bounded", "y bound")


def decorate(voxels, num, coors, vx, vy, xoff, yoff, radius, fault=None):
    """-> (d [N, T, D] float64 of the exact fp32 inputs, err [N, T, D] the fp32 decoration's bound, live [N, T]);
    fault "mean_nm1": each pillar's mean of x, y, z over its first num - 1 points"""
    v = voxels.double()
    N, T, F = v.shape
    dev = v.device
    num = num.to(dev).long()
    live = torch.arange(T, device=dev)[None, :] < num[:, None]
    p = torch.where(live[..., None], v, 0.0)
    fn = num.clamp_min(1).double()[:, None]
    if fault == "mean_nm1":
        keep = torch.arange(T, device=dev)[None, :] < (num - 1)[:, None]
        mean = (p[..., :3] * keep[..., None]).sum(1) / (num - 1).clamp_min(1).double()[:, None]
    else:
        mean = p[..., :3].sum(1) / fn
    mabs = p[..., :3].abs().sum(1) / fn
    e_mean = gamma(num)[:, None] * mabs + U * mean.abs()
    q = coors.to(dev).double()
    cv = torch.stack([q[:, 3] * float(vx), q[:, 2] * float(vy)], 1)
    off = torch.tensor([float(xoff), float(yoff)], dtype=torch.float64, device=dev)
    centre = cv + off
    e_centre = gamma(2) * (cv.abs() + off.abs())
    if radius:
        r = torch.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2)
        raw = torch.cat([r[..., None], p[..., 2:]], -1)
        e_raw = torch.cat([gamma(3) * r[..., None], torch.zeros_like(p[..., 2:])], -1)
    else:
        raw, e_raw = p, torch.zeros_like(p)
    d_mean = p[..., :3] - mean[:, None, :]
    d_centre = p[..., :2] - centre[:, None, :]
    d = torch.cat([raw, d_mean, d_centre], -1)
    err = torch.cat([e_raw, (1 + U) * e_mean[:, None, :] + U * d_mean.abs(),
                     (1 + U) * e_centre[:, None, :] + U * d_centre.abs()], -1)
    m = live[..., None]
    return torch.where(m, d, 0.0), torch.where(m, err, 0.0), live


def closed_form(d, live, w, g, b, rm, rv, momentum, eps, dout=None, fault=None):
    """the contract in float64 on decorated inputs d [N, T, D] (0 at padded slots) -> dict with out [N, C], arg [N, C]
    (T = the padded slot), mean, var, s, running_mean, running_var and, with dout [N, C], dW, dgamma, dbeta."""
    N, T, D = d.shape
    w, g, b = w.double(), g.double(), b.double()
    dev = d.device
    M = float(N * T)
    flat = d.reshape(-1, D)
    n_real = float(live.sum())
    if fault == "count_sum":              # M counted as the real slots only
        mu = flat[live.reshape(-1)].sum(0) / n_real
    else:
        mu = flat.sum(0) / M
    if fault == "count_sum":
        rows = flat[live.reshape(-1)]
        C = (rows - mu).t() @ (rows - mu) / n_real
    else:
        C = (flat - mu).t() @ (flat - mu) / M
    mean = w @ mu
    var = ((w @ C) * w).sum(1)
    s = 1.0 / torch.sqrt(var + eps)
    y = d @ w.t()                                                                   # [N, T, C]
    xh = (y - mean) * s
    yh = g * xh + b
    val = torch.relu(yh).masked_fill(~live[..., None], -float("inf"))
    pad_val = torch.relu(b - g * mean * s).expand(N, -1)
    padded = live.sum(1) < T
    if fault == "pad_drop":
        padded = torch.zeros_like(padded)
    vmax, arg = val.max(1)
    if fault == "second":
        top = val.topk(min(2, T), dim=1)
        arg = top.indices[:, -1]
        vmax = torch.where(torch.isfinite(top.values[:, -1]), top.values[:, -1], vmax)
    use_pad = padded[:, None] & (pad_val >= vmax)
    out = torch.where(use_pad, pad_val, vmax)
    arg = torch.where(use_pad, torch.full_like(arg, T), arg)
    unb = var * (M / (M - 1.0)) if fault != "biased_var" else var
    res = dict(out=out, arg=arg, mean=mean, var=var, s=s, mu=mu, C=C, y=y, xh=xh, yh=yh,
               running_mean=(1 - momentum) * rm.double() + momentum * mean,
               running_var=(1 - momentum) * rv.double() + momentum * unb)
    if dout is None:
        return res
    delta = dout.double() * (out > 0)
    ai = arg.clamp_max(T - 1)
    x_at = torch.gather(xh, 1, ai[:, None, :])[:, 0]                                # [N, C]
    x_at = torch.where(use_pad, -mean * s, x_at)
    d_at = d[torch.arange(N, device=dev)[:, None], ai]                              # [N, C, D]
    d_at = torch.where(use_pad[..., None], 0.0, d_at)
    A = delta.sum(0)
    B = (delta * x_at).sum(0)
    G = (delta[..., None] * d_at).sum(0)                                            # [C, D]
    K = G - A[:, None] * mu[None, :] - (B * s)[:, None] * (w @ C)
    res.update(dW=(g * s)[:, None] * K, dgamma=B, dbeta=A, A=A, B=B, G=G, K=K, delta=delta)
    return res


def reference(voxels, num, coors, w, g, b, rm, rv, momentum, eps, vx, vy, xoff, yoff, radius, dout, fault=None):
    """-> dict of Bounded for out, running_mean, running_var, dW, dgamma, dbeta (float64 on voxels' device)"""
    d, err, live = decorate(voxels, num, coors, vx, vy, xoff, yoff, radius)
    dev = d.device
    if fault == "mean_nm1":
        d = decorate(voxels, num, coors, vx, vy, xoff, yoff, radius, fault)[0]
    args = [t.to(dev) for t in (w, g, b, rm, rv)]
    r = closed_form(d, live, *args, float(momentum), float(eps), dout.to(dev), fault=fault)
    N, T, D = d.shape
    M = float(N * T)
    wd, gd = w.to(dev).double(), g.to(dev).double()
    wa = wd.abs()
    mu, C, mean, var, s = r["mu"], r["C"], r["mean"], r["var"], r["s"]
    # statistics
    dmu = err.reshape(-1, D).sum(0) / M
    dmean = wa @ dmu
    e_slot = (err + torch.where(live[..., None], dmu, 0.0)) @ wa.t()                # [N, T, C]; padded: 0 (exact zeros)
    yc = (r["y"] - mean).abs()
    pad_n = M - float(live.sum())
    dvar = ((2 * yc * e_slot + e_slot ** 2) * live[..., None]).sum((0, 1)) / M \
        + pad_n / M * (2 * mean.abs() * dmean + dmean ** 2)
    dvar = dvar + 2.0 ** -40 * (wa @ C.abs() @ wa.t()).diagonal()
    s_lo = 1.0 / torch.sqrt((var - dvar).clamp_min(0) + eps)
    ds = s_lo ** 3 / 2 * dvar
    gs = gd * s
    dscale = gd.abs() * ds + U * gs.abs()
    shift = b.to(dev).double() - mean * gs
    dshift = gd.abs() * (mean.abs() * ds + s * dmean + dmean * ds) + U * shift.abs() + 2.0 ** -40 * (mean * gs).abs()
    # forward
    S1 = d.abs() @ wa.t()
    E = err @ wa.t()
    ey = gamma(D) * (S1 + E) + E + D * ETA
    scale_hi = gs.abs() + dscale
    yh = r["yh"]
    b_slot = scale_hi * ey + r["y"].abs() * dscale + dshift + U * (yh.abs() + scale_hi * ey + r["y"].abs() * dscale
                                                                   + dshift) + ETA
    b_slot = b_slot.masked_fill(~live[..., None], 0.0)
    out = r["out"]
    val = torch.relu(yh).masked_fill(~live[..., None], -float("inf"))
    padded = (live.sum(1) < T)[:, None]
    pad_val = torch.relu(shift).expand(N, -1)
    # admissible slots: value within the two bounds of the maximum
    b_max = torch.maximum(b_slot.max(1).values, torch.where(padded, dshift.expand(N, -1), torch.zeros_like(out)))
    adm = val >= (out - b_max)[:, None, :] - b_slot
    adm_pad = padded & (pad_val >= out - b_max - dshift)
    out_b = Bounded(out, b_max)
    # fp32_ref's aggregate: unit |scale| S1, rest = everything in the bound but the chain's gamma_D (S1 + E) term
    rest_slot = b_slot - scale_hi * gamma(D) * (S1 + E)
    out_rest = torch.maximum(torch.where(adm, rest_slot, 0.0).max(1).values,
                             torch.where(adm_pad, dshift.expand(N, -1), torch.zeros_like(out)))
    out_unit = torch.where(live[..., None], gs.abs() * S1, 0.0).max(1).values
    # backward: the reference argmax's contribution and the spread of the admissible ones
    dlt = r["delta"]
    g_abs = dout.to(dev).double().abs()
    x_slot, x_pad = r["xh"], (-mean * s).expand(N, -1)
    pre = torch.maximum(yh.masked_fill(~live[..., None], -float("inf")).max(1).values,
                        torch.where(padded, shift.expand(N, -1), torch.full_like(out, -float("inf"))))
    relu_open = pre.abs() <= b_max                                                     # the gate may be either way
    ai = r["arg"].clamp_max(T - 1)
    use_pad = r["arg"] == T
    x_ref = torch.where(use_pad, x_pad, torch.gather(x_slot, 1, ai[:, None, :])[:, 0])
    d_ref = torch.where(use_pad[..., None], 0.0, d[torch.arange(N, device=dev)[:, None], ai])
    big = -float("inf")
    sB = torch.maximum(torch.where(adm, (x_slot - x_ref[:, None, :]).abs(), big).max(1).values,
                       torch.where(adm_pad, (x_pad - x_ref).abs(), big)).clamp_min(0)
    sG = torch.empty_like(d_ref)                                                       # [N, C, D]
    er = torch.empty_like(d_ref)
    for i in range(0, N, 2048):                                                        # [rows, T, C, D] at a time
        j = min(N, i + 2048)
        dd = (d[i:j, :, None, :] - d_ref[i:j, None, :, :]).abs()
        sG[i:j] = torch.maximum(torch.where(adm[i:j, ..., None], dd, big).max(1).values,
                                torch.where(adm_pad[i:j, ..., None], d_ref[i:j].abs(), big)).clamp_min(0)
        er[i:j] = torch.where(adm[i:j, ..., None], err[i:j, :, None, :], 0.0).max(1).values
    sA_n = torch.where(relu_open, g_abs, 0.0)
    sB_n = g_abs * sB + sA_n * x_ref.abs()
    sG_n = g_abs[..., None] * sG + sA_n[..., None] * d_ref.abs()
    # the kernel's own errors at its slot: xhat = ((double) y32 - mean') s', d32
    ex_slot = s * (ey + dmean) + yc * ds + (ey + dmean) * ds
    ex_pad = (s * dmean + mean.abs() * ds + dmean * ds).expand(N, -1)
    ex = torch.maximum(torch.where(adm, ex_slot, 0.0).max(1).values, torch.where(adm_pad, ex_pad, 0.0))
    Aabs, Babs = r["A"].abs(), r["B"].abs()
    eA = sA_n.sum(0) + 2.0 ** -40 * dlt.abs().sum(0)
    eB = (sB_n + (g_abs + sA_n) * ex).sum(0) + 2.0 ** -40 * (dlt.abs() * x_ref.abs()).sum(0)
    eG = (sG_n + (g_abs + sA_n)[..., None] * er).sum(0) + 2.0 ** -40 * (dlt.abs()[..., None] * d_ref.abs()).sum(0)
    # dC: centred products with the inputs' and the mean's errors (padded slots: |0 - mu| and dmu)
    dc = torch.where(live[..., None], (d - mu).abs(), mu.abs()).reshape(-1, D)
    ec = torch.where(live[..., None], err + dmu, dmu.expand_as(err)).reshape(-1, D)
    dC = (dc.t() @ ec + ec.t() @ dc + ec.t() @ ec) / M + 2.0 ** -40 * C.abs()
    Cw = wd @ C
    eK = eG + eA[:, None] * mu.abs() + Aabs[:, None] * dmu + ((eB * s + Babs * ds) * Cw.abs().t()).t() \
        + (Babs * s)[:, None] * (wa @ dC)
    K = r["K"].abs()
    dW = r["dW"]
    edW = gd.abs()[:, None] * (ds[:, None] * (K + eK) + s[:, None] * eK) + U * (dW.abs() + gd.abs()[:, None] * (
        ds[:, None] * (K + eK) + s[:, None] * eK)) + 2.0 ** -40 * (gs.abs()[:, None] * (
            r["G"].abs() + Aabs[:, None] * mu.abs() + (Babs * s)[:, None] * (wa @ C.abs())))
    # running buffers: fp32(mean), fp32(unbiased var), two products and a sum in fp32
    mom = float(momentum)
    rmd, rvd = rm.to(dev).double(), rv.to(dev).double()
    unb = M / (M - 1.0)
    e_rm = mom * (dmean + U * mean.abs()) + 3 * U * (mom * mean.abs() + (1 - mom) * rmd.abs()) + 2 * U * rmd.abs()
    e_rv = mom * unb * (dvar + U * var) + 3 * U * (mom * unb * var + (1 - mom) * rvd.abs()) + 2 * U * rvd.abs()
    return dict(out=out_b, out_aggregate=R.Ref(out, b_max, out_unit, out_rest), running_mean=Bounded(r["running_mean"], e_rm), running_var=Bounded(r["running_var"], e_rv),
                dW=Bounded(dW, edW), dgamma=Bounded(r["B"], eB + U * (Babs + eB)),
                dbeta=Bounded(r["A"], eA + U * (Aabs + eA)), raw=r)


def ratio(got, ref):
    """max |got - y| / bound (0 where both are equal)"""
    err = (got.to(ref.y.device, torch.float64) - ref.y).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / ref.bound).max()) if err.numel() else 0.0


# ---- test data ----------------------------------------------------------------------------------------------------
def voxels_of(points, slots, num):
    """fp32_ref.pillars' (points, slots, num) -> voxels [n, T, F] with zero rows past num (VoxelGeneratorV2's layout)"""
    n, T = slots.shape
    sl = torch.as_tensor(slots).long()
    pts = torch.as_tensor(points)
    live = torch.arange(T)[None, :] < torch.as_tensor(num).long()[:, None]
    return torch.where(live[..., None], pts[sl.clamp_min(0)], 0.0).float().contiguous()


def case(seed, n, T, F, radius, batch=1, dup=True):
    """(voxels, num, coors, w, gamma, beta, running_mean, running_var, dout) of n pillars over `batch` frames: counts 1,
    T - 1, T and random (fp32_ref.pillars), duplicate points in some pillars, channels 0..7 reading only x (or |xy|) with
    gamma < 0 so the padded slot holds their maximum, channel 8 all negative (beta << 0)"""
    import numpy as np
    import fp32_ref as R
    rng = np.random.default_rng(seed)
    pts, slots, num, coors = R.pillars(rng, n, T, F)
    vox = voxels_of(pts, slots, num)
    if dup:
        for i in range(3, n, 11):
            if num[i] >= 2:
                vox[i, num[i] - 1] = vox[i, 0]
    coors[:, 0] = rng.integers(batch, size=n)
    D = F + (4 if radius else 5)
    w = (rng.standard_normal((64, D)) * 0.3).astype(np.float32)
    g = (rng.uniform(0.5, 1.5, 64) * rng.choice([-1, 1], 64)).astype(np.float32)
    b = (rng.standard_normal(64) * 0.1).astype(np.float32)
    w[:8] = 0
    w[:8, 0] = 1
    g[:8] = -1
    b[:8] = rng.uniform(0.2, 0.5, 8)
    g[8], b[8] = 0.1, -5.0
    rm = (rng.standard_normal(64) * 0.1).astype(np.float32)
    rv = rng.uniform(0.5, 2.0, 64).astype(np.float32)
    dout = rng.standard_normal((n, 64)).astype(np.float32)
    t = torch.from_numpy
    return vox, t(num.astype(np.int32)), t(coors.astype(np.int32)), t(w), t(g), t(b), t(rm), t(rv), t(dout)
