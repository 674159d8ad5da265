"""TEST INFRASTRUCTURE: float64 references of the tensor-core convolutions and the per-element error bound of the 3xF16
split they use (csrc/tc_common.cuh).  CPU-importable; the GPU tests call it on CUDA float64 tensors.

A kernel result y of  y = s * sum(a * w) + shift  (a, w fp32, each carried as fp16 hi/lo planes, w pre-scaled by the
power of two ws = b2second.tc.pow2_scale) must satisfy, element by element,

    |y - y64| <= |s| * (ALPHA * 2^-23 * S1 + 2^-25 * (Sw + Sa / ws)) + 2^-22 * |y64| + 2^-25

with y64 the float64 value computed from the fp32 inputs and, over exactly the terms that feed the element,
S1 = sum|a * w|, Sa = sum|a|, Sw = sum|w|.  The terms: the three-product truncation and the fp32 accumulation chains;
the lo plane of an activation (weight) below 2^-3 (2^-3 / ws) is an fp16 subnormal, good to 2^-25 absolute only; the
output rounding to fp32 or to hi + lo.  ReLU is 1-Lipschitz, so the bound of the pre-activation value holds after it.
On top of it, a fault spread thinly over all outputs is caught by the aggregate check
rms(e) / rms(|s| * S1) <= RHO, e = |y - y64| beyond the bound's terms other than the ALPHA one.

ALPHA and RHO are the smallest powers of two that the unmodified kernels meet with at least a 2x margin on every case of
tests/test_gpu_tc_fp64.py.  The fault helpers (F1 to F3) simulate, in float64 from the actual hi/lo planes, the faults
the check must reject: F1 drops A_lo*W_hi of one 16-channel K step of one tap everywhere (thin), F2 drops one tap of
one output row (local), F3 zeroes the lo plane of one output channel.  The weight gradient of the sparse conv has the
same three faults over its reduction of output rows (wgrad_ref, wgrad_f1, wgrad_f2).
"""
import collections

import numpy as np
import torch
import torch.nn.functional as F

ALPHA = 8.0
RHO = 2.0 ** -23
# F1 is only a fault the bound can see while the activations' lo planes are mostly normal fp16 (|a| >= 2^-3): below,
# A_lo * W_hi is itself within the 2^-25 * Sw term, so inputs of randn * 2^e with e < F1_MIN_EXP skip F1.
F1_MIN_EXP = -3

Ref = collections.namedtuple("Ref", "y pre S1 Sa Sw s")


def _bcast(v, like, dim):
    """per-channel vector -> broadcastable against `like` along `dim` (float64)."""
    shape = [1] * like.dim()
    shape[dim] = -1
    return v.to(like.device, torch.float64).reshape(shape)


def _finish(y, S1, Sa, Sw, scale, shift, relu, cdim):
    s = torch.ones(y.shape[cdim], dtype=torch.float64, device=y.device) if scale is None else \
        scale.to(y.device, torch.float64)
    pre = y * _bcast(s, y, cdim)
    if shift is not None:
        pre = pre + _bcast(shift, y, cdim)
    s = _bcast(s, y, cdim).abs().expand_as(y)
    return Ref(torch.relu(pre) if relu else pre, pre, S1, Sa, Sw, s)


def _conv(transpose, stride, padding):
    if transpose:
        return lambda x, w: F.conv_transpose2d(x, w, stride=stride)
    return lambda x, w: F.conv2d(x, w, stride=stride, padding=padding)


def dense_ref(x, w, scale=None, shift=None, relu=False, stride=1, padding=0, transpose=False):
    """x [B, Cin, H, W] fp32, w in torch layout (conv [Cout, Cin, kh, kw], transpose [Cin, Cout, k, k]; stride = k, no
    padding) -> Ref, every field NCHW float64 (s broadcast to the output shape)."""
    conv = _conv(transpose, stride, padding)
    xd, wd = x.double(), w.double()
    y = conv(xd, wd)
    S1 = conv(xd.abs(), wd.abs())
    Sa = conv(xd.abs(), torch.ones_like(wd))
    Sw = conv(torch.ones_like(xd), wd.abs())
    return _finish(y, S1, Sa, Sw, scale, shift, relu, 1)


def sparse_ref(x, w, nbr, scale=None, shift=None, relu=False):
    """gather-GEMM straight from the kernel's table: y[o] = sum_k W[k]^T x[nbr[o, k]] (nbr < 0: no neighbour).
    x [n_in, Cin] fp32, w [K, Cin, Cout], nbr [n_out, K] -> Ref with [n_out, Cout] float64 fields."""
    xd, wd = x.double(), w.double()
    n_out, K = nbr.shape
    y = torch.zeros(n_out, wd.shape[2], dtype=torch.float64, device=xd.device)
    S1, Sa, Sw = y.clone(), y.clone(), y.clone()
    for k in range(K):
        src = nbr[:, k].long()
        ok = src >= 0
        if not bool(ok.any()):
            continue
        a = xd[src[ok]]
        y[ok] += a @ wd[k]
        S1[ok] += a.abs() @ wd[k].abs()
        Sa[ok] += a.abs().sum(1, keepdim=True)
        Sw[ok] += wd[k].abs().sum(0, keepdim=True)
    return _finish(y, S1, Sa, Sw, scale, shift, relu, 1)


def wgrad_ref(x, g, nbr):
    """weight gradient straight from the table: dW[k] = sum_o x[nbr[o, k]]^T g[o].  x [n_in, Cin], g [n_out, Cout],
    nbr [n_out, K] -> Ref with [K, Cin, Cout] fields and s = 1.  In the bound x plays the activation and g the weight:
    Sa = sum|x| and Sw = sum|g| over the rows o that feed the element (those with a neighbour through k)."""
    xd, gd = x.double(), g.double()
    K = nbr.shape[1]
    y = torch.zeros(K, xd.shape[1], gd.shape[1], dtype=torch.float64, device=xd.device)
    S1, Sa, Sw = y.clone(), y.clone(), y.clone()
    for k in range(K):
        src = nbr[:, k].long()
        ok = src >= 0
        a, b = xd[src[ok]], gd[ok]
        y[k] = a.t() @ b
        S1[k] = a.abs().t() @ b.abs()
        Sa[k] = a.abs().sum(0)[:, None]
        Sw[k] = b.abs().sum(0)[None, :]
    return _finish(y, S1, Sa, Sw, None, None, False, 2)


def _terms(ref, ws):
    """(the chain-error unit |s| * 2^-23 * S1, everything else of the bound)"""
    unit = ref.s * 2.0 ** -23 * ref.S1
    rest = ref.s * 2.0 ** -25 * (ref.Sw + ref.Sa / ws) + 2.0 ** -22 * ref.pre.abs() + 2.0 ** -25
    return unit, rest


def error_stats(got, ref, ws, alpha=None):
    """-> {"ratio": max |y - y64| / bound, "alpha": the least ALPHA the element-wise bound needs,
    "rms": the aggregate ratio} of a kernel result `got` (same shape as ref.y)."""
    alpha = ALPHA if alpha is None else alpha
    err = (got.to(ref.y.device, torch.float64) - ref.y).abs()
    unit, rest = _terms(ref, ws)
    bound = alpha * unit + rest
    need = ((err - rest) / unit.clamp_min(1e-300)).clamp_min(0.0)
    need = torch.where(unit > 0, need, torch.where(err > rest, torch.full_like(need, float("inf")), need))
    # aggregate: the error beyond the subnormal / output-rounding terms (which dominate at small magnitudes and are
    # not relative to S1)
    excess = (err - rest).clamp_min(0.0)
    den = float((ref.s * ref.S1).pow(2).mean().sqrt())
    rms = float(excess.pow(2).mean().sqrt()) / den if den > 0 else (0.0 if float(excess.max()) == 0.0 else float("inf"))
    return {"ratio": float((err / bound).max()) if err.numel() else 0.0,
            "alpha": float(need.max()) if err.numel() else 0.0, "rms": rms}


def assert_accurate(got, ref, ws, what=""):
    st = error_stats(got, ref, ws)
    assert st["ratio"] <= 1.0, "%s: |y - y64| reaches %.3g x the bound (needs ALPHA %.3g)" % (what, st["ratio"],
                                                                                           st["alpha"])
    assert st["rms"] <= RHO, "%s: rms error %.3g x rms(|s| S1), above RHO = %.3g" % (what, st["rms"], RHO)
    return st


def assert_rejected(got, ref, ws, what=""):
    st = error_stats(got, ref, ws)
    assert not (st["ratio"] <= 1.0 and st["rms"] <= RHO), "%s: a simulated fault passes the check (%r)" % (what, st)
    return st


# ---- simulated faults ----------------------------------------------------------------------------------------------

def hi_lo(t, scale=1.0):
    """float64 values of the fp16 hi / lo planes the kernels get for t * scale (b2second.tc.split_f16)."""
    t = t.detach().to(torch.float32) * float(scale)
    hi = t.clamp(-65504.0, 65504.0).half()
    lo = (t - hi.float()).clamp(-65504.0, 65504.0).half()
    return hi.double(), lo.double()


def _apply(got, delta, relu):
    out = got.to(delta.device, torch.float64) - delta
    return torch.relu(out) if relu else out


def dense_f1(got, x, w, ws, ref, relu, stride=1, padding=0, transpose=False, tap=None, k0=None):
    """F1: A_lo * W_hi of one 16-channel K step (input channels k0 .. k0+15, default the last step) of one tap (kernel
    position (dy, dx), default the centre) dropped at every output pixel."""
    conv = _conv(transpose, stride, padding)
    _, a_lo = hi_lo(x)
    w_hi, _ = hi_lo(w, ws)
    kh, kw = w.shape[2], w.shape[3]
    dy, dx = tap if tap is not None else (kh // 2, kw // 2)
    cin = x.shape[1]
    k0 = cin - 16 if k0 is None else k0
    wm = torch.zeros_like(w_hi)
    if transpose:
        wm[k0:k0 + 16, :, dy, dx] = w_hi[k0:k0 + 16, :, dy, dx] / ws
    else:
        wm[:, k0:k0 + 16, dy, dx] = w_hi[:, k0:k0 + 16, dy, dx] / ws
    return _apply(got, conv(a_lo, wm) * ref.s, relu)


def dense_f2(got, x, w, ws, ref, relu, stride=1, padding=0, transpose=False, tap=None):
    """F2: the whole contribution of one tap (the three products) dropped for one output row of the bottom-right
    partial strip: the last output row, its last (W_out mod 8, or 8) pixels.  Default tap: the centre (a
    ConvTranspose2d: the last sub-grid position, the one that reaches the last output row)."""
    conv = _conv(transpose, stride, padding)
    a_hi, a_lo = hi_lo(x)
    w_hi, w_lo = hi_lo(w, ws)
    kh, kw = w.shape[2], w.shape[3]
    dy, dx = tap if tap is not None else ((kh - 1, kw - 1) if transpose else (kh // 2, kw // 2))
    sel = (slice(None), slice(None), dy, dx)
    m = torch.zeros_like(w_hi)
    mh, ml = m.clone(), m.clone()
    mh[sel], ml[sel] = w_hi[sel] / ws, w_lo[sel] / ws
    delta = (conv(a_hi, mh) + conv(a_hi, ml) + conv(a_lo, mh)) * ref.s
    Wo = delta.shape[3]
    w0 = Wo - (Wo % 8 or 8)
    keep = torch.zeros_like(delta)
    keep[:, :, -1, w0:] = 1.0
    return _apply(got, delta * keep, relu)


def f3(got, lo, ch=None, cdim=1):
    """F3: the lo plane of output channel `ch` zeroed (lo None: an fp32 output, the channel rounded to fp16 instead).
    Default channel: the one whose lo plane carries the most (after a ReLU some channels are all zero)."""
    out = got.to(torch.float64).clone()
    if ch is None:
        rest = lo.to(out.device, torch.float64) if lo is not None else out - out.float().half().double()
        ch = int(rest.abs().transpose(0, cdim).reshape(out.shape[cdim], -1).sum(1).argmax())
    idx = [slice(None)] * out.dim()
    idx[cdim] = ch
    if lo is None:
        out[tuple(idx)] = out[tuple(idx)].float().half().double()
    else:
        out[tuple(idx)] -= lo.to(out.device, torch.float64)[tuple(idx)]
    return out


def sparse_f1(got, x, w, ws, nbr, ref, relu, cin_tc, tile=0, kb=None):
    """F1 of the sparse kernel: A_lo * W_hi of one 64-channel K block (the 64 / cin_tc kernel offsets packed into it)
    dropped for the rows of one 128-row tile.  Default block: the one with the most neighbours in the tile."""
    _, a_lo = hi_lo(x)
    w_hi, _ = hi_lo(w, ws)
    K = nbr.shape[1]
    pack = max(1, 64 // cin_tc)
    rows = slice(128 * tile, min(nbr.shape[0], 128 * tile + 128))
    t = nbr[rows].long()
    if kb is None:
        cnt = [(t[:, k0:k0 + pack] >= 0).sum().item() for k0 in range(0, K, pack)]
        kb = int(np.argmax(cnt))
    delta = torch.zeros_like(ref.y)
    for k in range(kb * pack, min(K, kb * pack + pack)):
        src = t[:, k]
        ok = src >= 0
        d = torch.zeros(t.shape[0], w.shape[2], dtype=torch.float64, device=delta.device)
        d[ok] = a_lo[src[ok]] @ (w_hi[k] / ws)
        delta[rows] += d
    return _apply(got, delta * ref.s, relu)


def sparse_f2(got, x, w, ws, nbr, ref, relu, row=None):
    """F2 of the sparse kernel: one neighbour (the first present offset) of one row (default the last) dropped."""
    a_hi, a_lo = hi_lo(x)
    w_hi, w_lo = hi_lo(w, ws)
    o = nbr.shape[0] - 1 if row is None else row
    ks = (nbr[o] >= 0).nonzero()
    assert ks.numel(), "row %d has no neighbour" % o
    k = int(ks[0])
    i = int(nbr[o, k])
    delta = torch.zeros_like(ref.y)
    delta[o] = (a_hi[i] @ (w_hi[k] / ws) + a_hi[i] @ (w_lo[k] / ws) + a_lo[i] @ (w_hi[k] / ws)) * ref.s[o]
    return _apply(got, delta, relu)


def wgrad_f1(got, x, g, nbr, ref, chunk=0):
    """F1 of the weight gradient: X_lo * dY_hi of one 64-row chunk of output rows (rows 64*chunk .. +63) dropped for
    every kernel offset.  x, g: the operands as the kernel splits them (already under their power-of-two scales)."""
    _, x_lo = hi_lo(x)
    g_hi, _ = hi_lo(g)
    rows = slice(64 * chunk, min(nbr.shape[0], 64 * chunk + 64))
    t = nbr[rows].long()
    delta = torch.zeros_like(ref.y)
    for k in range(nbr.shape[1]):
        ok = t[:, k] >= 0
        delta[k] = x_lo[t[ok, k]].t() @ g_hi[rows][ok]
    return got.to(delta.device, torch.float64) - delta


def wgrad_f2(got, x, g, nbr, ref, row=None):
    """F2 of the weight gradient: one (row, offset) pair -- the last row's first neighbour -- left out of dW."""
    x_hi, x_lo = hi_lo(x)
    g_hi, g_lo = hi_lo(g)
    o = nbr.shape[0] - 1 if row is None else row
    k = int((nbr[o] >= 0).nonzero()[0])
    i = int(nbr[o, k])
    delta = torch.zeros_like(ref.y)
    delta[k] = torch.outer(x_hi[i], g_hi[o]) + torch.outer(x_hi[i], g_lo[o]) + torch.outer(x_lo[i], g_hi[o])
    return got.to(delta.device, torch.float64) - delta
