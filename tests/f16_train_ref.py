"""TEST INFRASTRUCTURE: the per-element error bound of the f16 training mode (training.enable_sparse_backward /
enable_rpn_training with precision="f16") and the float64 reference of the dense weight gradient.  CPU-importable; the
GPU tests call it on CUDA float64 tensors.

A training contraction computes y = sum(a * b) over the terms that feed an element, with both operands split under their
own power of two: a is carried as fp16(a * sa) and b as fp16(b * sb), and the kernel multiplies the fp32 sum by
1 / (sa * sb) exactly.  The three contractions and their operands:
  forward y   a = the activation X (scale of b2s_split_f16_autoscale / _halo_), b = the weight W (scale of the pack);
  input dX    the forward contraction over the transposed table (sparse) or the flipped weights (dense): a = dY, b = W;
  weight dW   a = X, b = dY, the terms are the pairs (sparse) or pixels (dense): S1 = sum |x * dy| per (k, c_in, c_out).
With u = 2^-11 each fp16 rounding errs by at most u relative, or 2^-25 absolute below the fp16 normal range.  The
floors apply to the SCALED operands, so in unscaled units they are 2^-25 / sa and 2^-25 / sb, and one product errs by at
most (2u + u^2) |a b| + 2^-25 (1 + u) (|b| / sa + |a| / sb) + 2^-50 / (sa sb).  Over the n terms of an element:

    |y - y64| <= (2u + u^2) S1 + 2^-25 (1 + u) (Sw / sa + Sa / sb) + n 2^-50 / (sa sb) + ALPHA 2^-23 S1
                 + 2^-22 |y64| + 2^-25 / (sa sb)

with S1 = sum |a b|, Sa = sum |a|, Sw = sum |b| as in tests/tc_ref.py (its Ref), ALPHA 2^-23 S1 the fp32 accumulation
chains (tc_ref.ALPHA) and the last two terms the fp32 output rounding (its absolute part, like the floors, in the
scaled domain).  The comparison that shows the f16 bound is not vacuous is tc_ref's 3xF16 bound in the same scaled
domain, ALPHA 2^-23 S1 + 2^-25 (Sw / sa + Sa / sb) + 2^-22 |y64| + 2^-25 / (sa sb): on every layer shape some element
lies beyond it.  (In unscaled units its floors, 2^-25 Sw and 2^-25, would exceed a gradient of order 2^-20 outright.)
"""
import torch

import tc_ref

U = 2.0 ** -11


def bounds(ref, sa, sb, n):
    """-> (the f16 bound, the 3xF16 bound in the same scaled domain) per element of ref.y; sa, sb the operands' powers
    of two (floats), n an upper bound of the terms per element"""
    floors = ref.s * 2.0 ** -25 * (ref.Sw / sa + ref.Sa / sb)
    common = ref.s * tc_ref.ALPHA * 2.0 ** -23 * ref.S1 + 2.0 ** -22 * ref.pre.abs() + 2.0 ** -25 / (sa * sb)
    f16 = ref.s * ((2 * U + U * U) * ref.S1 + n * 2.0 ** -50 / (sa * sb)) + (1 + U) * floors + common
    return f16, floors + common


def check(got, ref, sa, sb, n, what="", mask=None):
    """assert the f16 bound element by element (where `mask`, if given); -> (max error / bound, share of elements
    beyond the 3xF16 bound), and assert that share is not zero"""
    err = (got.to(ref.y.device, torch.float64) - ref.y).abs()
    f16, three = bounds(ref, sa, sb, n)
    if mask is not None:
        err, f16, three = err[mask], f16[mask], three[mask]
    ratio = float((err / f16).max()) if err.numel() else 0.0
    assert ratio <= 1.0, "%s: |y - y64| reaches %.3g x the f16 bound" % (what, ratio)
    beyond = float((err > three).double().mean()) if err.numel() else 0.0
    assert beyond > 0, "%s: the f16 error never exceeds the 3xF16 bound (the bound would be vacuous)" % what
    return ratio, beyond


def dense_wgrad_ref(x, dy):
    """dW[co, ci, ky, kx] = sum_px dy[px, co] x[px + (ky - 1, kx - 1), ci] of a 3x3 stride-1 pad-1 conv (x [B, Cin, H, W],
    dy [B, Cout, H, W]) -> Ref with [Cout, Cin, 3, 3] float64 fields and s = 1: x plays the activation (Sa = sum |x|)
    and dy the weight (Sw = sum |dy|) over the pixels that feed the element.  One float64 GEMM per tap."""
    B, cin, H, W = x.shape
    cout = dy.shape[1]
    xp = torch.nn.functional.pad(x.double(), (1, 1, 1, 1))
    g = dy.double().permute(1, 0, 2, 3).reshape(cout, -1)                   # [Cout, pixels]
    y = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device=x.device)
    S1, Sa, Sw = y.clone(), y.clone(), y.clone()
    for ky in range(3):
        for kx in range(3):
            a = xp[:, :, ky:ky + H, kx:kx + W].permute(0, 2, 3, 1).reshape(-1, cin)   # [pixels, Cin]
            inside = torch.zeros(B, 1, H + 2, W + 2, dtype=torch.float64, device=x.device)
            inside[:, :, 1:-1, 1:-1] = 1
            m = inside[:, :, ky:ky + H, kx:kx + W].reshape(-1, 1)               # pixel reads the map, not the pad
            y[:, :, ky, kx] = g @ a
            S1[:, :, ky, kx] = g.abs() @ a.abs()
            Sa[:, :, ky, kx] = (a.abs().sum(0))[None, :]
            Sw[:, :, ky, kx] = (g.abs() @ m)
    return tc_ref._finish(y, S1, Sa, Sw, None, None, False, 1)
