"""CPU self-test of tests/tc_ref.py: a numpy emulation of the 3xF16 kernels (fp16 hi/lo planes, the three products
A_hi*W_hi + A_hi*W_lo + A_lo*W_hi summed in float64, epilogue and output rounding in fp32) passes the per-element
bound at the calibrated ALPHA / RHO, and the simulated faults F1 to F3 fail it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tc_ref
from b2second import tc


def planes(t, scale=1.0):
    """fp16 hi / lo planes of t * scale, made in numpy (float64 values)."""
    v = t.double().numpy().astype(np.float32) * np.float32(scale)
    hi = np.clip(v, -65504, 65504).astype(np.float16)
    lo = np.clip(v - hi.astype(np.float32), -65504, 65504).astype(np.float16)
    return torch.from_numpy(hi.astype(np.float64)), torch.from_numpy(lo.astype(np.float64))


def epilogue(acc, s_k, shift, relu, cdim, fp32_out):
    """fmaf(acc, scale / ws, shift) in fp32, ReLU, then fp32 or the hi + lo output planes -> (value, lo plane)"""
    sh = [1] * acc.dim()
    sh[cdim] = -1
    y = (acc.float() * s_k.view(sh) + (0.0 if shift is None else shift.view(sh))).float()
    if relu:
        y = torch.relu(y)
    if fp32_out:
        return y.double(), None
    hi, lo = planes(y)
    return hi + lo, lo


def emulate_dense(x, w, ws, scale, shift, relu, stride=1, padding=0, transpose=False, fp32_out=False):
    conv = (lambda a, b: F.conv_transpose2d(a, b, stride=stride)) if transpose else \
        (lambda a, b: F.conv2d(a, b, stride=stride, padding=padding))
    a_hi, a_lo = planes(x)
    w_hi, w_lo = planes(w, ws)
    acc = conv(a_hi, w_hi) + conv(a_hi, w_lo) + conv(a_lo, w_hi)
    cout = acc.shape[1]
    s_k = (torch.ones(cout) if scale is None else scale) / ws
    return epilogue(acc, s_k.float(), shift, relu, 1, fp32_out)


DENSE = [  # (B, Cin, Cout, H, W, k, stride, pad, transpose, relu, fp32 out, magnitude exponent)
    (1, 64, 32, 9, 11, 3, 1, 1, False, True, False, 0),
    (2, 128, 16, 5, 13, 3, 2, 1, False, True, False, 0),
    (1, 64, 16, 6, 10, 2, 2, 0, True, True, False, 0),
    (1, 128, 20, 7, 9, 1, 1, 0, False, False, True, 0),
    (1, 64, 32, 9, 11, 3, 1, 1, False, True, False, -12),
    (1, 64, 32, 9, 11, 3, 1, 1, False, False, False, 6),
]


@pytest.mark.parametrize("B,cin,cout,H,W,k,stride,pad,transpose,relu,fp32_out,e", DENSE)
def test_emulated_dense_passes_and_faults_fail(B, cin, cout, H, W, k, stride, pad, transpose, relu, fp32_out, e):
    g = torch.Generator().manual_seed(cin + cout + H + W + e)
    x = torch.randn(B, cin, H, W, generator=g) * 2.0 ** e
    wshape = (cin, cout, k, k) if transpose else (cout, cin, k, k)
    w = torch.randn(*wshape, generator=g) * (2.0 / (k * k * cin)) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5
    shift = None if fp32_out else torch.randn(cout, generator=g) * 0.1
    ws = tc.pow2_scale(w)
    got, lo = emulate_dense(x, w, ws, scale, shift, relu, stride, pad, transpose, fp32_out)
    ref = tc_ref.dense_ref(x, w, scale, shift, relu, stride, pad, transpose)
    st = tc_ref.assert_accurate(got, ref, ws, "emulation")
    assert st["alpha"] <= tc_ref.ALPHA / 2
    kw = dict(stride=stride, padding=pad, transpose=transpose)
    if e >= tc_ref.F1_MIN_EXP:
        tc_ref.assert_rejected(tc_ref.dense_f1(got, x, w, ws, ref, relu, **kw), ref, ws, "F1")
    tc_ref.assert_rejected(tc_ref.dense_f2(got, x, w, ws, ref, relu, **kw), ref, ws, "F2")
    tc_ref.assert_rejected(tc_ref.f3(got, lo), ref, ws, "F3")


def test_bound_needs_its_absolute_terms():
    """at activations of 2^-12 the lo plane is subnormal: the emulation passes only because of the 2^-25 * Sw term."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 64, 8, 8, generator=g) * 2.0 ** -12
    w = torch.randn(32, 64, 3, 3, generator=g) * 0.06
    ws = tc.pow2_scale(w)
    got, _ = emulate_dense(x, w, ws, None, None, False, 1, 1)
    ref = tc_ref.dense_ref(x, w, None, None, False, 1, 1)
    tc_ref.assert_accurate(got, ref, ws, "emulation")
    no_abs = ref._replace(Sw=torch.zeros_like(ref.Sw))
    assert tc_ref.error_stats(got, no_abs, ws)["ratio"] > 1.0


@pytest.mark.parametrize("cin,cout", [(8, 16), (16, 32), (64, 64)])
def test_emulated_sparse_passes_and_faults_fail(cin, cout):
    rng = np.random.default_rng(cin + cout)
    n_in, n_out, K = 400, 300, 27
    nbr = np.where(rng.random((n_out, K)) < 0.3, rng.integers(n_in, size=(n_out, K)), -1).astype(np.int32)
    nbr[:, 13] = np.arange(n_out)
    nbr = torch.from_numpy(nbr)
    x = torch.from_numpy(rng.standard_normal((n_in, cin)).astype(np.float32))
    w = torch.from_numpy((rng.standard_normal((K, cin, cout)) * 0.1).astype(np.float32))
    scale = torch.from_numpy((rng.random(cout) + 0.5).astype(np.float32))
    shift = torch.from_numpy((rng.standard_normal(cout) * 0.1).astype(np.float32))
    ws = tc.pow2_scale(w)
    a_hi, a_lo = planes(x)
    w_hi, w_lo = planes(w, ws)
    acc = torch.zeros(n_out, cout, dtype=torch.float64)
    for k in range(K):
        src = nbr[:, k].long()
        ok = src >= 0
        acc[ok] += a_hi[src[ok]] @ w_hi[k] + a_hi[src[ok]] @ w_lo[k] + a_lo[src[ok]] @ w_hi[k]
    got, lo = epilogue(acc, scale / ws, shift, True, 1, False)
    ref = tc_ref.sparse_ref(x, w, nbr, scale, shift, True)
    st = tc_ref.assert_accurate(got, ref, ws, "emulation")
    assert st["alpha"] <= tc_ref.ALPHA / 2
    tc_ref.assert_rejected(tc_ref.sparse_f1(got, x, w, ws, nbr, ref, True, cin), ref, ws, "F1")
    tc_ref.assert_rejected(tc_ref.sparse_f2(got, x, w, ws, nbr, ref, True), ref, ws, "F2")
    tc_ref.assert_rejected(tc_ref.f3(got, lo), ref, ws, "F3")


def test_emulated_wgrad_passes_and_faults_fail():
    rng = np.random.default_rng(3)
    n_in, n_out, K, cin, cout = 500, 400, 27, 32, 16
    nbr = np.where(rng.random((n_out, K)) < 0.3, rng.integers(n_in, size=(n_out, K)), -1).astype(np.int32)
    nbr = torch.from_numpy(nbr)
    x = torch.from_numpy((rng.standard_normal((n_in, cin)) * 2.0 ** 10).astype(np.float32))
    g = torch.from_numpy((rng.standard_normal((n_out, cout)) * 2.0 ** 10).astype(np.float32))
    x_hi, x_lo = planes(x)
    g_hi, g_lo = planes(g)
    got = torch.zeros(K, cin, cout, dtype=torch.float64)
    for k in range(K):
        ok = nbr[:, k] >= 0
        src = nbr[ok, k].long()
        got[k] = x_hi[src].t() @ g_hi[ok] + x_hi[src].t() @ g_lo[ok] + x_lo[src].t() @ g_hi[ok]
    got = got.float().double()
    ref = tc_ref.wgrad_ref(x, g, nbr)
    st = tc_ref.assert_accurate(got, ref, 1.0, "emulation")
    assert st["alpha"] <= tc_ref.ALPHA / 2
    tc_ref.assert_rejected(tc_ref.wgrad_f1(got, x, g, nbr, ref), ref, 1.0, "F1")
    tc_ref.assert_rejected(tc_ref.wgrad_f2(got, x, g, nbr, ref), ref, 1.0, "F2")
    tc_ref.assert_rejected(tc_ref.f3(got, None, cdim=2), ref, 1.0, "F3")
