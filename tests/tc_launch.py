"""TEST INFRASTRUCTURE: launches of the dense tensor-core convolution (b2s_conv2d_tc_ex2) into sentinel-filled output
maps, and the checks the float64 tests share (tests/test_gpu_tc_fp64.py, test_gpu_conv_tc.py, test_gpu_rpn_tc_bits.py)."""
import ctypes

import torch
import torch.nn.functional as F

import tc_ref

HI_SENT, LO_SENT, F32_SENT = -3.0, -5.0, 7.0


def pad_nhwc(x):
    return F.pad(x.permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).contiguous()


def _n_pad(c):
    return 32 if c <= 32 else (64 if c <= 64 else 128)


def launch_dense(product, x, w, ws, k, stride=1, pad=0, transpose=False, scale=None, shift=None, relu=False,
                 planes=2, out_stride=None, coff=0, n_pad=None, in_planes=None, lists=None):
    """one layer as b2s_conv2d_tc_ex2 launches (output channels cut into slices of <= 128, a ConvTranspose2d k = s as
    k*k sub-grid launches) into a sentinel-filled output map of out_stride channels at channel offset coff.
    scale None: the kernel gets scale = NULL (then ws must be 1).  lists: (R, work, wn, bg, bn, field_hi, field_lo,
    margin) for a strip-list launch.  -> (out planes, status, (Ho, Wo))"""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, cin, H, W = x.shape
    cout = w.shape[1] if transpose else w.shape[0]
    hi, lo = in_planes if in_planes is not None else tc.split_f16(pad_nhwc(x))
    Ho, Wo = (H * k, W * k) if transpose else ((H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1)
    out_stride = out_stride or coff + cout
    if planes == 2:
        out = [torch.full((B, Ho + 2, Wo + 2, out_stride), v, dtype=torch.float16, device="cuda")
               for v in (HI_SENT, LO_SENT)]
    else:
        out = [torch.full((B, Ho, Wo, out_stride), F32_SENT, dtype=torch.float32, device="cuda")]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert scale is not None or ws == 1.0
    keep = []
    for c0 in range(0, cout, 128):
        c1 = min(cout, c0 + 128)
        npd = n_pad or _n_pad(c1 - c0)
        sk = None if scale is None else (scale[c0:c1] / ws).float().contiguous()
        sh = None if shift is None else shift[c0:c1].float().contiguous()
        if transpose:
            subs = [((a, c), w[:, c0:c1, a, c].t().unsqueeze(0)) for a in range(k) for c in range(k)]
            geo = dict(kh=1, kw=1, stride=1, pad=0, Hg=H, Wg=W, mul=k)
        else:
            subs = [((0, 0), w[c0:c1].permute(2, 3, 0, 1).reshape(k * k, c1 - c0, cin))]
            geo = dict(kh=k, kw=k, stride=stride, pad=pad, Hg=Ho, Wg=Wo, mul=1)
        for (oh, ow), wt in subs:
            w_hi, w_lo = tc.split_f16(tc._pad_rows(wt.contiguous().float(), npd), ws)
            esz = out[0].element_size()
            o_hi = ctypes.c_void_p(out[0].data_ptr() + esz * (coff + c0))
            o_lo = ctypes.c_void_p(out[1].data_ptr() + esz * (coff + c0)) if planes == 2 else None
            R, wl, wn, bl, bn, fh, fl, margin = lists if lists is not None else (8, None, None, None, None, None, None, -1)
            keep.append((w_hi, w_lo, sk, sh))
            L.check(lib.b2s_conv2d_tc_ex2(
                L.ptr(hi), L.ptr(lo), B, H, W, cin, L.ptr(w_hi), L.ptr(w_lo), geo["kh"], geo["kw"], geo["stride"],
                geo["pad"], c1 - c0, npd, L.ptr(sk), L.ptr(sh), 1 if relu else 0, geo["Hg"], geo["Wg"], o_hi, o_lo,
                Ho, Wo, 1 if planes == 2 else 0, out_stride, geo["mul"], oh, ow, L.ptr(wl), L.ptr(wn), L.ptr(bl),
                L.ptr(bn), L.ptr(fh), L.ptr(fl), margin, R, L.ptr(status), L.stream()), "b2s_conv2d_tc_ex2")
    torch.cuda.synchronize()
    return out, int(status.item()), (Ho, Wo)


def interior(out, planes, coff, cout):
    """-> (merged value NCHW float64, lo plane NCHW float64 or None) of channels coff .. coff+cout"""
    if planes == 2:
        hi, lo = (o[:, 1:-1, 1:-1, coff:coff + cout].permute(0, 3, 1, 2).double() for o in out)
        return hi + lo, lo
    return out[0][..., coff:coff + cout].permute(0, 3, 1, 2).double(), None


def assert_sentinels(out, planes, coff, cout):
    """everything outside channels coff .. coff+cout of the interior still holds the sentinel"""
    for p, o in enumerate(out):
        sent = (HI_SENT, LO_SENT)[p] if planes == 2 else F32_SENT
        m = torch.ones(o.shape, dtype=torch.bool, device=o.device)
        if planes == 2:
            m[:, 1:-1, 1:-1, coff:coff + cout] = False
        else:
            m[..., coff:coff + cout] = False
        assert bool((o[m] == sent).all()), "plane %d written outside its output" % p


def assert_faults_rejected(got, lo, x, w, ws, ref, relu, what, e=0, **conv):
    if e >= tc_ref.F1_MIN_EXP:
        tc_ref.assert_rejected(tc_ref.dense_f1(got, x, w, ws, ref, relu, **conv), ref, ws, what + " F1")
    tc_ref.assert_rejected(tc_ref.dense_f2(got, x, w, ws, ref, relu, **conv), ref, ws, what + " F2")
    tc_ref.assert_rejected(tc_ref.f3(got, lo), ref, ws, what + " F3")
