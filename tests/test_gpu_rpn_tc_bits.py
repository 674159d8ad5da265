"""Bit-level regression of the dense RPN kernels (k_conv3x3_tc2, k_conv_tc, k_rpn_tail): the output planes of fixed
seeded layers must be the exact bits recorded in tests/golden/rpn_tc_bits.json.  A change to scheduling, background
skipping or tiling may not change a single bit; a change that means to change results re-records the fixture:
    python tests/test_gpu_rpn_tc_bits.py OUT.json

Cases: the 3x3 stride-1 layer (dense launches at 200x176 and 21x36, B = 3, Cin 128 and 256, one into channel 128 of a
256-channel map; the 21x36 layer again as strip-list launches of R = 8, 4 and 2 rows with background lists and a
bg_margin, whose listed strips must equal the dense planes), a 3x3 stride-2 conv, a ConvTranspose2d k = 2 sub-grid
launch set into a channel offset, the fp32 heads with a second slice at channel 128, and b2s_rpn_tail_tc.
Inputs come from seeded numpy and are split into hi/lo planes on the host (b2second.tc.split_f16)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

from tc_launch import launch_dense, pad_nhwc

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rpn_tc_bits.json")
# name: (B, Cin, Cout, H, W, k, stride, pad, transpose, planes, out_stride, coff)
LAYERS = {
    "v2_200x176_cin128": (3, 128, 128, 200, 176, 3, 1, 1, False, 2, None, 0),
    "v2_21x36_cin256_coff128": (3, 256, 128, 21, 36, 3, 1, 1, False, 2, 256, 128),
    "v2_21x36_cin128": (3, 128, 128, 21, 36, 3, 1, 1, False, 2, None, 0),
    "conv_3x3_s2": (3, 128, 128, 17, 23, 3, 2, 1, False, 2, None, 0),
    "deconv_k2_coff128": (2, 128, 128, 21, 36, 2, 2, 0, True, 2, 256, 128),
    "heads_fp32_148": (2, 384, 148, 21, 36, 1, 1, 0, False, 1, 160, 0),
}
LIST_ROWS = (8, 4, 2)
CASES = sorted(list(LAYERS) + ["v2_21x36_cin128_list%d" % r for r in LIST_ROWS] + ["rpn_tail"])


def _digest(ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def _layer(name):
    B, cin, cout, H, W, k, stride, pad, transpose, planes, out_stride, coff = LAYERS[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x = torch.from_numpy(rng.standard_normal((B, cin, H, W)).astype(np.float32))
    wshape = (cin, cout, k, k) if transpose else (cout, cin, k, k)
    w = torch.from_numpy((rng.standard_normal(wshape) * (2.0 / (k * k * cin)) ** 0.5).astype(np.float32))
    scale = torch.from_numpy((rng.random(cout) + 0.5).astype(np.float32))
    shift = torch.from_numpy((rng.standard_normal(cout) * 0.1).astype(np.float32))
    from b2second import tc
    hi, lo = tc.split_f16(pad_nhwc(x))
    return dict(x=x.cuda(), w=w.cuda(), ws=tc.pow2_scale(w), k=k, stride=stride, pad=pad, transpose=transpose,
                scale=scale.cuda(), shift=None if planes == 1 else shift.cuda(), relu=planes == 2, planes=planes,
                out_stride=out_stride, coff=coff, in_planes=(hi.cuda(), lo.cuda()))


def _run_layer(product, d, lists=None):
    out, status, hw = launch_dense(product, d["x"], d["w"], d["ws"], d["k"], d["stride"], d["pad"], d["transpose"],
                                   d["scale"], d["shift"], d["relu"], d["planes"], d["out_stride"], d["coff"],
                                   in_planes=d["in_planes"], lists=lists)
    assert status == 0
    return out


def _list_case(product, R):
    """the v2_21x36_cin128 layer as a strip-list launch; listed strips checked against the dense planes"""
    L = product._lib
    lib = L.load()
    d = _layer("v2_21x36_cin128")
    B, _, H, W = d["x"].shape
    C = 128
    rng = np.random.default_rng(77)
    occ = (rng.random((B, H, W)) < 0.02).astype(np.uint8)
    occ[1] = 0
    occ[2, H - 1, W - 1] = 1
    sh_n, sw_n = -(-H // R), -(-W // 8)
    ns = B * sh_n * sw_n
    scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device="cuda")
    flags, work, bg = (torch.zeros(1, ns, dtype=torch.int32, device="cuda") for _ in range(3))
    counts = torch.zeros(1, 2, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_strip_plan(L.ptr(torch.from_numpy(occ).cuda()), B, H, W, 1, R, L.ptr(scratch), L.ptr(flags),
                                   L.ptr(work), L.ptr(bg), L.ptr(counts), L.stream()), "b2s_rpn_strip_plan")
    margin = 2
    field = torch.from_numpy(rng.standard_normal((2, H + 2, W + 2, C)).astype(np.float16))
    field[:, 1 + margin:H + 1 - margin, 1 + margin:W + 1 - margin] = field[:, 1 + H // 2, 1 + W // 2][:, None, None]
    field = field.cuda()
    lists = (R, work[0], counts[0, 0:1].contiguous(), bg[0], counts[0, 1:2].contiguous(), field[0], field[1], margin)
    got = _run_layer(product, d, lists)
    dense = _run_layer(product, d)
    nw = int(counts[0, 0])
    assert 0 < nw < ns
    for s in work[0, :nw].tolist():
        b, sh, sw = s // (sh_n * sw_n), (s // sw_n) % sh_n, s % sw_n
        sl = (b, slice(1 + sh * R, 1 + min(H, sh * R + R)), slice(1 + sw * 8, 1 + min(W, sw * 8 + 8)))
        for p in range(2):
            assert torch.equal(got[p][sl], dense[p][sl]), (R, s)
    return got


def _tail_case(product):
    from b2second import tc
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(31)
    B, H, W, cin, cmid, cout = 2, 20, 33, 128, 128, 20
    x = torch.from_numpy(rng.standard_normal((B, cin, H, W)).astype(np.float32))
    f = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32))
    w1, w2 = f(cmid, cin) * (2.0 / cin) ** 0.5, f(cout, cmid) * 0.1
    scale1 = torch.from_numpy((rng.random(cmid) + 0.5).astype(np.float32))
    shift1, bias2 = f(cmid) * 0.1, f(cout) * 0.1
    hi, lo = (t.cuda() for t in tc.split_f16(pad_nhwc(x)))
    wp1, wp2 = tc._pad_rows(w1.unsqueeze(0), 128), tc._pad_rows(w2.unsqueeze(0), 32)
    ws1, ws2 = tc.pow2_scale(wp1), tc.pow2_scale(wp2)
    w1_hi, w1_lo = (t.cuda() for t in tc.split_f16(wp1, ws1))
    w2_hi, w2_lo = (t.cuda() for t in tc.split_f16(wp2, ws2))
    s1, sh1 = (scale1 / ws1).cuda(), shift1.cuda()
    s2, b2 = (torch.ones(cout) / ws2).cuda(), bias2.cuda()
    out = torch.full((B, H, W, 32), 7.0, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_tail_tc(L.ptr(hi), L.ptr(lo), B, H, W, cin, L.ptr(w1_hi), L.ptr(w1_lo), cmid, L.ptr(s1),
                                L.ptr(sh1), L.ptr(w2_hi), L.ptr(w2_lo), cout, 32, L.ptr(s2), L.ptr(b2), L.ptr(out), 32,
                                L.ptr(status), L.stream()), "b2s_rpn_tail_tc")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return [out]


def run_case(product, name):
    if name == "rpn_tail":
        out = _tail_case(product)
    elif name.startswith("v2_21x36_cin128_list"):
        out = _list_case(product, int(name[len("v2_21x36_cin128_list"):]))
    else:
        out = _run_layer(product, _layer(name))
    return _digest(out)


@pytest.mark.parametrize("name", CASES)
def test_rpn_tc_bits_unchanged(product, name):
    with open(FIXTURE) as f:
        want = json.load(f)[name]
    assert run_case(product, name) == want


if __name__ == "__main__":
    REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
    from b2second import loader
    sp = loader.product_spconv()
    rec = {}
    for c in CASES:
        rec[c] = run_case(sp, c)
        print(c, rec[c])
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
