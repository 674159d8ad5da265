"""GPU parity of the tensor-core RPN convolution (b2s_conv2d_tc, wgmma f16 + 3xF16 hi/lo split) against float64 with
the per-element 3xF16 bound of tests/tc_ref.py (single layers), and against torch fp32 conv2d with TF32 disabled (whole
RPN programs, bar 1e-4 on the head outputs)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tc_ref
from tc_launch import assert_faults_rejected

pytestmark = pytest.mark.gpu


def pad_nhwc(x):
    """[B,C,H,W] -> NHWC with one-pixel zero halo [B,H+2,W+2,C]."""
    return F.pad(x.permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).contiguous()


def run_tc(product, x, w_tco_ci, taps, cout, n_pad, scale, shift, relu, out_padded, out_stride, want_lo=True):
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, C, H, W = x.shape
    hi, lo = tc.split_f16(pad_nhwc(x))
    wp = tc._pad_rows(w_tco_ci, n_pad)
    ws = tc.pow2_scale(wp)                                    # power-of-two weight pre-scale, undone by `scale`
    w_hi, w_lo = tc.split_f16(wp, ws)
    scale_k = ((scale if scale is not None else torch.ones(cout, device="cuda")) / ws).contiguous()
    shape = (B, H + 2, W + 2, out_stride) if out_padded else (B, H, W, out_stride)
    o_hi = torch.zeros(shape, device="cuda", dtype=torch.float16 if want_lo else torch.float32)
    o_lo = torch.zeros(shape, device="cuda", dtype=torch.float16) if want_lo else None
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_conv2d_tc(L.ptr(hi), L.ptr(lo), B, H, W, C, L.ptr(w_hi), L.ptr(w_lo), taps, cout, n_pad,
                              L.ptr(scale_k), L.ptr(shift), 1 if relu else 0, L.ptr(o_hi), L.ptr(o_lo),
                              1 if out_padded else 0, out_stride, L.ptr(status), L.stream()), "b2s_conv2d_tc")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return o_hi, o_lo


@pytest.fixture(autouse=True)
def _fp32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,H,W,cin,cout", [(1, 8, 16, 64, 128), (2, 24, 40, 128, 128), (1, 200, 176, 128, 128),
                                            (1, 16, 32, 64, 64), (3, 35, 21, 256, 128), (1, 16, 16, 64, 32)])
def test_conv3x3_bn_relu(product, B, H, W, cin, cout):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    x = torch.randn(B, cin, H, W, device="cuda", generator=g)
    w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * (2.0 / (9 * cin)) ** 0.5
    scale = torch.rand(cout, device="cuda", generator=g) + 0.5
    shift = torch.randn(cout, device="cuda", generator=g) * 0.1
    wt = w.permute(2, 3, 0, 1).reshape(9, cout, cin).contiguous()
    n_pad = 128 if cout > 64 else (64 if cout > 32 else 32)
    o_hi, o_lo = run_tc(product, x, wt, 9, cout, n_pad, scale, shift, True, True, cout)
    got = (o_hi.float() + o_lo.float())[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2)
    from b2second import tc
    ws = tc.pow2_scale(tc._pad_rows(wt, n_pad))
    r64 = tc_ref.dense_ref(x, w, scale, shift, True, padding=1)
    tc_ref.assert_accurate(got.double(), r64, ws)
    assert_faults_rejected(got.double(), o_lo[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2).double(), x, w, ws, r64, True, "",
                           padding=1)
    # halo untouched (stays zero); hi is the fp16 rounding of the value and lo the fp16 rounding of the rest
    assert float(o_hi[:, 0].float().abs().sum() + o_hi[:, -1].float().abs().sum() + o_hi[:, :, 0].float().abs().sum()
                 + o_hi[:, :, -1].float().abs().sum()) == 0.0
    hi_in = o_hi.float()[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2)
    assert float(((hi_in - got).abs() - (2.0 ** -11 * got.abs() + 2.0 ** -25)).max()) <= 0.0      # |lo| <= ulp(hi)/2


@pytest.mark.timeout(120)
def test_conv1x1_heads_packed(product):
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, W, cin, cout = 2, 20, 33, 128, 20
    x = torch.randn(B, cin, H, W, device="cuda", generator=g)
    w = torch.randn(cout, cin, 1, 1, device="cuda", generator=g) * 0.1
    bias = torch.randn(cout, device="cuda", generator=g)
    wt = w[:, :, 0, 0].unsqueeze(0).contiguous()
    o, _ = run_tc(product, x, wt, 1, cout, 32, None, bias, False, False, 32, want_lo=False)
    assert o.dtype == torch.float32
    got = o[..., :cout].permute(0, 3, 1, 2).double()
    from b2second import tc
    ws = tc.pow2_scale(tc._pad_rows(wt, 32))
    r64 = tc_ref.dense_ref(x, w, None, bias)
    tc_ref.assert_accurate(got, r64, ws)
    assert_faults_rejected(got, None, x, w, ws, r64, False, "")
    assert float(o[..., cout:].abs().sum()) == 0.0


def run_rpn_plan(product, plan, x_nchw):
    """execute a tc.plan_rpn program with b2s_conv2d_tc_ex; returns the packed heads tensor [B, H, W, S]."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B = x_nchw.shape[0]
    bufs = {"in": tc.split_f16(pad_nhwc(x_nchw))}
    for name, (h, w, c) in plan["buffers"].items():
        bufs[name] = (torch.zeros(B, h + 2, w + 2, c, device="cuda", dtype=torch.float16),
                      torch.zeros(B, h + 2, w + 2, c, device="cuda", dtype=torch.float16))
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    hd = plan["heads"]
    heads = torch.zeros(B, hd["H"], hd["W"], hd["stride"], device="cuda")
    bufs["heads"] = (heads, None)
    keep = []
    for op in plan["ops"]:
        src, dst = bufs[op["src"]], bufs[op["dst"]]
        esz = dst[0].element_size()
        o_hi = ctypes.c_void_p(dst[0].data_ptr() + esz * op["dst_coff"])
        o_lo = ctypes.c_void_p(dst[1].data_ptr() + esz * op["dst_coff"]) if op["planes"] == 2 else None
        keep.append((op["scale"], op["shift"]))
        L.check(lib.b2s_conv2d_tc_ex(
            L.ptr(src[0]), L.ptr(src[1]), B, op["Hin"], op["Win"], op["cin"], L.ptr(op["w_hi"]), L.ptr(op["w_lo"]),
            op["kh"], op["kw"], op["stride"], op["pad"], op["cout"], op["n_pad"],
            L.ptr(op["scale"]),
            L.ptr(op["shift"]) if op["shift"] is not None else None, 1 if op["relu"] else 0, op["Hg"], op["Wg"], o_hi, o_lo,
            op["Hout"], op["Wout"], 1 if op["padded"] else 0, dst[0].shape[-1], op["out_mul"], op["off_h"], op["off_w"],
            None, None, None, None, None, None, L.ptr(status), L.stream()), "b2s_conv2d_tc_ex")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return heads


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,H,W", [("car.fhd", 40, 48), ("all.fhd", 40, 48), ("pointpillars.car.xyres_16", 48, 40),
                                       ("nuscenes.all.pp.largea", 48, 64)])
def test_rpn_program_matches_torch(product, name, H, W):
    """whole RPNV2 of each config family (stride-1 / stride-2 blocks, k=1/2/4 ConvTranspose2d and k=2/4 strided
    Conv2d deblocks, channel concat, 1x1 heads) as a b2s_conv2d_tc_ex program vs the torch modules (fp32)."""
    from b2second import config, models, tc
    cfg = config.get_config(name)
    net = models.build_network(cfg, product).eval()
    models.synthetic_weights_(net, name, seed=0)
    rpn = net.rpn.cuda()
    assert tc.supported(rpn)
    B = 2
    cin = rpn.blocks[0][1].in_channels
    x = torch.relu(torch.randn(B, cin, H, W, device="cuda"))
    x = x * (torch.rand(B, 1, H, W, device="cuda") < 0.15)        # sparse BEV-like input
    with torch.no_grad():
        feat = rpn.backbone(x)
        heads = [rpn.conv_box(feat), rpn.conv_cls(feat)] + ([rpn.conv_dir_cls(feat)] if rpn._use_direction_classifier else [])
        ref = torch.cat(heads, 1)
    plan = tc.plan_rpn(rpn, H, W)
    out = run_rpn_plan(product, plan, x)
    n = ref.shape[1]
    got = out[..., :n].permute(0, 3, 1, 2)
    assert got.shape == ref.shape
    err = (got - ref).abs().max().item()
    assert err <= 1e-4 * max(1.0, ref.abs().max().item()), "head tensors differ by %g (bar 1e-4 on the regression outputs)" % err
    offs = plan["heads"]["offsets"]
    assert offs[-1] == n and offs[0] == 0


@pytest.mark.timeout(120)
def test_fp16_range_guard_raises_status(product):
    """an activation beyond the fp16 range is clamped and reported (B2S_STATUS_F16_RANGE), never turned into inf."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, H, W, cin, cout = 1, 16, 16, 64, 128
    x = torch.full((B, cin, H, W), 30.0, device="cuda")
    w = torch.full((cout, cin, 3, 3), 8.0, device="cuda")          # 64 * 9 * 30 * 8 = 138240 > 65504
    wt = w.permute(2, 3, 0, 1).reshape(9, cout, cin).contiguous()
    hi, lo = tc.split_f16(pad_nhwc(x))
    ws = tc.pow2_scale(wt)
    w_hi, w_lo = tc.split_f16(wt, ws)
    scale = torch.full((cout,), 1.0 / ws, device="cuda")
    o_hi = torch.zeros(B, H + 2, W + 2, cout, device="cuda", dtype=torch.float16)
    o_lo = torch.zeros_like(o_hi)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_conv2d_tc(L.ptr(hi), L.ptr(lo), B, H, W, cin, L.ptr(w_hi), L.ptr(w_lo), 9, cout, 128, L.ptr(scale),
                              None, 0, L.ptr(o_hi), L.ptr(o_lo), 1, cout, L.ptr(status), L.stream()), "b2s_conv2d_tc")
    torch.cuda.synchronize()
    assert int(status.item()) & 16
    assert bool(torch.isfinite(o_hi.float()).all()) and float(o_hi.float().max()) == 65504.0


@pytest.mark.timeout(180)
@pytest.mark.parametrize("B,H,W", [(2, 20, 33), (1, 200, 176), (3, 8, 16), (1, 5, 7)])
def test_fused_rpn_tail_is_bit_identical_to_two_launches(product, B, H, W):
    """b2s_rpn_tail_tc (deblock 1x1 + BN + ReLU -> packed heads in one kernel, the deblock output stays in shared memory)
    against the two b2s_conv2d_tc launches it replaces: same MMA sequences, same epilogue arithmetic => identical bits;
    and both against torch fp32 (rpn.py:264-299, 386-420)."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(B * 100 + H)
    cin, cmid, cout = 128, 128, 20
    x = torch.randn(B, cin, H, W, device="cuda", generator=g)
    w1 = torch.randn(cmid, cin, device="cuda", generator=g) * (2.0 / cin) ** 0.5          # [y channel, x channel]
    scale1 = torch.rand(cmid, device="cuda", generator=g) + 0.5
    shift1 = torch.randn(cmid, device="cuda", generator=g) * 0.1
    w2 = torch.randn(cout, cmid, device="cuda", generator=g) * 0.1
    bias2 = torch.randn(cout, device="cuda", generator=g) * 0.1
    # two launches
    y_hi, y_lo = run_tc(product, x, w1.unsqueeze(0).contiguous(), 1, cmid, 128, scale1, shift1, True, True, cmid)
    hi, lo = tc.split_f16(pad_nhwc(x))
    wp2 = tc._pad_rows(w2.unsqueeze(0).contiguous(), 32)
    ws2 = tc.pow2_scale(wp2)
    w2_hi, w2_lo = tc.split_f16(wp2, ws2)
    scale2 = (torch.ones(cout, device="cuda") / ws2).contiguous()
    two = torch.zeros(B, H, W, 32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_conv2d_tc(L.ptr(y_hi), L.ptr(y_lo), B, H, W, cmid, L.ptr(w2_hi), L.ptr(w2_lo), 1, cout, 32,
                              L.ptr(scale2), L.ptr(bias2), 0, L.ptr(two), None, 0, 32, L.ptr(status), L.stream()),
            "b2s_conv2d_tc")
    # one launch
    wp1 = tc._pad_rows(w1.unsqueeze(0).contiguous(), 128)
    ws1 = tc.pow2_scale(wp1)
    w1_hi, w1_lo = tc.split_f16(wp1, ws1)
    scale1_k = (scale1 / ws1).contiguous()
    one = torch.full((B, H, W, 32), 7.0, device="cuda")
    L.check(lib.b2s_rpn_tail_tc(L.ptr(hi), L.ptr(lo), B, H, W, cin, L.ptr(w1_hi), L.ptr(w1_lo), cmid, L.ptr(scale1_k),
                                L.ptr(shift1), L.ptr(w2_hi), L.ptr(w2_lo), cout, 32, L.ptr(scale2), L.ptr(bias2),
                                L.ptr(one), 32, L.ptr(status), L.stream()), "b2s_rpn_tail_tc")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(one[..., :cout], two[..., :cout]), "fused tail differs from the two-launch path"
    assert bool((one[..., cout:] == 7.0).all())                       # channels past Cout are not written
    # against float64, stage by stage: the deblock output (the first launch's planes) from x, the heads from those planes
    # (the values the fused kernel consumes, bit-identical to the first launch's)
    r1 = tc_ref.dense_ref(x, w1.view(cmid, cin, 1, 1), scale1, shift1, True)
    y = (y_hi.float() + y_lo.float())[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2)
    y_lo64 = y_lo[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2).double()
    tc_ref.assert_accurate(y.double(), r1, ws1, "deblock")
    assert_faults_rejected(y.double(), y_lo64, x, w1.view(cmid, cin, 1, 1), ws1, r1, True, "deblock")
    r2 = tc_ref.dense_ref(y, w2.view(cout, cmid, 1, 1), None, bias2)
    got = one[..., :cout].permute(0, 3, 1, 2).double()
    tc_ref.assert_accurate(got, r2, ws2, "heads")
    assert_faults_rejected(got, None, y, w2.view(cout, cmid, 1, 1), ws2, r2, False, "heads")
