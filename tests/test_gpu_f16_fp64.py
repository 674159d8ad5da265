"""The single-product (f16 mode) tensor-core kernels against a float64 reference, on every layer shape of car.fhd,
car.lite, all.fhd, pointpillars.car.xyres_16 and nuscenes.all.pp.largea: the dense RPN ops (k_conv3x3_tc2, k_conv_tc),
the sparse middle encoder (k_sparse_conv_tc), the fused deblock + heads tail (k_rpn_tail) and the plane producers.

In the f16 mode every operand is ONE fp16 plane: an activation a is carried as fp16(a), a weight w (pre-scaled by the
power of two ws = b2second.tc.pow2_scale) as fp16(w * ws) / ws.  With u = 2^-11 each rounding errs by at most u
relative, or 2^-25 absolute below the fp16 normal range (2^-25 / ws for a weight), so one product errs by at most
(2u + u^2) |a w| + 2^-25 (1 + u) (|w| + |a| / ws) + 2^-50 / ws, and the per-element bound is

    |y - y64| <= |s| ((2u + u^2) S1 + 2^-25 (1 + u) (Sw + Sa / ws) + ALPHA 2^-23 S1) + out

with S1, Sa, Sw and the fp32 accumulation term ALPHA 2^-23 S1 as in tests/tc_ref.py (the 3xF16 bound), and out the
output rounding: u |y64| + 2^-25 for an fp16 plane, 2^-22 |y64| + 2^-25 for fp32 records.  The bound is not vacuous:
every case also shows elements whose error exceeds the 3xF16 bound of tc_ref.
"""
import ctypes

import pytest
import torch

import engine_ref as E
import tc_ref
from tc_launch import F32_SENT, HI_SENT, pad_nhwc

pytestmark = pytest.mark.gpu

U = 2.0 ** -11
CONFIGS = ["car.fhd", "car.lite", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea"]


@pytest.fixture(autouse=True)
def _fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def f16_check(got, ref, ws, f16_out, extra=0.0, what=""):
    """the per-element f16 bound (module docstring); -> share of elements beyond the 3xF16 bound of tc_ref"""
    err = (got.to(ref.y.device, torch.float64) - ref.y).abs()
    unit, rest3 = tc_ref._terms(ref, ws)
    rounding = ref.s * ((2 * U + U * U) * ref.S1 + 2.0 ** -25 * (1 + U) * (ref.Sw + ref.Sa / ws) + 2.0 ** -40)
    out = (U if f16_out else 2.0 ** -22) * ref.pre.abs() + 2.0 ** -25
    bound = tc_ref.ALPHA * unit + rounding + out + extra
    ratio = float((err / bound).max()) if err.numel() else 0.0
    assert ratio <= 1.0, "%s: |y - y64| reaches %.3g x the f16 bound" % (what, ratio)
    beyond = float((err > tc_ref.ALPHA * unit + rest3 + extra).double().mean())
    assert beyond > 0, "%s: the f16 error never exceeds the 3xF16 bound (the bound would be vacuous)" % what
    return beyond


# ---- shapes --------------------------------------------------------------------------------------------------------
_SHAPES = {}


def shapes(product, name):
    """(the f16 engine's RPN ops, its tensor-pipe sparse layers) for config `name` at batch 1"""
    if name not in _SHAPES:
        from b2second import config, models
        from b2second.engine import InferenceEngine
        net = models.build_network(config.get_config(name), product).eval()
        models.synthetic_weights_(net, name, seed=0)
        eng = InferenceEngine(net.cuda(), batch_size=1, max_points=2000, precision="f16")
        ops = [{k: v for k, v in op.items() if not isinstance(v, torch.Tensor)} for op in eng.tc_plan]
        sparse = [(l["cin"], l["cin_tc"], l["cout"], l["K"]) for l in eng.layers if l["tc"]]
        _SHAPES[name] = (ops, sparse, eng.tc_tail_fused)
        del eng
    return _SHAPES[name]


def launch_f16(product, x, w, ws, k, stride, pad, transpose, scale, shift, relu, planes, out_stride, n_pad):
    """one layer as b2s_conv2d_tc_ex3 launches with products = 1 (output channels in slices of <= 128, a
    ConvTranspose2d k = s as k*k sub-grid launches) -> (output map, status)"""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, cin, H, W = x.shape
    cout = w.shape[1] if transpose else w.shape[0]
    xin = tc.split_f16(pad_nhwc(x))[0]
    Ho, Wo = (H * k, W * k) if transpose else ((H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1)
    if planes == 2:
        out = torch.full((B, Ho + 2, Wo + 2, out_stride), HI_SENT, dtype=torch.float16, device="cuda")
    else:
        out = torch.full((B, Ho, Wo, out_stride), F32_SENT, dtype=torch.float32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    keep = []
    for c0 in range(0, cout, 128):
        c1 = min(cout, c0 + 128)
        npd = n_pad or tc._n_pad(c1 - c0)
        sk = None if scale is None else (scale[c0:c1] / ws).float().contiguous()
        sh = None if shift is None else shift[c0:c1].float().contiguous()
        if transpose:
            subs = [((a, c), w[:, c0:c1, a, c].t().unsqueeze(0)) for a in range(k) for c in range(k)]
            geo = dict(kh=1, kw=1, stride=1, pad=0, Hg=H, Wg=W, mul=k)
        else:
            subs = [((0, 0), w[c0:c1].permute(2, 3, 0, 1).reshape(k * k, c1 - c0, cin))]
            geo = dict(kh=k, kw=k, stride=stride, pad=pad, Hg=Ho, Wg=Wo, mul=1)
        for (oh, ow), wt in subs:
            w_hi, w_lo = tc.weight_planes(tc._pad_rows(wt.contiguous().float(), npd), ws, 1)
            assert w_lo is None
            keep.append((w_hi, sk, sh))
            L.check(lib.b2s_conv2d_tc_ex3(
                L.ptr(xin), None, B, H, W, cin, L.ptr(w_hi), None, geo["kh"], geo["kw"], geo["stride"], geo["pad"],
                c1 - c0, npd, L.ptr(sk), L.ptr(sh), 1 if relu else 0, geo["Hg"], geo["Wg"],
                ctypes.c_void_p(out.data_ptr() + out.element_size() * c0), None, Ho, Wo, 1 if planes == 2 else 0,
                out_stride, geo["mul"], oh, ow, None, None, None, None, None, None, -1, 8, 1,
                0 if planes == 2 else 1, L.ptr(status), L.stream()), "b2s_conv2d_tc_ex3")
    torch.cuda.synchronize()
    return out, int(status.item())


def op_geometry(op):
    """(k, stride, pad, transpose) of the layer a tc_plan op belongs to"""
    if op["out_mul"] > 1 and op["kh"] == 1:
        return op["out_mul"], op["out_mul"], 0, True
    return op["kh"], op["stride"], op["pad"], False


def check_dense_f16(product, B, cin, cout, H, W, k, stride, pad, transpose, planes, n_pad, seed, what):
    from b2second import tc
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, cin, H, W, device="cuda", generator=g)
    if planes == 2:
        x = torch.relu(x)                          # RPN activations: ReLU outputs (the first layer's BEV included)
    w = torch.randn(*((cin, cout, k, k) if transpose else (cout, cin, k, k)), device="cuda", generator=g)
    w = w * (2.0 / (k * k * cin)) ** 0.5
    scale = torch.rand(cout, device="cuda", generator=g) + 0.5
    shift = torch.randn(cout, device="cuda", generator=g) * 0.1
    relu = planes == 2
    ws = tc.pow2_scale(w)
    out_stride = cout + (-cout) % 8 if planes == 2 else max(32, cout + (-cout) % 4)
    out, status = launch_f16(product, x, w, ws, k, stride, pad, transpose, scale, shift, relu, planes, out_stride,
                             n_pad)
    assert status == 0
    if planes == 2:
        got = out[:, 1:-1, 1:-1, :cout].permute(0, 3, 1, 2).double()
        m = torch.ones(out.shape, dtype=torch.bool, device="cuda")
        m[:, 1:-1, 1:-1, :cout] = False
        assert bool((out[m] == HI_SENT).all()), "written outside the output"
    else:
        got = out[..., :cout].permute(0, 3, 1, 2).double()
    ref = tc_ref.dense_ref(x, w, scale, shift, relu, stride=stride, padding=pad, transpose=transpose)
    return f16_check(got, ref, ws, planes == 2, what=what)


@pytest.mark.parametrize("name", CONFIGS)
def test_dense_ops_of_each_config(product, name):
    """every distinct RPN layer of the config (the fused tail's two ops included, as separate launches)"""
    ops, _, _ = shapes(product, name)
    seen = set()
    for i, op in enumerate(ops):
        if op["kind"] == "crop":
            continue
        k, stride, pad, transpose = op_geometry(op)
        cout = op["cout"]
        key = (op["cin"], cout, op["Hin"], op["Win"], k, stride, pad, transpose, op["planes"], op["n_pad"])
        if key in seen:
            continue
        seen.add(key)
        check_dense_f16(product, 1, op["cin"], cout, op["Hin"], op["Win"], k, stride, pad, transpose, op["planes"],
                        op["n_pad"] if not transpose else None, i, "%s op %d (%s)" % (name, i, op["kind"]))
    assert seen


@pytest.mark.parametrize("B,H,W", [(2, 9, 17), (1, 1, 1), (3, 21, 36)])
def test_dense_small_and_ragged_maps(product, B, H, W):
    """partial tiles and strips at the map edge, several frames"""
    check_dense_f16(product, B, 128, 128, H, W, 3, 1, 1, False, 2, 128, 7, "3x3 v2")
    check_dense_f16(product, B, 64, 64, H, W, 3, 1, 1, False, 2, 64, 8, "3x3 n_pad 64")
    check_dense_f16(product, B, 128, 128, H, W, 3, 2, 1, False, 2, None, 9, "3x3 stride 2")
    check_dense_f16(product, B, 128, 128, H, W, 2, 2, 0, True, 2, None, 10, "deblock k = 2")
    check_dense_f16(product, B, 128, 20, H, W, 1, 1, 0, False, 1, 32, 11, "heads")


# ---- sparse ----------------------------------------------------------------------------------------------------------
def run_sparse_f16(product, x, w, nbr, scale, shift, relu, cin_tc, n_out):
    from b2second import tc
    L = product._lib
    lib = L.load()
    n_in, cin = x.shape
    K, _, cout = w.shape
    wp = tc.pack_sparse_weights(w)
    ws = tc.pow2_scale(wp)
    w_hi, w_lo = tc.weight_planes(wp, ws, 1)
    assert w_lo is None
    rows = torch.full((n_in, cin_tc), HI_SENT, dtype=torch.float16, device="cuda")
    n_in_dev = torch.tensor([n_in], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_split_f16_ex(L.ptr(x), L.ptr(rows), None, L.ptr(n_in_dev), n_in, cin, cin_tc, cin_tc, 1,
                                 L.stream()), "b2s_split_f16_ex")
    torch.cuda.synchronize()
    assert torch.equal(rows[:, :cin].view(torch.int16), tc.split_f16(x)[0].view(torch.int16))
    assert bool((rows[:, cin:] == 0).all())
    out = torch.full((n_out + 5, cout), HI_SENT, dtype=torch.float16, device="cuda")
    n_out_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    sk = (scale / ws).float().contiguous()
    L.check(lib.b2s_sparse_conv_tc_plan_ex(L.ptr(rows), None, cin_tc, n_in, cin_tc, L.ptr(w_hi), None, L.ptr(nbr), K,
                                           L.ptr(n_out_dev), n_out + 5, None, None, L.ptr(sk), L.ptr(shift),
                                           1 if relu else 0, L.ptr(out), None, cout, cout, 1, L.ptr(status),
                                           L.stream()), "b2s_sparse_conv_tc_plan_ex")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert bool((out[n_out:] == HI_SENT).all()), "rows past the live count written"
    return out[:n_out], ws


@pytest.mark.parametrize("name", CONFIGS)
def test_sparse_layers_of_each_config(product, name):
    _, sparse, _ = shapes(product, name)
    if not sparse:
        pytest.skip("%s has no sparse middle encoder" % name)
    for j, (cin, cin_tc, cout, K) in enumerate(sorted(set(sparse))):
        g = torch.Generator(device="cuda").manual_seed(100 + j)
        n_in, n_out = 4000, 3000
        x = torch.randn(n_in, cin, device="cuda", generator=g)
        if j:
            x = torch.relu(x)
        w = torch.randn(K, cin, cout, device="cuda", generator=g) * (2.0 / (K * cin)) ** 0.5
        nbr = torch.randint(0, n_in, (n_out, K), device="cuda", generator=g, dtype=torch.int32)
        nbr[torch.rand(n_out, K, device="cuda", generator=g) < 0.6] = -1
        scale = torch.rand(cout, device="cuda", generator=g) + 0.5
        shift = torch.randn(cout, device="cuda", generator=g) * 0.1
        got, ws = run_sparse_f16(product, x, w, nbr, scale, shift, True, cin_tc, n_out)
        ref = tc_ref.sparse_ref(x, w, nbr, scale, shift, True)
        f16_check(got.double(), ref, ws, True, what="%s sparse %d -> %d, K %d" % (name, cin, cout, K))


# ---- fused tail ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["car.fhd", "car.lite"])
def test_fused_tail_equals_the_two_launches(product, name):
    """b2s_rpn_tail_tc_ex2 (products 1) writes, bit for bit, what the deblock and heads launches of the f16 mode write
    (each checked against float64 above), with and without a tile work list"""
    from b2second import tc
    ops, _, fused = shapes(product, name)
    assert fused
    d, h = ops[-2], ops[-1]
    L = product._lib
    lib = L.load()
    B, H, W = 2, d["Hin"], d["Win"]
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.relu(torch.randn(B, H + 2, W + 2, 128, device="cuda", generator=g)).half()
    x[:, 0], x[:, -1], x[:, :, 0], x[:, :, -1] = 0, 0, 0, 0
    w1 = torch.randn(1, 128, 128, device="cuda", generator=g) * 0.1
    w2 = tc._pad_rows(torch.randn(1, h["cout"], 128, device="cuda", generator=g) * 0.1, 32)
    ws1, ws2 = tc.pow2_scale(w1), tc.pow2_scale(w2)
    w1h, w2h = tc.weight_planes(w1, ws1, 1)[0], tc.weight_planes(w2, ws2, 1)[0]
    s1 = (torch.rand(128, device="cuda", generator=g) + 0.5) / ws1
    sh1 = torch.randn(128, device="cuda", generator=g) * 0.1
    s2 = torch.ones(h["cout"], device="cuda") / ws2
    sh2 = torch.randn(h["cout"], device="cuda", generator=g) * 0.1
    stride = 32
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    # two launches
    y = torch.zeros(B, H + 2, W + 2, 128, dtype=torch.float16, device="cuda")
    L.check(lib.b2s_conv2d_tc_ex3(L.ptr(x), None, B, H, W, 128, L.ptr(w1h), None, 1, 1, 1, 0, 128, 128, L.ptr(s1),
                                  L.ptr(sh1), 1, H, W, L.ptr(y), None, H, W, 1, 128, 1, 0, 0, None, None, None, None,
                                  None, None, -1, 8, 1, 0, L.ptr(status), L.stream()), "deblock")
    two = torch.full((B, H, W, stride), F32_SENT, dtype=torch.float32, device="cuda")
    L.check(lib.b2s_conv2d_tc_ex3(L.ptr(y), None, B, H, W, 128, L.ptr(w2h), None, 1, 1, 1, 0, h["cout"], 32, L.ptr(s2),
                                  L.ptr(sh2), 0, H, W, L.ptr(two), None, H, W, 0, stride, 1, 0, 0, None, None, None,
                                  None, None, None, -1, 8, 1, 1, L.ptr(status), L.stream()), "heads")
    fused_out = torch.full_like(two, F32_SENT)
    L.check(lib.b2s_rpn_tail_tc_ex2(L.ptr(x), None, B, H, W, 128, L.ptr(w1h), None, 128, L.ptr(s1), L.ptr(sh1),
                                    L.ptr(w2h), None, h["cout"], 32, L.ptr(s2), L.ptr(sh2), L.ptr(fused_out), stride,
                                    None, None, None, None, None, -1, 1, L.ptr(status), L.stream()), "tail")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(fused_out.view(torch.int32), two.view(torch.int32))
    # a work list of every other tile: those tiles equal, the others untouched
    tiles = B * (-(-H // 8)) * (-(-W // 16))
    work = torch.arange(0, tiles, 2, dtype=torch.int32, device="cuda")
    cnt = torch.tensor([work.numel()], dtype=torch.int32, device="cuda")
    part = torch.full_like(two, F32_SENT)
    L.check(lib.b2s_rpn_tail_tc_ex2(L.ptr(x), None, B, H, W, 128, L.ptr(w1h), None, 128, L.ptr(s1), L.ptr(sh1),
                                    L.ptr(w2h), None, h["cout"], 32, L.ptr(s2), L.ptr(sh2), L.ptr(part), stride,
                                    L.ptr(work), L.ptr(cnt), None, None, None, -1, 1, L.ptr(status), L.stream()),
            "tail (work list)")
    torch.cuda.synchronize()
    tw, th = -(-W // 16), -(-H // 8)
    for t in range(tiles):
        b, r = divmod(t, th * tw)
        sl = (b, slice((r // tw) * 8, (r // tw) * 8 + 8), slice((r % tw) * 16, (r % tw) * 16 + 16))
        if t % 2 == 0:
            assert torch.equal(part[sl].view(torch.int32), two[sl].view(torch.int32)), t
        else:
            assert bool((part[sl] == F32_SENT).all()), t


# ---- plane producers -------------------------------------------------------------------------------------------------
def test_bev_scatter_and_crop_single_plane(product):
    """b2s_to_bev_tc_ex2 and b2s_crop_nhwc_ex with products 1 write exactly the hi planes of the 3xF16 calls and
    nothing else"""
    L = product._lib
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(2)
    B, D, H, W, C, n = 2, 2, 20, 24, 64, 300
    coors = torch.stack([torch.randint(0, B, (n,)), torch.randint(0, D, (n,)), torch.randint(0, H, (n,)),
                         torch.randint(0, W, (n,))], 1).int().cuda()
    coors = torch.unique(coors, dim=0).contiguous()
    n = coors.shape[0]
    feats = torch.randn(n, C, device="cuda", generator=g) * 3
    n_dev = torch.tensor([n], dtype=torch.int32, device="cuda")
    planes3 = [torch.zeros(B, H + 2, W + 2, C * D, dtype=torch.float16, device="cuda") for _ in range(2)]
    occ3 = torch.zeros(B, H, W, dtype=torch.uint8, device="cuda")
    plane1 = torch.zeros(B, H + 2, W + 2, C * D, dtype=torch.float16, device="cuda")
    occ1 = torch.zeros_like(occ3)
    for _ in range(2):           # the second call clears what the first wrote
        L.check(lib.b2s_to_bev_tc_ex(L.ptr(feats), None, None, 0, L.ptr(coors), L.ptr(n_dev), n, C, B, D, H, W,
                                     L.ptr(planes3[0]), L.ptr(planes3[1]), L.ptr(occ3), L.stream()), "3xF16")
        L.check(lib.b2s_to_bev_tc_ex2(L.ptr(feats), None, None, 0, L.ptr(coors), L.ptr(n_dev), n, C, B, D, H, W,
                                      L.ptr(plane1), None, L.ptr(occ1), 1, L.stream()), "f16")
        torch.cuda.synchronize()
        assert torch.equal(plane1.view(torch.int16), planes3[0].view(torch.int16)) and torch.equal(occ1, occ3)
        feats = feats[:n // 2].contiguous()
        n_dev.fill_(n // 2)
    # from single-plane rows
    rows = torch.randn(n, C, device="cuda", generator=g).half()
    L.check(lib.b2s_to_bev_tc_ex2(None, L.ptr(rows), None, C, L.ptr(coors), L.ptr(n_dev), n, C, B, D, H, W,
                                  L.ptr(plane1), None, L.ptr(occ1), 1, L.stream()), "f16 rows")
    torch.cuda.synchronize()
    m = n // 2
    q = coors[:m].long()
    got = plane1[q[:, 0], q[:, 2] + 1, q[:, 3] + 1].view(m, C, D)[torch.arange(m), :, q[:, 1]]
    assert torch.equal(got.view(torch.int16), rows[:m].view(torch.int16))
    # crop
    c = E.crop_size(H)
    dst3 = [torch.full((B, H - 2 * c + 2, W - 2 * c + 2, C * D), 9.0, dtype=torch.float16, device="cuda")
            for _ in range(2)]
    dst1 = torch.full_like(dst3[0], 9.0)
    L.check(lib.b2s_crop_nhwc(L.ptr(planes3[0]), L.ptr(planes3[1]), B, H, W, C * D, c, L.ptr(dst3[0]), L.ptr(dst3[1]),
                              L.stream()), "crop 3xF16")
    L.check(lib.b2s_crop_nhwc_ex(L.ptr(plane1), None, B, H, W, C * D, c, L.ptr(dst1), None, 1, L.stream()),
            "crop f16")
    torch.cuda.synchronize()
    want = torch.zeros_like(dst1)
    want[:, 1:-1, 1:-1] = plane1[:, 1 + c:H + 1 - c, 1 + c:W + 1 - c]
    assert torch.equal(dst1.view(torch.int16), want.view(torch.int16))
