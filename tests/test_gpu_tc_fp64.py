"""The tensor-core convolutions against a float64 reference with the per-element 3xF16 bound of tests/tc_ref.py:
  b2s_conv2d_tc_ex2 (k_conv3x3_tc2 and k_conv_tc) at the launch shapes of the RPN programs: channel-offset outputs in
      a wider map, Cout < n_pad, Cin 64 .. 384, maps smaller than one tile, strided and k = s convs, ConvTranspose2d
      sub-grids, fp32 head records past 128 channels; strip-list launches of b2s_rpn_strip_plan
  b2s_sparse_conv_tc / _plan on SubM, strided and (3,1,1)-stride-(2,1,1) tables
  a magnitude sweep of the activations (the bound's absolute terms), the fp16 range boundary of the hi/lo outputs.
Every case writes into sentinel-filled buffers and checks that nothing outside its outputs changed, and asserts that
the simulated faults F1 (thin), F2 (local) and F3 (output lo plane) fail the same check."""
import numpy as np
import pytest
import torch

import tc_ref
from tc_launch import F32_SENT, HI_SENT, LO_SENT, assert_faults_rejected, assert_sentinels, interior, launch_dense

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def check_dense(product, B, cin, cout, H, W, k, stride=1, pad=0, transpose=False, plain=False, planes=2,
                out_stride=None, coff=0, n_pad=None, seed=0, e=0, relu=None, faults=True):
    """random layer -> kernel vs float64, sentinels, status, faults rejected; -> error_stats"""
    from b2second import tc
    g = torch.Generator(device="cuda").manual_seed(seed * 1000 + cin + cout + H * 7 + W + k)
    x = torch.randn(B, cin, H, W, device="cuda", generator=g) * 2.0 ** e
    wshape = (cin, cout, k, k) if transpose else (cout, cin, k, k)
    w = torch.randn(*wshape, device="cuda", generator=g)
    if plain:
        # scale = NULL: the weights go in unscaled (ws = 1), so they are drawn at unit size, where their lo planes are
        # mostly normal fp16 (the bound's 2^-25 * Sa / ws term would otherwise hide F1)
        scale, shift, relu, ws = None, None, False, 1.0
    else:
        w = w * (2.0 / (k * k * cin)) ** 0.5
        scale = torch.rand(cout, device="cuda", generator=g) + 0.5
        shift = None if planes == 1 else torch.randn(cout, device="cuda", generator=g) * 0.1
        relu = planes == 2 if relu is None else relu
        ws = tc.pow2_scale(w)
    out, status, _ = launch_dense(product, x, w, ws, k, stride, pad, transpose, scale, shift, relu, planes,
                                  out_stride, coff, n_pad)
    assert status == 0
    assert_sentinels(out, planes, coff, cout)
    got, lo = interior(out, planes, coff, cout)
    conv = dict(stride=stride, padding=pad, transpose=transpose)
    ref = tc_ref.dense_ref(x, w, scale, shift, relu, **conv)
    assert got.shape == ref.y.shape
    st = tc_ref.assert_accurate(got, ref, ws, "kernel")
    if faults:
        assert_faults_rejected(got, lo, x, w, ws, ref, relu, "", e, **conv)
    return st


# ---- k_conv3x3_tc2: 3x3 stride 1 pad 1, n_pad 128 -----------------------------------------------------------------
# (B, Cin, Cout, H, W, channel offset into a 256-channel map (0: a map of Cout channels), plain: relu 0 / NULL scale
# and shift)
V2_CASES = [
    (1, 64, 128, 1, 1, 0, False), (3, 128, 128, 3, 7, 128, False), (1, 192, 96, 8, 8, 0, False),
    (3, 256, 128, 9, 17, 0, True), (1, 384, 128, 21, 36, 128, False), (3, 128, 96, 200, 176, 0, False),
    (1, 384, 96, 3, 7, 0, True), (3, 64, 128, 21, 36, 0, False), (1, 256, 128, 200, 176, 128, False),
    (3, 192, 128, 9, 17, 128, False), (1, 128, 128, 1, 1, 0, True), (3, 384, 128, 8, 8, 0, False),
    (1, 64, 96, 9, 17, 128, True), (3, 256, 96, 1, 1, 0, False),
]


@pytest.mark.parametrize("B,cin,cout,H,W,coff,plain", V2_CASES)
def test_conv3x3_v2(product, B, cin, cout, H, W, coff, plain):
    check_dense(product, B, cin, cout, H, W, 3, 1, 1, plain=plain, coff=coff, out_stride=256 if coff else None,
                n_pad=128)


# ---- k_conv_tc: every other shape -------------------------------------------------------------------------------
# (B, Cin, Cout, H, W, k, stride, pad, transpose, planes, out_stride, coff, plain)
CONV_CASES = [
    # 3x3 s1 p1 at n_pad 64 / 32: the small head's 64 -> 64 layers
    (2, 64, 64, 17, 23, 3, 1, 1, False, 2, None, 0, False),
    (1, 128, 32, 9, 9, 3, 1, 1, False, 2, None, 0, True),
    (1, 64, 64, 1, 1, 3, 1, 1, False, 2, None, 0, True),
    # 3x3 s2 p1, odd input sizes, 256 outputs as two slices
    (2, 64, 128, 17, 23, 3, 2, 1, False, 2, None, 0, False),
    (1, 128, 256, 200, 176, 3, 2, 1, False, 2, None, 0, False),
    (1, 256, 256, 17, 23, 3, 2, 1, False, 2, None, 0, True),
    # deblock k = s = 1
    (2, 128, 128, 21, 36, 1, 1, 0, False, 2, None, 0, False),
    (1, 256, 128, 9, 17, 1, 1, 0, False, 2, None, 0, True),
    # 1x1 heads into fp32 records wider than Cout; 148 channels: a second slice at dst_coff 128
    (2, 128, 20, 20, 33, 1, 1, 0, False, 1, 32, 0, False),
    (1, 384, 104, 21, 36, 1, 1, 0, False, 1, 128, 0, True),
    (1, 384, 148, 9, 17, 1, 1, 0, False, 1, 160, 0, False),
    # ConvTranspose2d k = s into a channel offset of a wider concat map
    (2, 64, 128, 9, 17, 2, 2, 0, True, 2, 384, 128, False),
    (1, 128, 128, 5, 7, 4, 4, 0, True, 2, 384, 256, True),
    (1, 128, 128, 21, 36, 2, 2, 0, True, 2, 256, 0, False),
    # Conv2d k = s, pad 0, input not divisible by k
    (2, 128, 128, 21, 35, 2, 2, 0, False, 2, 256, 128, False),
    (1, 256, 128, 23, 30, 4, 4, 0, False, 2, None, 0, True),
    # 4x4 stride 4 (16 taps: the kernel's tap limit)
    (1, 64, 64, 33, 47, 4, 4, 0, False, 2, None, 0, False),
]


@pytest.mark.parametrize("B,cin,cout,H,W,k,stride,pad,transpose,planes,out_stride,coff,plain", CONV_CASES)
def test_conv_general(product, B, cin, cout, H, W, k, stride, pad, transpose, planes, out_stride, coff, plain):
    check_dense(product, B, cin, cout, H, W, k, stride, pad, transpose, plain, planes, out_stride, coff)


# ---- strip-list launches ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [8, 4, 2])
def test_strip_list_launch_against_fp64(product, R):
    """work / background lists of b2s_rpn_strip_plan on random occupancy: listed strips against float64 directly,
    background strips = the field, nothing else written."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, cin, C, H, W = 2, 128, 128, 37, 45
    rng = np.random.default_rng(R)
    occ = (rng.random((B, H, W)) < 0.01).astype(np.uint8)
    occ[1, H - 1, W - 1] = 1                                   # data in the partial corner strip
    sh_n, sw_n = -(-H // R), -(-W // 8)
    ns = B * sh_n * sw_n
    d_occ = torch.from_numpy(occ).cuda()
    scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(1, ns, dtype=torch.int32, device="cuda")
    work = torch.zeros(1, ns, dtype=torch.int32, device="cuda")
    bg = torch.zeros(1, ns, dtype=torch.int32, device="cuda")
    counts = torch.zeros(1, 2, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_strip_plan(L.ptr(d_occ), B, H, W, 1, R, L.ptr(scratch), L.ptr(flags), L.ptr(work), L.ptr(bg),
                                   L.ptr(counts), L.stream()), "b2s_rpn_strip_plan")
    torch.cuda.synchronize()
    nw, nb = int(counts[0, 0]), int(counts[0, 1])
    assert 0 < nw < ns and nw + nb == ns
    g = torch.Generator(device="cuda").manual_seed(40 + R)
    x = torch.randn(B, cin, H, W, device="cuda", generator=g)
    w = torch.randn(C, cin, 3, 3, device="cuda", generator=g) * (2.0 / (9 * cin)) ** 0.5
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.1
    ws = tc.pow2_scale(w)
    field = torch.randn(2, H + 2, W + 2, C, device="cuda", generator=g).half()
    lists = (R, work[0], counts[0, 0:1].contiguous(), bg[0], counts[0, 1:2].contiguous(), field[0], field[1], -1)
    out, status, _ = launch_dense(product, x, w, ws, 3, 1, 1, scale=scale, shift=shift, relu=True, n_pad=128,
                                  lists=lists)
    assert status == 0
    listed = torch.zeros(B, H, W, dtype=torch.bool, device="cuda")
    for s in work[0, :nw].tolist():
        b, sh, sw = s // (sh_n * sw_n), (s // sw_n) % sh_n, s % sw_n
        listed[b, sh * R:sh * R + R, sw * 8:sw * 8 + 8] = True
    for s in bg[0, :nb].tolist():
        b, sh, sw = s // (sh_n * sw_n), (s // sw_n) % sh_n, s % sw_n
        for p in range(2):
            assert torch.equal(out[p][b, 1 + sh * R:1 + min(H, sh * R + R), 1 + sw * 8:1 + min(W, sw * 8 + 8)],
                               field[p][1 + sh * R:1 + min(H, sh * R + R), 1 + sw * 8:1 + min(W, sw * 8 + 8)])
    for p in range(2):                                          # the halo is never written
        for t in (out[p][:, 0], out[p][:, -1], out[p][:, :, 0], out[p][:, :, -1]):
            assert bool((t == (HI_SENT, LO_SENT)[p]).all())
    got, lo = interior(out, 2, 0, C)
    ref = tc_ref.dense_ref(x, w, scale, shift, True, 1, 1)
    sub = lambda t: t.permute(0, 2, 3, 1)[listed]               # [listed pixels, C]
    sref = tc_ref.Ref(*[sub(f) for f in ref])
    tc_ref.assert_accurate(sub(got), sref, ws, "listed strips")
    # faults on the listed strips
    for name, bad in (("F1", tc_ref.dense_f1(got, x, w, ws, ref, True, padding=1)),
                      ("F3", tc_ref.f3(got, lo))):
        tc_ref.assert_rejected(sub(bad), sref, ws, name)
    f2 = tc_ref.dense_f2(got, x, w, ws, ref, True, padding=1)
    f2 = torch.where(listed[:, None], f2, got)                  # only where the kernel computed
    if bool((f2 != got).any()):
        tc_ref.assert_rejected(sub(f2), sref, ws, "F2")
    else:
        bad = got.clone()
        i = listed.nonzero()[-1]
        bad[i[0], :, i[1], i[2]] = tc_ref.dense_f2(got, x, w, ws, ref, True, padding=1)[i[0], :, -1, -1]
        tc_ref.assert_rejected(sub(bad), sref, ws, "F2")


# ---- magnitude sweep --------------------------------------------------------------------------------------------
SWEEP = (-14, -10, -6, -3, 0, 4, 8)


@pytest.mark.parametrize("e", SWEEP)
@pytest.mark.parametrize("kernel", ["v2", "conv_tc"])
def test_dense_magnitude_sweep(product, kernel, e):
    """activations randn * 2^e: the per-element bound holds with its absolute terms (the lo plane of an activation
    below 2^-3 is an fp16 subnormal) while max|y| stays in the fp16 range."""
    if kernel == "v2":
        st = check_dense(product, 2, 128, 128, 21, 36, 3, 1, 1, seed=7, e=e, relu=False)
    else:
        st = check_dense(product, 2, 128, 128, 17, 23, 3, 2, 1, seed=7, e=e, relu=False)
    assert st["ratio"] <= 1.0


# ---- fp16 range boundary ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [3, 1])
def test_fp16_range_boundary(product, k):
    """an output of exactly +-65504 raises no status bit; the next fp32 value beyond raises B2S_STATUS_F16_RANGE and its
    hi plane is clamped to +-65504 (3x3 n_pad 128: k_conv3x3_tc2; 1x1: k_conv_tc)."""
    B, cin, C, H, W = 1, 64, 128, 9, 10
    x = torch.zeros(B, cin, H, W, device="cuda")
    w = torch.zeros(C, cin, k, k, device="cuda")
    scale = torch.ones(C, device="cuda")
    top = float(np.nextafter(np.float32(65504.0), np.float32(np.inf)))
    for v, bad in ((65504.0, False), (top, True)):
        shift = torch.full((C,), v, device="cuda")
        shift[1::2] = -v
        out, status, _ = launch_dense(product, x, w, 1.0, k, 1, k // 2, scale=scale, shift=shift, relu=False)
        assert status == (16 if bad else 0), (v, status)
        hi = out[0][:, 1:-1, 1:-1].float()
        assert bool((hi[..., 0::2] == 65504.0).all()) and bool((hi[..., 1::2] == -65504.0).all())
        if not bad:
            assert bool((out[1][:, 1:-1, 1:-1] == 0).all())


# ---- sparse -----------------------------------------------------------------------------------------------------
TABLES = {"subm": ([3, 3, 3], [1, 1, 1], [1, 1, 1], True), "strided": ([3, 3, 3], [2, 2, 2], [1, 1, 1], False),
          "k311": ([3, 1, 1], [2, 1, 1], [0, 0, 0], False)}
SPARSE_CASES = [(cin, cout, t) for cin in (3, 4, 8, 16, 32, 64) for cout in (16, 32, 64) for t in TABLES]
NUM_OUT = (1, 127, 128, 129, 5000)


def sparse_table(product, table, n_out, seed):
    """coordinates of a noisy surface and the rulebook of `table`, cut to exactly n_out output rows"""
    rng = np.random.default_rng(seed)
    shape, batch = (9, 64, 56), 2
    ks, st, pd, subm = TABLES[table]
    n = 4 * n_out + 64
    b = rng.integers(batch, size=4 * n)
    y = rng.integers(shape[1], size=4 * n)
    x = rng.integers(shape[2], size=4 * n)
    z = np.clip(np.round(shape[0] / 2 + 2 * np.sin(x / 5.0) + rng.normal(0, 0.9, size=4 * n)), 0, shape[0] - 1)
    idx = np.unique(np.stack([b, z, y, x], 1).astype(np.int32), axis=0)
    idx = idx[rng.permutation(idx.shape[0])[:n]]
    idx = idx[np.lexsort(idx.T[::-1])]
    feats = torch.zeros(idx.shape[0], 1, device="cuda")
    t = product.SparseConvTensor(feats, torch.from_numpy(idx).cuda(), shape, batch)
    rb = product.ops.build_rulebook(t, ks, st, pd, [1, 1, 1], subm)
    assert rb.num_out >= n_out
    return idx.shape[0], rb.nbr[:n_out].contiguous(), ks


def run_sparse(product, x, w, ws, nbr, ks, scale, shift, relu, cin_tc):
    """-> (hi/lo value [n_out, Cout] float64, lo plane, fp32 output), the planned launch bit-identical to the plain one"""
    from b2second import tc
    L = product._lib
    lib = L.load()
    n_in, cin = x.shape
    n_out, K = nbr.shape
    cout = w.shape[2]
    w_hi, w_lo = tc.split_f16(tc.pack_sparse_weights(w), ws)
    fbuf = torch.full((n_in, 2, cin_tc), 9.0, dtype=torch.float16, device="cuda")
    n_dev = torch.tensor([n_in], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_split_f16(L.ptr(x), L.ptr(fbuf[:, 0]), L.ptr(fbuf[:, 1]), L.ptr(n_dev), n_in, cin, cin_tc,
                              2 * cin_tc, L.stream()), "b2s_split_f16")
    out_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    sk, sh = (scale / ws).contiguous(), shift.contiguous()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    perm = torch.zeros(n_out, dtype=torch.int32, device="cuda")
    tmask = torch.zeros((n_out + 127) // 128, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_sparse_tile_plan(L.ptr(nbr), None, K, L.i3(ks), L.ptr(out_dev), n_out, 1, L.ptr(perm),
                                     L.ptr(tmask), L.stream()), "b2s_sparse_tile_plan")
    res = []
    for pm, tm in ((None, None), (perm, tmask)):
        # interleaved [row][hi | lo | spare] rows with a sentinel in the spare channels
        obuf = torch.full((n_out + 1, 3, cout), HI_SENT, dtype=torch.float16, device="cuda")
        L.check(lib.b2s_sparse_conv_tc_plan(L.ptr(fbuf[:, 0]), L.ptr(fbuf[:, 1]), 2 * cin_tc, n_in, cin_tc,
                                            L.ptr(w_hi), L.ptr(w_lo), L.ptr(nbr), K, L.ptr(out_dev), n_out, L.ptr(pm),
                                            L.ptr(tm), L.ptr(sk), L.ptr(sh), 1 if relu else 0, L.ptr(obuf[:, 0]),
                                            L.ptr(obuf[:, 1]), 3 * cout, cout, L.ptr(status), L.stream()),
                "b2s_sparse_conv_tc_plan")
        res.append(obuf)
    o32 = torch.full((n_out + 1, cout), F32_SENT, device="cuda")                # fp32 rows: [n_out, Cout], dense
    L.check(lib.b2s_sparse_conv_tc(L.ptr(fbuf[:, 0]), L.ptr(fbuf[:, 1]), 2 * cin_tc, n_in, cin_tc, L.ptr(w_hi),
                                   L.ptr(w_lo), L.ptr(nbr), K, L.ptr(out_dev), n_out, L.ptr(sk), L.ptr(sh),
                                   1 if relu else 0, L.ptr(o32), None, 0, cout, L.ptr(status), L.stream()),
            "b2s_sparse_conv_tc")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert torch.equal(res[0], res[1]), "tile plan changed the result"
    obuf = res[0]
    assert bool((obuf[:, 2] == HI_SENT).all()) and bool((obuf[n_out] == HI_SENT).all())
    assert bool((o32[n_out] == F32_SENT).all())
    lo = obuf[:n_out, 1].double()
    return obuf[:n_out, 0].double() + lo, lo, o32[:n_out, :cout].double()


def check_sparse(product, cin, cout, table, n_out, seed, e=0):
    from b2second import tc
    n_in, nbr, ks = sparse_table(product, table, n_out, seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    K = nbr.shape[1]
    x = torch.randn(n_in, cin, device="cuda", generator=g) * 2.0 ** e
    w = torch.randn(K, cin, cout, device="cuda", generator=g) * (2.0 / (K * cin)) ** 0.5
    scale = torch.rand(cout, device="cuda", generator=g) + 0.5
    shift = torch.randn(cout, device="cuda", generator=g) * 0.1
    cin_tc = tc.sparse_tc_cin(cin)
    ws = tc.pow2_scale(tc.pack_sparse_weights(w))
    got, lo, o32 = run_sparse(product, x, w, ws, nbr, ks, scale, shift, True, cin_tc)
    ref = tc_ref.sparse_ref(x, w, nbr, scale, shift, True)
    st = tc_ref.assert_accurate(got, ref, ws, "hi/lo planes")
    tc_ref.assert_accurate(o32, ref, ws, "fp32 rows")
    if e >= tc_ref.F1_MIN_EXP:
        tc_ref.assert_rejected(tc_ref.sparse_f1(got, x, w, ws, nbr, ref, True, cin_tc), ref, ws, "F1")
    tc_ref.assert_rejected(tc_ref.sparse_f2(got, x, w, ws, nbr, ref, True), ref, ws, "F2")
    tc_ref.assert_rejected(tc_ref.f3(got, lo), ref, ws, "F3")
    tc_ref.assert_rejected(tc_ref.f3(o32, None), ref, ws, "F3 fp32")
    return st


@pytest.mark.parametrize("cin,cout,table", SPARSE_CASES)
def test_sparse_conv_tc(product, cin, cout, table):
    i = SPARSE_CASES.index((cin, cout, table))
    n_out = NUM_OUT[i % len(NUM_OUT)]
    check_sparse(product, cin, cout, table, n_out, seed=100 + i)


@pytest.mark.parametrize("e", SWEEP)
def test_sparse_magnitude_sweep(product, e):
    st = check_sparse(product, 32, 32, "subm", 5000, seed=9, e=e)
    assert st["ratio"] <= 1.0


# ---- sparse weight gradient -------------------------------------------------------------------------------------
# (Cin, Cout, table, output rows); Cin 4 is zero-padded to 8 like the first layer of the middle encoders
WGRAD_CASES = [(64, 64, "subm", 5000), (16, 32, "strided", 3000), (4, 16, "subm", 2000), (32, 16, "k311", 1500)]


@pytest.mark.parametrize("e", (-40, -24, -12, 0))
@pytest.mark.parametrize("cin,cout,table,n_out", WGRAD_CASES)
def test_sparse_wgrad_tc(product, cin, cout, table, n_out, e):
    """b2s_sparse_conv_wgrad_tc against float64 sum_o x[nbr[o, k]]^T dY[o], dY = randn * 2^e, both operands split by
    b2s_split_f16_autoscale; rows in storage order, in tile-plan order, and in plan order with tile masks (the last two
    bit-identical).  The check runs on the operands as the kernel splits them (x * 2^ex, dY * 2^eg: exact powers of two)
    and on dW * 2^(ex + eg)."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    n_in, nbr, ks = sparse_table(product, table, n_out, seed=300 + cin + cout)
    K = nbr.shape[1]
    g = torch.Generator(device="cuda").manual_seed(cin * 100 + cout)
    x = torch.randn(n_in, cin, device="cuda", generator=g)
    dy = torch.randn(n_out, cout, device="cuda", generator=g) * 2.0 ** e
    cin_tc = tc.sparse_tc_cin(cin)

    def split(t, ch):
        buf = torch.full((t.shape[0], 2, ch), 9.0, dtype=torch.float16, device="cuda")
        sc = torch.zeros(2, device="cuda")
        L.check(lib.b2s_split_f16_autoscale(L.ptr(t), L.ptr(buf[:, 0]), L.ptr(buf[:, 1]), None, t.shape[0], t.shape[1],
                                            ch, 2 * ch, L.ptr(sc), L.stream()), "b2s_split_f16_autoscale")
        return buf, sc

    xb, sx = split(x, cin_tc)
    gb, sg = split(dy, cout)
    scale = (sx[:1] * sg[:1]).contiguous()
    out_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    perm = torch.zeros(n_out, dtype=torch.int32, device="cuda")
    tmask = torch.zeros((n_out + 127) // 128, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_sparse_tile_plan(L.ptr(nbr), None, K, L.i3(ks), L.ptr(out_dev), n_out, 1, L.ptr(perm),
                                     L.ptr(tmask), L.stream()), "b2s_sparse_tile_plan")
    wbytes = lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(n_out, K, cin_tc, cout)
    work = torch.empty(max(wbytes, 1), dtype=torch.uint8, device="cuda")
    res = {}
    for name, pm, tm in (("storage order", None, None), ("plan order", perm, None), ("plan + masks", perm, tmask)):
        dw = torch.full((K, cin_tc, cout), F32_SENT, device="cuda")
        L.check(lib.b2s_sparse_conv_wgrad_tc(L.ptr(xb[:, 0]), L.ptr(xb[:, 1]), 2 * cin_tc, n_in, cin_tc,
                                             L.ptr(gb[:, 0]), L.ptr(gb[:, 1]), 2 * cout, cout, L.ptr(nbr), K,
                                             L.ptr(out_dev), n_out, L.ptr(pm), L.ptr(tm), L.ptr(scale), L.ptr(dw),
                                             L.ptr(work), wbytes, L.stream()), "b2s_sparse_conv_wgrad_tc")
        torch.cuda.synchronize()
        res[name] = dw
    assert torch.equal(res["plan order"], res["plan + masks"]), "tile masks changed the weight gradient"
    wx, wg = 1.0 / float(sx[0]), 1.0 / float(sg[0])
    assert np.log2(wx) == int(np.log2(wx)) and np.log2(wg) == int(np.log2(wg))
    xs, gs = x * wx, dy * wg                                      # exact in fp32: powers of two, no under/overflow
    assert torch.equal(xb[:, 0, :cin].double(), tc_ref.hi_lo(xs)[0]) and torch.equal(gb[:, 1].double(), tc_ref.hi_lo(gs)[1])
    ref = tc_ref.wgrad_ref(xs, gs, nbr)
    for name, dw in res.items():
        assert bool((dw[:, cin:] == 0).all()), name + ": zero-padded input channels"
        tc_ref.assert_accurate(dw[:, :cin].double() * (wx * wg), ref, 1.0, name)
    got = res["storage order"][:, :cin].double() * (wx * wg)
    tc_ref.assert_rejected(tc_ref.wgrad_f1(got, xs, gs, nbr, ref), ref, 1.0, "F1")
    tc_ref.assert_rejected(tc_ref.wgrad_f2(got, xs, gs, nbr, ref), ref, 1.0, "F2")
    tc_ref.assert_rejected(tc_ref.f3(got, None, cdim=2), ref, 1.0, "F3")
