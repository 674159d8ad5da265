"""The fp32 kernels against the float64 references and per-element bounds of tests/fp32_ref.py:
  b2s_sparse_conv          every k_sparse_conv instance and k_sparse_conv_generic (odd widths, K = 1, K = 125) on
                           SubM 3^3, 3^3-stride-2 and (3,1,1)-stride-(2,1,1) tables, across the 64-row tile edge, with
                           and without scale / shift / ReLU, activations from 2^-40 to 2^20
  b2s_sparse_conv_wgrad    across the 32-row chunk, the 2048-row slab and the 64-channel tile edges, dY down to 2^-130
                           (subnormal products, which must not be flushed), bit-reproducible
  input gradient           conv._dgrad on the fp32 pipe (this bound) and the tensor pipe (tests/tc_ref.py's bound, dY rows
                           of very different magnitude under one scale), b2s_rulebook_transpose against an index-level
                           transpose, K = 27 and K = 3
  b2s_pfn / b2s_pfn_ex     both decorations, 3 to 8 features, num in {1, T-1, T}, T = 1, the grid corners and x ~ 69 m,
                           channels that only the padded-slot rule decides
  b2s_vfe_mean, b2s_voxelize's fused mean   vfe_mode 1 and 2, 3 to 5 features, voxels of 1 and of T points
Outputs go into sentinel-filled buffers longer than the live count; table and feature rows past the live count are
poisoned (NaN features, table entries naming those NaN rows: out of the live range but inside the allocation) and every
sentinel must survive.  Every case asserts that its simulated faults fail the same check."""
import numpy as np
import pytest
import torch

import fp32_ref as R
import tc_ref

pytestmark = pytest.mark.gpu

SENT = 7.0
POISON = 8                      # NaN feature rows appended after the live ones


@pytest.fixture(autouse=True)
def _fp32():
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


_STATS = {}


@pytest.fixture(autouse=True)
def _record(request, monkeypatch):
    """keep the largest bound ratio and aggregate ratio of every case (written to fp32_fp64_stats.json under the test
    output directory: the measurement behind fp32_ref.RHO)"""
    real = R.assert_accurate

    def rec(got, ref, what=""):
        st = R.error_stats(got, ref)
        old = _STATS.get(request.node.name, {"ratio": 0.0, "rms": 0.0})
        _STATS[request.node.name] = {k: max(old[k], st[k]) for k in old}
        return real(got, ref, what)
    monkeypatch.setattr(R, "assert_accurate", rec)


@pytest.fixture(scope="module", autouse=True)
def _report(out_dir):
    yield
    import json
    import os
    worst = max(_STATS.items(), key=lambda kv: kv[1]["rms"]) if _STATS else None
    with open(os.path.join(out_dir, "fp32_fp64_stats.json"), "w") as f:
        json.dump({"rho": R.RHO, "worst_rms": worst, "cases": _STATS}, f, indent=1, sort_keys=True)


def _poisoned_rows(t, extra=POISON):
    """[n, C] -> a CUDA buffer [n + extra, C] whose rows past n are NaN"""
    buf = torch.full((t.shape[0] + extra,) + tuple(t.shape[1:]), float("nan"), device="cuda")
    buf[:t.shape[0]] = t.cuda()
    return buf


def _poisoned_table(nbr, n_in, extra):
    """[n_out, K] -> [n_out + extra, K] whose rows past n_out name the NaN rows n_in .. n_in + POISON - 1"""
    n_out, K = nbr.shape
    t = torch.empty(n_out + extra, K, dtype=torch.int32, device="cuda")
    t[:n_out] = torch.as_tensor(nbr).cuda()
    t[n_out:] = n_in + (torch.arange(extra * K, device="cuda", dtype=torch.int32) % POISON).view(extra, K)
    return t


# ---- b2s_sparse_conv ----------------------------------------------------------------------------------------------
def run_conv(product, x, w, nbr, scale=None, shift=None, relu=False, extra=67):
    """b2s_sparse_conv over n_out live rows of a table with `extra` poisoned rows (cap_out = n_out + extra) into a
    sentinel-filled buffer -> [n_out, Cout] fp32"""
    L = product._lib
    lib = L.load()
    n_in, cin = x.shape
    n_out, K = nbr.shape
    cout = w.shape[2]
    xb = _poisoned_rows(x)
    tb = _poisoned_table(nbr, n_in, extra)
    cap = n_out + extra
    out = torch.full((cap + 1, cout), SENT, device="cuda")
    n_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    sc = None if scale is None else scale.cuda().contiguous()
    sh = None if shift is None else shift.cuda().contiguous()
    L.check(lib.b2s_sparse_conv(L.ptr(xb), cin, L.ptr(w.cuda().contiguous()), L.ptr(tb), K, L.ptr(n_dev), cap, L.ptr(sc),
                                L.ptr(sh), 1 if relu else 0, L.ptr(out), cout, L.stream()), "b2s_sparse_conv")
    torch.cuda.synchronize()
    assert bool((out[n_out:] == SENT).all()), "rows past the live count were written"
    return out[:n_out]


def check_conv(product, cin, cout, table, n_out, epilogue, seed, e=0):
    """random layer on a table -> kernel vs float64 (bound + aggregate), F1 / F2 / F4 rejected; -> error_stats"""
    rng = np.random.default_rng(seed)
    n_in, nbr = R.table_rows(rng, table, n_out)
    K = nbr.shape[1]
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n_in, cin, device="cuda", generator=g) * 2.0 ** e
    w = torch.randn(K, cin, cout, device="cuda", generator=g) * (2.0 / (K * cin)) ** 0.5
    scale = shift = None
    if n_out == 1:
        # the ReLU outputs of one row can all be zero, and then no fault is visible: one row runs without it
        epilogue = {"bn_relu": "bn", "relu": "none"}.get(epilogue, epilogue)
    relu = epilogue in ("bn_relu", "relu")
    if epilogue in ("bn", "bn_relu"):
        scale = torch.rand(cout, device="cuda", generator=g) + 0.5
    if epilogue in ("bn", "bn_relu", "shift"):
        # scaled with the activations, so that a shift of unit size does not hide the faults in u * |pre|
        shift = torch.randn(cout, device="cuda", generator=g) * 0.1 * 2.0 ** e
    nbr = torch.from_numpy(nbr).cuda()
    got = run_conv(product, x, w, nbr, scale, shift, relu)
    ref = R.sparse_ref(x, w, nbr, scale, shift, relu)
    st = R.assert_accurate(got, ref, "b2s_sparse_conv")
    if n_out:
        R.assert_rejected(R.conv_f1(got, x, w, nbr, scale, relu), ref, "F1")
        R.assert_rejected(R.conv_f1(got, x, w, nbr, scale, relu, tile=(n_out - 1) // R.TILE), ref, "F1 last tile")
        R.assert_rejected(R.conv_f2(got, x, w, nbr, scale, relu), ref, "F2")
        R.assert_rejected(R.conv_f4(got, ref, x, w, nbr, scale, shift, relu), ref, "F4")
    return st


INSTANCES = [(3, 16), (4, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64)]
GENERIC = [(5, 7), (8, 64), (64, 128)]
TABLE_KINDS = ("subm", "strided", "k311")
NUM_OUT = (0, 1, 63, 64, 65, 5000)
EPILOGUES = ("bn_relu", "none", "bn", "shift", "relu")
CONV_CASES = [(ci, co, t) for ci, co in INSTANCES + GENERIC for t in TABLE_KINDS]


@pytest.mark.parametrize("cin,cout,table", CONV_CASES)
def test_sparse_conv(product, cin, cout, table):
    i = CONV_CASES.index((cin, cout, table))
    for j, n_out in enumerate(NUM_OUT):
        check_conv(product, cin, cout, table, n_out, EPILOGUES[(i + j) % len(EPILOGUES)], seed=1000 * i + j)


@pytest.mark.parametrize("cin,cout", [(16, 16), (5, 7), (64, 64)])
@pytest.mark.parametrize("table", ["subm5", "k1"])
def test_sparse_conv_k1_and_k125(product, cin, cout, table):
    """K = 125 (5^3 SubM) runs k_sparse_conv_generic even for the widths of a templated instance"""
    for j, n_out in enumerate((1, 65, 3000)):
        check_conv(product, cin, cout, table, n_out, EPILOGUES[j], seed=77 + cin + j)


@pytest.mark.parametrize("e", [-40, -30, -20, -10, 0, 10, 20])
@pytest.mark.parametrize("cin,cout", [(32, 32), (5, 7)])
def test_sparse_conv_magnitude_sweep(product, cin, cout, e):
    check_conv(product, cin, cout, "subm", 5000, "bn_relu", seed=9, e=e)


# ---- b2s_sparse_conv_wgrad ----------------------------------------------------------------------------------------
def run_wgrad(product, x, dy, nbr, extra=37):
    L = product._lib
    lib = L.load()
    n_in, cin = x.shape
    n_out, cout = dy.shape
    K = nbr.shape[1]
    xb = _poisoned_rows(x)
    gb = _poisoned_rows(dy, extra)
    tb = _poisoned_table(nbr, n_in, extra)
    cap = n_out + extra
    wbytes = lib.b2s_sparse_conv_wgrad_workspace_bytes(cap, K, cin, cout)
    work = torch.full((max(wbytes, 4) // 4 + 16,), SENT, device="cuda")
    n_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    res = []
    for _ in range(2):
        dw = torch.full((K * cin * cout + 64,), SENT, device="cuda")
        L.check(lib.b2s_sparse_conv_wgrad(L.ptr(xb), cin, L.ptr(gb), cout, L.ptr(tb), K, L.ptr(n_dev), cap, None,
                                          L.ptr(dw), L.ptr(work), wbytes, L.stream()), "b2s_sparse_conv_wgrad")
        torch.cuda.synchronize()
        assert bool((dw[K * cin * cout:] == SENT).all()), "written past dW"
        assert bool((work[wbytes // 4:] == SENT).all()), "written past the workspace"
        res.append(dw[:K * cin * cout].view(K, cin, cout))
    assert torch.equal(res[0], res[1]), "two runs differ"
    return res[0]


WGRAD_ROWS = (1, 31, 33, 2047, 2048, 2049, 4097)
WGRAD_WIDTHS = [(3, 5), (5, 80), (80, 3), (128, 128), (80, 128), (3, 3), (128, 5)]


@pytest.mark.parametrize("e", [0, -60, -126, -130])
@pytest.mark.parametrize("n_out,cin,cout", [(n, ci, co) for n, (ci, co) in zip(WGRAD_ROWS, WGRAD_WIDTHS)])
def test_sparse_conv_wgrad(product, n_out, cin, cout, e):
    """dY = randn * 2^e: at 2^-126 and 2^-130 the products are subnormal, and a flush to zero fails the bound"""
    table = TABLE_KINDS[WGRAD_ROWS.index(n_out) % 3]
    rng = np.random.default_rng(n_out + cin)
    n_in, nbr = R.table_rows(rng, table, n_out)
    nbr = torch.from_numpy(nbr).cuda()
    g = torch.Generator(device="cuda").manual_seed(n_out * 7 + cout)
    x = torch.randn(n_in, cin, device="cuda", generator=g) * (2.0 ** -6 if e <= -126 else 1.0)
    dy = torch.randn(n_out, cout, device="cuda", generator=g) * 2.0 ** e
    got = run_wgrad(product, x, dy, nbr)
    ref = R.wgrad_ref(x, dy, nbr)
    R.assert_accurate(got, ref, "b2s_sparse_conv_wgrad")
    R.assert_rejected(R.wgrad_f1(got, x, dy, nbr), ref, "F1")
    last = n_out - 1
    R.assert_rejected(R.wgrad_f1(got, x, dy, nbr, slab=last // R.SLAB, chunk=(last % R.SLAB) // R.CHUNK), ref,
                      "F1 last chunk")
    R.assert_rejected(R.wgrad_f2(got, x, dy, nbr), ref, "F2")
    if e > -100:
        R.assert_rejected(R.wgrad_f4(got, ref, x, dy, nbr), ref, "F4")
    else:
        # every product is subnormal (x is randn * 2^-6); flushing the subnormal dY inputs to zero must fail
        assert float(x.abs().max()) * float(dy.abs().max()) < 2.0 ** -126
        sub = torch.where(dy.abs() < 2.0 ** -126, dy, torch.zeros_like(dy))
        R.assert_rejected(got.double() - R.wgrad_ref(x, sub, nbr).y, ref, "flush to zero")


# ---- input gradient -----------------------------------------------------------------------------------------------
DGRAD_TABLES = {"subm": ([3, 3, 3], [1, 1, 1], [1, 1, 1], True), "strided": ([3, 3, 3], [2, 2, 2], [0, 1, 1], False),
                "k311": ([3, 1, 1], [2, 1, 1], [0, 0, 0], False)}


@pytest.mark.parametrize("tc_pipe", [False, True], ids=["fp32", "tc"])
@pytest.mark.parametrize("table", list(DGRAD_TABLES))
@pytest.mark.parametrize("cin,cout", [(16, 32), (64, 64), (5, 16)])
def test_dgrad(product, monkeypatch, tc_pipe, table, cin, cout):
    """conv._dgrad against float64 sum_k W[k] dY[nbrT[i, k]] over an index-level transpose of the table; dY rows scaled
    by 2^0 .. 2^-24 under one autoscale"""
    monkeypatch.setattr(product, "USE_TENSOR_CORES", tc_pipe)
    from b2second import tc
    ks, st, pd, subm = DGRAD_TABLES[table]
    rng = np.random.default_rng(cin + cout + len(table))
    idx = R.surface_coords(rng, 4000)
    n_in = idx.shape[0]
    x = product.SparseConvTensor(torch.zeros(n_in, cin, device="cuda"), torch.from_numpy(idx).cuda(), list(R.SHAPE),
                                 R.BATCH)
    rb = product.ops.build_rulebook(x, ks, st, pd, [1, 1, 1], subm)
    K, n_out = rb.K, rb.num_out
    nbr = rb.nbr.cpu().numpy()
    nbrT = torch.from_numpy(R.transpose_table(nbr, n_in)).cuda()
    conv = (product.SubMConv3d(cin, cout, ks, bias=False, indice_key="k") if subm else
            product.SparseConv3d(cin, cout, ks, st, padding=pd, bias=False)).cuda()
    g = torch.Generator(device="cuda").manual_seed(cin * cout)
    w = torch.randn(K, cin, cout, device="cuda", generator=g) * (2.0 / (K * cin)) ** 0.5
    with torch.no_grad():
        conv.weight.copy_(w.view(conv.weight.shape))
    rows = torch.from_numpy(rng.integers(-24, 1, n_out).astype(np.float32)).cuda()
    dy = (torch.randn(n_out, cout, device="cuda", generator=g) * torch.exp2(rows)[:, None]).contiguous()
    if not subm:
        assert torch.equal(product.ops.transpose_rulebook(rb, n_in), nbrT), "b2s_rulebook_transpose"
    wt = w.transpose(1, 2).contiguous()                                  # W'[k] = W[k]^T: [K, Cout, Cin]
    split = product._GradSplit(dy)
    dx = conv._dgrad(dy, conv.weight, rb, n_in, split)
    dx2 = conv._dgrad(dy, conv.weight, rb, n_in, split)
    torch.cuda.synchronize()
    assert dx.shape == (n_in, cin) and torch.equal(dx, dx2)
    used_tc = tc_pipe and tc.sparse_tc_cin(cout) == cout and bool(product._lib.load().b2s_sparse_conv_tc_supported(cout, cin))
    assert used_tc == (tc_pipe and cin != 5)
    if used_tc:
        inv = float(split.planes()[3])
        flip = subm
        ws = conv._dgrad_weights(conv.weight, flip)[2]
        ref = tc_ref.sparse_ref(dy * (1.0 / inv), wt, nbrT, torch.full((cin,), inv, device="cuda"))
        tc_ref.assert_accurate(dx, ref, ws, "tensor-pipe dgrad")
        tc_ref.assert_rejected(tc_ref.sparse_f2(dx, dy * (1.0 / inv), wt, ws, nbrT, ref, False), ref, ws, "F2")
    else:
        ref = R.sparse_ref(dy, wt, nbrT)
        R.assert_accurate(dx, ref, "fp32 dgrad")
        R.assert_rejected(R.conv_f1(dx, dy, wt, nbrT), ref, "F1")
        # F2 on the input row whose first neighbour is the largest dY row: dropping a 2^-24 row next to unit rows is
        # within the rounding of the sum, no fault the bound can see
        t = nbrT.long()
        first = t.gather(1, (t >= 0).int().argmax(1, keepdim=True))[:, 0]           # the first present offset
        size = torch.where(first >= 0, dy.abs().amax(1)[first.clamp_min(0)], torch.zeros_like(first, dtype=dy.dtype))
        R.assert_rejected(R.conv_f2(dx, dy, wt, nbrT, row=int(size.argmax())), ref, "F2")
        R.assert_rejected(R.conv_f4(dx, ref, dy, wt, nbrT), ref, "F4")


def test_rulebook_transpose_k3(product):
    """b2s_rulebook_transpose of the (3,1,1)-stride-(2,1,1) table (K = 3) against an index-level transpose, with table
    rows past the live count and a capacity past n_in left at -1"""
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(31)
    n_in, nbr = R.table_rows(rng, "k311", 3000)
    n_out = nbr.shape[0]
    assert nbr.shape[1] == 3
    tb = _poisoned_table(nbr, n_in, 40)
    out = torch.full((n_in + 9, 3), 12345, dtype=torch.int32, device="cuda")
    n_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rulebook_transpose(L.ptr(tb), L.ptr(n_dev), n_out + 40, 3, L.ptr(out), n_in + 9, L.ptr(status),
                                       L.stream()), "b2s_rulebook_transpose")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    want = np.full((n_in + 9, 3), -1, np.int32)
    want[:n_in] = R.transpose_table(nbr, n_in)
    assert np.array_equal(out.cpu().numpy(), want)


# ---- PFN ----------------------------------------------------------------------------------------------------------
VS, LO = (0.16, 0.16), (0.0, -39.68)
XOFF, YOFF = float(np.float32(VS[0] / 2 + LO[0])), float(np.float32(VS[1] / 2 + LO[1]))


def run_pfn(product, pts, slots, num, coors, w, scale, shift, radius, n_live, extra=9):
    """b2s_pfn (radius False) and b2s_pfn_ex over n_live live pillars of cap_rows = n + extra; rows past n_live are
    poisoned (slots name NaN points, counts T, coordinates off the grid) -> [n_live, 64] (b2s_pfn and b2s_pfn_ex with
    decoration 0 bit-identical)"""
    L = product._lib
    lib = L.load()
    n, T = slots.shape
    F = pts.shape[1]
    P = pts.shape[0]
    pb = _poisoned_rows(pts)
    cap = n + extra
    sl = torch.full((cap, T), P, dtype=torch.int32, device="cuda")
    sl[:n] = slots.cuda()
    sl[:n][slots.cuda() < 0] = P                                          # slots past num name a NaN point
    nm = torch.full((cap,), T, dtype=torch.int32, device="cuda")
    nm[:n] = num.cuda()
    co = torch.full((cap, 4), 100000, dtype=torch.int32, device="cuda")
    co[:n] = coors.cuda()
    n_dev = torch.tensor([n_live], dtype=torch.int32, device="cuda")
    args = (w.cuda().contiguous(), scale.cuda().contiguous(), shift.cuda().contiguous())
    outs = []
    calls = [(lib.b2s_pfn_ex, (1 if radius else 0,))] + ([] if radius else [(lib.b2s_pfn, ())])
    for fn, deco in calls:
        out = torch.full((cap + 1, 64), SENT, device="cuda")
        L.check(fn(L.ptr(pb), F, L.ptr(sl), L.ptr(nm), L.ptr(co), L.ptr(n_dev), cap, T, *[L.ptr(a) for a in args], 64,
                   VS[0], VS[1], XOFF, YOFF, *deco, L.ptr(out), L.stream()), "b2s_pfn")
        torch.cuda.synchronize()
        assert bool((out[n_live:] == SENT).all()), "rows past the live count were written"
        outs.append(out[:n_live])
    if len(outs) == 2:
        assert torch.equal(outs[0], outs[1])
    return outs[0]


PFN_CASES = [(F, T) for F, T in ((3, 1), (4, 20), (5, 100), (6, 2), (7, 32), (8, 60))]


@pytest.mark.parametrize("radius", [False, True], ids=["plain", "radius"])
@pytest.mark.parametrize("F,T", PFN_CASES)
def test_pfn(product, F, T, radius):
    rng = np.random.default_rng(F * 100 + T + radius)
    n = 700
    pts, slots, num, coors = R.pillars(rng, n, T, F)
    w, scale, shift = R.pfn_layer(rng, F, radius)
    t = torch.from_numpy
    args = (t(pts).cuda(), t(slots).cuda(), t(num).cuda(), t(coors).cuda(), t(w).cuda(), t(scale).cuda(),
            t(shift).cuda())
    n_live = n - 17
    got = run_pfn(product, *args, radius, n_live)
    live = [a[:n_live] if i in (1, 2, 3) else a for i, a in enumerate(args)]
    geo = (np.float32(VS[0]), np.float32(VS[1]), np.float32(XOFF), np.float32(YOFF))
    ref = R.pfn_ref(*live, *geo, radius=radius)
    R.assert_accurate(got, ref, "b2s_pfn")
    nm = live[2]
    part = nm < T
    assert torch.equal(got[part, :8].double(), ref.y[part, :8]), "channels decided by the padded-slot rule"
    for fault in R.PFN_FAULTS:
        if fault == "pad_drop" and not bool(part.any()):
            continue                                                  # T = 1: no pillar has a padded slot
        R.assert_rejected(R.pfn_fault(got, ref, fault, *live, *geo, radius=radius), ref, fault)


def test_pfn_no_live_rows(product):
    rng = np.random.default_rng(5)
    pts, slots, num, coors = R.pillars(rng, 40, 20, 4)
    w, scale, shift = R.pfn_layer(rng, 4, False)
    t = torch.from_numpy
    got = run_pfn(product, t(pts), t(slots), t(num), t(coors), t(w), t(scale), t(shift), False, 0)
    assert got.shape == (0, 64)


# ---- voxel mean ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vfe_mode", [1, 2])
@pytest.mark.parametrize("nf", [3, 4, 5])
def test_vfe_mean(product, vfe_mode, nf):
    """b2s_vfe_mean over gathered voxels (slots past num NaN), rows past the live count poisoned"""
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(nf * 3 + vfe_mode)
    n, T, F, extra = 3000, 5, 5, 11
    num = rng.integers(1, T + 1, n).astype(np.int32)
    num[:300], num[300:600] = 1, T
    vox = rng.uniform(-40, 70, (n, T, F)).astype(np.float32)
    vox[np.arange(T)[None, :] >= num[:, None]] = np.nan
    vb = torch.full((n + extra, T, F), float("nan"), device="cuda")
    vb[:n] = torch.from_numpy(vox).cuda()
    nm = torch.full((n + extra,), T, dtype=torch.int32, device="cuda")
    nm[:n] = torch.from_numpy(num).cuda()
    c = nf - (vfe_mode == 2)
    out = torch.full((n + extra + 1, c), SENT, device="cuda")
    n_dev = torch.tensor([n], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_vfe_mean(L.ptr(vb), L.ptr(nm), L.ptr(n_dev), n + extra, T, F, vfe_mode, nf, L.ptr(out), L.stream()),
            "b2s_vfe_mean")
    torch.cuda.synchronize()
    assert bool((out[n:] == SENT).all())
    got = out[:n]
    ref = R.vfe_ref(torch.from_numpy(vox).cuda(), torch.from_numpy(num).cuda(), nf, vfe_mode == 2)
    R.assert_accurate(got, ref, "b2s_vfe_mean")
    bad = R.vfe_ref(torch.from_numpy(vox).cuda(), torch.from_numpy(num).cuda(), nf, vfe_mode == 2, fault="mean")
    R.assert_rejected(got.double() + (bad.y - ref.y), ref, "mean over num - 1")


@pytest.mark.parametrize("vfe_mode", [1, 2])
@pytest.mark.parametrize("nf", [3, 4, 5])
def test_voxelize_fused_mean(product, vfe_mode, nf):
    """b2s_voxelize's fused mean (k_finish) against float64 over the voxels it gathered"""
    rng = np.random.default_rng(nf + 10 * vfe_mode)
    T, mv = 5, 6000
    pts = rng.uniform((0, -4, -3, 0, 0), (7, 4, 1, 1, 1), (20000, 5)).astype(np.float32)
    pts[::7] = pts[3]
    pts[5::11, :3] = pts[2, :3]
    gen = product.utils.VoxelGeneratorV2([0.05, 0.05, 0.1], [0, -4, -3, 7.04, 4, 1], T, mv)
    offs = torch.tensor([0, pts.shape[0]], dtype=torch.int32, device="cuda")
    res = gen.generate_device(torch.from_numpy(pts).cuda(), mv, frame_offsets=offs, batch=1, vfe_mode=vfe_mode,
                              vfe_num_features=nf)
    torch.cuda.synchronize()
    n = int(res["num_voxels"][0].item())
    num = res["num_points_per_voxel"][:n]
    assert bool((num == 1).any()) and bool((num == T).any())
    ref = R.vfe_ref(res["voxels"][:n], num, nf, vfe_mode == 2)
    got = res["vfe"][:n]
    R.assert_accurate(got, ref, "fused mean")
    bad = R.vfe_ref(res["voxels"][:n], num, nf, vfe_mode == 2, fault="mean")
    R.assert_rejected(got.double() + (bad.y - ref.y), ref, "mean over num - 1")
