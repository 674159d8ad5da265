"""The float64 references and error bounds of tests/fp32_ref.py, checked on the CPU before any kernel runs: emulations
of the fp32 kernels (float32 values, each fmaf as the exact float64 product and sum rounded once to float32, in the
kernels' order) meet every bound, and every simulated fault fails the same check."""
import numpy as np
import pytest
import torch

import fp32_ref as R


def _fma(acc, a, b):
    """fmaf(a, b, acc) elementwise: the exact product and the sum in float64, rounded once to float32"""
    return (acc.double() + a.double() * b.double()).float()


def emulate_conv(x, w, nbr, scale=None, shift=None, relu=False, ftz=False):
    """k_sparse_conv / k_sparse_conv_generic: per output element one chain, k ascending, then c ascending"""
    nbr = torch.as_tensor(nbr).long()
    K, cin, cout = w.shape
    acc = torch.zeros(nbr.shape[0], cout)
    for k in range(K):
        ok = nbr[:, k] >= 0
        a = torch.where(ok[:, None], x[nbr[:, k].clamp_min(0)], torch.zeros(()))
        for c in range(cin):
            acc = _fma(acc, a[:, c:c + 1], w[k, c][None])
    sh = torch.zeros(cout) if shift is None else shift
    v = _fma(sh[None].expand_as(acc), acc, scale[None]) if scale is not None else acc + sh
    return torch.relu(v) if relu else v


def emulate_wgrad(x, g, nbr, ftz=False):
    """b2s_sparse_conv_wgrad: rows ascending inside each 2048-row slab, then the slab partials added in order"""
    nbr = torch.as_tensor(nbr).long()
    n_out, K = nbr.shape
    total = torch.zeros(K, x.shape[1], g.shape[1])
    for j in range(0, n_out, R.SLAB):
        acc = torch.zeros_like(total)
        for o in range(j, min(n_out, j + R.SLAB)):
            ok = nbr[o] >= 0
            a = torch.where(ok[:, None], x[nbr[o].clamp_min(0)], torch.zeros(()))
            prod = a.double()[:, :, None] * g[o].double()[None, None, :]
            if ftz:
                prod = torch.where(prod.abs() < 2.0 ** -126, torch.zeros(()).double(), prod)
            acc = (acc.double() + prod).float()
        total = total + acc
    return total


def emulate_pfn(points, slots, num, coors, w, scale, shift, vx, vy, xoff, yoff, radius=False):
    """k_pfn: the mean summed in slot order, the centre and offsets rounded op by op, the Linear as one fmaf chain over
    the inputs in order, BN as fmaf, the max over the real slots and relu(shift) while num < T"""
    n, T = slots.shape
    f32 = torch.float32
    live = torch.arange(T)[None, :] < num[:, None].long()
    p = torch.where(live[..., None], points[slots.long().clamp_min(0)], torch.zeros((), dtype=f32))
    s = torch.zeros(n, 3)
    for t in range(T):
        s = s + p[:, t, :3]                       # +0 past num: exact
    m = s / num[:, None].to(f32)
    vxy = torch.tensor([vx, vy], dtype=f32)
    cxy = coors[:, [3, 2]].to(f32) * vxy + torch.tensor([xoff, yoff], dtype=f32)
    if radius:
        r = torch.sqrt(p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1])
        raw = torch.cat([r[..., None], p[..., 2:]], -1)
    else:
        raw = p
    inp = torch.cat([raw, p[..., :3] - m[:, None], p[..., :2] - cxy[:, None]], -1)
    acc = torch.zeros(n, T, w.shape[0])
    for f in range(inp.shape[-1]):
        acc = _fma(acc, inp[..., f:f + 1], w[:, f][None, None])
    v = torch.relu(_fma(shift.expand_as(acc), acc, scale))
    v = torch.where(live[..., None], v, torch.full((), -float("inf")))
    pad = torch.where((num < T)[:, None], torch.relu(shift)[None], torch.full((), -float("inf")))
    return torch.maximum(v.max(1).values, pad)


def emulate_vfe(voxels, num, nf, radius=False):
    n, T, _ = voxels.shape
    live = (torch.arange(T)[None, :] < num[:, None].long())[..., None]
    v = torch.where(live, voxels[..., :nf], torch.zeros(()))
    s = torch.zeros(n, nf)
    for t in range(T):
        s = s + v[:, t]
    m = s / num[:, None].float()
    if not radius:
        return m
    return torch.cat([torch.sqrt(m[:, :1] * m[:, :1] + m[:, 1:2] * m[:, 1:2]), m[:, 2:]], 1)


# ---- tables -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table", list(R.TABLES))
def test_table_against_brute_force(table):
    rng = np.random.default_rng(1)
    idx = R.surface_coords(rng, 300)
    ks, st, pd, subm = R.TABLES[table]
    out, nbr = R.build_table(idx, R.SHAPE, ks, st, pd, subm)
    pos = {tuple(p): i for i, p in enumerate(idx.tolist())}
    offs = R._offsets(ks)
    pad = np.array(ks) // 2 if subm else np.array(pd)
    for o in range(out.shape[0]):
        for k, d in enumerate(offs):
            p = (int(out[o, 0]),) + tuple(int(v) for v in out[o, 1:] * np.array(st) - pad + d)
            assert nbr[o, k] == pos.get(p, -1)
        assert (nbr[o] >= 0).any()
    if subm:
        assert np.array_equal(out, idx)
        c = nbr.shape[1] // 2
        assert np.array_equal(nbr[:, c], np.arange(idx.shape[0]))
    nT = R.transpose_table(nbr, idx.shape[0])
    o, k = np.nonzero(nT >= 0)
    assert np.array_equal(nbr[nT[o, k], k], o)
    assert (nT >= 0).sum() == (nbr >= 0).sum()


# ---- sparse convolution -------------------------------------------------------------------------------------------
CONV_CASES = [(3, 16, "subm", 70, True), (16, 32, "strided", 65, True), (8, 64, "k311", 64, False),
              (5, 7, "subm5", 40, True), (4, 16, "k1", 1, False), (64, 64, "subm", 130, True)]


def _conv_case(cin, cout, table, n_out, epilogue, e=0, seed=0):
    rng = np.random.default_rng(seed + cin + cout)
    n_in, nbr = R.table_rows(rng, table, n_out)
    K = nbr.shape[1]
    g = torch.Generator().manual_seed(seed + cin * cout)
    x = torch.randn(n_in, cin, generator=g) * 2.0 ** e
    w = torch.randn(K, cin, cout, generator=g) * (2.0 / (K * cin)) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5 if epilogue else None
    shift = torch.randn(cout, generator=g) * 0.1 * 2.0 ** e if epilogue else None
    return x, w, torch.from_numpy(nbr), scale, shift


@pytest.mark.parametrize("cin,cout,table,n_out,epilogue", CONV_CASES)
def test_conv_emulation_meets_the_bound_and_faults_fail(cin, cout, table, n_out, epilogue):
    x, w, nbr, scale, shift = _conv_case(cin, cout, table, n_out, epilogue)
    relu = epilogue
    ref = R.sparse_ref(x, w, nbr, scale, shift, relu)
    got = emulate_conv(x, w, nbr, scale, shift, relu)
    st = R.assert_accurate(got, ref, "emulated kernel")
    assert st["rms"] <= R.RHO / 2, "the 2x margin of RHO: %r" % st
    R.assert_rejected(R.conv_f1(got, x, w, nbr, scale, relu), ref, "F1")
    R.assert_rejected(R.conv_f2(got, x, w, nbr, scale, relu), ref, "F2")
    st4 = R.assert_rejected(R.conv_f4(got, ref, x, w, nbr, scale, shift, relu), ref, "F4")
    assert st4["rms"] > R.RHO, "F4 must fail the aggregate check (%r)" % st4


@pytest.mark.parametrize("e", [-40, -20, 0, 20])
def test_conv_emulation_magnitude_sweep(e):
    x, w, nbr, scale, shift = _conv_case(16, 16, "subm", 100, True, e=e, seed=5)
    ref = R.sparse_ref(x, w, nbr, scale, shift, True)
    got = emulate_conv(x, w, nbr, scale, shift, True)
    R.assert_accurate(got, ref, "2^%d" % e)
    R.assert_rejected(R.conv_f1(got, x, w, nbr, scale, True), ref, "F1")
    R.assert_rejected(R.conv_f2(got, x, w, nbr, scale, True), ref, "F2")
    R.assert_rejected(R.conv_f4(got, ref, x, w, nbr, scale, shift, True), ref, "F4")


def test_conv_precision_loss_is_caught_only_by_the_aggregate():
    """the worst-case bound alone lets F4 through at n = 27 * 64: the aggregate check is what rejects it"""
    x, w, nbr, scale, shift = _conv_case(64, 64, "subm", 300, False, seed=2)
    nbr = torch.from_numpy(np.broadcast_to(np.arange(27, dtype=np.int32)[None] % x.shape[0], (300, 27)).copy())
    ref = R.sparse_ref(x, w, nbr)
    got = emulate_conv(x, w, nbr)
    st = R.error_stats(R.conv_f4(got, ref, x, w, nbr), ref)
    assert st["ratio"] <= 1.0 and st["rms"] > R.RHO, st


# ---- weight gradient ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e", [0, -126, -130])
def test_wgrad_emulation_meets_the_bound_and_faults_fail(e):
    rng = np.random.default_rng(7)
    n_in, nbr = R.table_rows(rng, "subm", 2049)                    # two slabs, the second of one row
    nbr = torch.from_numpy(nbr)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(n_in, 5, generator=g)
    dy = torch.randn(2049, 3, generator=g) * 2.0 ** e
    ref = R.wgrad_ref(x, dy, nbr)
    got = emulate_wgrad(x, dy, nbr)
    st = R.assert_accurate(got, ref, "emulated kernel")
    assert st["rms"] <= R.RHO / 2
    R.assert_rejected(R.wgrad_f1(got, x, dy, nbr), ref, "F1")
    R.assert_rejected(R.wgrad_f1(got, x, dy, nbr, slab=1), ref, "F1 last slab")
    R.assert_rejected(R.wgrad_f2(got, x, dy, nbr), ref, "F2")
    if e >= -100:
        R.assert_rejected(R.wgrad_f4(got, ref, x, dy, nbr), ref, "F4")
    else:
        # subnormal products: flushing them to zero must fail
        R.assert_rejected(emulate_wgrad(x, dy, nbr, ftz=True), ref, "flush to zero")


# ---- PFN ----------------------------------------------------------------------------------------------------------
VS, LO = (0.16, 0.16), (0.0, -39.68)
XOFF, YOFF = VS[0] / 2 + LO[0], VS[1] / 2 + LO[1]


def _pfn_case(F, T, radius, n=60, seed=0):
    rng = np.random.default_rng(seed + F * 10 + T + radius)
    pts, slots, num, coors = R.pillars(rng, n, T, F)
    w, scale, shift = R.pfn_layer(rng, F, radius)
    t = torch.from_numpy
    return (t(pts), t(slots), t(num), t(coors), t(w), t(scale), t(shift), np.float32(VS[0]), np.float32(VS[1]),
            np.float32(XOFF), np.float32(YOFF))


@pytest.mark.parametrize("radius", [False, True], ids=["plain", "radius"])
@pytest.mark.parametrize("F,T", [(3, 1), (4, 20), (5, 2), (8, 32)])
def test_pfn_emulation_meets_the_bound_and_faults_fail(F, T, radius):
    args = _pfn_case(F, T, radius)
    ref = R.pfn_ref(*args, radius=radius)
    got = emulate_pfn(*args, radius=radius)
    st = R.assert_accurate(got, ref, "emulated kernel")
    assert st["rms"] <= R.RHO / 2
    num = args[2]
    for fault in R.PFN_FAULTS:
        if fault == "pad_drop" and not bool((num < T).any()):
            continue                                                # T = 1: no pillar has a padded slot
        R.assert_rejected(R.pfn_fault(got, ref, fault, *args, radius=radius), ref, fault)
    # in pillars with a padded slot, the padded-slot rule alone decides the first channels: they are exact
    part = num < T
    assert torch.equal(got[part, :8].double(), ref.y[part, :8])


# ---- voxel mean ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("radius", [False, True], ids=["mean", "radius"])
@pytest.mark.parametrize("nf", [3, 4, 5])
def test_vfe_emulation_meets_the_bound_and_faults_fail(nf, radius):
    rng = np.random.default_rng(nf)
    T = 5
    num = torch.from_numpy(rng.integers(1, T + 1, 200).astype(np.int32))
    num[:20], num[20:40] = 1, T
    vox = torch.from_numpy(rng.uniform(-40, 70, (200, T, 5)).astype(np.float32))
    ref = R.vfe_ref(vox, num, nf, radius)
    got = emulate_vfe(vox, num, nf, radius)
    st = R.assert_accurate(got, ref, "emulated kernel")
    assert st["rms"] <= R.RHO / 2
    R.assert_rejected(got.double() + (R.vfe_ref(vox, num, nf, radius, fault="mean").y - ref.y), ref, "mean fault")
