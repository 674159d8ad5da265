"""GPU parity of the tensor-pipe sparse convolution (b2s_sparse_conv_tc, wgmma f16 + 3xF16) against the CPU
oracle's sparse conv (fp32).  Same rulebook (b2s_rulebook_*), same BN/ReLU epilogue; bar 2e-5 * max|ref| per layer."""
import numpy as np
import pytest
import torch

import tc_ref

pytestmark = pytest.mark.gpu


def random_sparse(rng, shape, batch, n, cin):
    D, H, W = shape
    flat = rng.choice(batch * D * H * W, size=n, replace=False)
    b, r = np.divmod(flat, D * H * W)
    z, r = np.divmod(r, H * W)
    y, x = np.divmod(r, W)
    idx = np.stack([b, z, y, x], 1).astype(np.int32)
    feats = rng.standard_normal((n, cin)).astype(np.float32)
    return torch.from_numpy(feats), torch.from_numpy(idx)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("cin,cout", [(32, 32), (32, 64), (64, 64), (64, 32), (4, 16), (3, 16), (16, 16), (16, 32),
                                      (64, 16), (8, 64)])
@pytest.mark.parametrize("subm", [True, False])
@pytest.mark.parametrize("n", [5000, 100, 0])
def test_sparse_conv_tc_matches_oracle(product, oracle, cin, cout, subm, n):
    from b2second import tc
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(cin * 7 + cout + subm + n)
    shape, batch = (11, 40, 36), 2
    feats, idx = random_sparse(rng, shape, batch, n, cin)
    if subm:
        oc = oracle.SubMConv3d(cin, cout, 3, bias=False, indice_key="k")
        k, s, p = [3, 3, 3], [1, 1, 1], [1, 1, 1]
    else:
        oc = oracle.SparseConv3d(cin, cout, 3, 2, padding=[0, 1, 1], bias=False)
        k, s, p = [3, 3, 3], [2, 2, 2], [0, 1, 1]
    scale = torch.rand(cout) + 0.5
    shift = torch.randn(cout) * 0.1
    with torch.no_grad():
        yo = oc(oracle.SparseConvTensor(feats, idx, shape, batch))
        ref = torch.relu(yo.features * scale + shift)
    x = product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch)
    rb = product.ops.build_rulebook(x, k, s, p, [1, 1, 1], subm)
    assert rb.num_out == yo.features.shape[0]
    if rb.num_out == 0:
        return
    w = oc.weight.detach().view(27, cin, cout).cuda()
    cin_tc = tc.sparse_tc_cin(cin)
    assert lib.b2s_sparse_conv_tc_supported(cin_tc, cout)
    wp = tc.pack_sparse_weights(w)           # [K,Cout,64], or packed K blocks for Cin < 64 (Cin 3/4 padded to 8)
    ws = tc.pow2_scale(wp)
    w_hi, w_lo = tc.split_f16(wp, ws)
    n_in = feats.shape[0]
    fbuf = torch.zeros(max(n_in, 1), 2, cin_tc, dtype=torch.float16, device="cuda")   # interleaved [row][hi | lo]
    f_hi, f_lo, fstride = fbuf[:, 0], fbuf[:, 1], 2 * cin_tc
    feats_d = feats.cuda()
    n_in_dev = torch.tensor([n_in], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_split_f16(L.ptr(feats_d), L.ptr(f_hi), L.ptr(f_lo), L.ptr(n_in_dev), n_in, cin, cin_tc, fstride,
                              L.stream()), "b2s_split_f16")
    ref_hi, ref_lo = tc.split_f16(feats_d)
    torch.cuda.synchronize()
    assert torch.equal(f_hi[:n_in, :cin], ref_hi) and torch.equal(f_lo[:n_in, :cin], ref_lo)   # device split == host split
    assert float(f_hi[:, cin:].float().abs().sum()) == 0.0                                     # zero padding
    obuf = torch.zeros(rb.num_out, 2, cout, dtype=torch.float16, device="cuda")
    o_hi, o_lo = obuf[:, 0], obuf[:, 1]
    scale_d, shift_d, nbr = (scale / ws).cuda(), shift.cuda(), rb.nbr.contiguous()   # keep alive across the async launch
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_sparse_conv_tc(L.ptr(f_hi), L.ptr(f_lo), fstride, n_in, cin_tc, L.ptr(w_hi), L.ptr(w_lo), L.ptr(nbr),
                                   27, L.ptr(rb.num_out_dev), rb.num_out, L.ptr(scale_d), L.ptr(shift_d), 1,
                                   L.ptr(o_hi), L.ptr(o_lo), 2 * cout, cout, L.ptr(status), L.stream()),
            "b2s_sparse_conv_tc")
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    got = (o_hi.float() + o_lo.float()).cpu()
    err = (got - ref).abs().max().item()
    assert err <= 2e-5 * max(ref.abs().max().item(), 1.0), "max err %g (ref max %g)" % (err, ref.abs().max().item())
    # fp32 output variant (out_lo NULL) gives the same values before the split
    o32 = torch.zeros(rb.num_out, cout, device="cuda")
    L.check(lib.b2s_sparse_conv_tc(L.ptr(f_hi), L.ptr(f_lo), fstride, n_in, cin_tc, L.ptr(w_hi), L.ptr(w_lo), L.ptr(nbr),
                                   27, L.ptr(rb.num_out_dev), rb.num_out, L.ptr(scale_d), L.ptr(shift_d), 1,
                                   L.ptr(o32), None, 0, cout, L.ptr(status), L.stream()), "b2s_sparse_conv_tc")
    m = torch.zeros(rb.num_out, cout, device="cuda")
    L.check(lib.b2s_merge_f16(L.ptr(o_hi), L.ptr(o_lo), L.ptr(m), L.ptr(rb.num_out_dev), rb.num_out, cout, 2 * cout,
                              L.stream()), "b2s_merge_f16")
    torch.cuda.synchronize()
    assert torch.equal(m, o_hi.float() + o_lo.float())          # merge is exact
    assert float((o32 - m).abs().max()) <= 2e-7 * max(1.0, float(o32.abs().max())) + 6e-8   # split drops < 2^-22 rel / 2^-25 abs
    # fp32 rows against the float64 gather-GEMM of the same table, per element
    r64 = tc_ref.sparse_ref(feats_d, w, rb.nbr[:rb.num_out], scale, shift, True)
    tc_ref.assert_accurate(o32.double(), r64, ws, "fp32 rows")
    tc_ref.assert_rejected(tc_ref.sparse_f1(o32.double(), feats_d, w, ws, rb.nbr[:rb.num_out], r64, True, cin_tc),
                           r64, ws, "F1")
    tc_ref.assert_rejected(tc_ref.sparse_f2(o32.double(), feats_d, w, ws, rb.nbr[:rb.num_out], r64, True), r64, ws, "F2")
    tc_ref.assert_rejected(tc_ref.f3(o32.double(), None), r64, ws, "F3")


@pytest.mark.timeout(180)
def test_drop_in_sparse_sequential_runs_on_tensor_cores(product, oracle):
    """spconv.SparseSequential in eval mode (the reference's middle_conv) on the wgmma kernel: hi/lo planes flow from
    layer to layer, .features materialises fp32 lazily, results match the oracle package layer stack."""
    from torch import nn
    torch.manual_seed(0)
    rng = np.random.default_rng(5)
    shape, batch = (11, 40, 36), 2
    feats, idx = random_sparse(rng, shape, batch, 4000, 4)

    def build(sp):
        def bn(c):
            m = nn.BatchNorm1d(c, eps=1e-3, momentum=0.01)
            return m
        return sp.SparseSequential(
            sp.SubMConv3d(4, 16, 3, bias=False, indice_key="s0"), bn(16), nn.ReLU(),
            sp.SubMConv3d(16, 16, 3, bias=False, indice_key="s0"), bn(16), nn.ReLU(),
            sp.SparseConv3d(16, 32, 3, 2, padding=1, bias=False), bn(32), nn.ReLU(),
            sp.SubMConv3d(32, 32, 3, bias=False, indice_key="s1"), bn(32), nn.ReLU(),
            sp.SparseConv3d(32, 64, 3, 2, padding=[0, 1, 1], bias=False), bn(64), nn.ReLU(),
            sp.SubMConv3d(64, 64, 3, bias=False, indice_key="s2"), bn(64), nn.ReLU()).eval()
    ref_net = build(oracle)
    g = torch.Generator().manual_seed(1)
    for k, v in ref_net.state_dict().items():
        if v.dtype.is_floating_point:
            if k.endswith("running_var"):
                v.copy_(torch.rand(v.shape, generator=g) + 0.5)
            elif v.dim() >= 2:
                v.copy_((torch.rand(v.shape, generator=g) * 2 - 1) * (6.0 / np.prod(v.shape[:-1])) ** 0.5)
            else:
                v.copy_(torch.randn(v.shape, generator=g) * 0.3 + (1.0 if k.endswith("weight") else 0.0))
    net = build(product)
    net.load_state_dict(ref_net.state_dict())
    net = net.cuda()
    with torch.no_grad():
        yo = ref_net(oracle.SparseConvTensor(feats, idx, shape, batch))
        y = net(product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch))
    assert y._hilo is not None and y._features is None            # stayed on the tensor pipe, nothing merged yet
    assert torch.equal(y.indices.cpu(), yo.indices)
    got = y.features.cpu()
    assert float((got - yo.features).abs().max()) <= 1e-4 * max(1.0, float(yo.features.abs().max()))
    d = y.dense().cpu()
    assert float((d - yo.dense()).abs().max()) <= 1e-4 * max(1.0, float(yo.features.abs().max()))
    # training mode must fail loudly instead of returning gradient-free tensors
    net.train()
    with pytest.raises(NotImplementedError):
        net(product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch))
    with torch.no_grad():                                          # nothing to record: allowed
        net(product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch))


def _clustered_sparse(rng, shape, batch, n, cin):
    """surface-like occupancy (a noisy sheet per frame) so that rows have structured, differing neighbourhoods."""
    D, H, W = shape
    pts = set()
    while len(pts) < n:
        b = int(rng.integers(batch)); y = int(rng.integers(H)); x = int(rng.integers(W))
        z = int(np.clip(round(D / 2 + 2 * np.sin(x / 5.0) + rng.normal(0, 0.7)), 0, D - 1))
        pts.add((b, z, y, x))
    idx = np.array(sorted(pts), dtype=np.int32)
    feats = rng.standard_normal((idx.shape[0], cin)).astype(np.float32)
    return torch.from_numpy(feats), torch.from_numpy(idx)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("cin,cout", [(64, 64), (32, 32), (16, 32), (4, 16)])
@pytest.mark.parametrize("subm", [True, False])
@pytest.mark.parametrize("n", [20000, 300, 1])
def test_tile_plan_properties_and_bit_identity(product, cin, cout, subm, n):
    """b2s_sparse_tile_plan: perm is a permutation that only moves rows inside 8192-row chunks, tile_mask is exactly the
    OR of the tile's row masks (sorted and unsorted); b2s_sparse_conv_tc_plan gives BIT-IDENTICAL rows with no plan, with
    masks only and with grouped rows (fixed chain boundaries + exact zeros for missing neighbours)."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(cin + cout + subm + n)
    shape, batch = (9, 48, 40), 3
    feats, idx = _clustered_sparse(rng, shape, batch, n, cin)
    x = product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch)
    k = [3, 3, 3]
    s, p = ([1, 1, 1], [1, 1, 1]) if subm else ([2, 2, 2], [1, 1, 1])
    rb = product.ops.build_rulebook(x, k, s, p, [1, 1, 1], subm)
    n_out = rb.num_out
    assert n_out > 0
    nbr = rb.nbr.contiguous()
    ksz = L.i3(k)
    cap = n_out + 77                                  # capacity above the live row count
    nbr_cap = torch.full((cap, 27), -1, dtype=torch.int32, device="cuda"); nbr_cap[:n_out] = nbr[:n_out]
    ntiles = (cap + 127) // 128
    row_mask = ((nbr_cap[:n_out] >= 0).long() << torch.arange(27, device="cuda")).sum(1)        # [n_out]
    plans = {}
    for sort in (0, 1):
        perm = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        tmask = torch.full((ntiles,), -1, dtype=torch.int32, device="cuda")
        L.check(lib.b2s_sparse_tile_plan(L.ptr(nbr_cap), None, 27, ksz, L.ptr(rb.num_out_dev), cap, sort, L.ptr(perm),
                                         L.ptr(tmask), L.stream()), "b2s_sparse_tile_plan")
        # same plan from the row masks the rulebook builder wrote (no second pass over the table)
        perm2 = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        tmask2 = torch.full((ntiles,), -1, dtype=torch.int32, device="cuda")
        rm_cap = torch.zeros(cap, dtype=torch.int32, device="cuda"); rm_cap[:n_out] = rb.row_mask[:n_out]
        L.check(lib.b2s_sparse_tile_plan(None, L.ptr(rm_cap), 27, ksz, L.ptr(rb.num_out_dev), cap, sort, L.ptr(perm2),
                                         L.ptr(tmask2), L.stream()), "b2s_sparse_tile_plan")
        torch.cuda.synchronize()
        assert torch.equal(rb.row_mask[:n_out].long(), row_mask), "row masks from the rulebook builder"
        assert torch.equal(perm, perm2) and torch.equal(tmask[:(n_out + 127) // 128], tmask2[:(n_out + 127) // 128])
        order = perm[:n_out].long() if sort else torch.arange(n_out, device="cuda")
        if sort:
            assert torch.equal(torch.sort(order).values, torch.arange(n_out, device="cuda"))       # a permutation
            assert torch.equal(order // 8192, torch.arange(n_out, device="cuda") // 8192)           # chunk-local
            assert bool((perm[n_out:] == -7).all())                                                 # nothing past the rows
        else:
            assert bool((perm == -7).all())
        live_tiles = (n_out + 127) // 128
        pad = torch.zeros(live_tiles * 128, dtype=torch.long, device="cuda"); pad[:n_out] = row_mask[order]
        want = pad.view(live_tiles, 128)
        acc = want[:, 0].clone()
        for j in range(1, 128):
            acc |= want[:, j]
        assert torch.equal(tmask[:live_tiles].long() & 0x7FFFFFF, acc), "tile masks (sort=%d)" % sort
        plans[sort] = (perm if sort else None, tmask)
    if n >= 20000 and subm:
        # grouping must pay: fewer (tile, offset) blocks than storage order
        def blocks(t):
            return int(sum(bin(int(v) & 0x7FFFFFF).count("1") for v in t[:(n_out + 127) // 128].tolist()))
        assert blocks(plans[1][1]) <= blocks(plans[0][1])
    # ---- convolution: identical bits with every plan ----
    w = (torch.randn(27, cin, cout) * 0.1).cuda()
    cin_tc = tc.sparse_tc_cin(cin)
    wp = tc.pack_sparse_weights(w)
    ws = tc.pow2_scale(wp)
    w_hi, w_lo = tc.split_f16(wp, ws)
    n_in = feats.shape[0]
    fbuf = torch.zeros(n_in, 2, cin_tc, dtype=torch.float16, device="cuda")
    f_hi, f_lo, fstride = fbuf[:, 0], fbuf[:, 1], 2 * cin_tc
    feats_d = feats.cuda()
    n_in_dev = torch.tensor([n_in], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_split_f16(L.ptr(feats_d), L.ptr(f_hi), L.ptr(f_lo), L.ptr(n_in_dev), n_in, cin, cin_tc, fstride,
                              L.stream()), "b2s_split_f16")
    scale_d = (torch.rand(cout) + 0.5).cuda() / ws
    shift_d = (torch.randn(cout) * 0.1).cuda()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    outs = []
    for perm, tmask in [(None, None), (None, plans[0][1]), plans[1]]:
        obuf = torch.full((cap, 2, cout), 7.0, dtype=torch.float16, device="cuda")
        L.check(lib.b2s_sparse_conv_tc_plan(L.ptr(f_hi), L.ptr(f_lo), fstride, n_in, cin_tc, L.ptr(w_hi), L.ptr(w_lo),
                                            L.ptr(nbr_cap), 27, L.ptr(rb.num_out_dev), cap, L.ptr(perm), L.ptr(tmask),
                                            L.ptr(scale_d), L.ptr(shift_d), 1, L.ptr(obuf[:, 0]), L.ptr(obuf[:, 1]),
                                            2 * cout, cout, L.ptr(status), L.stream()), "b2s_sparse_conv_tc_plan")
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        assert bool((obuf[n_out:] == 7.0).all())          # rows past the live count untouched
        outs.append(obuf[:n_out].clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    # and they are the right values
    ref = torch.zeros(n_out, cout, device="cuda", dtype=torch.float64)
    fd = feats_d.double()
    for kk in range(27):
        src = nbr_cap[:n_out, kk].long()
        ok = src >= 0
        ref[ok] += fd[src[ok]] @ w[kk].double()
    ref = torch.relu(ref * (scale_d * ws).double() + shift_d.double())
    got = outs[0][:, 0].double() + outs[0][:, 1].double()
    assert float((got - ref).abs().max()) <= 2e-5 * max(1.0, float(ref.abs().max()))
