"""GPU tests of the sparse convolution backward (b2second.training.enable_sparse_backward) against the CPU oracle's
float64 autograd: the kernels (weight gradient, input gradient on the tensor pipe and in fp32, dense() backward), a
SparseSequential with BN/ReLU in train() mode, and SECOND's middle encoders (car.fhd, car.lite)."""
import numpy as np
import pytest
import torch
from torch import nn

import golden_util as gu
from b2second import config, models, training

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_torch():
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


@pytest.fixture(params=[True, False], ids=["tc", "fp32"])
def pipe(request, product, monkeypatch):
    """tensor pipe where the widths allow (the default), or B2S_SPCONV_TC=0 (fp32 FMA kernels everywhere)"""
    monkeypatch.setattr(product, "USE_TENSOR_CORES", request.param)
    return request.param


def random_sparse(rng, shape, batch, n, cin):
    D, H, W = shape
    flat = rng.choice(batch * D * H * W, size=n, replace=False)
    b, r = np.divmod(flat, D * H * W)
    z, r = np.divmod(r, H * W)
    y, x = np.divmod(r, W)
    idx = np.stack([b, z, y, x], 1).astype(np.int32)
    feats = rng.standard_normal((n, cin)).astype(np.float32)
    return torch.from_numpy(feats), torch.from_numpy(idx)


def _oracle_conv(oracle, cin, cout, subm, w):
    if subm:
        c = oracle.SubMConv3d(cin, cout, 3, bias=False, indice_key="k")
    else:
        c = oracle.SparseConv3d(cin, cout, 3, 2, padding=[0, 1, 1], bias=False)
    c = c.double()
    with torch.no_grad():
        c.weight.copy_(w.double().view(c.weight.shape))
    return c


def _oracle_grads(oracle, conv, feats, idx, shape, batch, g):
    """(out indices, dX, dW) of sum(out * g) through the oracle conv, float64"""
    conv.weight.grad = None
    x = feats.double().clone().requires_grad_()
    y = conv(oracle.SparseConvTensor(x, idx, shape, batch))
    (y.features * g.double()).sum().backward()
    return y.indices, x.grad, conv.weight.grad.view(-1, conv.in_channels, conv.out_channels).clone()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("cin,cout", [(64, 64), (32, 32), (16, 32), (4, 16)])
@pytest.mark.parametrize("subm", [True, False])
@pytest.mark.parametrize("n", [20000, 300, 1])
def test_dgrad_wgrad_kernels_match_oracle(product, oracle, pipe, cin, cout, subm, n):
    """weight gradient (b2s_sparse_conv_wgrad_tc on the tensor pipe, b2s_sparse_conv_wgrad in fp32) and input gradient
    (SubM: forward kernel over the same table with flipped weights; strided: over b2s_rulebook_transpose's table), dY at
    scales 1, 2^-30, 2^10.  Bar per element:
    |g - g64| <= 1e-5 * the same gradient of the absolute values (|X|^T |dY| for dW, |W| |dY| for dX)."""
    rng = np.random.default_rng(cin * 3 + cout + subm * 7 + n)
    shape, batch = (9, 48, 40), 3
    feats, idx = random_sparse(rng, shape, batch, n, cin)
    w = torch.from_numpy(rng.uniform(-1, 1, (27, cin, cout)).astype(np.float32)) * (6.0 / (27 * cin)) ** 0.5
    oc = _oracle_conv(oracle, cin, cout, subm, w)
    with torch.no_grad():
        n_out = oc(oracle.SparseConvTensor(feats.double(), idx, shape, batch)).features.shape[0]
    g = torch.from_numpy(rng.standard_normal((n_out, cout)).astype(np.float32))
    oidx, dx64, dw64 = _oracle_grads(oracle, oc, feats, idx, shape, batch, g)
    oc_abs = _oracle_conv(oracle, cin, cout, subm, w.abs())
    _, dx_abs, _ = _oracle_grads(oracle, oc_abs, feats, idx, shape, batch, g.abs())
    _, _, dw_abs = _oracle_grads(oracle, oc, feats.abs(), idx, shape, batch, g.abs())

    conv = (product.SubMConv3d(cin, cout, 3, bias=False, indice_key="k") if subm else
            product.SparseConv3d(cin, cout, 3, 2, padding=[0, 1, 1], bias=False)).cuda()
    with torch.no_grad():
        conv.weight.copy_(w.view(conv.weight.shape))
    x = product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch)
    k, s, p = ([3, 3, 3], [1, 1, 1], [1, 1, 1]) if subm else ([3, 3, 3], [2, 2, 2], [0, 1, 1])
    rb = product.ops.build_rulebook(x, k, s, p, [1, 1, 1], subm)
    assert rb.num_out == n_out and torch.equal(rb.out_indices.cpu(), oidx)
    fd = feats.cuda().contiguous()
    for scale in (1.0, 2.0 ** -30, 2.0 ** 10):
        dy = (g * scale).cuda().contiguous()
        dw = conv._wgrad(fd, dy, rb)
        dw2 = conv._wgrad(fd, dy, rb)
        dx = conv._dgrad(dy, conv.weight, rb, n)
        torch.cuda.synchronize()
        assert torch.equal(dw, dw2), "weight gradient is not deterministic"
        err_w = (dw.cpu().double() - dw64 * scale).abs()
        bad = err_w > 1e-5 * dw_abs * scale
        assert not bad.any(), "dW scale %g: %d elements over the bar, worst ratio %g" % (
            scale, int(bad.sum()), float((err_w / (dw_abs * scale).clamp_min(1e-300)).max()))
        err_x = (dx.cpu().double() - dx64 * scale).abs()
        bad = err_x > 1e-5 * dx_abs * scale
        assert not bad.any(), "dX scale %g: %d elements over the bar, worst ratio %g" % (
            scale, int(bad.sum()), float((err_x / (dx_abs * scale).clamp_min(1e-300)).max()))
        if subm and pipe and scale == 1.0 and rb.plan is not None and rb.plan[0] is not None:
            saved, rb.plan = rb.plan, (None, None)       # the tile plan does not change a bit
            dx_noplan = conv._dgrad(dy, conv.weight, rb, n)
            rb.plan = saved
            torch.cuda.synchronize()
            assert torch.equal(dx, dx_noplan)
        if subm and pipe and rb.plan is not None and rb.plan[1] is not None:
            saved, rb.plan = rb.plan, (rb.plan[0], None)  # tensor-pipe wgrad: skipping by tile_mask changes no bit
            dw_nomask = conv._wgrad(fd, dy, rb)
            rb.plan = saved
            torch.cuda.synchronize()
            assert torch.equal(dw, dw_nomask)


def test_rulebook_transpose(product):
    rng = np.random.default_rng(3)
    shape, batch = (9, 48, 40), 2
    feats, idx = random_sparse(rng, shape, batch, 3000, 16)
    x = product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch)
    rb = product.ops.build_rulebook(x, [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False)
    nbrT = product.ops.transpose_rulebook(rb, 3000).cpu()
    nbr = rb.nbr.cpu()
    want = torch.full((3000, 27), -1, dtype=torch.int32)
    o, kk = torch.nonzero(nbr >= 0, as_tuple=True)
    want[nbr[o, kk].long(), kk] = o.int()
    assert torch.equal(nbrT, want)
    assert product.ops.transpose_rulebook(rb, 3000) is rb.nbrT          # cached on the rulebook


@pytest.mark.parametrize("channels_first", [True, False])
def test_from_bev_is_exact(product, channels_first):
    """b2s_from_bev against torch indexing, NCHW and NHWC, D = 2"""
    lib = product._lib.load()
    L = product._lib
    rng = np.random.default_rng(11)
    B, C, D, H, W = 2, 24, 2, 30, 20
    _, idx = random_sparse(rng, (D, H, W), B, 700, 1)
    idx = idx.cuda()
    layout = 0 if channels_first else 1
    dmap = torch.randn(B, C * D, H, W, device="cuda") if channels_first else torch.randn(B, H, W, C * D, device="cuda")
    drows = torch.full((700, C), 7.0, device="cuda")
    n_dev = torch.tensor([700], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_from_bev(L.ptr(dmap), L.ptr(idx), L.ptr(n_dev), 700, C, B, D, H, W, layout, L.ptr(drows), L.stream()),
            "b2s_from_bev")
    il = idx.long()
    ch = torch.arange(C, device="cuda")[None, :] * D + il[:, 1:2]
    if channels_first:
        want = dmap[il[:, 0:1], ch, il[:, 2:3], il[:, 3:4]]
    else:
        want = dmap[il[:, 0:1], il[:, 2:3], il[:, 3:4], ch]
    assert torch.equal(drows, want)
    # and dense() is differentiable through it
    f = torch.randn(700, C, device="cuda", requires_grad=True)
    t = product.SparseConvTensor(f, idx, [D, H, W], B)
    g = torch.randn(B, C, D, H, W, device="cuda")
    (t.dense() * g).sum().backward()
    assert torch.equal(f.grad, g.view(B, C * D, H, W)[il[:, 0:1], ch, il[:, 2:3], il[:, 3:4]])


def _seq(sp):
    def bn(c):
        return nn.BatchNorm1d(c, eps=1e-3, momentum=0.01)
    return sp.SparseSequential(
        sp.SubMConv3d(4, 16, 3, bias=False, indice_key="s0"), bn(16), nn.ReLU(),
        sp.SubMConv3d(16, 16, 3, bias=False, indice_key="s0"), bn(16), nn.ReLU(),
        sp.SparseConv3d(16, 32, 3, 2, padding=1, bias=False), bn(32), nn.ReLU(),
        sp.SubMConv3d(32, 32, 3, bias=False, indice_key="s1"), bn(32), nn.ReLU(),
        sp.SparseConv3d(32, 64, 3, 2, padding=[0, 1, 1], bias=False), bn(64), nn.ReLU(),
        sp.SubMConv3d(64, 64, 3, bias=False, indice_key="s2"), bn(64), nn.ReLU())


def _rel_err(got, ref):
    return float((got.detach().cpu().double() - ref.detach().double()).abs().max()) / max(
        float(ref.detach().abs().max()), 1e-300)


@pytest.mark.timeout(300)
def test_sparse_sequential_trains_like_the_oracle(product, oracle, pipe):
    """train() mode with enable_sparse_backward: every parameter gradient, the input gradient and the running BN
    statistics against the same module on the oracle in float64.  Bar ||g - g64||_inf <= 2e-4 ||g64||_inf on the tensor
    pipe, 2e-5 in fp32."""
    bar = 2e-4 if pipe else 2e-5
    rng = np.random.default_rng(5)
    shape, batch = (11, 40, 36), 2
    feats, idx = random_sparse(rng, shape, batch, 4000, 4)
    torch.manual_seed(0)
    ref = _seq(oracle)
    net = _seq(product)
    net.load_state_dict(ref.state_dict())
    ref = ref.double().train()
    net = training.enable_sparse_backward(net.cuda()).train()
    # without the opt-in the module still refuses to record
    plain = _seq(product).cuda().train()
    with pytest.raises(NotImplementedError):
        plain(product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch))

    x64 = feats.double().clone().requires_grad_()
    y64 = ref(oracle.SparseConvTensor(x64, idx, shape, batch))
    d64 = y64.dense()
    g = torch.randn(d64.shape, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    (d64 * g).sum().backward()

    x = feats.cuda().requires_grad_()
    y = net(product.SparseConvTensor(x, idx.cuda(), shape, batch))
    assert torch.equal(y.indices.cpu(), y64.indices)
    (y.dense() * g.float().cuda()).sum().backward()
    torch.cuda.synchronize()
    errs = {"input": _rel_err(x.grad, x64.grad)}
    for (name, p), (_, p64) in zip(net.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, name
        errs[name] = _rel_err(p.grad, p64.grad)
    for (name, b), (_, b64) in zip(net.named_buffers(), ref.named_buffers()):
        if b.dtype.is_floating_point:
            errs["buffer " + name] = _rel_err(b, b64)
    bad = {k: v for k, v in errs.items() if v > bar}
    assert not bad, "over the bar %g: %s" % (bar, bad)
    # eval() keeps the fused inference path (no autograd recorded, hi/lo planes between layers)
    net.eval()
    ye = net(product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch))
    assert ye.features.grad_fn is None


def _smooth(module):
    """every ReLU under `module` -> SiLU.  Measured on car.fhd seed 0 with ReLU (H100, float64 oracle): the forward's
    pre-activations differ from the oracle's by up to 4.8e-5 (tensor pipe) and 6.7e-5 (fp32 kernels, BN batch statistics
    in fp32) -- the fp32 pipe is NOT more accurate here -- and on each pipe one pre-activation in 10^6 lies closer to
    zero than that (|x64| = 1.5e-8 / 3.7e-7 on the tensor pipe, 3.2e-6 on the fp32 pipe) and lands on the other side of
    the kink.  Train-mode BatchNorm spreads that one element over every gradient below it: 1e-3 (up to 9e-3 for the
    conv just below it) relative, against 1e-6 when the float64 oracle is compared with itself in fp32.  A property of
    the comparison, not of the backward; a smooth activation compares the backward itself."""
    for name, m in list(module.named_modules()):
        for key, child in list(m._modules.items()):
            if isinstance(child, nn.ReLU):
                m._modules[key] = nn.SiLU()
    return module


def _middle_inputs(name, seed, n, oracle):
    cfg = config.get_config(name)
    onet = models.build_network(cfg, oracle)
    models.synthetic_weights_(onet, name, seed=0)
    res = onet.voxel_generator.generate(gu.make_cloud(name, seed, n), cfg.max_voxels)
    coords = torch.from_numpy(np.pad(res["coordinates"], ((0, 0), (1, 0))))
    with torch.no_grad():
        vf = onet.voxel_feature_extractor(torch.from_numpy(res["voxels"]), torch.from_numpy(res["num_points_per_voxel"]),
                                          coords)
    return cfg, onet, vf.float(), coords


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name,act", [("car.fhd", "silu"), ("car.lite", "relu"), ("car.lite", "silu")])
def test_middle_encoder_gradients_match_oracle(product, oracle, pipe, name, act):
    """SpMiddleFHD / SpMiddleFHDLite in train mode, loss = sum(dense_out * G): every middle gradient (and the voxel
    feature gradient) meets the module bar against the oracle in float64 (car.fhd with SiLU, see _smooth)"""
    bar = 2e-4 if pipe else 2e-5
    cfg, onet, vf, coords = _middle_inputs(name, 0, 20000, oracle)
    mid64 = onet.middle_feature_extractor.double().train()
    net = models.build_network(cfg, product)
    net.load_state_dict(onet.state_dict())
    mid = training.enable_sparse_backward(net.middle_feature_extractor.cuda()).train()
    if act == "silu":
        mid, mid64 = _smooth(mid), _smooth(mid64)
    v64 = vf.double().requires_grad_()
    o64 = mid64(v64, coords, 1)
    g = torch.randn(o64.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    (o64 * g).sum().backward()
    v = vf.cuda().requires_grad_()
    o = mid(v, coords.cuda(), 1)
    assert _rel_err(o, o64) <= bar
    (o * g.float().cuda()).sum().backward()
    torch.cuda.synchronize()
    errs = {"voxel features": _rel_err(v.grad, v64.grad)}
    for (pname, p), (_, p64) in zip(mid.named_parameters(), mid64.named_parameters()):
        errs[pname] = _rel_err(p.grad, p64.grad)
    bad = {k: e for k, e in errs.items() if e > bar}
    assert not bad, "over the bar %g: %s" % (bar, bad)


@pytest.mark.timeout(600)
def test_car_lite_sgd_trajectory_matches_oracle(product, oracle):
    """three SGD steps of car.lite's middle encoder (loss = sum(dense_out * G), SiLU: see _smooth) on the tensor pipe
    stay on the oracle's float64 trajectory: ||dp - dp64||_inf <= 2e-4 ||dp64||_inf for the change of every parameter.
    The steps are large (lr 0.1): with small ones the fp32 storage of a BN weight near 1 (2^-24 resolution) is itself a
    few 1e-4 of the change."""
    cfg, onet, vf, coords = _middle_inputs("car.lite", 1, 29000, oracle)
    mid64 = _smooth(onet.middle_feature_extractor.double().train())
    net = models.build_network(cfg, product)
    net.load_state_dict(onet.state_dict())
    mid = _smooth(training.enable_sparse_backward(net.middle_feature_extractor.cuda()).train())
    p0 = {k: v.detach().clone().double().cpu() for k, v in mid64.named_parameters()}
    opt64 = torch.optim.SGD(mid64.parameters(), lr=0.1, momentum=0.9)
    opt = torch.optim.SGD(mid.parameters(), lr=0.1, momentum=0.9)
    gen = torch.Generator().manual_seed(4)
    cuda_coords, cuda_vf, v64 = coords.cuda(), vf.cuda(), vf.double()
    for _ in range(3):
        o64 = mid64(v64, coords, 1)
        g = torch.randn(o64.shape, generator=gen, dtype=torch.float64) / o64.numel() ** 0.5
        opt64.zero_grad()
        (o64 * g).sum().backward()
        opt64.step()
        opt.zero_grad()
        (mid(cuda_vf, cuda_coords, 1) * g.float().cuda()).sum().backward()
        opt.step()
    torch.cuda.synchronize()
    errs = {}
    for (k, p), (_, p64) in zip(mid.named_parameters(), mid64.named_parameters()):
        errs[k] = _rel_err(p.detach().cpu().double() - p0[k], p64.detach() - p0[k])
    bad = {k: e for k, e in errs.items() if e > 2e-4}
    assert not bad, bad


@pytest.mark.parametrize("cin,cout", [(64, 64), (64, 16), (32, 32), (16, 32), (16, 64), (8, 16)])
def test_wgrad_tc_operand_layout_known_answer(product, cin, cout):
    """b2s_sparse_conv_wgrad_tc on integer X and one-hot dY rows (every product and sum exact in fp16 / fp32): the
    result equals the float64 contraction bit for bit, which pins the transposed SWIZZLE_128B staging of both operands,
    the packing of PACK = 64/Cin offsets into one K block and the unpacking into [K, Cin, Cout]"""
    L = product._lib
    lib = L.load()
    g = torch.Generator().manual_seed(cin + cout)
    n_in, n_out, K = 700, 3000, 27
    x = torch.randint(-8, 9, (n_in, cin), generator=g).float()
    dy = torch.zeros(n_out, cout)
    dy[torch.arange(n_out), torch.randint(0, cout, (n_out,), generator=g)] = 2.0 ** torch.randint(-3, 4, (n_out,),
                                                                                                  generator=g).float()
    nbr = torch.randint(0, n_in, (n_out, K), generator=g, dtype=torch.int32)
    nbr[torch.rand(n_out, K, generator=g) < 0.6] = -1
    want = torch.zeros(K, cin, cout, dtype=torch.float64)
    for k in range(K):
        ok = nbr[:, k] >= 0
        want[k] = x[nbr[ok, k].long()].double().t() @ dy[ok].double()
    xb = torch.zeros(n_in, 2, cin, dtype=torch.float16); xb[:, 0] = x.half()          # integers: lo plane zero
    gb = torch.zeros(n_out, 2, cout, dtype=torch.float16); gb[:, 0] = dy.half()
    xb, gb, nbr_d = xb.cuda(), gb.cuda(), nbr.cuda()
    n_dev = torch.tensor([n_out], dtype=torch.int32, device="cuda")
    ws = lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(n_out, K, cin, cout)
    work = torch.empty(ws, dtype=torch.uint8, device="cuda")
    dw = torch.full((K, cin, cout), 7.0, device="cuda")
    L.check(lib.b2s_sparse_conv_wgrad_tc(L.ptr(xb[:, 0]), L.ptr(xb[:, 1]), 2 * cin, n_in, cin, L.ptr(gb[:, 0]),
                                         L.ptr(gb[:, 1]), 2 * cout, cout, L.ptr(nbr_d), K, L.ptr(n_dev), n_out, None, None,
                                         None, L.ptr(dw), L.ptr(work), ws, L.stream()), "b2s_sparse_conv_wgrad_tc")
    torch.cuda.synchronize()
    assert torch.equal(dw.cpu().double(), want)


@pytest.mark.timeout(900)
def test_car_lite_loss_through_rpn_matches_oracle(product, oracle):
    """car.lite in train mode, one graph: middle encoder -> dense() -> RPN (cuDNN, TF32 off) -> loss = sum over the
    head maps of preds * G, one loss.backward().  Every middle and RPN gradient and the voxel feature gradient meet
    ||g - g64||_inf <= 2e-4 ||g64||_inf against the oracle network in float64 (tensor pipe; SiLU for ReLU, see _smooth:
    the RPN holds ~10^8 activations)."""
    cfg, onet, vf, coords = _middle_inputs("car.lite", 0, 20000, oracle)
    net = models.build_network(cfg, product)
    net.load_state_dict(onet.state_dict())
    parts64 = [_smooth(onet.middle_feature_extractor.double().train()), _smooth(onet.rpn.double().train())]
    parts = [_smooth(training.enable_sparse_backward(net.middle_feature_extractor.cuda()).train()),
             _smooth(net.rpn.cuda().train())]
    gen = torch.Generator().manual_seed(3)

    def run(mid, rpn, v, c, dev, dt):
        preds = rpn(mid(v, c, 1))
        keys = sorted(k for k, t in preds.items() if torch.is_tensor(t) and t.is_floating_point())
        return sum((preds[k] * gs[k].to(dev, dt)).sum() for k in keys), keys

    v64 = vf.double().requires_grad_()
    with torch.no_grad():
        shapes = {k: t.shape for k, t in parts64[1](parts64[0](vf.double(), coords, 1)).items() if torch.is_tensor(t)}
    gs = {k: torch.randn(shp, generator=gen, dtype=torch.float64) for k, shp in sorted(shapes.items())}
    loss64, keys = run(parts64[0], parts64[1], v64, coords, "cpu", torch.float64)
    assert keys
    loss64.backward()
    v = vf.cuda().requires_grad_()
    loss, _ = run(parts[0], parts[1], v, coords.cuda(), "cuda", torch.float32)
    loss.backward()
    torch.cuda.synchronize()
    errs = {"voxel features": _rel_err(v.grad, v64.grad)}
    for m, m64 in zip(parts, parts64):
        for (k, p), (_, p64) in zip(m.named_parameters(), m64.named_parameters()):
            errs[k] = _rel_err(p.grad, p64.grad)
    bad = {k: e for k, e in errs.items() if e > 2e-4}
    assert not bad, bad
