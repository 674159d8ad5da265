"""Train-mode BatchNorm + ReLU pairs (b2second.bn_train, csrc/bn_train.cu) on the CPU: the formulas of
tests/bn_train_ref.py equal torch autograd in float64; enable_bn_relu_training selects the pairs of every config on the
mirror and on the reference's own networks; enable_rpn_training selects the same convs on the reference's networks as
on the mirror; the C-ABI entry points reject bad arguments before any CUDA call; uncovered cases run the torch forward."""
import ctypes

import pytest
import torch
import torch.nn as nn

import bn_train_ref as R
from b2second import bn_train, config, loader, models, refcompat, rpn_train, training

CONFIGS = {   # name -> (BatchNorm1d pairs, BatchNorm2d pairs, channels)
    "car.fhd": (14, 7, [16, 32, 64, 128]),
    "car.lite": (4, 7, [16, 32, 64, 128]),
    "all.fhd": (14, 14, [16, 32, 64, 128]),
    "pointpillars.car.xyres_16": (0, 19, [64, 128, 256]),
    "nuscenes.all.pp.largea": (0, 19, [64, 128, 256]),
    "nuscenes.all.pp.mhead": (0, 22, [64, 128, 256]),
}
REF_CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"]


@pytest.mark.parametrize("shape,cl", [((37, 16), False), ((3, 8, 5, 7), False), ((3, 8, 5, 7), True), ((2, 12, 9), False),
                                      ((2, 4), False)])
def test_reference_equals_autograd(shape, cl):
    """y, the running buffers, dX, dgamma and dbeta of bn_train_ref within 1e-12 of torch autograd through BatchNorm +
    ReLU in float64; channel 1 is all negative after the BN shift (no gradient through the ReLU), channel 2 has
    |mean| / std = 1e4"""
    torch.manual_seed(0)
    C = shape[1]
    x = torch.randn(shape, dtype=torch.float64)
    x[:, 2] = x[:, 2] + 1e4
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    bn = (nn.BatchNorm2d if len(shape) == 4 else nn.BatchNorm1d)(C, eps=1e-3, momentum=0.01).double().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.2, 0.2)
        bn.bias[1] = -100.0
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
    g0, b0, rm0, rv0 = (t.detach().clone() for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
    y = torch.relu(bn(x))
    dy = torch.randn(shape, dtype=torch.float64)
    (y * dy).sum().backward()
    xr = R.rows(x)
    fw = R.forward(xr, g0, b0, rm0, rv0, 0.01, 1e-3)
    bw = R.backward(xr, R.rows(dy), fw["y"], g0, fw)

    # float64 itself resolves x - mean of the shifted channel only to 2^-53 |mean|: that term scales the tolerance too
    shifted = float((fw["mean"].abs() * (g0 * fw["s"]).abs()).max()) * (1.0 + float(dy.abs().max()))

    def close(got, want, what):
        scale = float(want.abs().max()) or 1.0
        assert float((got.detach().double() - want).abs().max()) <= 1e-12 * scale + 1e-15 * shifted, what
    close(R.rows(y), fw["y"], "y")
    close(bn.running_mean, fw["running_mean"], "running_mean")
    close(bn.running_var, fw["running_var"], "running_var")
    close(R.rows(x.grad), bw["dx"], "dx")
    close(bn.weight.grad, bw["dgamma"], "dgamma")
    close(bn.bias.grad, bw["dbeta"], "dbeta")
    assert bool((fw["y"][:, 1] == 0).all()) and float(bw["dbeta"][1]) == 0.0
    assert torch.equal(R.unrows(R.rows(x), x), x.detach())


def _counts(net):
    ps = bn_train.select(net)
    n1 = sum(isinstance(bn, nn.BatchNorm1d) for bn, _ in ps)
    n2 = sum(isinstance(bn, nn.BatchNorm2d) for bn, _ in ps)
    return n1, n2, sorted({bn.num_features for bn, _ in ps})


def _check_enable(net):
    keys = sorted(net.state_dict())
    classes = [type(m) for m in net.modules()]
    ps = bn_train.select(net)
    assert training.enable_bn_relu_training(net) is net
    assert training.enable_bn_relu_training(net) is net                 # idempotent
    for bn, relu in ps:
        assert bn.forward.__func__ is bn_train._bn_forward
        assert relu.forward.__func__ is bn_train._relu_forward and relu._b2s_bn is bn
    assert sorted(net.state_dict()) == keys
    assert [type(m) for m in net.modules()] == classes


@pytest.mark.parametrize("name", list(CONFIGS))
def test_selection_on_the_mirror(name):
    net = models.build_network(config.get_config(name), loader.oracle_spconv())
    assert _counts(net) == CONFIGS[name]
    assert pfn_bn_is_not_a_pair(net)
    _check_enable(net)


def pfn_bn_is_not_a_pair(net):
    vfe = net.voxel_feature_extractor
    layers = getattr(vfe, "pfn_layers", None)
    return layers is None or all(l.norm not in {bn for bn, _ in bn_train.pairs(net)} for l in layers)


def test_uncovered_pairs_stay_torch():
    seqs = [nn.Sequential(nn.BatchNorm2d(8, momentum=None), nn.ReLU()),
            nn.Sequential(nn.BatchNorm2d(8, affine=False), nn.ReLU()),
            nn.Sequential(nn.BatchNorm2d(8, track_running_stats=False), nn.ReLU()),
            nn.Sequential(nn.BatchNorm2d(8), nn.ReLU(inplace=True)),
            nn.Sequential(nn.BatchNorm2d(6), nn.ReLU()),
            nn.Sequential(nn.GroupNorm(2, 8), nn.ReLU()),
            nn.Sequential(nn.BatchNorm2d(8), nn.Identity(), nn.ReLU())]

    class OwnForward(nn.BatchNorm2d):
        def forward(self, x):
            return super().forward(x)
    seqs.append(nn.Sequential(OwnForward(8), nn.ReLU()))
    for s in seqs:
        assert bn_train.select(s) == []
        training.enable_bn_relu_training(s)
        assert all("forward" not in m.__dict__ for m in s)
    assert len(bn_train.pairs(seqs[0])) == 1 and bn_train.pairs(seqs[-1]) == []      # an own forward is not matched


def test_fallbacks_run_the_torch_forward():
    """eval(), no_grad and CPU input (and, by geometry(), fp16 or a C % 4 != 0 tensor) give the torch modules' results;
    M = 1 raises torch's own ValueError"""
    torch.manual_seed(1)
    seq = nn.Sequential(nn.BatchNorm2d(8, eps=1e-3, momentum=0.01), nn.ReLU())
    with torch.no_grad():
        seq[0].weight.uniform_(0.5, 1.5)
    ref = nn.Sequential(nn.BatchNorm2d(8, eps=1e-3, momentum=0.01), nn.ReLU())
    ref.load_state_dict(seq.state_dict())
    training.enable_bn_relu_training(seq)
    x = torch.randn(2, 8, 4, 5)
    for mode in ("train", "eval"):
        getattr(seq, mode)(), getattr(ref, mode)()
        assert torch.equal(seq(x), ref(x))
        with torch.no_grad():
            assert torch.equal(seq(x), ref(x))
    assert torch.equal(seq[0].running_mean, ref[0].running_mean)
    assert int(seq[0].num_batches_tracked) == int(ref[0].num_batches_tracked) == 2
    seq.train()
    with pytest.raises(ValueError):
        seq(torch.randn(1, 8, 1, 1))
    assert bn_train.geometry(torch.randn(2, 8, 3, 3).half()) is not None      # dtype is _active's test, not layout's
    assert not bn_train._active(seq[0], torch.randn(2, 8, 3, 3).half())
    assert bn_train.geometry(torch.randn(2, 6, 3, 3)) is None
    assert bn_train.geometry(torch.randn(1, 8, 1, 1)) is None
    assert bn_train.geometry(torch.randn(3, 8, 5, 7).transpose(2, 3)) is None
    assert bn_train.geometry(torch.randn(3, 8, 5, 7).contiguous(memory_format=torch.channels_last)) == (1, 3, 35)
    assert bn_train.geometry(torch.randn(3, 8, 5, 7)) == (0, 3, 35)
    assert bn_train.geometry(torch.randn(300, 16)) == (1, 300, 1)


def test_abi_rejects_bad_arguments_without_cuda():
    from spconv import _lib
    lib = _lib.load()
    assert lib.b2s_bn_relu_train_workspace_bytes(1, 281600, 128, 1) > lib.b2s_bn_relu_train_workspace_bytes(1, 8, 16, 1) > 0
    assert lib.b2s_bn_relu_train_workspace_bytes(0, 2, 64, 53568) > 0
    assert lib.b2s_bn_relu_train_workspace_bytes(2, 8, 16, 1) == 0
    assert lib.b2s_bn_relu_train_workspace_bytes(1, 8, 18, 1) == 0
    p = ctypes.c_void_p(256)                     # never dereferenced: every call below fails its argument check
    odd = ctypes.c_void_p(260)
    ws = lib.b2s_bn_relu_train_workspace_bytes(1, 100, 64, 1)

    def fwd(layout=1, B=100, C=64, S=1, x=p, y=p, mom=0.01, eps=1e-3, wsb=ws, nbt=p):
        return lib.b2s_bn_relu_train_forward(x, layout, B, C, S, p, p, p, p, nbt, mom, eps, y, p, wsb, None)

    def bwd(layout=1, B=100, C=64, S=1, x=p, dy=p, wsb=ws, dg=p):
        return lib.b2s_bn_relu_train_backward(x, dy, layout, B, C, S, p, p, wsb, p, dg, p, None)
    for call in (fwd, bwd):
        assert call(x=None) == -2 and b"NULL" in lib.b2s_last_error()
        assert call(layout=2) == -2 and b"layout" in lib.b2s_last_error()
        assert call(B=1) == -2 and b"M >= 2" in lib.b2s_last_error()
        assert call(B=0) == -2 and call(S=0) == -2
        assert call(C=18) == -2 and b"multiple of 4" in lib.b2s_last_error()
        assert call(C=0) == -2 and call(C=2048) == -2
        assert call(wsb=ws - 1) == -2 and b"workspace" in lib.b2s_last_error()
        assert call(x=odd) == -2 and b"16-byte" in lib.b2s_last_error()
    assert fwd(nbt=None) == -2 and b"NULL" in lib.b2s_last_error()
    assert bwd(dg=None) == -2 and b"NULL" in lib.b2s_last_error()
    assert fwd(y=odd) == -2 and bwd(dy=odd) == -2
    assert fwd(eps=0.0) == -2 and fwd(eps=-1.0) == -2
    assert fwd(mom=1.5) == -2 and fwd(mom=-0.1) == -2 and b"momentum" in lib.b2s_last_error()


def _ref_net(name):
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    return refcompat.build_network(refcompat.load_config(f).model.second)


def _names(net, mods):
    names = {id(m): n for n, m in net.named_modules()}
    return [names[id(m)] for m in mods]


def _layer_shapes(ps):
    return [(type(bn).__mro__[1].__name__ if type(bn).__name__ == "DefaultArgLayer" else type(bn).__name__,
             bn.num_features, bn.eps, bn.momentum) for bn, _ in ps]


# last in the module: ref_env puts the CPU oracle under the name ``spconv`` until the module ends
@pytest.mark.skipif(not refcompat.reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("name", REF_CONFIGS)
def test_reference_networks_match_the_mirror(ref_env, name):
    """enable_bn_relu_training selects the same pairs (class, channels, eps, momentum, in order) on the reference's own
    network as on the mirror, and enable_rpn_training's select the same convs, layer by layer"""
    net = _ref_net(name)
    mirror = models.build_network(config.get_config(name), loader.oracle_spconv())
    ps, mps = bn_train.select(net), bn_train.select(mirror)
    assert len(ps) == sum(CONFIGS[name][:2])
    assert _layer_shapes(ps) == _layer_shapes(mps)
    assert any(type(bn).__name__ == "DefaultArgLayer" for bn, _ in ps)             # change_default_args
    _check_enable(net)
    convs, mconvs = rpn_train.select(net.rpn), rpn_train.select(mirror.rpn)
    assert len(convs) == len(mconvs) == {"car.fhd": 6, "all.fhd": 11}.get(name, 13)

    def desc(sel):
        return [(c.in_channels, c.out_channels, tuple(c.padding), p is not None) for c, p in sel]
    assert desc(convs) == desc(mconvs)
    assert _names(net.rpn, [c for c, _ in convs]) == _names(mirror.rpn, [c for c, _ in mconvs])
