"""PointPillars' pillar feature net in training (b2second.pfn_train, csrc/pfn_train.cu) on the CPU: the closed form the
kernels compute (tests/pfn_train_ref.py) equals torch autograd through the mirror's PillarFeatureNet /
PillarFeatureNetRadius in float64; enable_pfn_training selects the same modules on the mirror and on the reference's own
networks; the C-ABI entry points reject bad arguments before any CUDA call."""
import ctypes

import pytest
import torch

import pfn_train_ref as P
from b2second import config, loader, models, pfn_train, refcompat, training

GEOM = (0.16, 0.16, 0.08, -39.6)          # vx, vy, x_offset, y_offset of fp32_ref.pillars' KITTI grid
PP_CONFIGS = ["pointpillars.car.xyres_16", "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"]


def _torch_layer(radius, F, w, g, b, rm, rv):
    cls = models.PillarFeatureNetRadius if radius else models.PillarFeatureNet
    vfe = cls(num_input_features=F, num_filters=(64,), voxel_size=(GEOM[0], GEOM[1], 4),
              pc_range=(0.0, -39.68, -3, 69.12, 39.68, 1)).double().train()
    lyr = vfe.pfn_layers[0]
    with torch.no_grad():
        lyr.linear.weight.copy_(w.double())
        lyr.norm.weight.copy_(g.double())
        lyr.norm.bias.copy_(b.double())
        lyr.norm.running_mean.copy_(rm.double())
        lyr.norm.running_var.copy_(rv.double())
    return vfe


@pytest.mark.parametrize("radius", [False, True])
@pytest.mark.parametrize("F,T,n", [(4, 12, 40), (5, 7, 33), (3, 1, 9)])
def test_closed_form_equals_autograd(radius, F, T, n):
    """out, dW, dgamma, dbeta and the three buffers of the closed form within 1e-10 of autograd through the mirror;
    cases: the padded-slot maximum (channels 0..7), 1-point and full pillars, duplicate points, an all-negative channel"""
    vox, num, coors, w, g, b, rm, rv, dout = P.case(n, n, T, F, radius)
    vfe = _torch_layer(radius, F, w, g, b, rm, rv)
    assert abs(vfe.x_offset - GEOM[2]) < 1e-12 and abs(vfe.y_offset - GEOM[3]) < 1e-12
    out = vfe(vox.double(), num, coors).reshape(n, 64)
    (out * dout.double()).sum().backward()
    lyr = vfe.pfn_layers[0]
    d, _, live = P.decorate(vox, num, coors, *GEOM, radius)
    r = P.closed_form(d, live, w, g, b, rm, rv, 0.01, 1e-3, dout)
    assert bool((r["arg"] == T).any()) == (T > 1), "some maximum is the padded-slot value"
    assert bool((r["out"][:, 8] == 0).all()), "channel 8 is all negative"

    def close(got, want, what):
        scale = float(want.abs().max()) or 1.0
        assert float((got.detach() - want).abs().max()) <= 1e-10 * scale, what
    close(out, r["out"], "out")
    close(lyr.linear.weight.grad, r["dW"], "dW")
    close(lyr.norm.weight.grad, r["dgamma"], "dgamma")
    close(lyr.norm.bias.grad, r["dbeta"], "dbeta")
    close(lyr.norm.running_mean, r["running_mean"], "running_mean")
    close(lyr.norm.running_var, r["running_var"], "running_var")
    assert int(lyr.norm.num_batches_tracked) == 1


def test_faults_change_the_closed_form():
    vox, num, coors, w, g, b, rm, rv, dout = P.case(1, 60, 10, 4, False)
    d, _, live = P.decorate(vox, num, coors, *GEOM, False)
    ok = P.closed_form(d, live, w, g, b, rm, rv, 0.01, 1e-3, dout)
    for f in P.FAULTS:
        df = P.decorate(vox, num, coors, *GEOM, False, fault=f)[0]
        bad = P.closed_form(df, live, w, g, b, rm, rv, 0.01, 1e-3, dout, fault=f)
        moved = [k for k in ("out", "running_mean", "running_var", "dW") if not torch.allclose(bad[k], ok[k], rtol=1e-6)]
        assert moved, f


def _check_selection(net, covered):
    vfe, scatter = pfn_train.select(net)
    assert (vfe is not None) == covered
    assert scatter is net.middle_feature_extractor
    before = net.voxel_feature_extractor.__dict__.get("forward")
    assert training.enable_pfn_training(net) is net
    assert training.enable_pfn_training(net) is net                 # idempotent
    fwd = net.voxel_feature_extractor.__dict__.get("forward")
    if covered:
        assert fwd is not None and fwd.__func__ is pfn_train._vfe_forward
    else:
        assert fwd is before
    assert net.middle_feature_extractor.forward.__func__ is pfn_train._scatter_forward


@pytest.mark.parametrize("name", PP_CONFIGS)
def test_enable_selects_the_mirror_pfn(name):
    net = models.build_network(config.get_config(name), loader.oracle_spconv())
    keys = sorted(net.state_dict())
    _check_selection(net, True)
    assert sorted(net.state_dict()) == keys
    assert pfn_train.num_features(net.voxel_feature_extractor) == 4        # x, y, z, r (NuScenes: time lag for r)


def test_uncovered_vfes_stay_torch():
    sp = loader.oracle_spconv()
    for vfe in (models.PillarFeatureNet(4, num_filters=(64,), with_distance=True),
                models.PillarFeatureNet(4, num_filters=(32, 64)), models.SimpleVoxel(4), models.SimpleVoxelRadius(4)):
        assert pfn_train.num_features(vfe) is None
    net = models.build_network(config.get_config("car.fhd"), sp)
    assert pfn_train.select(net) == (None, None)
    training.enable_pfn_training(net)
    assert "forward" not in net.voxel_feature_extractor.__dict__
    assert "forward" not in net.middle_feature_extractor.__dict__


def test_eval_and_cpu_keep_the_torch_forward():
    net = models.build_network(config.get_config("pointpillars.car.xyres_16"), loader.oracle_spconv())
    vfe = net.voxel_feature_extractor
    vox, num, coors, *_ = P.case(3, 20, 100, 4, False, dup=False)
    net.eval()
    want = type(vfe).forward(vfe, vox.clone(), num, coors)
    training.enable_pfn_training(net)
    net.eval()
    assert torch.equal(vfe(vox.clone(), num, coors), want)
    net.train()
    with torch.no_grad():
        torch.manual_seed(0)
        got = vfe(vox.clone(), num, coors)                       # CPU input: the torch forward
    assert got.shape == (20, 64)


def test_abi_rejects_bad_arguments_without_cuda():
    from spconv import _lib
    lib = _lib.load()
    assert lib.b2s_pfn_train_workspace_bytes(24000) > lib.b2s_pfn_train_workspace_bytes(8) > 0
    assert lib.b2s_pfn_train_workspace_bytes(0) == 0
    p = ctypes.c_void_p(256)                    # never dereferenced: every call below fails its argument check
    ws = lib.b2s_pfn_train_workspace_bytes(100)

    def fwd(N=100, T=32, F=4, cout=64, deco=0, wsb=ws, mom=0.01, eps=1e-3, vox=p):
        return lib.b2s_pfn_train_forward(vox, N, T, F, p, p, p, p, p, cout, p, p, p, mom, eps, 0.16, 0.16, 0.08, -39.6,
                                         deco, p, p, p, wsb, None, None)

    def bwd(N=100, T=32, F=4, cout=64, deco=0, wsb=ws):
        return lib.b2s_pfn_train_backward(p, N, T, F, p, p, p, p, cout, 0.16, 0.16, 0.08, -39.6, deco, p, p, p, p, wsb,
                                          p, p, p, None)
    for call in (fwd, bwd):
        assert call(T=255) == -2 and b"max_points <= 254" in lib.b2s_last_error()
        assert call(T=0) == -2
        assert call(N=0) == -2
        assert call(N=1, T=1) == -2 and b"more than one value" in lib.b2s_last_error()
        assert call(F=9) == -2 and call(F=2) == -2
        assert call(cout=32) == -2 and b"Cout=64" in lib.b2s_last_error()
        assert call(deco=2) == -2
        assert call(wsb=ws - 1) == -2 and b"workspace" in lib.b2s_last_error()
    assert fwd(vox=None) == -2 and b"NULL" in lib.b2s_last_error()
    assert fwd(eps=0.0) == -2 and fwd(mom=1.5) == -2


# last in the module: ref_env puts the CPU oracle under the name ``spconv`` until the module ends
@pytest.mark.skipif(not refcompat.reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("name", PP_CONFIGS)
def test_enable_selects_the_reference_pfn(ref_env, name):
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    net = refcompat.build_network(refcompat.load_config(f).model.second)
    _check_selection(net, True)
    assert type(net.voxel_feature_extractor.pfn_layers[0].norm) is not torch.nn.BatchNorm1d    # change_default_args
    from second.pytorch.models import pointpillars as pp
    for cls in (pp.PillarFeatureNetOld, pp.PillarFeatureNetRadiusHeight):
        assert pfn_train.num_features(cls(4, num_filters=(64,))) is None

