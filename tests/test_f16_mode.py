"""The half-precision mode of the fused engine (precision="f16") on the CPU: the keyword and its refusals, the host
packing of single weight planes, and the host-side argument checks of the products-taking entry points."""
import ctypes

import pytest
import torch

from b2second import config, engine, fastpath, models, tc


def _net(oracle, name="car.fhd"):
    net = models.build_network(config.get_config(name), oracle).eval()
    models.synthetic_weights_(net, name, seed=0)
    return net


@pytest.mark.parametrize("precision,products", [("fp32", 3), ("f16", 1)])
def test_precision_selects_the_product_count(precision, products):
    assert engine.check_precision(precision) == products
    assert engine.check_precision(precision, "tc", "tc") == products


@pytest.mark.parametrize("precision", ["fp16", "half", "bf16", "F16", None, 16])
def test_unknown_precision_is_refused(oracle, precision):
    with pytest.raises(ValueError, match="precision"):
        engine.check_precision(precision)
    net = _net(oracle)
    with pytest.raises(ValueError, match="precision"):
        fastpath.accelerate(net, precision=precision)
    assert getattr(net, "b2s_fastpath", None) is None


@pytest.mark.parametrize("kw", [{"sparse_impl": "fma"}, {"rpn_impl": "cudnn"},
                                {"sparse_impl": "fma", "rpn_impl": "cudnn"}])
def test_f16_with_an_fp32_reference_path_is_refused(oracle, kw):
    with pytest.raises(ValueError, match="fp32 reference"):
        engine.check_precision("f16", kw.get("sparse_impl", "tc"), kw.get("rpn_impl", "auto"))
    with pytest.raises(ValueError, match="fp32 reference"):
        fastpath.accelerate(_net(oracle), precision="f16", **kw)
    # the same paths stay available in the default mode
    assert engine.check_precision("fp32", kw.get("sparse_impl", "tc"), kw.get("rpn_impl", "auto")) == 3


def test_accelerate_forwards_the_keyword(oracle):
    net = fastpath.accelerate(_net(oracle), precision="f16")
    assert net.b2s_fastpath.engine_kw == {"precision": "f16"}
    assert fastpath.accelerate(_net(oracle)).b2s_fastpath.engine_kw == {}


def test_single_weight_planes_are_the_hi_planes(oracle):
    """weight_planes(products = 1) is, bit for bit, the hi plane of the 3xF16 split, and carries no lo plane"""
    g = torch.Generator().manual_seed(3)
    w = torch.randn(27, 64, 64, generator=g) * torch.logspace(-12, 2, 64)
    wp = tc.pack_sparse_weights(w)
    ws = tc.pow2_scale(wp)
    hi3, lo3 = tc.weight_planes(wp, ws, 3)
    hi1, lo1 = tc.weight_planes(wp, ws, 1)
    assert lo1 is None and lo3 is not None
    assert torch.equal(hi1.view(torch.int16), hi3.view(torch.int16))
    assert torch.equal(hi3.view(torch.int16), tc.split_f16(wp, ws)[0].view(torch.int16))


@pytest.mark.parametrize("name", ["car.fhd", "car.lite", "all.fhd", "pointpillars.car.xyres_16",
                                  "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"])
def test_rpn_plan_single_planes(oracle, name):
    """plan_rpn* in the f16 mode: the same layout, every op's w_hi the 3xF16 plan's w_hi bit for bit, no w_lo, the same
    epilogue scale and shift"""
    from b2second import spec
    net = _net(oracle, name)
    s = spec.spec_from_module(net)
    H, W = 40, 48

    def plan(products):
        if getattr(s, "heads", None) is None:
            return tc.plan_rpn(s.rpn, H, W, products=products)
        return tc.plan_rpn_multihead(s.rpn, dict(s.heads), H, W, products=products)
    p3, p1 = plan(3), plan(1)
    assert tc.plan_layout(p3) == tc.plan_layout(p1)
    n = 0
    for a, b in zip(p3["ops"], p1["ops"]):
        if "w_hi" not in a:
            continue
        n += 1
        assert b["w_lo"] is None and a["w_lo"] is not None
        assert torch.equal(a["w_hi"].view(torch.int16), b["w_hi"].view(torch.int16))
        assert torch.equal(a["scale"], b["scale"]) and a["w_scale"] == b["w_scale"]
        assert (a["shift"] is None and b["shift"] is None) or torch.equal(a["shift"], b["shift"])
    assert n >= 3


def test_products_argument_checks_run_before_any_cuda_call():
    """the products-taking entry points reject a product count other than 3 or 1, and a lo plane in the f16 mode, with
    -2 before any CUDA call"""
    from spconv import _lib
    lib = _lib.load()
    d = ctypes.c_void_p(256)
    lo = ctypes.c_void_p(512)

    def conv(products, in_lo=None, out_lo=None, out_fp32=0):
        return lib.b2s_conv2d_tc_ex3(d, in_lo, 1, 8, 8, 64, d, None, 3, 3, 1, 1, 128, 128, None, None, 0, 8, 8, d, out_lo,
                                     8, 8, 1, 128, 1, 0, 0, None, None, None, None, None, None, -1, 8, products,
                                     out_fp32, None, None)
    for p in (0, 2, 4):
        assert conv(p) == -2 and b"products" in lib.b2s_last_error()
    assert conv(1, in_lo=lo) == -2 and conv(1, out_lo=lo) == -2 and conv(1, out_fp32=2) == -2
    assert conv(3, in_lo=lo, out_lo=lo, out_fp32=1) == -2

    def sparse(products, feat_lo=None, w_lo=None, out_lo=None):
        return lib.b2s_sparse_conv_tc_plan_ex(d, feat_lo, 128, 1000, 64, d, w_lo, d, 27, d, 1000, None, None, None, None,
                                              1, d, out_lo, 64, 64, products, None, None)
    assert sparse(2) == -2 and sparse(1, feat_lo=lo) == -2 and sparse(1, w_lo=lo) == -2 and sparse(1, out_lo=lo) == -2
    assert lib.b2s_rpn_tail_tc_ex2(d, lo, 1, 8, 8, 128, d, None, 128, None, None, d, None, 32, 32, None, None, d, 32,
                                   None, None, None, None, None, -1, 1, None, None) == -2
    assert lib.b2s_rpn_tail_tc_ex2(d, None, 1, 8, 8, 128, d, None, 128, None, None, d, None, 32, 32, None, None, d, 32,
                                   None, None, None, None, None, -1, 2, None, None) == -2
    assert lib.b2s_to_bev_tc_ex2(None, d, lo, 64, d, d, 10, 64, 1, 1, 8, 8, d, None, d, 1, None) == -2
    assert lib.b2s_to_bev_tc_ex2(None, d, None, 64, d, d, 10, 64, 1, 1, 8, 8, d, lo, d, 1, None) == -2
    assert lib.b2s_crop_nhwc_ex(d, lo, 1, 8, 8, 64, 1, d, None, 1, None) == -2
    assert lib.b2s_crop_nhwc_ex(d, None, 1, 8, 8, 64, 1, d, None, 0, None) == -2
    assert lib.b2s_split_f16_ex(d, d, lo, None, 10, 8, 8, 8, 1, None) == -2
    assert lib.b2s_split_f16_ex(d, d, None, None, 10, 8, 8, 8, 2, None) == -2


def test_graph_capture_runs_without_the_cyclic_collector():
    """engine.no_cyclic_gc, which InferenceEngine.run captures its CUDA graphs in: the collector is off in the block and
    restored after it, also when the block raises, and left off when it was off before"""
    import gc
    assert gc.isenabled()
    with engine.no_cyclic_gc():
        assert not gc.isenabled()
    assert gc.isenabled()
    with pytest.raises(RuntimeError):
        with engine.no_cyclic_gc():
            raise RuntimeError("capture failed")
    assert gc.isenabled()
    gc.disable()
    try:
        with engine.no_cyclic_gc():
            assert not gc.isenabled()
        assert not gc.isenabled()
    finally:
        gc.enable()
