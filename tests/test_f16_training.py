"""The f16 training mode's host side (no GPU needed): the precision keyword of training.enable_sparse_backward and
enable_rpn_training and its refusals, the layers each mode puts on the tensor pipe (the same in both), the weight-plane
caches keyed on the product count, and the argument checks of the products-taking entry points, which run before any
CUDA call."""
import ctypes

import pytest
import torch
import torch.nn as nn

CONFIGS = ["car.fhd", "car.lite", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea"]


def _net(product, name):
    from b2second import config, models
    net = models.build_network(config.get_config(name), product)
    models.synthetic_weights_(net, name, seed=0)
    return net


def _sparse_convs(product, net):
    return [m for m in net.modules() if isinstance(m, product.SparseConvolution)]


def test_keyword_and_refusals(product, monkeypatch):
    from b2second import rpn_train, training
    net = _net(product, "car.fhd")
    convs = _sparse_convs(product, net)
    for bad in ("fp16", "bf16", None, 1):
        with pytest.raises(ValueError, match="precision"):
            training.enable_sparse_backward(net, precision=bad)
        with pytest.raises(ValueError, match="precision"):
            training.enable_rpn_training(net, precision=bad)
    assert not any(m._b2s_backward for m in convs)            # a refused call marks nothing
    training.enable_sparse_backward(net)
    assert all(m._b2s_backward and m._b2s_products == 3 for m in convs)
    training.enable_sparse_backward(net, precision="f16")
    assert all(m._b2s_products == 1 for m in convs)
    training.enable_sparse_backward(net, precision="fp32")     # a second call switches back
    assert all(m._b2s_products == 3 for m in convs)
    rpn = [c for c, _ in rpn_train.select(net.rpn)]
    training.enable_rpn_training(net, precision="f16")
    assert rpn and all(c._b2s_rpn_train and c._b2s_products == 1 for c in rpn)
    training.enable_rpn_training(net)
    assert all(c._b2s_products == 3 for c in rpn)
    # f16 runs on the tensor pipe only: the FMA kernels (B2S_SPCONV_TC=0) are the fp32 reference path
    monkeypatch.setattr(product, "USE_TENSOR_CORES", False)
    with pytest.raises(ValueError, match="fp32 reference"):
        training.enable_sparse_backward(net, precision="f16")
    assert all(m._b2s_products == 3 for m in convs)
    training.enable_sparse_backward(net, precision="fp32")


@pytest.mark.parametrize("name", CONFIGS)
def test_coverage_is_the_same_in_both_modes(product, name):
    """rpn_train.select and the sparse convs' tensor-pipe widths (forward / wgrad, and dgrad) do not depend on the
    precision: the f16 mode changes how covered layers compute, not which layers are covered"""
    from b2second import rpn_train, tc, training
    lib = product._lib.load()
    seen = {}
    for precision in ("fp32", "f16"):
        net = _net(product, name)
        training.enable_rpn_training(training.enable_sparse_backward(net, precision=precision), precision=precision)
        rpn = getattr(net, "rpn", net)
        marked = [n for n, m in rpn.named_modules() if getattr(m, "_b2s_rpn_train", False)]
        assert marked == [n for n, m in rpn.named_modules() if any(m is c for c, _ in rpn_train.select(rpn))]
        sparse = []
        for n, m in net.named_modules():
            if isinstance(m, product.SparseConvolution):
                K = int(torch.tensor(m.kernel_size).prod())
                sparse.append((n, m._wgrad_tc_cin(lib, K), tc.sparse_tc_channels(lib, m.out_channels, m.in_channels, K)))
        seen[precision] = (marked, sparse)
    assert seen["fp32"] == seen["f16"]


def test_sparse_weight_caches_are_keyed_on_products(product, monkeypatch):
    """_tc_weights and _dgrad_weights repack when the product count changes, and only then (or when the weight does)"""
    calls = []

    def fake_pack(w, transpose=False, flip=False, products=3):
        calls.append((transpose, flip, products))
        hi = torch.zeros(1)
        return hi, (None if products == 1 else torch.zeros(1)), torch.ones(1), torch.ones(1)

    monkeypatch.setattr(product, "_pack_tc_weights", fake_pack)
    conv = product.SubMConv3d(16, 16, 3, bias=False)
    for p in (3, 3, 1, 1, 3):
        conv._tc_weights(16, p)
    assert calls == [(False, False, 3), (False, False, 1), (False, False, 3)]
    with torch.no_grad():
        conv.weight.add_(1.0)                      # a new weight version: repacked in the same mode
    conv._tc_weights(16, 3)
    assert len(calls) == 4 and conv._b2s_tc_w[0][-1] == 3
    calls.clear()
    for p in (1, 1, 3):
        conv._dgrad_weights(conv.weight, True, p)
    assert calls == [(True, True, 1), (True, True, 3)]
    assert conv._tc_weights(16, 1)[1] is None and conv._dgrad_weights(conv.weight, True, 1)[1] is None


def test_rpn_weight_cache_is_keyed_on_products(monkeypatch):
    """rpn_train.pack_weights: one b2s_pack_conv2d_weights(_ex) call per (weight version, transpose, product count)"""
    from b2second import rpn_train
    calls = []

    class FakeLib:
        def b2s_pack_conv2d_weights(self, *a):
            calls.append(3)
            return 0

        def b2s_pack_conv2d_weights_ex(self, *a):
            assert a[5] is None and a[7] == 1            # no lo plane, products = 1
            calls.append(1)
            return 0

    class FakeL:
        check = staticmethod(lambda rc, what: rc)
        ptr = staticmethod(lambda t: None if t is None else ctypes.c_void_p(t.data_ptr()))
        stream = staticmethod(lambda: None)

    monkeypatch.setattr(rpn_train, "_lib", lambda: (FakeL, FakeLib()))
    conv = nn.Conv2d(64, 64, 3, padding=1, bias=False)
    for p in (3, 3, 1, 1, 3):
        hi, lo, _ = rpn_train.pack_weights(conv, False, p)
        assert (lo is None) == (p == 1)
    assert calls == [3, 1, 3]
    rpn_train.pack_weights(conv, True, 3)
    rpn_train.pack_weights(conv, False, 3)         # the transposed planes are cached separately
    assert calls == [3, 1, 3, 3]


def test_argument_checks_run_before_any_cuda_call():
    from spconv import _lib
    lib = _lib.load()
    d = ctypes.c_void_p(256)                  # never dereferenced: every call below fails its argument check
    err = lib.b2s_last_error

    # sparse weight gradient
    ws = lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(5000, 27, 64, 64)

    def swg(products=1, x_lo=None, g_lo=None, cin=64, cout=64, K=27, plane=256, nbytes=ws):
        p = ctypes.c_void_p(plane)
        return lib.b2s_sparse_conv_wgrad_tc_ex(p, x_lo, 64, 100, cin, p, g_lo, 64, cout, d, K, d, 5000, None, None, d,
                                               d, d, nbytes, products, None)
    assert swg(products=2) == -2 and b"products" in err()
    assert swg(x_lo=d) == -2 and b"products" in err()
    assert swg(g_lo=d) == -2
    assert swg(cin=48) == -2 and b"built for" in err()
    assert swg(K=28) == -2 and b"K must be" in err()
    assert swg(plane=258) == -2 and b"16-byte" in err()
    assert swg(nbytes=ws - 1) == -2 and b"workspace too small" in err()

    # dense weight gradient
    ws2 = lib.b2s_conv2d_wgrad_tc_workspace_bytes(2, 16, 16, 128, 128)

    def dwg(products=1, x_lo=None, g_lo=None, cin=128, cout=128, plane=256, nbytes=ws2):
        p = ctypes.c_void_p(plane)
        return lib.b2s_conv2d_wgrad_tc_ex(p, x_lo, p, g_lo, 2, 16, 16, cin, cout, d, d, d, d, nbytes, products, None)
    assert dwg(products=0) == -2 and b"products" in err()
    assert dwg(x_lo=d) == -2 and dwg(g_lo=d) == -2
    assert dwg(cout=192) == -2 and b"Cout 64, 128 or 256" in err()
    assert dwg(plane=264) == -2 and b"16-byte" in err()
    assert dwg(nbytes=ws2 - 1) == -2 and b"workspace too small" in err()

    # splits
    def split(products=1, lo=None, C=64, scale=d, hi=256):
        return lib.b2s_split_f16_autoscale_ex(d, ctypes.c_void_p(hi), lo, None, 10, C, C, C, scale, products, None)
    assert split(lo=d) == -2 and b"products" in err()
    assert split(products=2) == -2
    assert split(C=12) == -2 and b"multiples of 8" in err()
    assert split(hi=264) == -2 and b"16-byte" in err()
    assert split(scale=None) == -2 and b"scale_dev" in err()

    def halo(products=1, lo=None, layout=0, C=64, hi=256):
        return lib.b2s_split_halo_f16_autoscale_ex(d, layout, 2, C, 8, 8, ctypes.c_void_p(hi), lo, d, None, products,
                                                   None)
    assert halo(lo=d) == -2 and b"products" in err()
    assert halo(layout=2) == -2 and b"layout" in err()
    assert halo(C=12) == -2 and b"multiple of 8" in err()
    assert halo(hi=264) == -2 and b"16-byte" in err()

    # weight packs
    def psw(products=1, lo=None, cin=16, transpose=0, hi=256):
        return lib.b2s_pack_sparse_weights_ex(d, 27, cin, 16, transpose, 0, ctypes.c_void_p(hi), lo, d, products, None)
    assert psw(lo=d) == -2 and b"products" in err()
    assert psw(cin=48) == -2 and b"packed input channels" in err()
    assert psw(transpose=2) == -2
    assert psw(hi=264) == -2 and b"16-byte" in err()

    def pcw(products=1, lo=None, cin=128, transpose=0, hi=256):
        return lib.b2s_pack_conv2d_weights_ex(d, 128, cin, transpose, ctypes.c_void_p(hi), lo, d, products, None)
    assert pcw(lo=d) == -2 and b"products" in err()
    assert pcw(cin=96) == -2 and b"multiples of 64" in err()
    assert pcw(transpose=2) == -2
    assert pcw(hi=258) == -2

    # the sparse forward's fp32 output
    def fwd(products=1, out_fp32=1, lo=None, cin=64):
        return lib.b2s_sparse_conv_tc_plan_ex2(d, lo, 64, 100, cin, d, lo, d, 27, d, 100, None, None, None, None, 0, d,
                                               lo, 64, 64, products, out_fp32, None, None)
    assert fwd(products=3, out_fp32=1, lo=d) == -2 and b"out_fp32" in err()
    assert fwd(out_fp32=2) == -2 and b"out_fp32" in err()
    assert fwd(lo=d) == -2 and b"products" in err()
    assert fwd(cin=48) == -2 and b"built for" in err()
