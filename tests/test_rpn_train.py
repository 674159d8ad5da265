"""enable_rpn_training on the host: which RPN layers it takes over in the mirror networks, the ZeroPad2d pairing, the
state dict, idempotence, the torch path off the GPU, and the host-side argument checks of the new C entry points."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn

from b2second import config, loader, models, rpn_train, training

# config -> (covered layers, of which ZeroPad2d(1) + padding-0 pairs, 3x3 layers of the RPN)
EXPECTED = {
    "car.fhd": (6, 1, 6),
    "car.lite": (6, 1, 6),
    "all.fhd": (11, 1, 12),                       # the 64 -> 128 stride-2 layer stays torch
    "pointpillars.car.xyres_16": (13, 0, 16),     # three stride-2 first layers stay torch
    "nuscenes.all.pp.largea": (13, 0, 16),
}


def _net(name):
    return models.build_network(config.get_config(name), loader.product_spconv())


def _convs3(rpn):
    return [m for m in rpn.modules() if type(m) is nn.Conv2d and tuple(m.kernel_size) == (3, 3)]


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_selection_in_the_mirror_networks(name):
    net = _net(name)
    sel = rpn_train.select(net.rpn)
    n, pairs, total = EXPECTED[name]
    assert len(sel) == n and sum(p is not None for _, p in sel) == pairs and len(_convs3(net.rpn)) == total
    chosen = {id(c) for c, _ in sel}
    for c in _convs3(net.rpn):
        covered = (c.stride == (1, 1) and c.in_channels % 64 == 0 and c.out_channels in (64, 128, 256)
                   and c.bias is None)
        assert (id(c) in chosen) == covered, c
    for c, pad in sel:
        assert (pad is None) == (c.padding == (1, 1))
        if pad is not None:
            assert type(pad) is nn.ZeroPad2d and tuple(pad.padding) == (1, 1, 1, 1)


def test_zeropad_pairing_needs_the_adjacent_pad():
    seq = nn.Sequential(nn.ZeroPad2d(1), nn.Conv2d(64, 64, 3, bias=False),      # paired
                        nn.ZeroPad2d(2), nn.Conv2d(64, 64, 3, bias=False),      # pad 2: not a pad-1 conv
                        nn.Conv2d(64, 64, 3, bias=False),                       # padding 0, no pad: not covered
                        nn.ZeroPad2d(1), nn.ReLU(), nn.Conv2d(64, 64, 3, bias=False),   # not adjacent
                        nn.Conv2d(64, 64, 3, padding=1, bias=True),             # bias: not covered
                        nn.Conv2d(64, 96, 3, padding=1, bias=False),            # Cout 96: not built
                        nn.Conv2d(96, 64, 3, padding=1, bias=False),            # Cin 96: not a multiple of 64
                        nn.Conv2d(64, 64, 3, padding=1, bias=False, dilation=1, groups=2))
    sel = rpn_train.select(seq)
    assert [(list(seq).index(c), list(seq).index(p) if p is not None else None) for c, p in sel] == [(1, 0)]


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16"])
def test_state_dict_classes_and_idempotence(name):
    net = _net(name)
    models.synthetic_weights_(net, name, seed=0)
    before = net.state_dict()
    classes = [type(m) for m in net.modules()]
    out = training.enable_rpn_training(net)
    assert out is net
    forwards = {id(m): m.__dict__.get("forward") for m in net.modules()}
    training.enable_rpn_training(net)
    assert {id(m): m.__dict__.get("forward") for m in net.modules()} == forwards      # nothing rebound twice
    after = net.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], before[k]) for k in before)
    assert [type(m) for m in net.modules()] == classes
    n = sum(1 for m in net.modules() if getattr(m, "_b2s_rpn_train", False))
    assert n == EXPECTED[name][0]


def test_never_raises_on_a_network_it_cannot_cover():
    seq = nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.BatchNorm2d(8), nn.ConvTranspose2d(8, 8, 2, stride=2))
    assert training.enable_rpn_training(seq) is seq
    assert not any(getattr(m, "_b2s_rpn_train", False) for m in seq.modules())


@pytest.mark.parametrize("train", [False, True])
def test_cpu_tensors_take_the_torch_path(train):
    """off the GPU (and in eval) the rebound modules compute exactly what nn.Conv2d / nn.ZeroPad2d compute"""
    torch.manual_seed(0)
    seq = nn.Sequential(nn.ZeroPad2d(1), nn.Conv2d(64, 64, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(),
                        nn.Conv2d(64, 128, 3, padding=1, bias=False))
    ref = copy.deepcopy(seq)
    rpn_train.enable(seq)
    seq = copy.deepcopy(seq)                                                         # still copyable
    seq.train(train)
    ref.train(train)
    x = torch.randn(2, 64, 9, 11)
    assert torch.equal(seq(x), ref(x))
    assert torch.equal(seq[0](x), ref[0](x))                                         # the pad alone still pads


def test_argument_checks_run_before_any_cuda_call():
    from spconv import _lib
    lib = _lib.load()
    d = ctypes.c_void_p(256)                  # never dereferenced: every call below fails its argument check

    def split(layout=0, B=2, C=64, H=8, W=8, hi=256, x=256, scale=d):
        return lib.b2s_split_halo_f16_autoscale(ctypes.c_void_p(x), layout, B, C, H, W, ctypes.c_void_p(hi),
                                                ctypes.c_void_p(hi), scale, None, None)
    assert split(layout=2) == -2 and b"layout" in lib.b2s_last_error()
    assert split(C=12) == -2 and b"multiple of 8" in lib.b2s_last_error()
    assert split(B=0) == -2 and split(H=0) == -2
    assert split(hi=264) == -2 and b"16-byte" in lib.b2s_last_error()
    assert split(layout=1, x=260) == -2
    assert split(scale=None) == -2
    assert split(B=64, C=256, H=512, W=512) == -2 and b"too large" in lib.b2s_last_error()

    def pack(cout=128, cin=128, transpose=0, hi=256):
        return lib.b2s_pack_conv2d_weights(d, cout, cin, transpose, ctypes.c_void_p(hi), ctypes.c_void_p(hi), d, None)
    assert pack(cin=96) == -2 and b"multiples of 64" in lib.b2s_last_error()
    assert pack(cout=32) == -2
    assert pack(transpose=2) == -2
    assert pack(hi=258) == -2

    assert lib.b2s_conv2d_wgrad_tc_workspace_bytes(2, 200, 176, 128, 128) == 4 * 9 * 128 * 128 * ((2 * 25 * 22 + 31) // 32)
    assert lib.b2s_conv2d_wgrad_tc_workspace_bytes(0, 200, 176, 128, 128) == 0
    ws = lib.b2s_conv2d_wgrad_tc_workspace_bytes(2, 16, 16, 128, 128)

    def wg(cin=128, cout=128, B=2, H=16, W=16, nbytes=ws, plane=256):
        p = ctypes.c_void_p(plane)
        return lib.b2s_conv2d_wgrad_tc(p, p, p, p, B, H, W, cin, cout, d, d, d, d, nbytes, None)
    assert wg(cout=192) == -2 and b"Cout 64, 128 or 256" in lib.b2s_last_error()
    assert wg(cin=96) == -2
    assert wg(H=0) == -2
    assert wg(plane=264) == -2 and b"16-byte" in lib.b2s_last_error()
    assert wg(nbytes=ws - 1) == -2 and b"workspace too small" in lib.b2s_last_error()
