"""Sparse convolution backward, host side (no GPU needed): the argument checks of the new entry points run before any
CUDA call, and the gradient reference -- the CPU oracle's autograd -- equals F.conv3d's on the dense grid in float64."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F


def test_backward_argument_checks_run_before_any_cuda_call():
    from spconv import _lib
    lib = _lib.load()
    dummy = ctypes.c_void_p(256)                      # never dereferenced: every call below fails its argument check
    # weight gradient: sizes, workspace query and size check
    assert lib.b2s_sparse_conv_wgrad_workspace_bytes(4096, 27, 64, 64) == 4 * 2 * 27 * 64 * 64   # two 2048-row slabs
    assert lib.b2s_sparse_conv_wgrad_workspace_bytes(4097, 27, 16, 32) == 4 * 3 * 27 * 16 * 32
    assert lib.b2s_sparse_conv_wgrad_workspace_bytes(0, 27, 16, 32) == 0

    def wgrad(cin=64, cout=64, K=27, cap_out=1000, ws=None):
        ws = lib.b2s_sparse_conv_wgrad_workspace_bytes(cap_out, K, cin, cout) if ws is None else ws
        return lib.b2s_sparse_conv_wgrad(dummy, cin, dummy, cout, dummy, K, dummy, cap_out, None, dummy, dummy, ws, None)
    assert wgrad(cin=0) == -2 and b"bad sizes" in lib.b2s_last_error()
    assert wgrad(cout=0) == -2 and wgrad(K=0) == -2 and wgrad(cap_out=-1) == -2
    assert wgrad(ws=1000) == -2 and b"workspace too small" in lib.b2s_last_error()
    # tensor-pipe weight gradient: channel table, K range, alignment, workspace
    assert lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(4096, 27, 16, 32) == 4 * 2 * 7 * 64 * 32   # 7 K blocks of 4

    def wtc(cin=64, cout=64, K=27, in_stride=128, feat=256, ws=None):
        ws = lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(1000, K, cin, cout) if ws is None else ws
        return lib.b2s_sparse_conv_wgrad_tc(ctypes.c_void_p(feat), ctypes.c_void_p(feat + 128), in_stride, 1000, cin,
                                            dummy, ctypes.c_void_p(256 + 128), 128, cout, dummy, K, dummy, 1000, None,
                                            None, None, dummy, dummy, ws, None)
    assert wtc(cin=48) == -2 and b"built for Cin" in lib.b2s_last_error()
    assert wtc(cout=8) == -2
    assert wtc(K=28) == -2 and b"K must be 1..27" in lib.b2s_last_error()
    assert wtc(in_stride=60) == -2 and b"16-byte aligned" in lib.b2s_last_error()
    assert wtc(feat=264) == -2
    assert wtc(ws=100) == -2 and b"workspace too small" in lib.b2s_last_error()
    # rulebook transpose
    assert lib.b2s_rulebook_transpose(dummy, dummy, 100, 0, dummy, 100, None, None) == -2
    assert lib.b2s_rulebook_transpose(dummy, dummy, -1, 27, dummy, 100, None, None) == -2
    # dense() backward
    assert lib.b2s_from_bev(dummy, dummy, dummy, 10, 16, 1, 2, 8, 8, 2, dummy, None) == -2
    assert b"bad layout" in lib.b2s_last_error()
    assert lib.b2s_from_bev(dummy, dummy, dummy, 10, 0, 1, 2, 8, 8, 0, dummy, None) == -2
    # auto-scaled split: widths, alignment, the scale word
    sc = ctypes.c_void_p(4096)
    assert lib.b2s_split_f16_autoscale(dummy, dummy, ctypes.c_void_p(288), None, 10, 16, 12, 32, sc, None) == -2
    assert lib.b2s_split_f16_autoscale(dummy, dummy, ctypes.c_void_p(290), None, 10, 16, 16, 32, sc, None) == -2
    assert b"16-byte aligned" in lib.b2s_last_error()
    assert lib.b2s_split_f16_autoscale(dummy, dummy, ctypes.c_void_p(288), None, 10, 16, 16, 32, None, None) == -2
    assert b"scale_dev" in lib.b2s_last_error()


def _random_sparse(rng, shape, batch, n, cin):
    D, H, W = shape
    flat = rng.choice(batch * D * H * W, size=n, replace=False)
    b, r = np.divmod(flat, D * H * W)
    z, r = np.divmod(r, H * W)
    y, x = np.divmod(r, W)
    idx = np.stack([b, z, y, x], 1).astype(np.int32)
    return torch.from_numpy(rng.standard_normal((n, cin))), torch.from_numpy(idx)


@pytest.mark.parametrize("layer", [
    dict(subm=True, k=3, s=1, p=1),
    dict(subm=False, k=3, s=2, p=1),
    dict(subm=False, k=3, s=2, p=[0, 1, 1]),
    dict(subm=False, k=(3, 1, 1), s=(2, 1, 1), p=0),
])
def test_oracle_gradients_equal_dense_conv3d(oracle, layer):
    """d/dX and d/dW of sum(out * G) through the oracle's sparse conv equal those of F.conv3d on the dense grid with G
    scattered at the active outputs (float64): the oracle is a sound reference for the CUDA backward."""
    rng = np.random.default_rng(7)
    shape, batch, cin, cout = (7, 9, 8), 2, 3, 5
    feats, idx = _random_sparse(rng, shape, batch, 120, cin)
    torch.manual_seed(0)
    if layer["subm"]:
        conv = oracle.SubMConv3d(cin, cout, layer["k"], bias=False, indice_key="s")
    else:
        conv = oracle.SparseConv3d(cin, cout, layer["k"], layer["s"], padding=layer["p"], bias=False)
    conv = conv.double()
    x = feats.clone().requires_grad_()
    y = conv(oracle.SparseConvTensor(x, idx, shape, batch))
    g = torch.from_numpy(rng.standard_normal(tuple(y.features.shape)))
    (y.features * g).sum().backward()
    # dense restatement
    w = conv.weight.detach().clone().requires_grad_()                      # [kD, kH, kW, Cin, Cout]
    il = idx.long()
    xs = torch.zeros(batch, cin, *shape, dtype=torch.float64)
    xs[il[:, 0], :, il[:, 1], il[:, 2], il[:, 3]] = feats
    xs.requires_grad_()
    pad = [conv.kernel_size[i] // 2 for i in range(3)] if layer["subm"] else conv.padding
    stride = [1, 1, 1] if layer["subm"] else conv.stride
    yd = F.conv3d(xs, w.permute(4, 3, 0, 1, 2), stride=stride, padding=pad)
    gd = torch.zeros_like(yd)
    ol = y.indices.long()
    gd[ol[:, 0], :, ol[:, 1], ol[:, 2], ol[:, 3]] = g
    # the forward agrees at the active outputs, and the loss is the same
    assert torch.allclose(yd[ol[:, 0], :, ol[:, 1], ol[:, 2], ol[:, 3]], y.features, rtol=1e-12, atol=1e-12)
    (yd * gd).sum().backward()
    dx_dense = xs.grad[il[:, 0], :, il[:, 1], il[:, 2], il[:, 3]]
    assert torch.allclose(x.grad, dx_dense, rtol=1e-12, atol=1e-12)
    assert torch.allclose(conv.weight.grad, w.grad, rtol=1e-12, atol=1e-12)
