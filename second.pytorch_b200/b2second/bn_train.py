"""Training of BatchNorm + ReLU pairs on the GPU (csrc/bn_train.cu).

``training.enable_bn_relu_training(net)`` rebinds every covered (BatchNorm1d or BatchNorm2d, ReLU) pair of consecutive
children of a sequential container under ``net`` (``nn.Sequential``, torchplus' ``Sequential`` and the ``spconv``
``SparseSequential``, which run their children in ``_modules`` order; see ``rpn_train.sequences``).  Modules match by
``isinstance`` when their class does not override ``forward``, so the reference's ``change_default_args`` BatchNorm
subclasses are covered as well as the mirror's.  Covered: BatchNorm with ``affine``, ``track_running_stats`` and a
numeric ``momentum``, followed by a ReLU that is not in place.  Anything else (GroupNorm, the PFN's BatchNorm1d, whose
ReLU is functional) stays torch.

The BatchNorm's forward becomes ``BNReLUTrain``, which returns relu(BN(x)) in x's memory format; the ReLU's forward
passes its input through unchanged when that input is the tensor its BatchNorm just returned from ``BNReLUTrain``
(ReLU of that tensor is that tensor) and is ``nn.ReLU.forward`` otherwise.  The kernels run only in ``train()`` mode
with grad enabled, on float32 CUDA input with C % 4 == 0 in one of two layouts: rows [M, C] (a BatchNorm1d input, or a
channels_last map) or NCHW contiguous; otherwise, and for M < 2 (where torch raises its ValueError), the BatchNorm runs
its torch forward.  ``eval()``, the fused engine, the drop-in's eval-mode folding and the state dict do not change.

BNReLUTrain, on the caller's stream without a host sync:
  forward   b2s_bn_relu_train_forward: batch statistics in float64, the running buffers and num_batches_tracked updated
            in place, y = relu(BN(x)); saves x and the workspace (the per-channel statistics), nothing else;
  backward  b2s_bn_relu_train_backward: the ReLU mask recomputed from x, dgamma, dbeta and dX.
"""
import types
import weakref

import torch
import torch.nn as nn
from torch.autograd.graph import increment_version

from . import loader, rpn_train

LAYOUT_NCHW, LAYOUT_ROWS = 0, 1      # B2S_LAYOUT_NCHW, B2S_LAYOUT_NHWC
MAX_CHANNELS = 1024


def _lib():
    sp = loader.product_spconv()
    return sp._lib, sp._lib.load()


def is_bn(m):
    return any(rpn_train.plain(m, cls) for cls in (nn.BatchNorm1d, nn.BatchNorm2d))


def is_relu(m):
    return rpn_train.plain(m, nn.ReLU)


def covered(bn, relu):
    return (bn.affine and bn.track_running_stats and bn.momentum is not None and not relu.inplace
            and bn.num_features % 4 == 0 and bn.num_features <= MAX_CHANNELS)


def pairs(net):
    """-> [(bn, relu)] of every (BatchNorm1d / BatchNorm2d, ReLU) pair of consecutive children of a sequential
    container under ``net``, covered or not, in module order."""
    out = []
    for mods in rpn_train.sequences(net):
        out += [(a, b) for a, b in zip(mods, mods[1:]) if is_bn(a) and is_relu(b)]
    return out


def select(net):
    """-> [(bn, relu)] of the covered pairs under ``net``, in module order."""
    return [(bn, relu) for bn, relu in pairs(net) if covered(bn, relu)]


def geometry(x):
    """(layout, batch, spatial) of a tensor the kernels take, or None: rows [M, C] -> (ROWS, M, 1), a channels_last
    [B, C, H, W] -> (ROWS, B, H * W), a contiguous [B, C, L...] -> (NCHW, B, L...)."""
    if x.dim() < 2 or x.dim() > 4:
        return None
    B, C = int(x.shape[0]), int(x.shape[1])
    spatial = 1
    for v in x.shape[2:]:
        spatial *= int(v)
    if x.dim() == 2:
        layout = LAYOUT_ROWS if x.is_contiguous() else None
    elif x.is_contiguous():
        layout = LAYOUT_NCHW
    elif x.dim() == 4 and x.is_contiguous(memory_format=torch.channels_last):
        layout = LAYOUT_ROWS
    else:
        layout = None
    if layout is None or (layout == LAYOUT_ROWS and x.data_ptr() % 16):
        return None
    if C % 4 or C > MAX_CHANNELS or B * spatial < 2:
        return None
    return layout, B, spatial


def _active(bn, x):
    return bn.training and torch.is_grad_enabled() and x.is_cuda and x.dtype == torch.float32


def _bn_forward(self, x):
    geom = geometry(x) if _active(self, x) and int(x.shape[1]) == self.num_features else None
    if geom is None:
        self.__dict__.pop("_b2s_bn_out", None)
        return type(self).forward(self, x)
    y = BNReLUTrain.apply(x, self.weight, self.bias, self, geom)
    self.__dict__["_b2s_bn_out"] = weakref.ref(y)
    return y


def _relu_forward(self, x):
    # relu of the fused pair's output is that output: pass it through; anything else is a plain ReLU
    ref = self._b2s_bn.__dict__.get("_b2s_bn_out")
    if ref is not None and ref() is x:
        return x
    return nn.ReLU.forward(self, x)


def enable(net):
    """rebind the covered pairs under ``net``; idempotent, leaves anything it does not cover untouched.  Returns
    ``net``."""
    for bn, relu in select(net):
        if getattr(bn, "_b2s_bn_train", False):
            continue
        relu.__dict__["_b2s_bn"] = bn            # a plain attribute: not a submodule, not in the state dict
        relu.forward = types.MethodType(_relu_forward, relu)
        bn.forward = types.MethodType(_bn_forward, bn)
        bn._b2s_bn_train = True
    return net


# ---- the layer ------------------------------------------------------------------------------------------------------

def _like(t, x, layout):
    """t in x's layout, 16-byte aligned (a gradient may arrive as a strided or offset view)"""
    fmt = torch.channels_last if layout == LAYOUT_ROWS and x.dim() == 4 else torch.contiguous_format
    if not t.is_contiguous(memory_format=fmt) or t.data_ptr() % 16:
        t = t.clone(memory_format=fmt)
    return t


class BNReLUTrain(torch.autograd.Function):
    """relu(bn(x)) of a covered BatchNorm ``bn`` in training; see the module docstring."""

    @staticmethod
    def forward(ctx, x, weight, bias, bn, geom):
        L, lib = _lib()
        layout, B, S = geom
        C = int(x.shape[1])
        nbytes = int(lib.b2s_bn_relu_train_workspace_bytes(layout, B, C, S))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        y = torch.empty_like(x)
        L.check(lib.b2s_bn_relu_train_forward(
            L.ptr(x), layout, B, C, S, L.ptr(weight.detach()), L.ptr(bias.detach()), L.ptr(bn.running_mean),
            L.ptr(bn.running_var), L.ptr(bn.num_batches_tracked), float(bn.momentum), float(bn.eps), L.ptr(y), L.ptr(ws),
            nbytes, L.stream()), "b2s_bn_relu_train_forward")
        increment_version(bn.num_batches_tracked)          # as the torch forward's num_batches_tracked.add_(1)
        ctx.save_for_backward(x, weight, ws)
        ctx.geom = (layout, B, C, S)
        return y

    @staticmethod
    def backward(ctx, dy):
        L, lib = _lib()
        x, weight, ws = ctx.saved_tensors
        layout, B, C, S = ctx.geom
        dy = _like(dy.float(), x, layout)
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dg = torch.empty(C, dtype=torch.float32, device=x.device)
        db = torch.empty_like(dg)
        L.check(lib.b2s_bn_relu_train_backward(
            L.ptr(x), L.ptr(dy), layout, B, C, S, L.ptr(weight.detach()), L.ptr(ws), ws.numel(), L.ptr(dx), L.ptr(dg),
            L.ptr(db), L.stream()), "b2s_bn_relu_train_backward")
        return (dx, dg if ctx.needs_input_grad[1] else None, db if ctx.needs_input_grad[2] else None, None, None)
