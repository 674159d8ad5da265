"""Training of the PointPillars feature net on the GPU (csrc/pfn_train.cu).

``training.enable_pfn_training(net)`` rebinds ``net.voxel_feature_extractor.forward`` when the VFE is covered and
``net.middle_feature_extractor.forward`` when it is a ``PointPillarsScatter``.  Modules are found by class name and
attribute names, so the reference's own network (its ``change_default_args`` BatchNorm1d subclass) is covered as well as
the mirror in b2second.models.  Covered: ``PillarFeatureNet`` and ``PillarFeatureNetRadius`` with one PFNLayer
(Linear(D -> 64) without bias, a BatchNorm1d with affine parameters, running statistics and a momentum),
``with_distance=False`` and 3 to 8 point features.  Anything else keeps its torch forward.

The rebound forwards take the kernels only in ``train()`` mode with grad enabled on float32 CUDA input; otherwise they
are the class's own ``forward``, so ``eval()``, the fused engine and the state dict do not change.

PFNTrain, all on the caller's stream without a host sync (the layer can be captured):
  forward   b2s_pfn_train_forward: the BN batch statistics from the float64 mean and covariance of the decorated
            inputs, the running buffers updated in place, out [N, 64] and the argmax slot of every (pillar, channel);
  backward  b2s_pfn_train_backward: dW, dgamma, dbeta in closed form from the argmax slots; no voxel gradient.
ScatterBEV: PointPillarsScatter's canvas through b2s_to_bev (NCHW) and its backward through b2s_from_bev.
"""
import types

import torch
import torch.nn as nn

from . import loader

PLAIN, RADIUS = 0, 1            # B2S_PFN_*
COUT = 64
VFE_DECORATION = {"PillarFeatureNet": PLAIN, "PillarFeatureNetRadius": RADIUS}


def _lib():
    sp = loader.product_spconv()
    return sp._lib, sp._lib.load()


def num_features(vfe):
    """the number of point features F a covered ``vfe`` takes, or None when the kernels do not cover it."""
    deco = VFE_DECORATION.get(type(vfe).__name__)
    if deco is None or getattr(vfe, "_with_distance", True):
        return None
    if not all(hasattr(vfe, a) for a in ("vx", "vy", "x_offset", "y_offset", "pfn_layers")):
        return None
    layers = vfe.pfn_layers
    if len(layers) != 1:
        return None
    lin, bn = getattr(layers[0], "linear", None), getattr(layers[0], "norm", None)
    if not (isinstance(lin, nn.Linear) and lin.bias is None and lin.out_features == COUT):
        return None
    if not (isinstance(bn, nn.BatchNorm1d) and bn.affine and bn.track_running_stats and bn.momentum is not None
            and bn.num_features == COUT):
        return None
    F = lin.in_features - (5 if deco == PLAIN else 4)
    return F if 3 <= F <= 8 else None


def is_scatter(m):
    return type(m).__name__ == "PointPillarsScatter" and all(hasattr(m, a) for a in ("ny", "nx", "nchannels"))


def select(net):
    """-> (the covered VFE or None, the PointPillarsScatter or None) of ``net``."""
    vfe = getattr(net, "voxel_feature_extractor", None)
    mid = getattr(net, "middle_feature_extractor", None)
    return (vfe if vfe is not None and num_features(vfe) is not None else None,
            mid if mid is not None and is_scatter(mid) else None)


def _active(module, x):
    return module.training and torch.is_grad_enabled() and x.is_cuda and x.dtype == torch.float32


def _vfe_forward(self, features, num_voxels, coors):
    if _active(self, features) and features.dim() == 3:
        return PFNTrain.apply(features, num_voxels, coors, self.pfn_layers[0].linear.weight,
                              self.pfn_layers[0].norm.weight, self.pfn_layers[0].norm.bias, self).squeeze()
    return type(self).forward(self, features, num_voxels, coors)


def _scatter_forward(self, voxel_features, coords, batch_size):
    if _active(self, voxel_features) and voxel_features.dim() == 2:
        return ScatterBEV.apply(voxel_features, coords, int(batch_size), int(self.ny), int(self.nx))
    return type(self).forward(self, voxel_features, coords, batch_size)


def enable(net):
    """rebind the covered VFE and the PointPillarsScatter of ``net``; idempotent, leaves anything it does not cover
    untouched.  Returns ``net``."""
    vfe, scatter = select(net)
    if vfe is not None and not getattr(vfe, "_b2s_pfn_train", False):
        vfe.forward = types.MethodType(_vfe_forward, vfe)
        vfe._b2s_pfn_train = True
    if scatter is not None and not getattr(scatter, "_b2s_pfn_train", False):
        scatter.forward = types.MethodType(_scatter_forward, scatter)
        scatter._b2s_pfn_train = True
    return net


# ---- the layer ------------------------------------------------------------------------------------------------------

def _int32(t, dev):
    return t.to(device=dev, dtype=torch.int32).contiguous()


def geometry(vfe):
    return float(vfe.vx), float(vfe.vy), float(vfe.x_offset), float(vfe.y_offset)


class PFNTrain(torch.autograd.Function):
    """the [N, 64] output of a covered VFE in training (before the reference's ``.squeeze()``); see the module
    docstring.  The status word of the last forward (B2S_STATUS_BAD_INPUT for a count outside [1, T]) is left in
    ``vfe._b2s_pfn_status`` for the caller to read when it next syncs."""

    @staticmethod
    def forward(ctx, voxels, num, coors, weight, gamma, beta, vfe):
        L, lib = _lib()
        N, T, F = (int(v) for v in voxels.shape)
        if F != num_features(vfe):
            raise RuntimeError("PFNTrain: voxels have %d features, the PFN takes %d" % (F, num_features(vfe)))
        dev = voxels.device
        voxels = voxels.contiguous()
        num, coors = _int32(num, dev), _int32(coors, dev)
        bn = vfe.pfn_layers[0].norm
        deco = VFE_DECORATION[type(vfe).__name__]
        ws = torch.empty(max(int(lib.b2s_pfn_train_workspace_bytes(N)), 1), dtype=torch.uint8, device=dev)
        out = torch.empty(N, COUT, dtype=torch.float32, device=dev)
        arg = torch.empty(N, COUT, dtype=torch.uint8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        w = weight.detach().contiguous()
        L.check(lib.b2s_pfn_train_forward(
            L.ptr(voxels), N, T, F, L.ptr(num), L.ptr(coors), L.ptr(w), L.ptr(gamma.detach()), L.ptr(beta.detach()),
            COUT, L.ptr(bn.running_mean), L.ptr(bn.running_var), L.ptr(bn.num_batches_tracked), float(bn.momentum),
            float(bn.eps), *geometry(vfe), deco, L.ptr(out), L.ptr(arg), L.ptr(ws), ws.numel(), L.ptr(status),
            L.stream()), "b2s_pfn_train_forward")
        vfe.__dict__["_b2s_pfn_status"] = status
        ctx.save_for_backward(voxels, num, coors, w, gamma, out, arg, ws)
        ctx.geom = geometry(vfe) + (deco,)
        return out

    @staticmethod
    def backward(ctx, dout):
        L, lib = _lib()
        voxels, num, coors, w, gamma, out, arg, ws = ctx.saved_tensors
        N, T, F = (int(v) for v in voxels.shape)
        dout = dout.float().contiguous()
        dw = torch.empty_like(w)
        dg = torch.empty(COUT, dtype=torch.float32, device=w.device)
        db = torch.empty_like(dg)
        vx, vy, xo, yo, deco = ctx.geom
        L.check(lib.b2s_pfn_train_backward(
            L.ptr(voxels), N, T, F, L.ptr(num), L.ptr(coors), L.ptr(w), L.ptr(gamma.detach()), COUT, vx, vy, xo, yo,
            deco, L.ptr(out), L.ptr(arg), L.ptr(dout), L.ptr(ws), ws.numel(), L.ptr(dw), L.ptr(dg), L.ptr(db),
            L.stream()), "b2s_pfn_train_backward")
        return None, None, None, dw, dg, db, None


class ScatterBEV(torch.autograd.Function):
    """PointPillarsScatter.forward: rows [N, C] -> canvas [B, C, ny, nx] (b2s_to_bev, NCHW, D = 1); the backward
    gathers each row's gradient from its pixel (b2s_from_bev)."""

    @staticmethod
    def forward(ctx, feats, coords, batch_size, ny, nx):
        L, lib = _lib()
        dev = feats.device
        feats = feats.contiguous()
        coords = _int32(coords, dev)
        n, C = (int(v) for v in feats.shape)
        n_dev = torch.full((1,), n, dtype=torch.int32, device=dev)
        out = torch.empty(batch_size, C, ny, nx, dtype=torch.float32, device=dev)
        L.check(lib.b2s_to_bev(L.ptr(feats), L.ptr(coords), L.ptr(n_dev), n, C, batch_size, 1, ny, nx, L.ptr(out), 0,
                               L.stream()), "b2s_to_bev")
        ctx.save_for_backward(coords, n_dev)
        ctx.shape = (n, C, batch_size, ny, nx)
        return out

    @staticmethod
    def backward(ctx, grad):
        L, lib = _lib()
        coords, n_dev = ctx.saved_tensors
        n, C, B, ny, nx = ctx.shape
        grad = grad.float().contiguous()
        drows = torch.empty(n, C, dtype=torch.float32, device=grad.device)
        if n > 0:
            L.check(lib.b2s_from_bev(L.ptr(grad), L.ptr(coords), L.ptr(n_dev), n, C, B, 1, ny, nx, 0, L.ptr(drows),
                                     L.stream()), "b2s_from_bev")
        return drows, None, None, None, None
