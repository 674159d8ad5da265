"""The training loss on the GPU: ``VoxelNet.loss`` (second/pytorch/models/voxelnet.py:239-312) and its gradient, in
csrc/loss.cu.

    net = loss.enable_gpu_loss(training.enable_sparse_backward(net)).train()
    ret = net(example)                      # the reference's dict: loss, cls_loss, loc_loss, cls_pos_loss, ...
    ret["loss"].backward()

``plan`` reads the loss settings only through the reference's attribute names (``_cls_loss_ftor._alpha``,
``_loc_loss_ftor._sigma``, ``_loss_norm_type``, ``_dir_offset`` ...), so it takes the reference's own VoxelNet or the
mirror in b2second.models.  What every config uses is covered: sigmoid focal classification, smooth-L1 localization
with the yaw sin-encoded, NormByNumPositives weights, background encoded as zeros and the softmax direction
classifier, box code size 7.  Anything else raises ``spec.UnsupportedNetwork``.

``LossPlan.loss(example, preds_dict)`` returns the reference's dict.  ``loss`` and the three ``*_reduced`` scalars are
differentiable (one autograd node whose backward is ``b2s_detection_loss_backward``); ``cls_loss``, ``loc_loss``,
``cared``, ``cls_pos_loss`` and ``cls_neg_loss`` are not.  Sums run in one fixed order: two calls on the same inputs
give the same bits.  Preds must be float32 CUDA tensors (no fp16/AMP).
"""
import types
from dataclasses import dataclass
from typing import Tuple

import numpy as np
import torch

from .spec import UnsupportedNetwork

CODE_SIZE = 7


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


@dataclass(frozen=True)
class LossSettings:
    """the loss settings one kernel call takes, as the float32 values the kernel sees"""
    alpha: float
    gamma: float
    sigma: float
    code_weight: Tuple[float, ...]
    pos_cls_weight: float
    neg_cls_weight: float
    loc_weight: float
    cls_weight: float
    dir_weight: float
    sin_factor: float
    dir_offset: float
    num_dir_bins: int
    num_class: int


def _f32(v):
    return float(np.float32(float(v)))


def _norm_type_name(t):
    return getattr(t, "name", None) or str(t)


def plan(net):
    """-> LossPlan for a VoxelNet (the reference's or the mirror), read through the reference's attribute names."""
    cls_f, loc_f = net._cls_loss_ftor, net._loc_loss_ftor
    if type(cls_f).__name__ != "SigmoidFocalClassificationLoss":
        raise UnsupportedNetwork("classification loss %s is not supported (weighted_sigmoid_focal is)"
                                 % type(cls_f).__name__)
    if type(loc_f).__name__ != "WeightedSmoothL1LocalizationLoss":
        raise UnsupportedNetwork("localization loss %s is not supported (weighted_smooth_l1 is)" % type(loc_f).__name__)
    if _norm_type_name(net._loss_norm_type) != "NormByNumPositives":
        raise UnsupportedNetwork("loss_norm_type %s is not supported (NormByNumPositives is)"
                                 % _norm_type_name(net._loss_norm_type))
    if not net._encode_rad_error_by_sin:
        raise UnsupportedNetwork("encode_rad_error_by_sin = false is not supported")
    if not net._encode_background_as_zeros:
        raise UnsupportedNetwork("encode_background_as_zeros = false is not supported")
    if not net._use_direction_classifier:
        raise UnsupportedNetwork("use_direction_classifier = false is not supported")
    code_size = int(net._box_coder.code_size)
    if code_size != CODE_SIZE:
        raise UnsupportedNetwork("box code size %d is not supported (7 is)" % code_size)
    cw = loc_f._code_weights
    cw = [1.0] * code_size if cw is None else [float(v) for v in (cw.tolist() if hasattr(cw, "tolist") else cw)]
    if len(cw) != code_size:
        raise UnsupportedNetwork("code_weight has %d entries for a box code of %d" % (len(cw), code_size))
    gamma = cls_f._gamma or 0.0
    if cls_f._alpha is None:
        raise UnsupportedNetwork("sigmoid focal loss without alpha is not supported")
    s = LossSettings(
        alpha=_f32(cls_f._alpha), gamma=_f32(gamma), sigma=_f32(loc_f._sigma), code_weight=tuple(_f32(v) for v in cw),
        pos_cls_weight=_f32(net._pos_cls_weight), neg_cls_weight=_f32(net._neg_cls_weight),
        loc_weight=_f32(net._loc_loss_weight), cls_weight=_f32(net._cls_loss_weight),
        dir_weight=_f32(net._direction_loss_weight), sin_factor=_f32(net._sin_error_factor),
        dir_offset=_f32(net._dir_offset), num_dir_bins=int(net._num_direction_bins), num_class=int(net._num_class))
    if s.sigma <= 0 or s.pos_cls_weight == 0 or s.neg_cls_weight == 0:
        raise UnsupportedNetwork("sigma must be > 0 and the class weights nonzero")
    return LossPlan(s)


class _Loss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, box, cls, dir_, labels, reg, imp, anchors, lp):
        L, lib = _lib()
        B, A = int(labels.shape[0]), int(labels.shape[1])
        dev = box.device
        reduced = torch.empty(4, dtype=torch.float32, device=dev)
        pos_neg = torch.empty(2, dtype=torch.float32, device=dev)
        cls_loss = torch.empty(B, A, lp.settings.num_class, dtype=torch.float32, device=dev)
        loc_loss = torch.empty(B, A, CODE_SIZE, dtype=torch.float32, device=dev)
        cared = torch.empty(B, A, dtype=torch.bool, device=dev)
        norms = torch.empty(B, 2, dtype=torch.float32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        ws_bytes = lib.b2s_detection_loss_workspace_bytes(B, A)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2s_detection_loss(
                L.ptr(box), L.ptr(cls), L.ptr(dir_), lp.settings.num_class, lp.settings.num_dir_bins, L.ptr(labels),
                int(labels.dtype == torch.int64), L.ptr(reg), L.ptr(imp), L.ptr(anchors), B, A, lp.params_ref(),
                L.ptr(reduced), L.ptr(pos_neg), L.ptr(cls_loss), L.ptr(loc_loss), L.ptr(cared), L.ptr(norms),
                L.ptr(ws), ws_bytes, L.ptr(status), L.stream()), "b2s_detection_loss")
        lp.last_status = status            # device word; nonzero: a label outside [-1, num_class]
        ctx.lp = lp
        ctx.save_for_backward(box, cls, dir_, labels, reg, imp, anchors, norms)
        ctx.mark_non_differentiable(pos_neg, cls_loss, loc_loss, cared)
        return reduced, pos_neg, cls_loss, loc_loss, cared

    @staticmethod
    def backward(ctx, d_reduced, *_):
        L, lib = _lib()
        box, cls, dir_, labels, reg, imp, anchors, norms = ctx.saved_tensors
        lp = ctx.lp
        B, A = int(labels.shape[0]), int(labels.shape[1])
        d_box, d_cls, d_dir = torch.empty_like(box), torch.empty_like(cls), torch.empty_like(dir_)
        dr = d_reduced.to(torch.float32).contiguous() if d_reduced is not None else None
        with torch.cuda.device(box.device):
            L.check(lib.b2s_detection_loss_backward(
                L.ptr(box), L.ptr(cls), L.ptr(dir_), lp.settings.num_class, lp.settings.num_dir_bins, L.ptr(labels),
                int(labels.dtype == torch.int64), L.ptr(reg), L.ptr(imp), L.ptr(anchors), B, A, lp.params_ref(),
                L.ptr(norms), L.ptr(dr), L.ptr(d_box), L.ptr(d_cls), L.ptr(d_dir), L.stream()),
                "b2s_detection_loss_backward")
        return d_box, d_cls, d_dir, None, None, None, None, None


class LossPlan:
    """the loss of one network (see ``plan``)."""

    def __init__(self, settings: LossSettings):
        self.settings = settings
        self.last_status = None
        self._params = None

    def params(self):
        """b2s_loss_params as a ctypes structure (host memory, read by the call)."""
        if self._params is None:
            L, _ = _lib()
            s = self.settings
            p = L.LossParams()
            p.alpha, p.gamma, p.sigma = s.alpha, s.gamma, s.sigma
            for i, v in enumerate(s.code_weight):
                p.code_weight[i] = v
            p.pos_cls_weight, p.neg_cls_weight = s.pos_cls_weight, s.neg_cls_weight
            p.loc_weight, p.cls_weight, p.dir_weight = s.loc_weight, s.cls_weight, s.dir_weight
            p.sin_factor, p.dir_offset, p.num_dir_bins = s.sin_factor, s.dir_offset, s.num_dir_bins
            self._params = p
        return self._params

    def params_ref(self):
        import ctypes
        return ctypes.byref(self.params())

    def loss(self, example, preds_dict):
        """VoxelNet.loss's result dict for a batch (voxelnet.py:299-312), computed by csrc/loss.cu."""
        L, _ = _lib()
        s = self.settings
        labels = example["labels"]
        B = int(labels.shape[0])
        box = preds_dict["box_preds"]
        cls = preds_dict["cls_preds"]
        dir_ = preds_dict["dir_cls_preds"]
        for name, t in (("box_preds", box), ("cls_preds", cls), ("dir_cls_preds", dir_)):
            L.require_cuda(t, name)
            if t.dtype != torch.float32:
                raise TypeError("%s must be float32, got %s (fp16/AMP is not supported)" % (name, t.dtype))
        box = box.contiguous().view(B, -1, CODE_SIZE)
        A = int(box.shape[1])
        cls = cls.contiguous().view(B, A, s.num_class)
        dir_ = dir_.contiguous().view(B, A, s.num_dir_bins)
        if labels.dtype not in (torch.int32, torch.int64):
            labels = labels.to(torch.int64)
        labels = labels.contiguous().view(B, A)
        reg = example["reg_targets"].to(torch.float32).contiguous().view(B, A, CODE_SIZE)
        imp = example["importance"].to(torch.float32).contiguous().view(B, A)
        anchors = example["anchors"].to(torch.float32).contiguous().view(B, A, -1)
        if anchors.shape[-1] != CODE_SIZE:
            raise ValueError("anchors must be [B, A, 7], got %s" % (tuple(example["anchors"].shape),))
        for name, t in (("labels", labels), ("reg_targets", reg), ("importance", imp), ("anchors", anchors)):
            L.require_cuda(t, name)
        reduced, pos_neg, cls_loss, loc_loss, cared = _Loss.apply(box, cls, dir_, labels, reg, imp, anchors, self)
        return {
            "loss": reduced[0],
            "cls_loss": cls_loss,
            "loc_loss": loc_loss,
            "cls_pos_loss": pos_neg[0],
            "cls_neg_loss": pos_neg[1],
            "cls_preds": preds_dict["cls_preds"],
            "cls_loss_reduced": reduced[1],
            "loc_loss_reduced": reduced[2],
            "cared": cared,
            "dir_loss_reduced": reduced[3],
        }


def enable_gpu_loss(net):
    """make ``net(example)`` in ``train()`` mode return the GPU loss; returns ``net``.

    On the reference's VoxelNet this rebinds ``net.loss`` on the instance, so its own ``forward`` calls it.  On the
    mirror (b2second.models.VoxelNet) it also switches on the training branch of ``forward``, which otherwise
    raises ``NotImplementedError``."""
    lp = plan(net)
    net.b2s_loss = lp
    net.loss = types.MethodType(lambda self, example, preds_dict: lp.loss(example, preds_dict), net)
    return net
