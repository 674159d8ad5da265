"""Training targets on the GPU: ``TargetAssigner.assign`` (second/core/target_assigner.py:38-167) through
``create_target_np`` (second/core/target_ops.py:29-229) for a whole batch, in csrc/targets.cu.

    tp = targets.plan(net.target_assigner, feature_map_size)      # once per anchor set
    example.update(tp.assign_batch(gt_boxes, gt_offsets, gt_classes, importance, anchors_mask))

``plan`` reads the assigner only through the reference's attribute names, so it takes the reference's own
``TargetAssigner`` or b2second.models.MirrorTargetAssigner.  A segment is one class's anchor range
(``assign_per_class``) or every anchor (``assign_all``, which uses ``_sim_calcs[0]`` for all classes).  What matches
the reference, per segment:
  * labels, importance and the + - * / sqrt components of the box targets bit for bit; the log / sin / cos components
    (GroundBox3dCoder.encode, box_np_ops.py:36-83) within a few float32 ulp, as libm implementations differ;
  * the reference's quirks: a forced anchor takes the class of its own best GT; per-class importance indexes the
    frame-wide array with the class-local GT index (target_assigner.py:140).
Divergence: when every anchor of a segment is pruned and the segment has ground truth, the reference raises (numpy
argmax over an empty axis); here that segment comes out as label -1, targets 0, importance 0.
Refused (spec.UnsupportedNetwork), as no config uses them: positive_fraction, RotateIouSimilarity,
DistanceSimilarity(with_rotation=True), BevBoxCoder.
"""
import ctypes
from dataclasses import dataclass
from typing import List

import numpy as np
import torch

from . import anchor_mask
from .spec import UnsupportedNetwork

KIND_IOU, KIND_DISTANCE = 0, 1
BLOCK = 256                                    # anchors per CTA of the kernel; a block never straddles two segments


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


@dataclass
class Segment:
    begin: int
    end: int
    kind: int
    distance_norm: float


class TargetPlan:
    """the anchor side of target assignment for one anchor set (see ``plan``)."""

    def __init__(self, anchors, matched, unmatched, segments: List[Segment], classes, assign_per_class, box_ndim,
                 code_size, linear_dim, vec_encode):
        self.anchors = np.ascontiguousarray(anchors, dtype=np.float32)
        self.matched_thresholds = np.ascontiguousarray(matched, dtype=np.float32)
        self.unmatched_thresholds = np.ascontiguousarray(unmatched, dtype=np.float32)
        self.segments = segments
        self.classes = list(classes)
        self.assign_per_class = bool(assign_per_class)
        self.box_ndim, self.code_size = int(box_ndim), int(code_size)
        self.linear_dim, self.vec_encode = bool(linear_dim), bool(vec_encode)
        # per anchor: rbbox2d_to_near_bbox (float32, box_np_ops.py:286-298) for IoU segments, (x, y, 0, 0) for distance
        sim = anchor_mask.near_bboxes(self.anchors) if len(self.anchors) else np.zeros((0, 4), np.float32)
        for s in segments:
            if s.kind == KIND_DISTANCE:
                sim[s.begin:s.end] = 0
                sim[s.begin:s.end, :2] = self.anchors[s.begin:s.end, :2]
        self.anchor_sim = np.ascontiguousarray(sim, dtype=np.float32)
        self.seg_info = np.array([[s.begin, s.end, s.kind, 0] for s in segments], np.int32).reshape(-1, 4)
        self.seg_param = np.array([s.distance_norm for s in segments], np.float64)
        self.blocks = np.array([[i, b, min(b + BLOCK, s.end), 0] for i, s in enumerate(segments)
                                for b in range(s.begin, s.end, BLOCK)], np.int32).reshape(-1, 4)
        self._dev = {}

    @property
    def num_anchors(self):
        return int(self.anchors.shape[0])

    def params(self):
        """everything the kernel is given about the anchors, as host arrays (for comparing two plans)."""
        return {"anchors": self.anchors, "matched_thresholds": self.matched_thresholds,
                "unmatched_thresholds": self.unmatched_thresholds, "anchor_sim": self.anchor_sim,
                "seg_info": self.seg_info, "seg_param": self.seg_param, "blocks": self.blocks,
                "assign_per_class": np.array(self.assign_per_class), "classes": np.array(self.classes),
                "coder": np.array([self.box_ndim, self.code_size, self.linear_dim, self.vec_encode], np.int32)}

    def _tables(self, device):
        key = str(torch.device(device))
        if key not in self._dev:
            t = {k: torch.from_numpy(getattr(self, k)).to(device) for k in
                 ("anchors", "matched_thresholds", "unmatched_thresholds", "anchor_sim", "seg_info", "seg_param",
                  "blocks")}
            self._dev[key] = t
        return self._dev[key]

    # -------------------------------------------------------------------------------------------- kernel call
    def _run(self, device, gt_boxes, gt_offsets, gt_seg, gt_class, importance, mask, batch, matched=None,
             unmatched=None, extra=False):
        L, lib = _lib()
        t = self._tables(device)
        A, G, S = self.num_anchors, int(gt_boxes.shape[0]), len(self.segments)
        if gt_boxes.dtype not in (torch.float32, torch.float64):
            raise TypeError("gt_boxes must be float32 or float64, got %s" % gt_boxes.dtype)
        if gt_boxes.dim() != 2 or gt_boxes.shape[1] != self.box_ndim:
            raise ValueError("gt_boxes must be [G, %d], got %s" % (self.box_ndim, tuple(gt_boxes.shape)))
        if mask is not None and tuple(mask.shape) != (batch, A):
            raise ValueError("anchors_mask must be [%d, %d], got %s" % (batch, A, tuple(mask.shape)))
        gt_boxes = gt_boxes.contiguous()
        labels = torch.empty(batch, A, dtype=torch.int32, device=device)
        targets = torch.empty(batch, A, self.code_size, dtype=torch.float32, device=device)
        imp = torch.empty(batch, A, dtype=torch.float32, device=device)
        gt_id = torch.empty(batch, A, dtype=torch.int32, device=device) if extra else None
        overlap = torch.empty(batch, A, dtype=torch.float32, device=device) if extra else None
        status = torch.zeros(1, dtype=torch.int32, device=device)
        ws_bytes = lib.b2s_assign_targets_workspace_bytes(batch, G, S)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        mt = t["matched_thresholds"] if matched is None else matched
        ut = t["unmatched_thresholds"] if unmatched is None else unmatched
        with torch.cuda.device(device):
            L.check(lib.b2s_assign_targets(
                L.ptr(t["anchors"]), L.ptr(t["anchor_sim"]), L.ptr(mt), L.ptr(ut), A, self.box_ndim,
                L.ptr(t["seg_info"]), L.ptr(t["seg_param"]), S, L.ptr(t["blocks"]), int(t["blocks"].shape[0]),
                L.ptr(gt_boxes) if G else None, int(gt_boxes.dtype == torch.float64), G, L.ptr(gt_offsets), batch,
                L.ptr(gt_seg) if G else None, L.ptr(gt_class) if G else None,
                L.ptr(importance) if (G and importance is not None) else None, L.ptr(mask), self.code_size,
                int(self.linear_dim) | (int(self.vec_encode) << 1), L.ptr(labels), L.ptr(targets), L.ptr(imp),
                L.ptr(gt_id), L.ptr(overlap), L.ptr(ws), ws_bytes, L.ptr(status), L.stream()), "b2s_assign_targets")
        self.last_status = status          # device word; nonzero: bad gt_offsets (see spconv._lib.STATUS_BITS)
        return labels, targets, imp, gt_id, overlap

    # -------------------------------------------------------------------------------------------- batch
    def assign_batch(self, gt_boxes, gt_offsets, gt_classes, importance=None, anchors_mask=None):
        """targets for a batch, without a host sync.
        gt_boxes CUDA float32/float64 [G, box_ndim], packed frame after frame; gt_offsets CUDA int32 [B+1];
        gt_classes CUDA int [G] (1-based class ids; per-class mode puts GT i in class gt_classes[i] - 1, as
        preprocess.py:269-272 builds them); importance CUDA float [G] or None; anchors_mask CUDA bool [B, A] (what
        b2second.inputs.anchor_area_mask returns) or None.
        -> {"labels": int32 [B, A], "reg_targets": float32 [B, A, code], "importance": float32 [B, A]}."""
        L, _ = _lib()
        for name, v in (("gt_boxes", gt_boxes), ("gt_offsets", gt_offsets), ("gt_classes", gt_classes),
                        ("importance", importance), ("anchors_mask", anchors_mask)):
            if v is not None:
                L.require_cuda(v, name)
        device = gt_boxes.device
        batch = int(gt_offsets.shape[0]) - 1
        if batch < 1:
            raise ValueError("gt_offsets must hold batch + 1 >= 2 entries")
        offs = gt_offsets.to(torch.int32).contiguous()
        cls = gt_classes.to(torch.int32).contiguous()
        seg = (cls - 1) if self.assign_per_class else torch.zeros_like(cls)
        imp = importance.to(torch.float32).contiguous() if importance is not None else None
        mask = anchors_mask.to(torch.uint8).contiguous() if anchors_mask is not None else None
        labels, targets, imp_out, _, _ = self._run(device, gt_boxes, offs, seg.contiguous(), cls, imp, mask, batch)
        return {"labels": labels, "reg_targets": targets, "importance": imp_out}

    # -------------------------------------------------------------------------------------------- one frame
    def assign(self, anchors, anchors_dict, gt_boxes, anchors_mask=None, gt_classes=None, gt_names=None,
               matched_thresholds=None, unmatched_thresholds=None, importance=None):
        """TargetAssigner.assign's signature and result dict for one frame, as CUDA tensors.  Host (numpy) arrays or
        CUDA tensors in; the anchors (``anchors`` or ``anchors_dict``) must be the plan's."""
        device = torch.device("cuda", torch.cuda.current_device())
        for v in (gt_boxes, anchors_mask, gt_classes, importance, matched_thresholds, unmatched_thresholds):
            if isinstance(v, torch.Tensor):
                if not v.is_cuda:
                    _lib()[0].require_cuda(v, "input")
                device = v.device
        if self.assign_per_class:
            got = np.concatenate([_host(d["anchors"]).reshape(-1, self.box_ndim) for d in anchors_dict.values()])
            mt = ut = None
            if not np.array_equal(got, self.anchors):
                raise ValueError("anchors_dict holds other anchors than the plan was built for")
        else:
            if not np.array_equal(_host(anchors).reshape(-1, self.box_ndim), self.anchors):
                raise ValueError("anchors are not the ones the plan was built for")
            # create_target_np's defaults (0.6 / 0.45) stand in for missing thresholds
            mt = _thresholds(matched_thresholds, 0.6, self.num_anchors, device)
            ut = _thresholds(unmatched_thresholds, 0.45, self.num_anchors, device)
        gt = _dev(gt_boxes, device)
        if gt.dtype not in (torch.float32, torch.float64):
            gt = gt.float()
        gt = gt.reshape(-1, self.box_ndim)
        G = int(gt.shape[0])
        cls = _dev(gt_classes, device).to(torch.int32) if gt_classes is not None else \
            torch.ones(G, dtype=torch.int32, device=device)
        if self.assign_per_class:
            names = list(gt_names) if gt_names is not None else []
            seg = torch.tensor([self.classes.index(n) if n in self.classes else -1 for n in names] or [],
                               dtype=torch.int32).reshape(-1).to(device)
        else:
            seg = torch.zeros(G, dtype=torch.int32, device=device)
        imp = _dev(importance, device).to(torch.float32).contiguous() if importance is not None else None
        mask = _dev(anchors_mask, device).reshape(1, -1).to(torch.uint8).contiguous() \
            if anchors_mask is not None else None
        offs = torch.tensor([0, G], dtype=torch.int32).to(device)
        labels, targets, imp_out, gt_id, overlap = self._run(device, gt, offs, seg, cls.contiguous(), imp, mask, 1,
                                                             mt, ut, extra=not self.assign_per_class)
        ret = {"labels": labels[0], "bbox_targets": targets[0], "importance": imp_out[0]}
        if not self.assign_per_class:
            inds = torch.nonzero(gt_id[0] >= 0).reshape(-1)
            ret["bbox_outside_weights"] = (labels[0] > 0).to(torch.float32)
            ret["assigned_anchors_overlap"] = overlap[0][inds] if G else None
            ret["positive_gt_id"] = gt_id[0][inds]
            ret["assigned_anchors_inds"] = inds
        return ret


def _host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _dev(x, device):
    if isinstance(x, torch.Tensor):
        return x.to(device)
    return torch.from_numpy(np.ascontiguousarray(x)).to(device)


def _thresholds(v, default, n, device):
    if v is None or isinstance(v, float):
        return torch.full((n,), default if v is None else v, dtype=torch.float32, device=device)
    return _dev(v, device).to(torch.float32).reshape(-1).contiguous()


# ------------------------------------------------------------------------------------------------ plan
def _similarity(sim, where):
    name = type(sim).__name__
    if hasattr(sim, "_distance_norm"):
        if getattr(sim, "_with_rotation", False):
            raise UnsupportedNetwork("%s: DistanceSimilarity with with_rotation=True is not supported" % where)
        return KIND_DISTANCE, float(sim._distance_norm)
    if "Nearest" in name:
        return KIND_IOU, 0.0
    raise UnsupportedNetwork("%s: region similarity %s is not supported (NearestIouSimilarity and "
                             "DistanceSimilarity are)" % (where, name))


def plan(target_assigner, feature_map_size):
    """-> TargetPlan for the anchors ``target_assigner.generate_anchors(feature_map_size)`` makes."""
    ta = target_assigner
    if getattr(ta, "_positive_fraction", None) is not None:
        raise UnsupportedNetwork("target_assigner.sample_positive_fraction = %r: random subsampling of positives is "
                                 "not supported" % ta._positive_fraction)
    coder = ta._box_coder
    if "Bev" in type(coder).__name__ or hasattr(coder, "z_fixed"):
        raise UnsupportedNetwork("box_coder: BevBoxCoder is not supported (ground_box3d_coder is)")
    gens = ta._anchor_generators
    custom = int(gens[0].custom_ndim)
    box_ndim = 7 + custom
    code_size = int(coder.custom_ndim if coder.custom_ndim is not None else custom) + (8 if coder.vec_encode else 7)
    anchors = np.asarray(ta.generate_anchors(feature_map_size)["anchors"], dtype=np.float32).reshape(-1, box_ndim)
    A = anchors.shape[0]
    matched = np.empty(A, np.float32)
    unmatched = np.empty(A, np.float32)
    classes = list(ta.classes)
    per_class = bool(ta._assign_per_class)
    segments = []
    if per_class:
        for c, g in enumerate(gens):
            b, e = (int(v) for v in ta.anchors_range(c))
            matched[b:e] = np.float32(g.match_threshold)
            unmatched[b:e] = np.float32(g.unmatch_threshold)
            kind, dn = _similarity(ta._sim_calcs[c], "class %s" % classes[c])
            segments.append(Segment(b, e, kind, dn))
        if segments and segments[-1].end != A:
            raise ValueError("anchors_range does not cover the %d anchors" % A)
    else:
        # generate_anchors (target_assigner.py:169-207): generator blocks in order, each on its own feature map
        fsizes = getattr(ta, "_feature_map_sizes", None) or [[]] * len(gens)
        b = 0
        for g, fs in zip(gens, fsizes):
            n = int(g.num_anchors_per_localization) * int(np.prod(list(fs) if len(fs) else list(feature_map_size)))
            matched[b:b + n] = np.float32(g.match_threshold)
            unmatched[b:b + n] = np.float32(g.unmatch_threshold)
            b += n
        if b != A:
            raise ValueError("anchor generators give %d anchors, generate_anchors %d" % (b, A))
        kind, dn = _similarity(ta._sim_calcs[0], "assign_all")
        segments.append(Segment(0, A, kind, dn))
    return TargetPlan(anchors, matched, unmatched, segments, classes, per_class, box_ndim, code_size,
                      bool(coder.linear_dim), bool(coder.vec_encode))
