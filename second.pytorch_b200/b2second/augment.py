"""Training augmentation on the GPU: what prep_pointcloud (second/data/preprocess.py:255-294) does to a frame after
ground-truth database sampling, for a whole batch, in csrc/augment.cu.

    ap = augment.plan(cfg.augment, cfg.point_cloud_range, class_names)       # once
    d = augment.draw(rs, cfg.augment, num_gt_per_frame, num_points_per_frame)  # host, per batch
    out = ap.augment_batch(points, point_offsets, gt_boxes, gt_offsets, gt_valid, gt_classes, importance, d)
    # out["points"] / point_offsets -> b2s_voxelize, out["boxes"] / out["gt_offsets"] / out["classes"] -> assign_batch

Steps, in the reference's order: noise_per_object_v3_ with 100 tries (second/core/preprocess.py:582-678), dropping the
boxes outside the class mask, random_flip, global_rotation_v2, global_scaling_v2, global_translate_ (:749-800, 885-899),
filter_gt_box_outside_range_by_center (:153-164), limit_period(0.5, 2 pi) and np.random.shuffle(points).

Random numbers come from one of two sources.  ``draw`` (the default) consumes a numpy RandomState exactly as the
reference's functions do, frame after frame, so a caller that samples the ground-truth database on the host first and
then calls ``draw`` on the same state gets the reference's augmentation.  ``DeviceDrawer`` (opt-in) draws them on the
device (csrc/augment_draws.cu) from a seeded Philox4x64-10 stream keyed by (seed, step) and counted by frame, with no
host work per frame and no host sync; its draws are reproducible from (seed, step), do not depend on how frames are
split over calls or data-parallel ranks, and replay inside a CUDA graph (INTEGRATION.md states the contract):

    dd = augment.DeviceDrawer(seed, "cuda")                                      # once; dd.step is the checkpoint
    d = dd.draw(cfg.augment, gt_offsets, point_offsets, G, P, frame_base=rank * B)  # device, per batch

Arithmetic follows the reference's dtypes (float32 points, float32 or float64 boxes, float64 draws); values that pass
through the reference's BLAS matmuls (per-object and global rotation) agree to a few float32 ulp, everything else bit
for bit, and every decision (selected try, point-in-box, range filter) is the reference's away from exact ties.
Refused (spec.UnsupportedNetwork), as no config uses them: a per-object global rotation range
(``global_random_rotation_range_per_object`` wider than 1e-3, noise_per_box_v2_) and ``use_group_id``.
Left on the host: database sampling and the row selections before augmentation (remove_environment, remove_unknown,
min_num_of_points_in_gt, the frustum crop, remove_outside_points); ``gt_valid`` and the packed inputs carry them.
"""
import ctypes
import math
import operator
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from .config import AugmentSettings  # noqa: F401  (re-exported: the settings type lives with the config parser)
from .spec import UnsupportedNetwork

NUM_TRY = 100                     # prep_pointcloud's num_try for noise_per_object_v3_ (preprocess.py:263)
MAX_BOXES = 1024                  # B2S_AUGMENT_MAX_BOXES: per-frame box cap of the pose-selection kernel
SEL_NONE, SEL_SKIPPED = -1, -2    # selected try: none was collision-free / the frame was over MAX_BOXES


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


def object_noise_enabled(s):
    """False where noise_per_object_v3_ returns before drawing anything (preprocess.py:611-612)."""
    grot = list(s.global_random_rotation_range_per_object)
    enable_grot = abs(grot[0] - grot[1]) >= 1e-3
    return not (all(c == 0 for c in s.groundtruth_localization_noise_std)
                and all(c == 0 for c in s.groundtruth_rotation_uniform_noise) and not enable_grot)


@dataclass
class Draws:
    """the random numbers of one batch, in the reference's terms: host numpy arrays from ``draw``, or CUDA tensors from
    ``DeviceDrawer.draw`` (whose num_gt and num_points are None: the counts stay on the device).
    loc_noise [G, 100, 3] / rot_noise [G, 100] float64 (None when the object noise returns early); frame [B, 8]
    float64: flip_y, flip_x, translate (0/1, as applied), rotation angle, scale, tx, ty, tz; perm [P] int32 frame-local
    source rows (None when not shuffling)."""
    loc_noise: Optional[np.ndarray]
    rot_noise: Optional[np.ndarray]
    frame: np.ndarray
    perm: Optional[np.ndarray]
    num_gt: List[int]
    num_points: List[int]


def draw(rs, settings, num_gt_per_frame, num_points_per_frame):
    """the draws prep_pointcloud makes for each frame, from ``rs`` (np.random.RandomState or the np.random module),
    consuming it in the reference's order: the object noise (normal, uniform, and the per-object global rotation uniform
    that is drawn and discarded), both flip choices, the rotation and scaling uniforms, the translation normals (only
    when a std is nonzero) and the shuffle."""
    s = settings
    rs = np.random if rs is None else rs
    noise = object_noise_enabled(s)
    std = np.array(s.groundtruth_localization_noise_std, dtype=np.float64)
    rot = list(s.groundtruth_rotation_uniform_noise)
    grot = list(s.global_random_rotation_range_per_object)
    tstd = list(s.global_translate_noise_std)
    translate = not all(e == 0 for e in tstd)
    locs, rots, frames, perms = [], [], [], []
    for n, npts in zip(num_gt_per_frame, num_points_per_frame):
        n, npts = int(n), int(npts)
        if noise:
            locs.append(rs.normal(scale=std, size=[n, NUM_TRY, 3]))
            rots.append(rs.uniform(rot[0], rot[1], size=[n, NUM_TRY]))
            rs.uniform(grot[0], grot[1], size=[n, NUM_TRY])       # global_rot_noises: only its stream use matters
        flip_x = rs.choice([False, True], replace=False, p=[0.5, 0.5])
        flip_y = rs.choice([False, True], replace=False, p=[0.5, 0.5])
        angle = rs.uniform(*s.global_rotation_uniform_noise)
        scale = rs.uniform(*s.global_scaling_uniform_noise)
        t = [0.0, 0.0, 0.0]
        if translate:
            t = [float(rs.normal(0, tstd[0], 1)[0]), float(rs.normal(0, tstd[1], 1)[0]),
                 float(rs.normal(0, tstd[0], 1)[0])]
        frames.append([float(bool(flip_y) and s.random_flip_y), float(bool(flip_x) and s.random_flip_x),
                       float(translate), float(angle), float(scale), *t])
        if s.shuffle_points:
            p = np.arange(npts)
            rs.shuffle(p)
            perms.append(p.astype(np.int32))
    return Draws(
        loc_noise=np.concatenate(locs) if noise and locs else (np.zeros((0, NUM_TRY, 3)) if noise else None),
        rot_noise=np.concatenate(rots) if noise and rots else (np.zeros((0, NUM_TRY)) if noise else None),
        frame=np.array(frames, np.float64).reshape(-1, 8),
        perm=np.concatenate(perms).astype(np.int32) if s.shuffle_points and perms else
        (np.zeros(0, np.int32) if s.shuffle_points else None),
        num_gt=[int(v) for v in num_gt_per_frame], num_points=[int(v) for v in num_points_per_frame])


def select(draws, start, stop):
    """-> the Draws of frames ``start .. stop - 1`` of ``draws``: a data-parallel rank's share of draws made for the
    whole batch in single-process order, so the augmentation does not depend on the number of ranks.  Device draws
    are refused: a rank draws its own frames with ``DeviceDrawer.draw(..., frame_base=start)`` instead."""
    if isinstance(draws.frame, torch.Tensor):
        raise ValueError("select takes host draws; DeviceDrawer.draw's frame_base gives a rank its frames' draws")
    g = np.cumsum([0] + list(draws.num_gt))
    p = np.cumsum([0] + list(draws.num_points))
    return Draws(
        loc_noise=None if draws.loc_noise is None else draws.loc_noise[g[start]:g[stop]],
        rot_noise=None if draws.rot_noise is None else draws.rot_noise[g[start]:g[stop]],
        frame=draws.frame[start:stop], perm=None if draws.perm is None else draws.perm[p[start]:p[stop]],
        num_gt=list(draws.num_gt[start:stop]), num_points=list(draws.num_points[start:stop]))


def _to_device(a, device, dtype):
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=dtype))
    if t.numel() == 0:
        return torch.empty(t.shape, dtype=t.dtype, device=device)
    return t.pin_memory().to(device, non_blocking=True)


def _draw_input(a, device, dtype):
    """one array of a Draws as b2s_augment reads it: host arrays are copied, DeviceDrawer's tensors used as they are"""
    if isinstance(a, torch.Tensor):
        if a.device != device or a.dtype != dtype:
            raise ValueError("device draws must be %s on %s, got %s on %s" % (dtype, device, a.dtype, a.device))
        return a.contiguous()
    return _to_device(a, device, np.float64 if dtype == torch.float64 else np.int32)


class AugmentPlan:
    """the fixed side of the augmentation for one config (see ``plan``)."""

    def __init__(self, settings, point_cloud_range, class_names):
        self.settings = settings
        self.point_cloud_range = np.asarray(point_cloud_range, dtype=np.float32)
        self.bv_range = np.ascontiguousarray(self.point_cloud_range[[0, 1, 3, 4]])
        self.class_names = list(class_names)
        self.object_noise = object_noise_enabled(settings)

    def augment_batch(self, points, point_offsets, gt_boxes, gt_offsets, gt_valid, gt_classes, importance, draws,
                      with_debug=False):
        """augment a batch without a host sync.
        points CUDA float32 [P, F] packed frame after frame, point_offsets CUDA int32 [B+1]; gt_boxes CUDA float32 or
        float64 [G, 7 or 9], gt_offsets CUDA int32 [B+1]; gt_valid CUDA bool [G] (the class mask); gt_classes CUDA int
        [G]; importance CUDA float [G] or None; draws: ``draw``'s result for these frames (copied to the device) or
        ``DeviceDrawer.draw``'s (read in place, so one CUDA graph can capture both calls).
        -> {"points": float32 [P, F] (frame rows in shuffled order), "boxes": [G, ndim] of the input dtype, "gt_offsets":
        int32 [B+1], "classes": int32 [G], "importance": float32 [G], "src_row": int32 [G]}: the kept boxes packed in
        input order, rows past gt_offsets[B] zero (src_row -1).  with_debug adds "selected" (int32 [G], the try each input box
        took: -1 none, -2 frame over MAX_BOXES) and "point_box" (int32 [P], the input box that moved each output
        point, -1 none)."""
        L, lib = _lib()
        for name, v in (("points", points), ("point_offsets", point_offsets), ("gt_boxes", gt_boxes),
                        ("gt_offsets", gt_offsets), ("gt_valid", gt_valid), ("gt_classes", gt_classes),
                        ("importance", importance)):
            if v is not None:
                L.require_cuda(v, name)
        device = points.device
        if gt_boxes.dtype not in (torch.float32, torch.float64):
            raise TypeError("gt_boxes must be float32 or float64, got %s" % gt_boxes.dtype)
        if gt_boxes.dim() != 2 or gt_boxes.shape[1] not in (7, 9):
            raise ValueError("gt_boxes must be [G, 7] or [G, 9], got %s" % (tuple(gt_boxes.shape),))
        if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] < 3:
            raise ValueError("points must be float32 [P, >= 3]")
        B = int(point_offsets.shape[0]) - 1
        if B < 1 or int(gt_offsets.shape[0]) != B + 1:
            raise ValueError("point_offsets and gt_offsets must both hold batch + 1 >= 2 entries")
        frames = draws.frame.shape[0] if draws.num_gt is None else len(draws.num_gt)
        if frames != B or draws.frame.shape[0] != B:
            raise ValueError("draws were made for %d frames, the batch has %d" % (frames, B))
        P, F = int(points.shape[0]), int(points.shape[1])
        G, ndim = int(gt_boxes.shape[0]), int(gt_boxes.shape[1])
        if self.object_noise and draws.loc_noise is None:
            raise ValueError("draws hold no object noise, the settings have it")
        if self.object_noise and draws.loc_noise.shape[0] != G:
            raise ValueError("draws hold object noise for %d boxes, gt_boxes has %d" % (draws.loc_noise.shape[0], G))
        if draws.perm is not None and draws.perm.shape[0] != P:
            raise ValueError("draws hold a permutation of %d points, points has %d" % (draws.perm.shape[0], P))
        points = points.contiguous()
        gt_boxes = gt_boxes.contiguous()
        poff = point_offsets.to(torch.int32).contiguous()
        goff = gt_offsets.to(torch.int32).contiguous()
        valid = gt_valid.to(torch.uint8).contiguous()
        cls = gt_classes.to(torch.int32).contiguous()
        imp = importance.to(torch.float32).contiguous() if importance is not None else None
        noise = self.object_noise and G > 0
        loc = _draw_input(draws.loc_noise, device, torch.float64) if noise else None
        rot = _draw_input(draws.rot_noise, device, torch.float64) if noise else None
        frame = _draw_input(draws.frame, device, torch.float64)
        perm = _draw_input(draws.perm, device, torch.int32) if draws.perm is not None else None
        pts_out = torch.empty_like(points)
        boxes_out = torch.empty_like(gt_boxes)
        offs_out = torch.empty(B + 1, dtype=torch.int32, device=device)
        cls_out = torch.empty(G, dtype=torch.int32, device=device)
        imp_out = torch.empty(G, dtype=torch.float32, device=device)
        src_out = torch.empty(G, dtype=torch.int32, device=device)
        selected = torch.empty(G, dtype=torch.int32, device=device)
        point_box = torch.empty(P, dtype=torch.int32, device=device) if with_debug else None
        status = torch.zeros(1, dtype=torch.int32, device=device)
        ws_bytes = lib.b2s_augment_workspace_bytes(B, G, ndim)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        rng = (ctypes.c_float * 4)(*[float(v) for v in self.bv_range])
        with torch.cuda.device(device):
            L.check(lib.b2s_augment(
                L.ptr(points) if P else None, P, F, L.ptr(poff), B, L.ptr(gt_boxes) if G else None,
                int(gt_boxes.dtype == torch.float64), ndim, G, L.ptr(goff), L.ptr(valid) if G else None,
                L.ptr(cls) if G else None, L.ptr(imp) if (G and imp is not None) else None, L.ptr(loc), L.ptr(rot),
                NUM_TRY, int(self.object_noise), L.ptr(frame), L.ptr(perm) if P else None, rng,
                L.ptr(pts_out) if P else None, L.ptr(point_box) if P else None, L.ptr(boxes_out) if G else None,
                L.ptr(offs_out), L.ptr(cls_out) if G else None, L.ptr(imp_out) if G else None,
                L.ptr(src_out) if G else None, L.ptr(selected) if G else None, L.ptr(ws), ws_bytes, L.ptr(status),
                L.stream()), "b2s_augment")
        self.last_status = status          # device word; nonzero: see spconv._lib.STATUS_BITS
        out = {"points": pts_out, "boxes": boxes_out, "gt_offsets": offs_out, "classes": cls_out,
               "importance": imp_out, "src_row": src_out}
        if with_debug:
            out["selected"] = selected
            out["point_box"] = point_box
        return out

    def augment_frame(self, points, gt_boxes, gt_names, importance=None, rs=None, device=None, with_debug=False):
        """one frame in the reference's terms: host numpy points [N, F] float32, gt_boxes [G, 7 or 9] (float32 or
        float64), gt_names [G] and gt_importance [G] (None: ones) as prep_pointcloud holds them after database sampling.
        DontCare rows are dropped and the class mask comes from the names (preprocess.py:196-211).
        -> (points, gt_dict) as prep_pointcloud holds them at preprocess.py:294 (host arrays): gt_dict has gt_boxes,
        gt_names, gt_importance (box dtype) and gt_classes (int32, 1-based)."""
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        rs = np.random if rs is None else rs
        names = np.asarray(gt_names)
        boxes = np.asarray(gt_boxes)
        if boxes.dtype not in (np.float32, np.float64):
            boxes = boxes.astype(np.float32)
        imp = np.ones(len(names), boxes.dtype) if importance is None else np.asarray(importance)
        keep = names != "DontCare"
        names, boxes, imp = names[keep], np.ascontiguousarray(boxes[keep]), imp[keep]
        valid = np.array([n in self.class_names for n in names], dtype=np.bool_)
        classes = np.array([self.class_names.index(n) + 1 if v else 0 for n, v in zip(names, valid)], np.int32)
        pts = np.ascontiguousarray(points, dtype=np.float32)
        d = draw(rs, self.settings, [len(boxes)], [len(pts)])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)   # noqa: E731
        boxes = boxes.reshape(-1, boxes.shape[-1] if boxes.ndim == 2 else 7)
        out = self.augment_batch(t(pts), t(np.array([0, len(pts)], np.int32)), t(boxes),
                                 t(np.array([0, len(boxes)], np.int32)), t(valid), t(classes),
                                 t(imp.astype(np.float32)), d, with_debug=with_debug)
        n = int(out["gt_offsets"][1].item())
        src = out["src_row"][:n].cpu().numpy()
        gt_dict = {"gt_boxes": out["boxes"][:n].cpu().numpy(), "gt_names": names[src],
                   "gt_importance": imp[src].astype(boxes.dtype), "gt_classes": out["classes"][:n].cpu().numpy()}
        if with_debug:
            gt_dict["selected"] = out["selected"].cpu().numpy()
            gt_dict["point_box"] = out["point_box"].cpu().numpy()
            gt_dict["src_row"] = src
        return out["points"].cpu().numpy(), gt_dict


def plan(settings, point_cloud_range, class_names):
    """-> AugmentPlan.  settings: b2second.config.AugmentSettings (``cfg.augment``)."""
    _check_settings(settings)
    return AugmentPlan(settings, point_cloud_range, class_names)


def _check_settings(settings):
    grot = list(settings.global_random_rotation_range_per_object)
    if len(grot) != 2:
        raise ValueError("global_random_rotation_range_per_object must hold two values, got %r" % (grot,))
    if abs(grot[0] - grot[1]) >= 1e-3:
        raise UnsupportedNetwork("global_random_rotation_range_per_object = %r: per-object global rotation "
                                 "(noise_per_box_v2_) is not supported" % (grot,))
    if settings.use_group_id:
        raise UnsupportedNetwork("use_group_id: group noise (noise_per_box_group) is not supported")
    for key, n in (("groundtruth_localization_noise_std", 3), ("groundtruth_rotation_uniform_noise", 2),
                   ("global_rotation_uniform_noise", 2), ("global_scaling_uniform_noise", 2),
                   ("global_translate_noise_std", 3)):
        if len(getattr(settings, key)) != n and not (key == "global_translate_noise_std" and
                                                     not settings.global_translate_noise_std):
            raise ValueError("%s must hold %d values, got %r" % (key, n, getattr(settings, key)))


def draw_params(settings):
    """-> spconv._lib.AugmentDrawParams: the settings of b2s_augment_draws.  Refuses what ``plan`` refuses, and what
    ``draw``'s numpy calls reject: a negative std (numpy.random.normal) or a bound that is not finite (uniform)."""
    _check_settings(settings)
    s = settings
    tstd = [float(v) for v in s.global_translate_noise_std] or [0.0, 0.0, 0.0]
    std = [float(v) for v in s.groundtruth_localization_noise_std]
    # the translation's z normal uses std[0] (global_translate_), so std[2] only decides whether it happens
    for key, v in (("groundtruth_localization_noise_std", std), ("global_translate_noise_std", tstd[:2]),
                   ("groundtruth_rotation_uniform_noise", s.groundtruth_rotation_uniform_noise),
                   ("global_rotation_uniform_noise", s.global_rotation_uniform_noise),
                   ("global_scaling_uniform_noise", s.global_scaling_uniform_noise)):
        if not all(math.isfinite(float(x)) for x in v):
            raise ValueError("%s must be finite, got %r" % (key, list(v)))
        if key.endswith("_std") and any(x < 0 for x in v):
            raise ValueError("%s must be >= 0, got %r" % (key, list(v)))
    from spconv import _lib as L
    d = lambda v: (ctypes.c_double * len(v))(*[float(x) for x in v])   # noqa: E731
    return L.AugmentDrawParams(d(std), d(s.groundtruth_rotation_uniform_noise), d(s.global_rotation_uniform_noise),
                               d(s.global_scaling_uniform_noise), d(tstd), int(object_noise_enabled(s)),
                               int(bool(s.random_flip_x)), int(bool(s.random_flip_y)))


class DeviceDrawer:
    """the augmentation's random numbers drawn on the device (csrc/augment_draws.cu, b2s_augment_draws): an opt-in
    alternative to ``draw`` whose every value is a function of (seed, step, frame, stream, index) through Philox4x64-10
    (numpy.random.Philox's block function).  INTEGRATION.md states the contract.

    ``step`` is a uint64 counter in device memory: every ``draw`` keys its numbers with it and advances it by one on
    the device, so a CUDA graph that captures ``draw`` (with ``augment_batch``) draws the next step at every replay.
    A checkpoint that saves ``seed`` and ``step`` and restores them resumes the same stream."""

    def __init__(self, seed, device):
        seed = operator.index(seed)
        if not 0 <= seed < 2 ** 64:
            raise ValueError("seed must be in [0, 2**64), got %d" % seed)
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("DeviceDrawer draws on a CUDA device, got %s" % device)
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.seed, self.device = seed, device
        self._step = torch.zeros(1, dtype=torch.int64, device=device)     # the uint64 word's bits

    @property
    def step(self):
        """the step the next ``draw`` uses (reading it waits for the device: meant for checkpoints)"""
        return int(self._step.item()) % 2 ** 64

    @step.setter
    def step(self, value):
        value = operator.index(value)
        if not 0 <= value < 2 ** 64:
            raise ValueError("step must be in [0, 2**64), got %d" % value)
        self._step.fill_(value - 2 ** 64 if value >= 2 ** 63 else value)

    def draw(self, settings, gt_offsets, point_offsets, num_boxes, num_points, frame_base=0):
        """-> Draws of CUDA tensors (num_gt = num_points = None) for the frames frame_base + b, b < B, whose boxes and
        points gt_offsets / point_offsets (CUDA int [B+1]) delimit; num_boxes / num_points: their totals G and P (the
        shapes of loc_noise / rot_noise and perm).  No host sync."""
        params = draw_params(settings)
        L, lib = _lib()
        L.require_cuda(gt_offsets, "gt_offsets")
        L.require_cuda(point_offsets, "point_offsets")
        if gt_offsets.device != self.device or point_offsets.device != self.device:
            raise ValueError("the offsets must be on %s, got %s and %s" % (self.device, gt_offsets.device,
                                                                           point_offsets.device))
        B = int(gt_offsets.shape[0]) - 1
        if gt_offsets.dim() != 1 or point_offsets.shape != gt_offsets.shape or B < 1:
            raise ValueError("gt_offsets and point_offsets must both hold batch + 1 >= 2 entries")
        G, P, frame_base = operator.index(num_boxes), operator.index(num_points), operator.index(frame_base)
        if G < 0 or P < 0 or G >= 2 ** 31 or P >= 2 ** 31:
            raise ValueError("num_boxes and num_points must be in [0, 2**31), got %d and %d" % (G, P))
        if not 0 <= frame_base <= 2 ** 64 - 1 - B:
            raise ValueError("frame_base must be in [0, 2**64 - batch], got %d" % frame_base)
        goff = gt_offsets.to(torch.int32).contiguous()
        poff = point_offsets.to(torch.int32).contiguous()
        dev = self.device
        noise = bool(params.object_noise)
        loc = torch.empty((G, NUM_TRY, 3), dtype=torch.float64, device=dev) if noise else None
        rot = torch.empty((G, NUM_TRY), dtype=torch.float64, device=dev) if noise else None
        frame = torch.empty((B, 8), dtype=torch.float64, device=dev)
        perm = torch.empty(P, dtype=torch.int32, device=dev) if settings.shuffle_points else None
        with torch.cuda.device(dev):
            L.check(lib.b2s_augment_draws(
                self.seed, L.ptr(self._step), frame_base, B, L.ptr(goff), G, L.ptr(poff), P, ctypes.byref(params),
                L.ptr(loc) if (noise and G) else None, L.ptr(rot) if (noise and G) else None, L.ptr(frame),
                L.ptr(perm) if (perm is not None and P) else None, L.stream()), "b2s_augment_draws")
        return Draws(loc_noise=loc, rot_noise=rot, frame=frame, perm=perm, num_gt=None, num_points=None)
