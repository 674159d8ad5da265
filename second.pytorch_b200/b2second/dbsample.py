"""Ground-truth database sampling on the GPU: what prep_pointcloud (second/data/preprocess.py:210-249) does with
DataBaseSamplerV2 (second/core/sample_ops.py:14-285) before the augmentation, for a whole batch, in csrc/dbsample.cu.

    db = dbsample.load(cfg.db_sampler, db_infos, root_path, cfg.num_point_features, class_names, device)   # once
    ds = dbsample.DatabaseSampler(db, cfg.db_sampler, class_names, rs)                                      # once
    cand = dbsample.draw(rs, ds.state, gt_names_per_frame)                       # host, per batch, no device work
    res = ds.sample_batch(points, point_offsets, gt_boxes, gt_offsets, gt_valid, gt_classes, importance, cand)
    num_boxes, num_points = res.counts()                                         # the one device-to-host read
    d = augment.draw(rs, cfg.augment, num_boxes, num_points)
    out = augment_plan.augment_batch(*res.augment_inputs(num_boxes, num_points), d)

``load`` applies the database prep steps on the host in the reference's order and reads every remaining object of a
sampled class once; the points, boxes and classes stay on the device.  ``draw`` restates prep.BatchSampler
(second/core/preprocess.py:17-55) as index bookkeeping on a caller-given RandomState: one sampler per key of db_infos,
shuffled at construction in the dict's order; a sampler asked for ``num`` at ``idx`` with ``idx + num >= N`` returns
only the remainder and reshuffles; ``sampled_num = round_half_even(rate * (max_num - count(gt_names == class)))`` and a
class is skipped when that is <= 0.  The kernel then rejects colliding candidates (the rule is stated in
csrc/dbsample.cu), drops the frame points inside accepted boxes when ``remove_points_after_sample`` is set and
concatenates, in ``augment_batch``'s input layout.

Stream order.  The reference interleaves, frame after frame, the sampler's shuffles and the augmentation's draws on
np.random.  The batch path makes every frame's sampler draws first and then ``augment.draw``.  A sampler only touches
the stream when it reshuffles, so the two orders give the same numbers unless a sampler wraps at a frame after the
first of the batch; then the reshuffle comes before the earlier frames' augmentation draws instead of after them.
``sample_frame`` followed by ``AugmentPlan.augment_frame`` on the same state is the reference's order exactly.

``SampleResult.counts()`` is the pipeline's only sync: ``augment.draw`` needs each frame's box and point counts.

Refused (spec.UnsupportedNetwork), as no config uses them: group sampling (a sample group of more than one name), a
per-object global rotation range of 1e-3 or more (rot_transform), ``random_crop``, a sampled class outside
class_names.
"""
import os
import pickle
from dataclasses import dataclass
from typing import List

import numpy as np
import torch

from .config import DatabaseSamplerSettings  # noqa: F401  (re-exported: the settings type lives with the config parser)
from .spec import UnsupportedNetwork

MAX_BOXES = 1024                  # B2S_DBSAMPLE_MAX_BOXES: per-frame cap on ground truths plus candidates


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


# ------------------------------------------------------------------------------------------------ database
def prep_infos(settings, db_infos):
    """DataBasePreprocessor of settings.database_prep_steps (second/core/preprocess.py:58-105) on a copy of db_infos:
    DBFilterByMinNumPoint keeps ``num_points_in_gt >= min_num`` where min_num > 0, DBFilterByDifficulty drops the listed
    difficulties; in file order.  -> dict of the same keys, in the same order."""
    out = {k: list(v) for k, v in db_infos.items()}
    for kind, arg in settings.database_prep_steps:
        if kind == "filter_by_min_num_points":
            for name, min_num in arg:
                if min_num > 0:
                    out[name] = [i for i in out[name] if i["num_points_in_gt"] >= min_num]
        elif kind == "filter_by_difficulty":
            out = {k: [i for i in v if i["difficulty"] not in arg] for k, v in out.items()}
        else:
            raise ValueError("unknown database prep step %r" % (kind,))
    return out


def sampled_classes(settings):
    """[(name, max_num)] in sample-group order"""
    return [(n, int(m)) for g in settings.sample_groups for n, m in g.items()]


@dataclass
class Database:
    """the filtered database (``load``).  keys / counts: every key of db_infos in the dict's order and its number of
    infos after the prep steps (each gets a sampler); objects[key]: the global object ids of a sampled class's infos,
    in info order.  Per object on the device: points [NP, F] float32 relative to the box centre, point_offsets int64
    [N+1], boxes [N, ndim] (the infos' dtype), classes int32 (class_names.index + 1), difficulty int32; host copies
    of the offsets, boxes, difficulty and the names and paths."""
    keys: List[str]
    counts: dict
    objects: dict
    points: torch.Tensor
    point_offsets: torch.Tensor
    boxes: torch.Tensor
    classes: torch.Tensor
    difficulty: torch.Tensor
    point_offsets_host: np.ndarray
    boxes_host: np.ndarray
    difficulty_host: np.ndarray
    names: np.ndarray
    paths: List[str]

    @property
    def num_objects(self):
        return int(self.boxes_host.shape[0])

    @property
    def nbytes(self):
        """device bytes held"""
        return sum(t.numel() * t.element_size() for t in (self.points, self.point_offsets, self.boxes, self.classes,
                                                           self.difficulty))


def load(settings, db_infos, root_path, num_point_features, class_names, device=None):
    """-> Database.  db_infos: the database pickle's dict ({name: [info]}), or its path.  Reads each remaining object
    of a sampled class once from ``root_path / info["path"]`` (float32 [n, num_point_features]); the infos of classes
    that are never sampled are only counted."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if isinstance(db_infos, (str, os.PathLike)):
        with open(db_infos, "rb") as f:
            db_infos = pickle.load(f)
    _check_settings(settings, class_names)
    infos = prep_infos(settings, db_infos)
    sampled = [n for n, _ in sampled_classes(settings)]
    for n in sampled:
        if n not in infos:
            raise KeyError("sampled class %r has no database infos (have %s)" % (n, list(infos)))
    objects, pts, offs, boxes, cls, diff, names, paths = {}, [], [0], [], [], [], [], []
    for key, lst in infos.items():
        if key not in sampled:
            continue
        objects[key] = np.arange(len(boxes), len(boxes) + len(lst), dtype=np.int64)
        for info in lst:
            p = np.fromfile(os.path.join(str(root_path), info["path"]), dtype=np.float32)
            p = p.reshape([-1, num_point_features])
            pts.append(p)
            offs.append(offs[-1] + len(p))
            boxes.append(np.asarray(info["box3d_lidar"]))
            cls.append(class_names.index(key) + 1)
            diff.append(int(info["difficulty"]))
            names.append(info["name"])
            paths.append(info["path"])
    if boxes:
        boxes_host = np.ascontiguousarray(np.stack(boxes))
    else:
        boxes_host = np.zeros((0, 7), np.float32)
    if boxes_host.dtype not in (np.float32, np.float64):
        boxes_host = boxes_host.astype(np.float32)
    pts_host = np.concatenate(pts) if pts else np.zeros((0, num_point_features), np.float32)
    offs_host = np.asarray(offs, np.int64)
    diff_host = np.asarray(diff, np.int32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)   # noqa: E731
    return Database(keys=list(infos), counts={k: len(v) for k, v in infos.items()}, objects=objects,
                    points=t(pts_host), point_offsets=t(offs_host), boxes=t(boxes_host),
                    classes=t(np.asarray(cls, np.int32)), difficulty=t(diff_host), point_offsets_host=offs_host,
                    boxes_host=boxes_host, difficulty_host=diff_host, names=np.asarray(names), paths=paths)


# ------------------------------------------------------------------------------------------------ host draws
class SamplerState:
    """prep.BatchSampler's bookkeeping for every key of the database (indices, idx), the sample groups and the rate"""

    def __init__(self, rs, db, settings):
        rs = np.random if rs is None else rs
        self.groups = sampled_classes(settings)
        self.rate = settings.rate
        self.objects = db.objects
        self.indices, self.idx = {}, {}
        for key in db.keys:                   # sample_ops.py:78-80: every key, in the dict's order
            ind = np.arange(db.counts[key])
            rs.shuffle(ind)
            self.indices[key] = ind
            self.idx[key] = 0

    def sample(self, rs, key, num):
        """BatchSampler._sample: info indices of ``key``"""
        ind, i, n = self.indices[key], self.idx[key], len(self.indices[key])
        if i + num >= n:
            ret = ind[i:].copy()
            rs.shuffle(ind)                   # _reset
            self.idx[key] = 0
        else:
            ret = ind[i:i + num]
            self.idx[key] = i + num
        return ret


def sample_counts(state, gt_names):
    """sample_all's sampled_num per class of ``state.groups`` (sample_ops.py:103-111)"""
    names = list(gt_names)
    out = []
    for name, max_num in state.groups:
        n = int(max_num - np.sum([x == name for x in names]))
        out.append(int(np.round(state.rate * n).astype(np.int64)))
    return out


@dataclass
class Candidates:
    """the candidates of one batch (host arrays): objects int32 [C] global object ids, group int32 [C] the sample
    group of each, offsets int32 [B+1]; per frame, class by class in sample-group order."""
    objects: np.ndarray
    group: np.ndarray
    offsets: np.ndarray


def draw(rs, state, gt_names_per_frame):
    """the candidates sample_all draws for each frame, frame after frame, consuming ``rs`` (np.random.RandomState or
    the np.random module) as the reference's samplers consume np.random."""
    rs = np.random if rs is None else rs
    objs, grp, offs = [], [], [0]
    for names in gt_names_per_frame:
        for g, ((name, _), num) in enumerate(zip(state.groups, sample_counts(state, names))):
            if num > 0:
                idx = state.sample(rs, name, num)
                objs.append(state.objects[name][idx])
                grp.append(np.full(len(idx), g, np.int32))
        offs.append(sum(len(o) for o in objs))
    return Candidates(objects=np.concatenate(objs).astype(np.int32) if objs else np.zeros(0, np.int32),
                      group=np.concatenate(grp).astype(np.int32) if grp else np.zeros(0, np.int32),
                      offsets=np.asarray(offs, np.int32))


def select(candidates, start, stop):
    """-> the Candidates of frames ``start .. stop - 1``: a data-parallel rank's share of candidates drawn for the whole
    batch in single-process order, so the sampling does not depend on the number of ranks."""
    o = candidates.offsets
    return Candidates(objects=candidates.objects[o[start]:o[stop]], group=candidates.group[o[start]:o[stop]],
                      offsets=(o[start:stop + 1] - o[start]).astype(np.int32))


# ------------------------------------------------------------------------------------------------ device
class SampleResult(dict):
    """device outputs of ``sample_batch``: points float32 [P + CP, F], point_offsets int32 [B+1], boxes [G + C, ndim],
    gt_offsets int32 [B+1], gt_valid bool, classes int32, importance float32, src_object int32 [G + C] (-1: the
    frame's own row), accepted bool [C], status int32 [1]; rows past the offsets' last entry are zeros."""

    def counts(self):
        """-> (boxes per frame, points per frame) as lists: the one device-to-host read of the pipeline (it waits for
        the sampling kernels)"""
        both = torch.stack([self["gt_offsets"], self["point_offsets"]]).cpu().numpy()
        return np.diff(both[0]).tolist(), np.diff(both[1]).tolist()

    def augment_inputs(self, num_boxes, num_points):
        """the positional inputs of AugmentPlan.augment_batch (before the draws), trimmed to the counts"""
        g, p = int(sum(num_boxes)), int(sum(num_points))
        return (self["points"][:p], self["point_offsets"], self["boxes"][:g], self["gt_offsets"],
                self["gt_valid"][:g], self["classes"][:g], self["importance"][:g])


def pack_candidates(candidates, db):
    """-> (int32 host array, C, CP): the candidate arrays of one batch as ``sample_batch`` copies them to the device in
    one transfer (objects [C], group [C], offsets [B+1], the prefix of their point counts [C+1]), with the candidate
    count C and their point total CP.  A caller that replays a captured ``sample_batch`` refills its staging buffer
    with this."""
    obj = np.ascontiguousarray(candidates.objects, np.int32)
    C = len(obj)
    npts = np.diff(db.point_offsets_host)[obj] if C else np.zeros(0, np.int64)
    cpo = np.concatenate([[0], np.cumsum(npts)]).astype(np.int64)
    CP = int(cpo[-1])
    if CP >= 2 ** 31:
        raise ValueError("the candidates' points must fit in int32")
    host = np.concatenate([obj, np.asarray(candidates.group, np.int32), np.asarray(candidates.offsets, np.int32),
                           cpo.astype(np.int32)])
    return host, C, CP


def _check_settings(settings, class_names):
    groups = settings.sample_groups
    if any(len(g) > 1 for g in groups):
        raise UnsupportedNetwork("group sampling (a sample group of more than one name) is not supported")
    grot = list(settings.global_random_rotation_range_per_object)
    if len(grot) not in (0, 2):
        raise ValueError("global_random_rotation_range_per_object must hold two values, got %r" % (grot,))
    if grot and abs(grot[0] - grot[1]) >= 1e-3:
        raise UnsupportedNetwork("global_random_rotation_range_per_object = %r: per-object rotation of samples "
                                 "(rot_transform) is not supported" % (grot,))
    for name, _ in sampled_classes(settings):
        if name not in class_names:
            raise UnsupportedNetwork("sampled class %r is not in class_names %r" % (name, list(class_names)))


class DatabaseSampler:
    """DataBaseSamplerV2 on a device-resident Database.  The samplers are built (and shuffled) at construction from
    ``rs`` (None: np.random), as the reference builds them from np.random."""

    def __init__(self, db, settings, class_names, rs=None):
        _check_settings(settings, class_names)
        self.db = db
        self.settings = settings
        self.class_names = list(class_names)
        self.state = SamplerState(rs, db, settings)

    def sample_batch(self, points, point_offsets, gt_boxes, gt_offsets, gt_valid, gt_classes, importance, candidates,
                     staging=None):
        """sample a batch without a host sync.  points CUDA float32 [P, F] packed frame after frame, point_offsets
        CUDA int32 [B+1]; gt_boxes CUDA [G, 7 or 9] in the database's box dtype, gt_offsets CUDA int32 [B+1]; gt_valid
        CUDA bool [G] (the class mask); gt_classes CUDA int [G]; importance CUDA float [G] or None (ones);
        candidates: ``draw``'s result for these frames.  -> SampleResult.

        The candidate arrays (``pack_candidates``) go to the device in one copy from pinned host memory.  staging: a
        pinned int32 CPU tensor the caller owns (at least as long as the packed array) to copy from; without it a
        temporary pinned buffer is used.  Under CUDA-graph capture staging is required: the captured copy reads it at
        every replay, so the caller keeps it alive and refills it with ``pack_candidates`` of the next candidates, which
        must keep the captured candidate count, point total and batch size (they set the output shapes and grids)."""
        L, lib = _lib()
        db = self.db
        for name, v in (("points", points), ("point_offsets", point_offsets), ("gt_boxes", gt_boxes),
                        ("gt_offsets", gt_offsets), ("gt_valid", gt_valid), ("gt_classes", gt_classes),
                        ("importance", importance)):
            if v is not None:
                L.require_cuda(v, name)
        device = points.device
        if gt_boxes.dtype != db.boxes.dtype:
            raise TypeError("gt_boxes are %s, the database's boxes %s" % (gt_boxes.dtype, db.boxes.dtype))
        if gt_boxes.dim() != 2 or gt_boxes.shape[1] not in (7, 9) or (db.num_objects and
                                                                      gt_boxes.shape[1] != db.boxes.shape[1]):
            raise ValueError("gt_boxes must be [G, 7] or [G, 9] like the database's, got %s" % (tuple(gt_boxes.shape),))
        if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] < 3:
            raise ValueError("points must be float32 [P, >= 3]")
        P, F = int(points.shape[0]), int(points.shape[1])
        if db.num_objects and int(db.points.shape[1]) != F:
            raise ValueError("points have %d features, the database's %d" % (F, int(db.points.shape[1])))
        B = int(point_offsets.shape[0]) - 1
        if B < 1 or int(gt_offsets.shape[0]) != B + 1:
            raise ValueError("point_offsets and gt_offsets must both hold batch + 1 >= 2 entries")
        if len(candidates.offsets) != B + 1:
            raise ValueError("candidates were drawn for %d frames, the batch has %d" % (len(candidates.offsets) - 1, B))
        G, ndim = int(gt_boxes.shape[0]), int(gt_boxes.shape[1])
        host, C, CP = pack_candidates(candidates, db)
        if P + CP >= 2 ** 31 or G + C >= 2 ** 31:
            raise ValueError("the batch's output rows must fit in int32")
        if staging is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("capturing sample_batch in a CUDA graph needs a caller-owned pinned staging buffer")
            cand = torch.from_numpy(host).pin_memory().to(device, non_blocking=True)
        else:
            if staging.device.type != "cpu" or staging.dtype != torch.int32 or not staging.is_pinned() or \
                    staging.numel() < len(host):
                raise ValueError("staging must be a pinned int32 CPU tensor of at least %d elements" % len(host))
            src = staging.view(-1)[:len(host)]
            src.copy_(torch.from_numpy(host))
            cand = src.to(device, non_blocking=True)
        c_obj, c_grp = cand[:C], cand[C:2 * C]
        c_off, c_pto = cand[2 * C:2 * C + B + 1], cand[2 * C + B + 1:]
        points = points.contiguous()
        gt_boxes = gt_boxes.contiguous()
        poff = point_offsets.to(torch.int32).contiguous()
        goff = gt_offsets.to(torch.int32).contiguous()
        valid = gt_valid.to(torch.uint8).contiguous()
        cls = gt_classes.to(torch.int32).contiguous()
        imp = importance.to(torch.float32).contiguous() if importance is not None else None
        pts_out = torch.empty(P + CP, F, dtype=torch.float32, device=device)
        poff_out = torch.empty(B + 1, dtype=torch.int32, device=device)
        boxes_out = torch.empty(G + C, ndim, dtype=gt_boxes.dtype, device=device)
        goff_out = torch.empty(B + 1, dtype=torch.int32, device=device)
        valid_out = torch.empty(G + C, dtype=torch.bool, device=device)
        cls_out = torch.empty(G + C, dtype=torch.int32, device=device)
        imp_out = torch.empty(G + C, dtype=torch.float32, device=device)
        src_out = torch.empty(G + C, dtype=torch.int32, device=device)
        accepted = torch.empty(C, dtype=torch.bool, device=device)
        status = torch.zeros(1, dtype=torch.int32, device=device)
        ws_bytes = lib.b2s_db_sample_workspace_bytes(B, P, C)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        s = self.settings
        with torch.cuda.device(device):
            L.check(lib.b2s_db_sample(
                L.ptr(points) if P else None, P, F, L.ptr(poff), B, L.ptr(gt_boxes) if G else None,
                int(gt_boxes.dtype == torch.float64), ndim, G, L.ptr(goff), L.ptr(valid) if G else None,
                L.ptr(cls) if G else None, L.ptr(imp) if (G and imp is not None) else None,
                L.ptr(c_obj) if C else None, L.ptr(c_grp) if C else None, L.ptr(c_off), L.ptr(c_pto), C, CP,
                L.ptr(db.points) if db.points.numel() else None, L.ptr(db.point_offsets), L.ptr(db.boxes),
                L.ptr(db.classes), db.num_objects, float(s.sample_importance), int(bool(s.remove_points_after_sample)),
                L.ptr(pts_out) if P + CP else None, L.ptr(poff_out), L.ptr(boxes_out) if G + C else None,
                L.ptr(goff_out), L.ptr(valid_out) if G + C else None, L.ptr(cls_out) if G + C else None,
                L.ptr(imp_out) if G + C else None, L.ptr(src_out) if G + C else None, L.ptr(accepted) if C else None,
                L.ptr(ws), ws_bytes, L.ptr(status), L.stream()), "b2s_db_sample")
        self.last_status = status          # device word; nonzero: see spconv._lib.STATUS_BITS
        return SampleResult(points=pts_out, point_offsets=poff_out, boxes=boxes_out, gt_offsets=goff_out,
                            gt_valid=valid_out, classes=cls_out, importance=imp_out, src_object=src_out,
                            accepted=accepted, status=status)

    def _one_frame(self, points, boxes, names, importance, rs):
        """one frame through draw and sample_batch; -> (SampleResult, candidates)"""
        device = self.db.boxes.device
        valid = np.array([n in self.class_names for n in names], dtype=np.bool_)
        classes = np.array([self.class_names.index(n) + 1 if v else 0 for n, v in zip(names, valid)], np.int32)
        cand = draw(rs, self.state, [names])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)   # noqa: E731
        imp = np.ones(len(boxes), np.float32) if importance is None else np.asarray(importance, np.float32)
        res = self.sample_batch(t(points), t(np.array([0, len(points)], np.int32)), t(boxes),
                                t(np.array([0, len(boxes)], np.int32)), t(valid), t(classes), t(imp), cand)
        return res, cand

    def _boxes(self, gt_boxes):
        ndim = int(self.db.boxes.shape[1]) if self.db.num_objects else 7
        boxes = np.asarray(gt_boxes).reshape(-1, ndim)
        if boxes.dtype != self.db.boxes_host.dtype:
            raise TypeError("gt_boxes are %s, the database's boxes %s" % (boxes.dtype, self.db.boxes_host.dtype))
        return np.ascontiguousarray(boxes)

    def sample_all(self, root_path, gt_boxes, gt_names, num_point_features, random_crop=False, gt_group_ids=None,
                   calib=None, rs=None):
        """DataBaseSamplerV2.sample_all's signature and result: {"gt_names", "difficulty", "gt_boxes", "points",
        "gt_masks", "group_ids"} of the accepted samples, or None.  Reads from the device database (root_path is not
        used); ``rs`` (None: np.random) drives the samplers."""
        if random_crop:
            raise UnsupportedNetwork("random_crop (a frustum crop of the sampled points) is not supported")
        rs = np.random if rs is None else rs
        boxes = self._boxes(gt_boxes)
        F = int(num_point_features)
        res, cand = self._one_frame(np.zeros((0, F), np.float32), boxes, list(gt_names), None, rs)
        n_g, n_p = res.counts()
        G = len(boxes)
        if n_g[0] == G:
            return None
        src = res["src_object"][G:n_g[0]].cpu().numpy()
        return {"gt_names": self.db.names[src], "difficulty": self.db.difficulty_host[src],
                "gt_boxes": res["boxes"][G:n_g[0]].cpu().numpy(), "points": res["points"][:n_p[0]].cpu().numpy(),
                "gt_masks": np.ones(len(src), dtype=np.bool_), "group_ids": np.arange(G, G + len(src))}

    def sample_frame(self, points, gt_dict, rs=None, with_debug=False):
        """one frame in the reference's terms: host points [N, F] float32 and gt_dict (gt_boxes, gt_names and
        optionally gt_importance and further keys) as prep_pointcloud holds them before sampling; DontCare rows are
        dropped first, from every per-box array of the dict (preprocess.py:191).  -> (points, gt_dict) as at
        preprocess.py:249: gt_boxes, gt_names and gt_importance (box dtype) with the samples appended, gt_boxes_mask,
        group_ids (when given) extended by the samples' ids, every other key carried over as the reference leaves it.
        with_debug adds "accepted", "candidates" and "src_object"."""
        rs = np.random if rs is None else rs
        names = np.asarray(gt_dict["gt_names"])
        boxes = self._boxes(gt_dict["gt_boxes"])
        imp = gt_dict.get("gt_importance")
        imp = np.ones(len(names), boxes.dtype) if imp is None else np.asarray(imp)
        keep = names != "DontCare"
        n_in = len(names)
        names, boxes, imp = names[keep], np.ascontiguousarray(boxes[keep]), imp[keep]
        rest = {k: (v[keep] if isinstance(v, np.ndarray) and v.ndim >= 1 and len(v) == n_in else v)
                for k, v in gt_dict.items() if k not in ("gt_boxes", "gt_names", "gt_importance")}
        res, cand = self._one_frame(np.ascontiguousarray(points, dtype=np.float32), boxes, names, imp, rs)
        n_g, n_p = res.counts()
        G = len(boxes)
        src = res["src_object"][G:n_g[0]].cpu().numpy()
        out = dict(rest)
        if "group_ids" in rest:                   # preprocess.py:239-242, sample_all's ids (sample_ops.py:212-213)
            out["group_ids"] = np.concatenate([rest["group_ids"], np.arange(G, G + len(src))])
        out.update({"gt_boxes": res["boxes"][:n_g[0]].cpu().numpy(),
               "gt_names": np.concatenate([names, self.db.names[src]]) if len(src) else names,
               "gt_importance": np.concatenate([imp, np.full(len(src), self.settings.sample_importance,
                                                             boxes.dtype)]).astype(boxes.dtype),
               "gt_boxes_mask": res["gt_valid"][:n_g[0]].cpu().numpy()})
        if with_debug:
            out["accepted"] = res["accepted"].cpu().numpy()
            out["candidates"] = cand.objects
            out["src_object"] = res["src_object"][:n_g[0]].cpu().numpy()
        return res["points"][:n_p[0]].cpu().numpy(), out


def sampler(settings, db_infos, root_path, num_point_features, class_names, device=None, rs=None):
    """load + DatabaseSampler, as dbsampler_builder.build does it"""
    db = load(settings, db_infos, root_path, num_point_features, class_names, device)
    return DatabaseSampler(db, settings, class_names, rs)

