"""Generate tests/golden/augment/*.npz FROM THE UNMODIFIED REFERENCE (needs the reference tree; runs on the CPU).

    python tests/golden/make_augment_golden.py

For each config, each synthetic frame (tests/augment_ref.frame: no GT, one GT, a crowded block where tries collide and
some boxes find no free try, overlapping and nested GTs, 210 GTs, GTs near the range's edges; names outside the class
list act as obstacles and drop) runs, under np.random.seed(seed), the reference's own noise_per_object_v3_ (num_try
100), the class-mask selection, random_flip, global_rotation_v2, global_scaling_v2, global_translate_,
filter_gt_box_outside_range_by_center, limit_period and np.random.shuffle, with the config's train preprocess settings,
in prep_pointcloud's order (second/data/preprocess.py:255-294).  The shuffle runs on the points with their row index
appended as a column, which consumes the stream exactly as shuffling the points does and records the order.

Recorded per frame f: seed_f, kind_f, the outputs (points_f, boxes_f, classes_f, importance_f, src_row_f), the selected
try of each box (selected_f, from the reference's own noise_per_box on the same draws, checked against the boxes it
moved), the box that moved each output point (point_box_f, from the reference's own points_in_convex_polygon_3d_jit on
the center_to_corner_box3d surfaces), and state_f, a sha1 of np.random's state after the last step.

Seeds are rejected while any decision lies near a tie, so that a last-bit difference in the corner arithmetic (BLAS,
libm) cannot flip it: a point within 2e-4 m of a valid box's surface; a tried pose whose separating-axis gap (or
penetration) to another box is below 1e-4 m, unless the pose overlaps some other box by more than that; a kept or dropped box centre within 1e-4 of the range edge; a yaw within
1e-6 of limit_period's wrap.

Adaptation: points_in_convex_polygon_jit (second/core/geometry.py:273) is a ``numba.jit`` that only compiled in numba's
object mode, which current numba has removed; filter_gt_box_outside_range_by_center runs its ``.py_func`` instead
(the same Python code, uncompiled).  noise_per_object_v3_ compiles on first use (about half a minute).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))
OUT = os.path.join(HERE, "augment")

from b2second import augment, config, loader, refcompat  # noqa: E402

import augment_ref as ar  # noqa: E402

refcompat.install(loader.ORACLE_DIR)
from second.core import box_np_ops  # noqa: E402
from second.core import geometry  # noqa: E402
from second.core import preprocess as prep  # noqa: E402

prep.points_in_convex_polygon_jit = geometry.points_in_convex_polygon_jit.py_func

BASE_SEED = {"car.fhd": 1000, "all.fhd": 2000, "pointpillars.car.xyres_16": 3000, "nuscenes.all.pp.largea": 4000,
             "nuscenes.all.pp.mhead": 5000}
POINT_EPS, POSE_EPS, RANGE_EPS = 2e-4, 1e-4, 1e-4


def local_margin(points, boxes):
    """[N, G]: min over axes of (half extent - |local coordinate|) of each point in each box (origin 0.5 boxes)"""
    b = boxes.astype(np.float64)
    p = points[:, :3].astype(np.float64)
    dx = p[:, None, 0] - b[None, :, 0]
    dy = p[:, None, 1] - b[None, :, 1]
    dz = p[:, None, 2] - b[None, :, 2]
    c, s = np.cos(b[:, 6]), np.sin(b[:, 6])
    lx = dx * c - dy * s
    ly = dx * s + dy * c
    return np.minimum(np.minimum(b[:, 3] / 2 - np.abs(lx), b[:, 4] / 2 - np.abs(ly)), b[:, 5] / 2 - np.abs(dz))


def corners64(x, y, w, l, r):
    nx = np.array([-0.5, -0.5, 0.5, 0.5])
    ny = np.array([-0.5, 0.5, 0.5, -0.5])
    px, py = w[..., None] * nx, l[..., None] * ny
    c, s = np.cos(r)[..., None], np.sin(r)[..., None]
    return np.stack([px * c + py * s + x[..., None], -px * s + py * c + y[..., None]], -1)


def sat_gap(a, b):
    """largest separating-axis gap between convex quads a [..., 4, 2] and b [..., 4, 2] (negative: penetration)"""
    gap = np.full(np.broadcast_shapes(a.shape[:-2], b.shape[:-2]), -np.inf)
    for q in (a, b):
        for k in range(4):
            e = q[..., (k + 1) % 4, :] - q[..., k, :]
            n = np.stack([-e[..., 1], e[..., 0]], -1)
            n = n / np.linalg.norm(n, axis=-1, keepdims=True)
            pa = (a * n[..., None, :]).sum(-1)
            pb = (b * n[..., None, :]).sum(-1)
            g = np.maximum(pb.min(-1) - pa.max(-1), pa.min(-1) - pb.max(-1))
            gap = np.maximum(gap, g)
    return gap


def pose_ties(boxes, valid, loc, rot, sel):
    """True when a tried pose's collision decision lies within POSE_EPS of a tie (float64 replay of noise_per_box)"""
    b = boxes.astype(np.float64)
    cur = corners64(b[:, 0], b[:, 1], b[:, 3], b[:, 4], b[:, 6])
    n = len(b)
    for i in range(n):
        if not valid[i]:
            continue
        last = sel[i] if sel[i] >= 0 else loc.shape[1] - 1
        js = np.arange(last + 1)
        tc = corners64(b[i, 0] + loc[i, js, 0], b[i, 1] + loc[i, js, 1], np.full(len(js), b[i, 3]),
                       np.full(len(js), b[i, 4]), b[i, 6] + rot[i, js])
        others = np.array([k for k in range(n) if k != i], np.int64)
        if len(others):
            g = sat_gap(tc[:, None], cur[None, others])
            # a try that overlaps some box by more than POSE_EPS is rejected whatever its other pairs decide
            if ((np.abs(g) < POSE_EPS).any(1) & ~(g < -POSE_EPS).any(1)).any():
                return True
            free = (g > 0).all(1)
        else:
            free = np.ones(len(js), bool)
        want = np.zeros(len(js), bool)
        if sel[i] >= 0:
            want[-1] = True
        if not np.array_equal(free, want):
            raise AssertionError("float64 replay disagrees with the reference's selection at box %d" % i)
        if sel[i] >= 0:
            cur[i] = tc[-1]
    return False


def run_reference(name, kind, seed):
    cfg = config.get_config(name)
    s = cfg.augment
    classes = ar.class_names(name)
    points, boxes, names = ar.frame(name, kind, seed)
    keep = names != "DontCare"
    points, boxes, names = points.copy(), boxes[keep].copy(), names[keep]
    valid, _ = ar.class_mask(name, names)
    G = len(boxes)
    ties = []
    np.random.seed(seed)
    orig = boxes.copy()
    sel = np.full(G, -1, np.int32)
    point_box = np.full(len(points), -1, np.int32)
    if augment.object_noise_enabled(s):
        st0 = np.random.get_state()
        prep.noise_per_object_v3_(boxes, points, valid, rotation_perturb=list(s.groundtruth_rotation_uniform_noise),
                                  center_noise_std=list(s.groundtruth_localization_noise_std),
                                  global_random_rot_range=list(s.global_random_rotation_range_per_object),
                                  group_ids=None, num_try=augment.NUM_TRY)
        st1 = np.random.get_state()
        # the same draws again, for the reference's own noise_per_box and the tie checks
        np.random.set_state(st0)
        loc = np.random.normal(scale=np.array(s.groundtruth_localization_noise_std, dtype=orig.dtype),
                               size=[G, augment.NUM_TRY, 3])
        rot = np.random.uniform(*s.groundtruth_rotation_uniform_noise, size=[G, augment.NUM_TRY])
        np.random.set_state(st1)
        sel = prep.noise_per_box(orig[:, [0, 1, 3, 4, 6]], valid, loc, rot).astype(np.int32)
        for i in range(G):
            if valid[i]:
                lt = loc[i, sel[i]] if sel[i] >= 0 else np.zeros(3)
                want = (orig[i, :3].astype(np.float64) + lt).astype(orig.dtype)
                assert np.array_equal(boxes[i, :3], want), "selection does not explain box %d" % i
        if G:
            corners = box_np_ops.center_to_corner_box3d(orig[:, :3], orig[:, 3:6], orig[:, 6], origin=[0.5, 0.5, 0.5],
                                                        axis=2)
            mask = geometry.points_in_convex_polygon_3d_jit(ar.frame(name, kind, seed)[0][:, :3],
                                                            box_np_ops.corner_to_surfaces_3d_jit(corners))
            mask &= valid[None, :]
            point_box = np.where(mask.any(1), mask.argmax(1), -1).astype(np.int32)
            margin = local_margin(ar.frame(name, kind, seed)[0], orig)[:, valid]
            if (np.abs(margin) < POINT_EPS).any():
                ties.append("point")
            if pose_ties(orig, valid, loc, rot, sel):
                ties.append("pose")
    imp = np.ones(G, boxes.dtype)
    idx = np.arange(G, dtype=np.int32)
    boxes, names, imp, idx = boxes[valid], names[valid], imp[valid], idx[valid]
    cls = np.array([classes.index(n) + 1 for n in names], np.int32)
    boxes, points = prep.random_flip(boxes, points, 0.5, s.random_flip_x, s.random_flip_y)
    boxes, points = prep.global_rotation_v2(boxes, points, *s.global_rotation_uniform_noise)
    boxes, points = prep.global_scaling_v2(boxes, points, *s.global_scaling_uniform_noise)
    prep.global_translate_(boxes, points, list(s.global_translate_noise_std))
    bv = np.asarray(cfg.point_cloud_range, np.float32)[[0, 1, 3, 4]]
    m = prep.filter_gt_box_outside_range_by_center(boxes, bv)
    edge = np.minimum(np.minimum(np.abs(boxes[:, 0] - bv[0]), np.abs(boxes[:, 0] - bv[2])),
                      np.minimum(np.abs(boxes[:, 1] - bv[1]), np.abs(boxes[:, 1] - bv[3])))
    if (edge < RANGE_EPS).any():
        ties.append("range")
    boxes, cls, imp, idx = boxes[m], cls[m], imp[m], idx[m]
    w = boxes[:, 6].astype(np.float64) / (2 * np.pi) + 0.5
    if (np.abs(w - np.round(w)) < 1e-6).any():
        ties.append("period")
    boxes[:, 6] = box_np_ops.limit_period(boxes[:, 6], offset=0.5, period=2 * np.pi)
    order = np.arange(len(points))
    if s.shuffle_points:
        tagged = np.concatenate([points, np.arange(len(points), dtype=np.float32)[:, None]], 1)
        np.random.shuffle(tagged)
        points = np.ascontiguousarray(tagged[:, :-1])
        order = tagged[:, -1].astype(np.int64)
    state = ar.state_digest(np.random)
    out = {"points": points, "point_box": point_box[order], "selected": sel, "boxes": boxes, "classes": cls,
           "importance": imp.astype(np.float32), "src_row": idx, "state": np.array(state)}
    return out, ties


def main():
    os.makedirs(OUT, exist_ok=True)
    for name in ar.CONFIGS:
        z = {}
        for f, kind in enumerate(ar.KINDS):
            for attempt in range(400):
                seed = BASE_SEED[name] + 10000 * f + attempt
                out, ties = run_reference(name, kind, seed)
                if not ties:
                    break
            else:
                raise RuntimeError("%s %s: no tie-free seed" % (name, kind))
            for k, v in out.items():
                z["%s_%d" % (k, f)] = v
            z["seed_%d" % f] = np.int64(seed)
            z["kind_%d" % f] = np.array(kind)
            print("%s %-8s seed %d: %d boxes kept, sel %s, %d points moved" % (
                name, kind, seed, len(out["boxes"]), np.unique(out["selected"]).tolist()[:6],
                int((out["point_box"] >= 0).sum())), flush=True)
        z["num_frames"] = np.int64(len(ar.KINDS))
        np.savez_compressed(ar.fixture_path(name), **z)


if __name__ == "__main__":
    main()
