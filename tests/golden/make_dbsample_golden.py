"""Generate tests/golden/dbsample/*.npz FROM THE UNMODIFIED REFERENCE (needs the reference tree; runs on the CPU).

    python tests/golden/make_dbsample_golden.py

For each config a synthetic object database is written to a temporary directory: one ``.bin`` file per object (float32
points relative to the box centre, as create_groundtruth_database writes them) and a db_infos dict with a key for
every class of the config plus one key that is never sampled (``Misc``, first, so its sampler is built and shuffled
before the others), with difficulties and ``num_points_in_gt`` that both prep filters act on.  Half of each sampled
class's boxes sit in a small cluster, so candidates of one frame collide with each other (sample_class_v2's "later
candidate" rule) and with the frame points there.

The reference's own DataBaseSamplerV2 (with its DataBasePreprocessor) is built under np.random.seed(seed_init); then,
frame after frame and with the samplers carried over, each frame runs under np.random.seed(seed_f) through
sample_all and prep_pointcloud's lines 224-249 (concatenation, sample_importance, remove_points_after_sample).  Frames:
no GT; DontCare and out-of-class names; a crowded frame where most candidates collide; frames with many GTs of the
first class (small sampled_num); plain frames, the run long enough for the samplers to wrap.  The xyres_16 fixture
also runs one frame on through prep_pointcloud's augmentation (lines 255-294) on the same stream: the chain.  A rate
table records sample_all's per-class sample count for rates whose products end in .5 (numpy rounds half to even).

Recorded: the database (infos as arrays, all points), the infos that survive the prep steps, per frame the inputs, the
candidates each sampler returned and the accepted ones (as info ids), the sample_all dict, the frame at
preprocess.py:249 and a sha1 of np.random's state after the frame.  Seeds are rejected while a decision lies near a
tie: a candidate whose BEV separating-axis gap to a box it is tested against is under 1e-4 m, a frame point within
2e-4 m of an accepted box's surface, and the augmentation's ties (make_augment_golden) in the chain.
"""
import copy
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_augment_golden as mag  # noqa: E402  (installs the reference and its numba adaptation)

import augment_ref as ar  # noqa: E402
from b2second import augment, config  # noqa: E402

from second.core import box_np_ops  # noqa: E402
from second.core import preprocess as prep  # noqa: E402
from second.core import sample_ops  # noqa: E402

OUT = os.path.join(HERE, "dbsample")
CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"]
BASE_SEED = {"car.fhd": 100, "all.fhd": 200, "pointpillars.car.xyres_16": 300, "nuscenes.all.pp.mhead": 400}
KINDS = ["empty", "dontcare", "crowd", "plain", "many", "plain", "plain", "plain", "plain", "chain"]
EXTRA_KEY = "Misc"
OBJECTS_PER_CLASS, OBJECTS_OTHER = 28, 5
POINT_EPS, GAP_EPS = 2e-4, 1e-4


def is_nus(name):
    return name.startswith("nuscenes")


def make_database(name, root):
    """-> db_infos (dict, EXTRA_KEY first) and the arrays recorded in the fixture"""
    cfg = config.get_config(name)
    rng = np.random.default_rng(BASE_SEED[name])
    classes = ar.class_names(name)
    sampled = [n for g in cfg.db_sampler.sample_groups for n in g]
    F = cfg.num_point_features
    r = np.asarray(cfg.point_cloud_range, np.float64)
    ndim = 9 if is_nus(name) else 7
    dtype = np.float64 if is_nus(name) else np.float32
    cluster = rng.uniform(r[:2] + 8, r[3:5] - 18)
    infos, rec = {}, {k: [] for k in ("key", "name", "path", "box", "difficulty", "npig", "off")}
    pts_all, off = [], 0
    for key in [EXTRA_KEY] + classes:
        n = OBJECTS_PER_CLASS if key in sampled else OBJECTS_OTHER
        lst = []
        for i in range(n):
            b = np.zeros(ndim)
            if i % 2 == 0:
                b[:2] = cluster + rng.uniform(0, 10, 2)
            else:
                b[:2] = rng.uniform(r[:2] + 2, r[3:5] - 2)
            b[2] = rng.uniform(-1.9, -1.2)
            b[3:6] = rng.uniform([0.6, 0.8, 1.4], [2.2, 5.0, 1.9])
            b[6] = rng.uniform(-np.pi, np.pi)
            if ndim == 9:
                b[7:] = rng.normal(0, 3, 2)
            box = b.astype(dtype)
            npts = int(rng.integers(3, 60))
            loc = rng.uniform(-0.45, 0.45, (npts, 3)) * b[3:6]
            c, s = np.cos(b[6]), np.sin(b[6])
            xyz = np.stack([loc[:, 0] * c - loc[:, 1] * s, loc[:, 0] * s + loc[:, 1] * c, loc[:, 2]], 1)
            p = np.concatenate([xyz, rng.uniform(0, 1, (npts, F - 3))], 1).astype(np.float32)
            path = "%s_%03d.bin" % (key, i)
            p.tofile(os.path.join(root, path))
            uid = len(rec["key"])
            diff = int(rng.choice([-1, 0, 1, 2], p=[0.15, 0.45, 0.25, 0.15]))
            npig = int(rng.integers(0, 40))
            lst.append({"name": key, "path": path, "box3d_lidar": box, "difficulty": diff, "num_points_in_gt": npig,
                        "group_id": uid, "image_idx": i, "gt_idx": i, "uid": uid})
            for k, v in (("key", key), ("name", key), ("path", path), ("box", box), ("difficulty", diff),
                         ("npig", npig), ("off", off)):
                rec[k].append(v)
            pts_all.append(p)
            off += npts
        infos[key] = lst
    rec["off"].append(off)
    arrays = {"db_keys": np.array(list(infos)), "db_key": np.array(rec["key"]), "db_name": np.array(rec["name"]),
              "db_path": np.array(rec["path"]), "db_box": np.stack(rec["box"]),
              "db_difficulty": np.array(rec["difficulty"], np.int64), "db_npig": np.array(rec["npig"], np.int64),
              "db_point_off": np.array(rec["off"], np.int64), "db_points": np.concatenate(pts_all),
              "db_cluster": cluster}
    return infos, arrays


def make_frame(name, kind, seed, cluster):
    cfg = config.get_config(name)
    rng = np.random.default_rng(seed)
    r = np.asarray(cfg.point_cloud_range, np.float64)
    classes = ar.class_names(name)
    ndim = 9 if is_nus(name) else 7
    dtype = np.float64 if is_nus(name) else np.float32
    F = cfg.num_point_features

    def rand_boxes(n):
        b = np.zeros((n, ndim))
        b[:, :2] = rng.uniform(r[:2] + 2, r[3:5] - 2, (n, 2))
        b[:, 2] = rng.uniform(-1.9, -1.2, n)
        b[:, 3:6] = rng.uniform([1.5, 3.5, 1.4], [2.0, 4.6, 1.8], (n, 3))
        b[:, 6] = rng.uniform(-np.pi, np.pi, n)
        if ndim == 9:
            b[:, 7:] = rng.normal(0, 3, (n, 2))
        return b

    pool = classes + ["Truck", "Misc"]
    if kind == "empty":
        b, names = np.zeros((0, ndim)), []
    elif kind == "dontcare":
        b = rand_boxes(6)
        names = ["DontCare", "Misc", classes[0], "DontCare", "Truck", classes[-1]]
    elif kind == "crowd":
        # a grid of GTs over the whole range: most candidates collide with one
        gx, gy = np.meshgrid(np.linspace(r[0] + 3, r[3] - 3, 9), np.linspace(r[1] + 3, r[4] - 3, 9))
        b = rand_boxes(81)
        b[:, 0], b[:, 1] = gx.ravel() + rng.uniform(-1, 1, 81), gy.ravel() + rng.uniform(-1, 1, 81)
        b[:, 3:5] = rng.uniform([3.0, 6.0], [4.0, 8.0], (81, 2))
        names = [["Misc", "Truck"][i] for i in rng.integers(0, 2, 81)]     # obstacles only: sampled_num stays high
    elif kind == "many":
        b = rand_boxes(14)
        names = [classes[0]] * 13 + ["Misc"]
    else:
        n = int(rng.integers(2, 7))
        b = rand_boxes(n)
        names = [pool[i] for i in rng.integers(0, len(pool), n)]
    boxes = b.astype(dtype)
    pts = [rng.uniform(r[:3], r[3:], (800, 3)),
           np.concatenate([cluster + rng.uniform(-1, 11, (800, 2)), rng.uniform(-2.5, -0.5, (800, 1))], 1)]
    for bx in b:
        loc = rng.uniform(-0.7, 0.7, (20, 3)) * bx[3:6]
        c, s = np.cos(bx[6]), np.sin(bx[6])
        pts.append(np.stack([loc[:, 0] * c - loc[:, 1] * s + bx[0], loc[:, 0] * s + loc[:, 1] * c + bx[1],
                             loc[:, 2] + bx[2]], 1))
    xyz = np.concatenate(pts)
    points = np.concatenate([xyz, rng.uniform(0, 1, (len(xyz), F - 3))], 1).astype(np.float32)
    return points, boxes, np.array(names, dtype="<U20")


class Recorder:
    """hooks on the reference's BatchSampler._sample and sample_class_v2 recording what they return (as info uids)"""

    def __init__(self):
        self.cand, self.acc, self.nums = [], [], []
        orig_sample, orig_v2 = prep.BatchSampler._sample, sample_ops.DataBaseSamplerV2.sample_class_v2
        rec = self

        def _sample(sampler, num):
            ret = orig_sample(sampler, num)
            rec.cand += [sampler._sampled_list[i]["uid"] for i in ret]
            rec.nums.append((sampler._name, int(num), len(ret)))
            return ret

        def sample_class_v2(sampler, name, num, gt_boxes):
            ret = orig_v2(sampler, name, num, gt_boxes)
            rec.acc += [s["uid"] for s in ret]
            return ret
        prep.BatchSampler._sample = _sample
        sample_ops.DataBaseSamplerV2.sample_class_v2 = sample_class_v2

    def reset(self):
        self.cand, self.acc, self.nums = [], [], []


def bev_ties(boxes, cand_boxes):
    """True when a candidate's BEV gap to any other box of the frame is within GAP_EPS of zero"""
    allb = np.concatenate([boxes, cand_boxes]).astype(np.float64)
    if len(cand_boxes) == 0:
        return False
    cor = mag.corners64(allb[:, 0], allb[:, 1], allb[:, 3], allb[:, 4], allb[:, 6])
    g = mag.sat_gap(cor[len(boxes):, None], cor[None, :])
    n = len(cand_boxes)
    g[np.arange(n), len(boxes) + np.arange(n)] = np.inf
    return bool((np.abs(g) < GAP_EPS).any())


def run_frame(name, sampler, rec, points, boxes, names, seed, root, db_box_by_uid):
    cfg = config.get_config(name)
    s = cfg.db_sampler
    classes = ar.class_names(name)
    keep = names != "DontCare"
    boxes, names = boxes[keep].copy(), names[keep]
    imp = np.ones(len(boxes), boxes.dtype)
    mask = np.array([n in classes for n in names], np.bool_)
    rec.reset()
    np.random.seed(seed)
    sd = sampler.sample_all(root, boxes, names, cfg.num_point_features, False, gt_group_ids=None, calib=None)
    ties = []
    cand_boxes = np.array([db_box_by_uid[u] for u in rec.cand]).reshape(-1, boxes.shape[1]) if rec.cand else \
        np.zeros((0, boxes.shape[1]), boxes.dtype)
    if bev_ties(boxes, cand_boxes):
        ties.append("bev")
    out_pts, out_boxes, out_names, out_imp, out_mask = points, boxes, names, imp, mask
    if sd is not None:
        out_names = np.concatenate([names, sd["gt_names"]], 0)
        out_boxes = np.concatenate([boxes, sd["gt_boxes"]])
        out_mask = np.concatenate([mask, sd["gt_masks"]], 0)
        out_imp = np.concatenate([imp, np.full([len(sd["gt_boxes"])], s.sample_importance,
                                               dtype=sd["gt_boxes"].dtype)])
        if s.remove_points_after_sample:
            m = box_np_ops.points_in_rbbox(points, sd["gt_boxes"])
            out_pts = points[np.logical_not(m.any(-1))]
            if (np.abs(mag.local_margin(points, sd["gt_boxes"])) < POINT_EPS).any():
                ties.append("point")
        out_pts = np.concatenate([sd["points"], out_pts], axis=0)
    rec_out = {"cand": np.array(rec.cand, np.int64), "acc": np.array(rec.acc, np.int64),
               "requested": np.array([n for _, n, _ in rec.nums], np.int64),
               "out_points": out_pts, "out_boxes": out_boxes, "out_names": out_names, "out_importance": out_imp,
               "out_mask": out_mask, "sa_none": np.bool_(sd is None)}
    if sd is not None:
        for k in ("gt_names", "difficulty", "gt_boxes", "points", "gt_masks", "group_ids"):
            rec_out["sa_" + k] = sd[k]
    return rec_out, ties, (out_pts, out_boxes, out_names, out_imp, out_mask)


def run_chain(name, pts, boxes, names, imp, valid):
    """prep_pointcloud's lines 255-294 on the sampled frame, continuing np.random; as make_augment_golden.run_reference"""
    cfg = config.get_config(name)
    s = cfg.augment
    classes = ar.class_names(name)
    G = len(boxes)
    ties = []
    points = pts.copy()
    boxes = boxes.copy()
    orig = boxes.copy()
    st0 = np.random.get_state()
    prep.noise_per_object_v3_(boxes, points, valid, rotation_perturb=list(s.groundtruth_rotation_uniform_noise),
                              center_noise_std=list(s.groundtruth_localization_noise_std),
                              global_random_rot_range=list(s.global_random_rotation_range_per_object),
                              group_ids=None, num_try=augment.NUM_TRY)
    st1 = np.random.get_state()
    np.random.set_state(st0)
    loc = np.random.normal(scale=np.array(s.groundtruth_localization_noise_std, dtype=orig.dtype),
                           size=[G, augment.NUM_TRY, 3])
    rot = np.random.uniform(*s.groundtruth_rotation_uniform_noise, size=[G, augment.NUM_TRY])
    np.random.set_state(st1)
    sel = prep.noise_per_box(orig[:, [0, 1, 3, 4, 6]], valid, loc, rot).astype(np.int32)
    corners = box_np_ops.center_to_corner_box3d(orig[:, :3], orig[:, 3:6], orig[:, 6], origin=[0.5, 0.5, 0.5], axis=2)
    mask = mag.geometry.points_in_convex_polygon_3d_jit(pts[:, :3], box_np_ops.corner_to_surfaces_3d_jit(corners))
    mask &= valid[None, :]
    point_box = np.where(mask.any(1), mask.argmax(1), -1).astype(np.int32)
    if (np.abs(mag.local_margin(pts, orig)[:, valid]) < mag.POINT_EPS).any():
        ties.append("point")
    if mag.pose_ties(orig, valid, loc, rot, sel):
        ties.append("pose")
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
    if (edge < mag.RANGE_EPS).any():
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
    out = {"chain_points": points, "chain_point_box": point_box[order], "chain_selected": sel,
           "chain_boxes": boxes, "chain_classes": cls, "chain_importance": imp.astype(np.float32),
           "chain_src_row": idx}
    return out, ties


def rate_table(name, infos, root, rec):
    """sample_all's per-class count for rates whose products end in .5"""
    cfg = config.get_config(name)
    rows = []
    for rate in (0.5, 0.25, 0.3, 1.5):
        np.random.seed(7)
        smp = sample_ops.DataBaseSamplerV2(copy.deepcopy(infos), cfg.db_sampler.sample_groups, None, rate, [0.0, 0.0])
        first = next(iter(cfg.db_sampler.sample_groups[0]))
        box = infos[first][0]["box3d_lidar"]
        for k in range(0, 16):
            rec.reset()
            gt = np.zeros((k, len(box)), box.dtype)
            gt[:, 0] = np.arange(k) * 5.0 - 300.0              # far from every database box: only the counts matter
            gt[:, 3:6] = 1.0
            smp.sample_all(root, gt, np.array([first] * k), cfg.num_point_features)
            req = [n for nm, n, _ in rec.nums if nm == first]
            rows.append((rate, k, req[0] if req else 0))
    return np.array(rows, np.float64)


def main():
    os.makedirs(OUT, exist_ok=True)
    rec = Recorder()
    for name in CONFIGS:
        cfg = config.get_config(name)
        with tempfile.TemporaryDirectory() as root:
            infos, z = make_database(name, root)
            db_box_by_uid = dict(enumerate(z["db_box"]))
            prepors = []
            for kind, arg in cfg.db_sampler.database_prep_steps:
                prepors.append(prep.DBFilterByMinNumPoint(dict(arg)) if kind == "filter_by_min_num_points" else
                               prep.DBFilterByDifficulty(list(arg)))
            seed_init = BASE_SEED[name] * 1000
            np.random.seed(seed_init)
            sampler = sample_ops.DataBaseSamplerV2(copy.deepcopy(infos), cfg.db_sampler.sample_groups,
                                                   prep.DataBasePreprocessor(prepors), cfg.db_sampler.rate,
                                                   list(cfg.db_sampler.global_random_rotation_range_per_object))
            z["seed_init"] = np.int64(seed_init)
            z["state_init"] = np.array(ar.state_digest(np.random))
            filt = [np.array([i["uid"] for i in sampler.db_infos[k]], np.int64) for k in infos]
            z["filt_uid"] = np.concatenate(filt)
            z["filt_off"] = np.cumsum([0] + [len(f) for f in filt]).astype(np.int64)
            kinds = [k for k in KINDS if k != "chain" or name == "pointpillars.car.xyres_16"]
            wraps = 0
            for f, kind in enumerate(kinds):
                for attempt in range(200):
                    seed = BASE_SEED[name] * 1000 + 100 * (f + 1) + attempt
                    saved = copy.deepcopy({k: (v._indices.copy(), v._idx) for k, v in sampler._sampler_dict.items()})
                    pts, boxes, names = make_frame(name, kind, seed, z["db_cluster"])
                    out, ties, frame = run_frame(name, sampler, rec, pts, boxes, names, seed, root, db_box_by_uid)
                    nums = list(rec.nums)
                    if kind == "chain" and not ties:
                        cout, cties = run_chain(name, frame[0], frame[1], frame[2], frame[3], frame[4])
                        ties += cties
                        out.update(cout)
                    if not ties:
                        break
                    for k, (ind, idx) in saved.items():
                        sampler._sampler_dict[k]._indices = ind
                        sampler._sampler_dict[k]._idx = idx
                else:
                    raise RuntimeError("%s %s: no tie-free seed" % (name, kind))
                wraps += sum(1 for _, n, got in nums if got < n)
                out["state"] = np.array(ar.state_digest(np.random))
                out["in_points"], out["in_boxes"], out["in_names"] = pts, boxes, names
                for k, v in out.items():
                    z["%s_%d" % (k, f)] = v
                z["seed_%d" % f] = np.int64(seed)
                z["kind_%d" % f] = np.array(kind)
                print("%s %-8s seed %d: %d candidates, %d accepted, %d points out" % (
                    name, kind, seed, len(out["cand"]), len(out["acc"]), len(out["out_points"])), flush=True)
            assert wraps > 0, "%s: no sampler wrapped" % name
            z["num_frames"] = np.int64(len(kinds))
            z["rate_table"] = rate_table(name, infos, root, rec)
            np.savez_compressed(os.path.join(OUT, name + ".npz"), **z)


if __name__ == "__main__":
    main()
