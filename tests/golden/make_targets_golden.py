"""Generate tests/golden/targets/*.npz FROM THE UNMODIFIED REFERENCE (needs the reference tree; runs on the CPU).

    python tests/golden/make_targets_golden.py [--force]

For each config the reference's own builders (b2second.refcompat.build_network) make the TargetAssigner, and its
unmodified ``assign`` (second/core/target_assigner.py:38-167 -> create_target_np) runs on seeded synthetic frames:
  0  no ground truth
  1  a dozen GTs: random ones, a duplicated GT, a GT outside every anchor, GTs centred between two anchors (ties for
     the GT's max) and a copy of an anchor
  2  like 1 under a random anchors_mask, with importance in [0.5, 2] over two classes
  3  more GTs in one segment than one shared-memory chunk of the kernel (200)
KITTI configs take float32 ground truth, the NuScenes ones float64 (as their infos hold it).  For
pointpillars.car.xyres_16, frames 1-3 use the anchors_mask the reference's own sparse_sum_for_anchors_mask /
fused_get_anchors_area give for a seeded synthetic cloud (threshold 1); its voxel coordinates are stored as well.
Each file holds, per frame f: gt_boxes_f, gt_names_f, gt_classes_f, importance_f, mask_f (packed bits, or absent),
labels_f (int8), importance_out_f (float32), pos_f (indices with labels > 0) and targets_f (box targets at pos_f); for
assign_all also overlap_f, gt_id_f, inds_f; and sha1 digests of the TargetPlan arrays (b2second.targets.plan) built
from the reference assigner.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
OUT = os.path.join(HERE, "targets")

from b2second import config, loader, refcompat, synth, targets  # noqa: E402

CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"]
MASK_CLOUD = ("pointpillars.car.xyres_16", 0, 20000)


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def reference_assigner(name):
    from second.utils.config_tool import get_downsample_factor
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    cfgp = refcompat.load_config(f)
    net = refcompat.build_network(cfgp.model.second)
    grid = net.voxel_generator.grid_size
    fms = [int(v) for v in [*(grid[:2] // get_downsample_factor(cfgp.model.second)), 1][::-1]]
    return net, net.target_assigner, fms


def cloud_mask(net, anchors):
    """the reference preprocessing's anchors_mask (preprocess.py:345-357) for the seeded cloud, threshold 1"""
    from second.core import box_np_ops
    name, seed, npts = MASK_CLOUD
    b = config.get_config(name)
    pts = synth.kitti_cloud(seed, npts, b.point_cloud_range)
    vg = net.voxel_generator
    res = vg.generate(pts, b.max_voxels)
    coors = res["coordinates"]
    grid = vg.grid_size
    dense = box_np_ops.sparse_sum_for_anchors_mask(coors, tuple(grid[::-1][1:]))
    dense = dense.cumsum(0).cumsum(1)
    bv = box_np_ops.rbbox2d_to_near_bbox(anchors[:, [0, 1, 3, 4, 6]])
    area = box_np_ops.fused_get_anchors_area(dense, bv, vg.voxel_size, vg.point_cloud_range, grid)
    return area > 1, np.ascontiguousarray(coors, np.int32)


def frames(rng, ta, anchors, per_class_ranges, dtype):
    """the four synthetic frames: (gt_boxes, gt_names, gt_classes, importance)"""
    classes = list(ta.classes)
    anchored = [c for c in range(len(per_class_ranges)) if per_class_ranges[c][1] > per_class_ranges[c][0]]

    def rand_gt(n, cls=None):
        rows, names = [], []
        for _ in range(n):
            c = anchored[rng.integers(len(anchored))] if cls is None else cls
            b, e = per_class_ranges[c]
            a = anchors[rng.integers(b, e)].astype(np.float64)
            g = a.copy()
            g[0:2] += rng.uniform(-1.0, 1.0, 2)
            g[3:6] *= rng.uniform(0.85, 1.15, 3)
            g[6] = rng.uniform(-np.pi, np.pi)
            rows.append(g)
            names.append(classes[c])
        return rows, names

    out = [(np.zeros((0, anchors.shape[1]), dtype), np.array([], "<U32"))]
    for f in (1, 2):
        rows, names = rand_gt(8)
        rows.append(rows[0].copy())                                 # duplicate
        names.append(names[0])
        far = rows[1].copy()
        far[0] += 500.0                                              # outside every anchor
        rows.append(far)
        names.append(names[1])
        c = anchored[0]
        b, e = per_class_ranges[c]
        i = rng.integers(b, e - 1)
        a0, a1 = anchors[i].astype(np.float64), anchors[i + 1].astype(np.float64)
        mid = a0.copy()
        mid[:2] = (a0[:2] + a1[:2]) / 2                              # between two neighbouring anchors
        rows.append(mid)
        names.append(classes[c])
        rows.append(anchors[rng.integers(b, e)].astype(np.float64))  # a copy of an anchor
        names.append(classes[c])
        out.append((np.array(rows, dtype), np.array(names, "<U32")))
    rows, names = rand_gt(200, anchored[0])
    more, mnames = rand_gt(10)
    out.append((np.array(rows + more, dtype), np.array(names + mnames, "<U32")))
    res = []
    for f, (gt, names) in enumerate(out):
        gcls = np.array([classes.index(n) + 1 for n in names], np.int32)
        imp = np.ones(len(gt), np.float32)
        if f == 2:
            imp = rng.uniform(0.5, 2.0, len(gt)).astype(np.float32)
        res.append((gt, names, gcls, imp))
    return res


def main():
    refcompat.install(loader.ORACLE_DIR)
    force = "--force" in sys.argv
    os.makedirs(OUT, exist_ok=True)
    for ci, name in enumerate(CONFIGS):
        path = os.path.join(OUT, name + ".npz")
        if os.path.exists(path) and not force:
            continue
        rng = np.random.default_rng(1000 + ci)
        net, ta, fms = reference_assigner(name)
        tp = targets.plan(ta, fms)
        ret = ta.generate_anchors(fms)
        anchors = ret["anchors"].reshape(-1, ta.box_ndim)
        anchors_dict = ta.generate_anchors_dict(fms)
        if ta._assign_per_class:
            ranges = [tuple(int(v) for v in ta.anchors_range(c)) for c in range(len(ta.classes))]
        else:
            ranges, b = [], 0
            for g in ta._anchor_generators:
                n = int(np.prod(fms)) * g.num_anchors_per_localization
                ranges.append((b, b + n))
                b += n
            ranges += [(0, 0)] * (len(ta.classes) - len(ranges))
        dtype = np.float64 if name.startswith("nuscenes") else np.float32
        fix = {"name": name, "feature_map_size": np.array(fms), "per_class": ta._assign_per_class,
               "num_anchors": anchors.shape[0], "anchors_sha1": sha(anchors.astype(np.float32))}
        for k, v in tp.params().items():
            fix["plan_" + k + "_sha1"] = sha(v)
        cmask = None
        if name == MASK_CLOUD[0]:
            cmask, coors = cloud_mask(net, anchors)
            fix["cloud_coors"] = coors
            fix["cloud_mask"] = np.packbits(cmask)
        for f, (gt, names, gcls, imp) in enumerate(frames(rng, ta, anchors, ranges, dtype)):
            mask = None
            if cmask is not None and f > 0:
                mask = cmask
            elif f == 2:
                mask = rng.random(anchors.shape[0]) < 0.7
            r = ta.assign(anchors, anchors_dict, gt, anchors_mask=mask, gt_classes=gcls, gt_names=names,
                          matched_thresholds=ret["matched_thresholds"],
                          unmatched_thresholds=ret["unmatched_thresholds"], importance=imp)
            labels = np.asarray(r["labels"])
            pos = np.flatnonzero(labels > 0)
            fix.update({"gt_boxes_%d" % f: gt, "gt_names_%d" % f: names, "gt_classes_%d" % f: gcls,
                        "importance_%d" % f: imp, "labels_%d" % f: labels.astype(np.int8),
                        "importance_out_%d" % f: np.asarray(r["importance"], np.float32),
                        "pos_%d" % f: pos.astype(np.int32),
                        "targets_%d" % f: np.asarray(r["bbox_targets"])[pos].astype(np.float32)})
            assert np.asarray(r["bbox_targets"]).dtype == np.float32
            assert not np.asarray(r["bbox_targets"])[labels <= 0].any()
            if mask is not None:
                fix["mask_%d" % f] = np.packbits(mask)
            if not ta._assign_per_class:
                fix["overlap_%d" % f] = np.asarray(r["assigned_anchors_overlap"] if len(gt) else [], np.float32)
                fix["gt_id_%d" % f] = np.asarray(r["positive_gt_id"], np.int32)
                fix["inds_%d" % f] = np.asarray(r["assigned_anchors_inds"], np.int64)
                assert np.array_equal(np.asarray(r["bbox_outside_weights"]), (labels > 0).astype(np.float32))
            print(name, "frame", f, "gt", len(gt), "pos", len(pos), "neg", int((labels == 0).sum()),
                  "ignored", int((labels < 0).sum()), flush=True)
        fix["num_frames"] = f + 1
        np.savez_compressed(path, **fix)
        print("->", os.path.relpath(path, HERE), os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main()
