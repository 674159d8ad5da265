"""Generate tests/golden/kitti_eval/*.npz from the UNMODIFIED reference (needs the reference tree; runs on the CPU).

    python tests/golden/make_kitti_eval_golden.py

Evaluation cases run second.utils.eval.get_official_eval_result / get_coco_eval_result through b2second.refcompat
(numba's CUDA simulator stands in for the GPU); the eval_class_v3 arrays are recorded from those same calls.  The
conversion case runs KittiDataset.convert_detection_to_kitti_annos on the detections stored in tests/golden/car.fhd.*.

The rotated overlaps here are fp32 polygon clips whose last bits differ between implementations (up to ~3e-5), so a
case is rejected when any reference overlap lies within 1e-4 of a min_overlap it is compared with, or when a printed AP
lies within 1e-6 of a rounding tie: then no count and no printed digit can depend on those bits.
"""
import glob
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
OUT = os.path.join(HERE, "kitti_eval")

from b2second import loader, refcompat  # noqa: E402

refcompat.install(loader.ORACLE_DIR)
_linspace = np.linspace


def _linspace_float_num(start, stop, num=50, *a, **k):
    # do_coco_style_eval passes num as a float64 (eval.py:704), which numpy >= 1.18 rejects
    return _linspace(start, stop, int(num) if float(num).is_integer() else num, *a, **k)


np.linspace = _linspace_float_num
import torch  # noqa: E402
from second.core import box_np_ops  # noqa: E402
from second.utils import eval as E  # noqa: E402

KEYS = ("bbox", "location", "dimensions", "rotation_y", "alpha", "truncated", "occluded")
DIMS = {"Car": (3.9, 1.56, 1.6), "Van": (5.0, 2.2, 1.9), "Pedestrian": (0.8, 1.75, 0.6),
        "Person_sitting": (0.8, 1.3, 0.6), "Cyclist": (1.76, 1.74, 0.6), "DontCare": (1.0, 1.0, 1.0),
        "Truck": (10.0, 3.2, 2.5)}
GT_NAMES = ["Car", "Car", "Car", "Van", "Pedestrian", "Pedestrian", "Person_sitting", "Cyclist", "DontCare", "Truck"]
COCO = [np.linspace(0.5, 0.95, 10), np.linspace(0.25, 0.7, 10)]
THRESHOLDS = np.unique(np.concatenate([[0.7, 0.5, 0.25]] + COCO))


def _box(rng, name, lidar):
    l, h, w = np.array(DIMS[name]) * rng.uniform(0.9, 1.1, 3)
    x, z = rng.uniform(-12, 12), rng.uniform(4, 45)
    y = rng.uniform(1.4, 1.9)
    f = 720.0
    u, v = 610 + f * x / z, 173 + f * y / z
    bw, bh = f * max(l, w) / z * rng.uniform(0.6, 1.0), f * h / z
    bh *= rng.choice([0.6, 1.0, 1.0, 1.5])               # spread the heights across the difficulty limits
    loc = np.array([x, y, z]) if not lidar else np.array([z, -x, 1.0 - y + h / 2])
    dims = np.array([l, h, w]) if not lidar else np.array([l, w, h])
    return dict(bbox=np.array([u - bw / 2, v - bh, u + bw / 2, v]), location=loc, dimensions=dims,
                rotation_y=rng.uniform(-np.pi, np.pi), alpha=rng.uniform(-np.pi, np.pi),
                truncated=rng.choice([0.0, 0.1, 0.2, 0.4, 0.6]), occluded=int(rng.integers(0, 4)))


def _stack(boxes, names, score=None):
    a = {"name": np.array(names, dtype="<U14") if names else np.array([])}
    for k in KEYS:
        shape = {"bbox": (0, 4), "location": (0, 3), "dimensions": (0, 3)}.get(k, (0,))
        a[k] = np.stack([b[k] for b in boxes]).astype(np.float64 if k != "occluded" else np.int64) if boxes \
            else np.zeros(shape)
    if score is not None:
        a["score"] = np.asarray(score, dtype=np.float32) if boxes else np.array([])
    return a


def _jitter(rng, b, lidar):
    d = dict(b)
    d["location"] = b["location"] + rng.normal(0, 0.25, 3)
    d["dimensions"] = b["dimensions"] * rng.uniform(0.9, 1.1, 3)
    d["rotation_y"] = b["rotation_y"] + rng.normal(0, 0.15)
    d["alpha"] = b["alpha"] + rng.normal(0, 0.3)
    d["bbox"] = b["bbox"] + rng.normal(0, 4, 4)
    return d


def _bev(a, lidar):
    ax = [0, 1] if lidar else [0, 2]
    return np.concatenate([a["location"][:, ax], a["dimensions"][:, ax], a["rotation_y"][:, None]], 1)


def _clear(g, d, lidar, margin=1e-3):
    """True when no overlap (2D, BEV, 3D; float64 CPU estimate) of detection d with ground truth g lies near a
    threshold.  The exact reference values are checked again after the reference has run."""
    if not len(g["name"]):
        return True
    iou2 = E.image_box_overlap(d["bbox"], g["bbox"])
    gb, db = _bev(g, lidar), _bev(d, lidar)
    bev = box_np_ops.riou_cc(db, gb)
    z = 2 if lidar else 1
    zc = 0.5 if lidar else 1.0
    box = lambda a: np.concatenate([a["location"], a["dimensions"], a["rotation_y"][:, None]], 1)
    inc = box_np_ops.rinter_cc(db, gb)
    E.box3d_overlap_kernel(box(d), box(g), inc, -1, z, zc)
    vals = np.concatenate([iou2.ravel(), bev.ravel(), inc.ravel()])
    return not (np.abs(vals[:, None] - THRESHOLDS[None, :]) < margin).any()


def make_case(seed, n_frames, lidar=False, no_aos=False, big_frames=()):
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for f in range(n_frames):
        n_gt = 0 if f % 17 == 5 else int(rng.integers(1, 12))
        names = [str(rng.choice(GT_NAMES)) for _ in range(n_gt)]
        gboxes = [_box(rng, n, lidar) for n in names]
        g = _stack(gboxes, names)
        dboxes, dnames = [], []
        if f % 13 != 7:
            for b, n in zip(gboxes, names):
                if n == "DontCare" or rng.uniform() < 0.2:
                    continue
                det_name = {"Van": "Car", "Person_sitting": "Pedestrian", "Truck": "Car"}.get(n, n)
                for _ in range(100):
                    cand = _jitter(rng, b, lidar)
                    if _clear(g, _stack([cand], [det_name], [0.5]), lidar):
                        break
                else:
                    raise RuntimeError("could not place a detection away from the thresholds")
                dboxes.append(cand)
                dnames.append(det_name)
            n_total = 100 if f in big_frames else len(dboxes) + int(rng.integers(0, 6))
            while len(dboxes) < n_total:
                n = str(rng.choice(["Car", "Pedestrian", "Cyclist"]))
                cand = _box(rng, n, lidar)
                if _clear(g, _stack([cand], [n], [0.5]), lidar):
                    dboxes.append(cand)
                    dnames.append(n)
        scores = rng.permutation(np.linspace(0.05, 0.99, max(len(dboxes), 1)).astype(np.float32))[:len(dboxes)]
        d = _stack(dboxes, dnames, scores)
        if no_aos and len(dnames):
            d["alpha"][:] = -10
        gts.append(g)
        dts.append(d)
    return gts, dts


class _Recorder:
    """wraps the reference's eval_class_v3 / calculate_iou_partly to keep what they returned (code unchanged)."""

    def __init__(self):
        self.evals, self.overlaps = [], []
        self._ev, self._iou = E.eval_class_v3, E.calculate_iou_partly

        def ev(gt, dt, classes, diffs, metric, min_overlaps, compute_aos=False, **kw):
            r = self._ev(gt, dt, classes, diffs, metric, min_overlaps, compute_aos, **kw)
            self.evals.append((metric, compute_aos, r))
            return r

        def iou(*a, **kw):
            r = self._iou(*a, **kw)
            self.overlaps.append(r[0])
            return r
        E.eval_class_v3, E.calculate_iou_partly = ev, iou

    def close(self):
        E.eval_class_v3, E.calculate_iou_partly = self._ev, self._iou


def _flatten(prefix, annos, with_score):
    out = {}
    counts = np.array([len(a["name"]) for a in annos], dtype=np.int64)
    out[prefix + "offsets"] = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    out[prefix + "name"] = np.concatenate([np.asarray(a["name"], dtype="<U16") for a in annos])
    for k in KEYS + (("score",) if with_score else ()):
        width = {"bbox": 4, "location": 3, "dimensions": 3}.get(k, 1)
        parts = [np.asarray(a[k]).reshape(len(a["name"]), width) for a in annos]
        out[prefix + k] = np.concatenate(parts).astype(np.float32 if k == "score" else np.float64)
        if width == 1:
            out[prefix + k] = out[prefix + k][:, 0]
    return out


def _ap_ties(values):
    v = np.asarray(values, dtype=np.float64).ravel() * 100
    v = v[np.isfinite(v)]
    return bool((np.abs(v - np.floor(v) - 0.5) < 1e-4).any())


def run_eval_case(name, seed, n_frames, classes, lidar=False, no_aos=False, big_frames=()):
    z_axis, z_center = (2, 0.5) if lidar else (1, 1.0)
    for attempt in range(20):
        gts, dts = make_case(seed + 1000 * attempt, n_frames, lidar, no_aos, big_frames)
        rec = _Recorder()
        try:
            off = E.get_official_eval_result(gts, dts, classes, z_axis=z_axis, z_center=z_center)
            n_off = len(rec.evals)
            coco = E.get_coco_eval_result(gts, dts, classes, z_axis=z_axis, z_center=z_center)
        finally:
            rec.close()
        ovs = np.concatenate([o.ravel() for frames in rec.overlaps for o in frames])
        near = (np.abs(ovs[:, None] - THRESHOLDS[None, :]) < 1e-4).any()
        aps = [v for res in (off, coco) for c in res["detail"].values() for v in c.values()]
        if near or _ap_ties(aps):
            print("%s: attempt %d rejected (near threshold: %s)" % (name, attempt, near))
            continue
        out = {"classes": np.array(classes, dtype=np.int64), "z_axis": np.int64(z_axis), "z_center": np.float64(z_center),
               "official_result": np.array(off["result"]), "coco_result": np.array(coco["result"])}
        out.update(_flatten("gt_", gts, False))
        out.update(_flatten("dt_", dts, True))
        for i, (metric, aos, r) in enumerate(rec.evals):
            tag = "official" if i < n_off else "coco"
            for k in ("precision", "orientation", "thresholds"):
                out["%s_m%d_%s" % (tag, metric, k)] = r[k]
            out["%s_m%d_aos" % (tag, metric)] = np.bool_(aos)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
        print(name, "written", off["result"].splitlines()[1])
        return
    raise RuntimeError("no acceptable case for " + name)


def kitti_like_calibs():
    """KITTI-like calibration with principal points / image sizes chosen so that boxes cross every image border."""
    P2 = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791],
                   [0.0, 0.0, 1.0, 0.002745884], [0.0, 0.0, 0.0, 1.0]])
    rect = np.eye(4)
    rect[:3, :3] = np.array([[0.9999239, 0.00983776, -0.00744505], [-0.0098698, 0.9999421, -0.00427846],
                             [0.00740253, 0.00435161, 0.9999631]])
    Trv2c = np.eye(4)
    Trv2c[:3, :] = np.array([[0.00753374, -0.9999714, -0.00061660, -0.00406977],
                             [0.01480249, 0.00072807, -0.9998902, -0.07631618],
                             [0.9998621, 0.00752379, 0.01480755, -0.2717806]])
    out = []
    for cx, cy, shape in ((609.5593, 172.854, (375, 1242)), (300.0, 20.0, (200, 700)), (900.0, 330.0, (375, 1242))):
        p = P2.copy()
        p[0, 2], p[1, 2] = cx, cy
        out.append({"R0_rect": rect, "Tr_velo_to_cam": Trv2c, "P2": p, "shape": np.array(shape)})
    return out


def run_convert_case():
    import importlib.util
    import types
    # second.data imports these for image reading and command lines, neither used by the conversion
    for mod in ("skimage", "fire"):
        if importlib.util.find_spec(mod) is None:
            sys.modules[mod] = types.SimpleNamespace(io=None)
    from second.data.kitti_dataset import KittiDataset
    class_names = ["Car", "Pedestrian", "Cyclist"]
    dets, infos = [], []
    for i, path in enumerate(sorted(glob.glob(os.path.join(HERE, "car.fhd.seed*.npz")))):
        fix = np.load(path)
        for c in kitti_like_calibs():
            labels = (fix["label_preds"] + np.arange(len(fix["label_preds"]))) % 3   # all three names
            dets.append({"box3d_lidar": torch.from_numpy(fix["box3d_lidar"].copy()),
                         "scores": torch.from_numpy(fix["scores"].copy()),
                         "label_preds": torch.from_numpy(labels.astype(np.int64)),
                         "metadata": {"image_idx": len(dets)}})
            infos.append({"calib": {k: c[k] for k in ("R0_rect", "Tr_velo_to_cam", "P2")},
                          "image": {"image_idx": len(infos), "image_shape": c["shape"]}})
    dets.append({"box3d_lidar": torch.zeros(0, 7), "scores": torch.zeros(0), "label_preds": torch.zeros(0, dtype=torch.long),
                 "metadata": {"image_idx": len(dets)}})
    infos.append(dict(infos[0], image={"image_idx": len(infos), "image_shape": np.array([375, 1242])}))
    ds = KittiDataset.__new__(KittiDataset)
    ds._kitti_infos, ds._class_names = infos, class_names
    clones = [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in d.items()} for d in dets]
    annos = ds.convert_detection_to_kitti_annos(clones)
    # border coverage: for each border, a kept box crosses it and a box beyond it is dropped
    kept = np.concatenate([a["bbox"] for a in annos if len(a["name"])])
    W = np.concatenate([np.full(len(a["name"]), infos[i]["image"]["image_shape"][1]) for i, a in enumerate(annos)])
    H = np.concatenate([np.full(len(a["name"]), infos[i]["image"]["image_shape"][0]) for i, a in enumerate(annos)])
    assert (kept[:, 0] == 0).any() and (kept[:, 1] == 0).any() and (kept[:, 2] == W).any() and (kept[:, 3] == H).any()
    n_in = sum(len(d["scores"]) for d in dets)
    assert sum(len(a["name"]) for a in annos) < n_in
    out = {"class_names": np.array(class_names), "image_shape": np.stack([i["image"]["image_shape"] for i in infos]),
           "calib": np.stack([np.stack([i["calib"][k] for k in ("R0_rect", "Tr_velo_to_cam", "P2")]) for i in infos]),
           "det_offsets": np.concatenate([[0], np.cumsum([len(d["scores"]) for d in dets])]).astype(np.int64),
           "det_box3d_lidar": np.concatenate([d["box3d_lidar"].numpy() for d in dets]).astype(np.float32),
           "det_scores": np.concatenate([d["scores"].numpy() for d in dets]).astype(np.float32),
           "det_label_preds": np.concatenate([d["label_preds"].numpy() for d in dets]).astype(np.int64)}
    out.update(_flatten("anno_", annos, True))
    np.savez_compressed(os.path.join(OUT, "convert.car_fhd.npz"), **out)
    print("convert written: %d of %d boxes kept" % (sum(len(a["name"]) for a in annos), n_in))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    which = sys.argv[1:] or ["convert", "main", "noaos", "lidar"]
    if "convert" in which:
        run_convert_case()
    if "main" in which:
        run_eval_case("eval.main", 1, 120, [0, 1, 2], big_frames=(3, 40))
    if "noaos" in which:
        run_eval_case("eval.noaos", 2, 60, [0, 1], no_aos=True)
    if "lidar" in which:
        run_eval_case("eval.lidar", 3, 60, [0, 2], lidar=True)
