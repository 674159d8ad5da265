"""CUDA-event times of the KITTI formatting and evaluation (b2second.kitti_eval, csrc/kitti_eval.cu) on a seeded
synthetic set the size of KITTI val: 3769 frames, 8 ground truths and 50 detections per frame.

    python tools/kitti_eval_times.py [--frames 3769] [--gt 8] [--dt 50] [--repeats 3] [--out kitti_eval_times.json]

Reports conversion (detections -> annos, including the device-to-host copy), the three overlap passes, and the
official and COCO evaluations (each end to end: packing, copies, kernels, formatting), with the card's name and power
limit read in the same run and the SM clock sampled during it.  Needs a CUDA device.
"""
import argparse
import os

import _measure
import numpy as np
import torch


def synthetic(frames, n_gt, n_dt, seed=0):
    rng = np.random.default_rng(seed)
    names = np.array(["Car", "Car", "Pedestrian", "Cyclist", "Van", "DontCare"])
    gts, dts, dets = [], [], []
    for f in range(frames):
        loc = np.stack([rng.uniform(-15, 15, n_gt), rng.uniform(1.4, 1.9, n_gt), rng.uniform(5, 50, n_gt)], 1)
        dims = np.stack([rng.uniform(0.6, 4.5, n_gt), rng.uniform(1.4, 1.9, n_gt), rng.uniform(0.5, 1.9, n_gt)], 1)
        u, h = 610 + 720 * loc[:, 0] / loc[:, 2], 720 * dims[:, 1] / loc[:, 2]
        bbox = np.stack([u - h, 180 - h, u + h, 180 + 0 * h], 1)
        g = {"name": rng.choice(names, n_gt), "bbox": bbox, "location": loc, "dimensions": dims,
             "rotation_y": rng.uniform(-3, 3, n_gt), "alpha": rng.uniform(-3, 3, n_gt),
             "truncated": rng.choice([0.0, 0.2, 0.4], n_gt), "occluded": rng.integers(0, 3, n_gt)}
        pick = rng.integers(0, n_gt, n_dt)
        d = {k: (v[pick].copy() if k != "name" else rng.choice(names[:4], n_dt)) for k, v in g.items()}
        d["location"] += rng.normal(0, 0.3, d["location"].shape)
        d["bbox"] += rng.normal(0, 5, d["bbox"].shape)
        d["score"] = rng.uniform(0, 1, n_dt).astype(np.float32)
        gts.append(g)
        dts.append(d)
        box = np.concatenate([rng.uniform(0, 60, (n_dt, 1)), rng.uniform(-30, 30, (n_dt, 1)), rng.uniform(-2, 0, (n_dt, 1)),
                              rng.uniform(1.5, 2, (n_dt, 1)), rng.uniform(3.5, 4.5, (n_dt, 1)),
                              rng.uniform(1.4, 1.7, (n_dt, 1)), rng.uniform(-3, 3, (n_dt, 1))], 1)
        dets.append({"box3d_lidar": torch.from_numpy(box.astype(np.float32)).cuda(),
                     "scores": torch.from_numpy(d["score"]).cuda(),
                     "label_preds": torch.from_numpy(rng.integers(0, 3, n_dt)).cuda(), "metadata": {"image_idx": f}})
    return gts, dts, dets


def timed(fn, repeats):
    """median of CUDA-event times of single calls of fn() (ms), after one warm-up call."""
    fn()
    return float(np.median([_measure.timed(fn, 1, warmup=0) for _ in range(repeats)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3769)
    ap.add_argument("--gt", type=int, default=8)
    ap.add_argument("--dt", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _measure.require_gpu("kitti_eval_times")
    from b2second import kitti_eval as ke, loader
    loader.product_spconv()
    gts, dts, dets = synthetic(args.frames, args.gt, args.dt)
    P2 = np.array([[721.5377, 0, 609.5593, 44.85728], [0, 721.5377, 172.854, 0.2163791], [0, 0, 1, 0.002745884],
                   [0, 0, 0, 1]])
    Tr = np.eye(4)
    Tr[:3, :] = [[0, -1, 0, 0], [0, 0, -1, -0.08], [1, 0, 0, -0.27]]
    infos = [{"calib": {"R0_rect": np.eye(4), "Tr_velo_to_cam": Tr, "P2": P2},
              "image": {"image_idx": i, "image_shape": np.array([375, 1242])}} for i in range(args.frames)]
    classes = [0, 1, 2]
    res = {}
    with _measure.clocks() as clk:
        res["convert_ms"] = timed(lambda: ke.convert_detection_to_kitti_annos(dets, infos, ["Car", "Pedestrian",
                                                                                           "Cyclist"]), args.repeats)
        packed = ke._Packed(gts, dts, 1, 1.0, "cuda")
        for metric in range(3):
            def ov(metric=metric):
                packed._ov.pop(metric, None)
                packed.overlaps(metric)
            res["overlaps_m%d_ms" % metric] = timed(ov, args.repeats)
        res["official_ms"] = timed(lambda: ke.get_official_eval_result(gts, dts, classes), args.repeats)
        res["coco_ms"] = timed(lambda: ke.get_coco_eval_result(gts, dts, classes), args.repeats)
    line = _measure.report("kitti_eval_times", res, clk, frames=args.frames, gt_per_frame=args.gt,
                           dt_per_frame=args.dt, repeats=args.repeats)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
