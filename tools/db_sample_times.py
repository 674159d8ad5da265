"""CUDA-event time of DatabaseSampler.sample_batch (csrc/dbsample.cu): python tools/db_sample_times.py [iters]

Prints one JSON line.  Per config (car.fhd, nuscenes.all.pp.mhead) at batch 8 with a synthetic object database (400
objects per sampled class, 20 to 400 points each, written to a temporary directory): milliseconds per call on the
device (the candidates' host-to-device copy, four memsets and the kernels), the host time of ``draw`` for the batch,
and the database's device footprint; with the card, its power limit and the SM clock sampled during the run.  Frames
hold 20 k to 30 k points and 10 ground truths.  Where the reference tree is importable (refcompat), the same frames
also go through the reference's DataBaseSamplerV2.sample_all plus preprocess.py:224-249 (points_in_rbbox removal,
concatenation) on the host, one frame after another on one core.
"""
import os
import sys
import tempfile
import time

import _measure
import numpy as np
import torch

from b2second import config, dbsample, refcompat

B = 8


def database(cfg, root, rng):
    nus = cfg.name.startswith("nuscenes")
    r = np.asarray(cfg.point_cloud_range)
    infos = {}
    for key in [n for g in cfg.db_sampler.sample_groups for n in g]:
        lst = []
        for i in range(400):
            b = np.zeros(9 if nus else 7)
            b[:2] = rng.uniform(r[:2] + 2, r[3:5] - 2)
            b[2] = rng.uniform(-1.9, -1.2)
            b[3:6] = rng.uniform([1.5, 3.5, 1.4], [2.5, 8.0, 3.0])
            b[6] = rng.uniform(-np.pi, np.pi)
            n = int(rng.integers(20, 401))
            p = np.concatenate([rng.uniform(-0.45, 0.45, (n, 3)) * b[3:6], rng.random((n, cfg.num_point_features - 3))],
                               1).astype(np.float32)
            path = "%s_%d.bin" % (key, i)
            p.tofile(os.path.join(root, path))
            lst.append({"name": key, "path": path, "box3d_lidar": b.astype(np.float64 if nus else np.float32),
                        "difficulty": 0, "num_points_in_gt": n, "group_id": i})
        infos[key] = lst
    return infos


def frames(cfg, rng):
    nus = cfg.name.startswith("nuscenes")
    r = np.asarray(cfg.point_cloud_range)
    out = []
    for _ in range(B):
        b = np.zeros((10, 9 if nus else 7))
        b[:, :2] = rng.uniform(r[:2] + 2, r[3:5] - 2, (10, 2))
        b[:, 2] = -1.5
        b[:, 3:6] = [1.8, 4.2, 1.5]
        n = int(rng.integers(20000, 30001))
        pts = np.concatenate([rng.uniform(r[:3], r[3:], (n, 3)), rng.random((n, cfg.num_point_features - 3))],
                             1).astype(np.float32)
        out.append((pts, b.astype(np.float64 if nus else np.float32), np.array([cfg.classes[0].class_name] * 10)))
    return out


def reference_ms(cfg, infos, root, fr):
    refcompat.install(os.path.join(_measure.REPO, "oracle"))
    from second.core import box_np_ops
    from second.core.sample_ops import DataBaseSamplerV2
    np.random.seed(0)
    smp = DataBaseSamplerV2(infos, cfg.db_sampler.sample_groups, None, cfg.db_sampler.rate, [0.0, 0.0])
    for rep in range(2):                                   # the first pass compiles the numba kernels
        t0 = time.perf_counter()
        for pts, boxes, names in fr:
            sd = smp.sample_all(root, boxes, names, cfg.num_point_features)
            if sd is not None:
                if cfg.db_sampler.remove_points_after_sample:
                    pts = pts[np.logical_not(box_np_ops.points_in_rbbox(pts, sd["gt_boxes"]).any(-1))]
                pts = np.concatenate([sd["points"], pts])
        ms = (time.perf_counter() - t0) * 1e3
    return ms


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    _measure.require_gpu("db_sample_times")
    rng = np.random.default_rng(0)
    rows = []
    dev = "cuda:0"
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    with _measure.clocks() as clk:
        for name in ("car.fhd", "nuscenes.all.pp.mhead"):
            cfg = config.get_config(name)
            classes = [c.class_name for c in cfg.classes]
            with tempfile.TemporaryDirectory() as root:
                infos = database(cfg, root, rng)
                fr = frames(cfg, rng)
                ds = dbsample.sampler(cfg.db_sampler, infos, root, cfg.num_point_features, classes, dev,
                                      np.random.RandomState(0))
                names = [f[2] for f in fr]
                h0 = time.perf_counter()
                cand = dbsample.draw(np.random.RandomState(1), ds.state, names)
                draw_ms = (time.perf_counter() - h0) * 1e3
                P = np.concatenate([f[0] for f in fr])
                G = np.concatenate([f[1] for f in fr])
                args = (t(P), t(np.cumsum([0] + [len(f[0]) for f in fr]).astype(np.int32)), t(G),
                        t(np.arange(0, 10 * B + 1, 10, dtype=np.int32)), t(np.ones(10 * B, bool)),
                        t(np.ones(10 * B, np.int32)), None, cand)
                res = ds.sample_batch(*args)
                torch.cuda.synchronize()
                assert int(ds.last_status.item()) == 0
                nb, npts = res.counts()
                ms = _measure.timed(lambda: ds.sample_batch(*args), ITERS, warmup=2)
                row = {"config": name, "batch": B, "points_in": int(len(P)), "candidates": int(len(cand.objects)),
                       "accepted": int(res["accepted"].sum().item()), "points_out": int(sum(npts)),
                       "ms": round(ms, 4), "draw_host_ms": round(draw_ms, 3), "db_nbytes": ds.db.nbytes}
                if refcompat.reference_available():
                    row["reference_host_ms"] = round(reference_ms(cfg, infos, root, fr), 2)
                else:
                    row["reference_host_ms"] = "not measured (reference tree not importable here)"
                rows.append(row)
    _measure.report("db_sample_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
