"""CUDA-event time of AugmentPlan.augment_batch (csrc/augment.cu): python tools/augment_times.py [iters]

Prints one JSON line.  Per (config, batch, GTs per frame): milliseconds per call on the device (the draws' host-to-device
copies, one memset and the three kernels), the bytes the call must move (points read and written, boxes, the draws
read) and their floor at the H100 SXM data-sheet 3.35 TB/s (arithmetic, not a measurement), and separately the host time
of ``draw`` for the same batch.  Frames hold 20 k to 30 k points, half of them in and around the boxes.
"""
import sys
import time

import _measure
import numpy as np
import torch

from b2second import augment, config

HBM_BYTES_PER_S = 3.35e12


def batch(cfg, B, G, rng):
    r = np.asarray(cfg.point_cloud_range)
    nus = cfg.name.startswith("nuscenes")
    pts, boxes, npts = [], [], []
    for _ in range(B):
        b = np.zeros((G, 9 if nus else 7))
        b[:, :2] = rng.uniform(r[:2] + 2, r[3:5] - 2, (G, 2))
        b[:, 2] = rng.uniform(-2, -1, G)
        b[:, 3:6] = rng.uniform([1.5, 3.5, 1.4], [2.0, 4.6, 1.8], (G, 3))
        b[:, 6] = rng.uniform(-np.pi, np.pi, G)
        if nus:
            b[:, 7:] = rng.normal(0, 3, (G, 2))
        n = int(rng.integers(20000, 30001))
        near = b[rng.integers(0, G, n // 2)]
        p_in = near[:, :3] + rng.uniform(-0.7, 0.7, (n // 2, 3)) * near[:, 3:6]
        p_bg = rng.uniform(r[:3], r[3:], (n - n // 2, 3))
        xyz = np.concatenate([p_in, p_bg])
        pts.append(np.concatenate([xyz, rng.random((n, 2 if nus else 1))], 1).astype(np.float32))
        boxes.append(b.astype(np.float64 if nus else np.float32))
        npts.append(n)
    dev = "cuda:0"
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    P = np.concatenate(pts)
    Bx = np.concatenate(boxes)
    args = (t(P), t(np.cumsum([0] + npts).astype(np.int32)), t(Bx), t(np.arange(0, B * G + 1, G, dtype=np.int32)),
            t(np.ones(B * G, bool)), t(np.ones(B * G, np.int32)))
    return args, npts, P.nbytes, Bx.nbytes


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    _measure.require_gpu("augment_times")
    rng = np.random.default_rng(0)
    rows = []
    with _measure.clocks() as clk:
        for name in ("car.fhd", "nuscenes.all.pp.largea"):
            cfg = config.get_config(name)
            plan = augment.plan(cfg.augment, cfg.point_cloud_range, [c.class_name for c in cfg.classes])
            for B in (8, 32):
                for G in (30, 200):
                    args, npts, pbytes, bbytes = batch(cfg, B, G, rng)
                    rs = np.random.RandomState(0)
                    h0 = time.perf_counter()
                    draws = [augment.draw(rs, cfg.augment, [G] * B, npts) for _ in range(3)]
                    draw_ms = (time.perf_counter() - h0) * 1e3 / 3
                    ms = _measure.timed(lambda: plan.augment_batch(*args, None, draws[0]), ITERS)
                    assert int(plan.last_status.item()) == 0
                    draw_bytes = (B * G * 100 * 32 if plan.object_noise else 0) + B * 64 + \
                        (4 * sum(npts) if cfg.augment.shuffle_points else 0)
                    moved = 2 * pbytes + 2 * bbytes + draw_bytes
                    rows.append({"config": name, "batch": B, "gt_per_frame": G, "points": int(sum(npts)),
                                 "box_dtype": "float64" if name.startswith("nuscenes") else "float32",
                                 "object_noise": plan.object_noise, "ms": round(ms, 4),
                                 "draw_host_ms": round(draw_ms, 3),
                                 "bytes_moved": moved, "hbm_floor_ms": round(moved / HBM_BYTES_PER_S * 1e3, 4)})
    _measure.report("augment_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
