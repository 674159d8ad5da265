"""CUDA-event time of TargetPlan.assign_batch (csrc/targets.cu): python tools/target_assign_times.py [iters]

Prints one JSON line.  Per (config, batch, GTs per frame): milliseconds per call (the GT kernel and both passes, plus
the few small torch ops assign_batch issues), the algorithmic bytes -- 16 B per anchor read (the anchor's similarity
row; thresholds and the box encode only touch positives' neighbours), (8 + 4 * code) B per anchor and frame written
(label, importance, box target) -- the write floor at the H100 SXM data-sheet 3.35 TB/s (arithmetic, not a
measurement), and the anchor-GT pair evaluations (two per pair: one per pass).  GTs are drawn around random anchors.
"""
import sys

import _measure
import numpy as np
import torch

from b2second import config, models, targets

HBM_BYTES_PER_S = 3.35e12


def frames(plan, B, G, dtype, rng):
    a = plan.anchors[rng.integers(0, plan.num_anchors, B * G)].astype(np.float64)
    a[:, :2] += rng.uniform(-1.0, 1.0, (B * G, 2))
    a[:, 3:6] *= rng.uniform(0.85, 1.15, (B * G, 3))
    a[:, 6] = rng.uniform(-np.pi, np.pi, B * G)
    cls = rng.integers(1, len(plan.classes) + 1, B * G).astype(np.int32)
    dev = "cuda:0"
    return (torch.from_numpy(a.astype(dtype)).to(dev), torch.arange(0, B * G + 1, G, dtype=torch.int32, device=dev),
            torch.from_numpy(cls).to(dev))


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    _measure.require_gpu("target_assign_times")
    rng = np.random.default_rng(0)
    rows = []
    with _measure.clocks() as clk:
        for name, dtype in (("car.fhd", np.float32), ("all.fhd", np.float32), ("nuscenes.all.pp.largea", np.float64)):
            cfg = config.get_config(name)
            plan = targets.plan(models.MirrorTargetAssigner(cfg), cfg.feature_map_size)
            A = plan.num_anchors
            for B in (8, 32):
                for G in (30, 200):
                    gt, offs, cls = frames(plan, B, G, dtype, rng)
                    ms = _measure.timed(lambda: plan.assign_batch(gt, offs, cls), ITERS)
                    written = B * A * (8 + 4 * plan.code_size)
                    # pairs: each anchor against its segment's GTs of the frame (per class in per-class mode)
                    seg_of = (cls - 1).cpu().numpy() if plan.assign_per_class else np.zeros(B * G, np.int64)
                    pairs = 0
                    for b in range(B):
                        counts = np.bincount(seg_of[b * G:(b + 1) * G], minlength=len(plan.segments))
                        pairs += sum(int(counts[i]) * (s.end - s.begin) for i, s in enumerate(plan.segments))
                    rows.append({"config": name, "batch": B, "gt_per_frame": G, "anchors": A,
                                 "gt_dtype": np.dtype(dtype).name, "ms": round(ms, 4), "bytes_read": 16 * A,
                                 "bytes_written": written,
                                 "write_floor_ms": round(written / HBM_BYTES_PER_S * 1e3, 4),
                                 "pair_evaluations": 2 * pairs})
    _measure.report("target_assign_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
