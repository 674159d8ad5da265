"""The augmentation's random numbers, host against device: python tools/augment_draw_times.py [iters]

Prints one JSON line.  Per (config, batch, GTs per frame): the host-clock milliseconds of ``augment.draw`` (numpy, the
default) and the CUDA-event milliseconds of ``augment.DeviceDrawer.draw`` (csrc/augment_draws.cu) for the same frame
counts, the bytes the device call writes (loc_noise, rot_noise, frame, perm) and their floor at the H100 SXM
data-sheet 3.35 TB/s (arithmetic, not a measurement).  Frames hold 20 k to 30 k points, as in augment_times.py.
"""
import sys
import time

import _measure
import numpy as np
import torch

from b2second import augment, config

HBM_BYTES_PER_S = 3.35e12


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    _measure.require_gpu("augment_draw_times")
    rng = np.random.default_rng(0)
    dev = torch.device("cuda", 0)
    rows = []
    with _measure.clocks() as clk:
        for name in ("car.fhd", "nuscenes.all.pp.largea"):
            s = config.get_config(name).augment
            for B in (8, 32):
                for G in (30, 200):
                    npts = [int(v) for v in rng.integers(20000, 30001, B)]
                    goff = torch.arange(0, B * G + 1, G, dtype=torch.int32, device=dev)
                    poff = torch.tensor(np.cumsum([0] + npts), dtype=torch.int32, device=dev)
                    rs = np.random.RandomState(0)
                    augment.draw(rs, s, [G] * B, npts)
                    h0 = time.perf_counter()
                    for _ in range(3):
                        augment.draw(rs, s, [G] * B, npts)
                    host_ms = (time.perf_counter() - h0) * 1e3 / 3
                    dd = augment.DeviceDrawer(0, dev)
                    ms = _measure.timed(lambda: dd.draw(s, goff, poff, B * G, sum(npts)), ITERS)
                    noise = augment.object_noise_enabled(s)
                    written = (B * G * augment.NUM_TRY * 32 if noise else 0) + B * 64 + \
                        (4 * sum(npts) if s.shuffle_points else 0)
                    rows.append({"config": name, "batch": B, "gt_per_frame": G, "points": int(sum(npts)),
                                 "object_noise": noise, "shuffle": bool(s.shuffle_points),
                                 "draw_host_ms": round(host_ms, 3), "draw_device_ms": round(ms, 4),
                                 "speedup": round(host_ms / ms, 1), "bytes_written": written,
                                 "hbm_floor_ms": round(written / HBM_BYTES_PER_S * 1e3, 4)})
    _measure.report("augment_draw_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
