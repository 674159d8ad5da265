"""HBM bytes the car.fhd RPN spends on background pixels per step, from the bench clouds, on the CPU:
    python tools/rpn_band_bytes.py [batch]

The BEV occupancy is the voxel grid of each cloud (synth.kitti_cloud, seeds 0 .. batch-1, 29 000 points) taken through
the middle encoder's three k3 s2 pad-1 downsamples in y and x.  The strip plan and the bands are the numpy
restatements of b2s_rpn_strip_plan (8 x 4 strips, six layers) and b2s_rpn_strip_bands (tests/rpn_bands_ref.py).
Printed per step:
  - the BEV zero-fill of b2s_to_bev_tc (both planes) against b2s_to_bev_tc_ex (the pixels the previous step wrote,
    taken as this step's count, plus the occupancy map);
  - the fill stores of the six k_conv3x3_tc2 launches: every background strip, against the bands;
  - the fused tail's reads of layer 6: every tile, against the computed tiles.
A map is B x 200 x 176 pixels of 2 planes x 128 channels x 2 bytes."""
import sys

import _measure  # noqa: F401  (the path set-up)
import numpy as np
from rpn_bands_ref import strip_bands, strip_flags, tail_tiles

from b2second import config, synth

ROWS, LAYERS, PIXEL_BYTES = 4, 6, 2 * 128 * 2


def bev_occupancy(cfg, seed, points):
    pts = synth.kitti_cloud(seed, points, cfg.point_cloud_range)
    lo, vs = np.array(cfg.point_cloud_range[:3]), np.array(cfg.voxel_size)
    gx, gy = int(cfg.grid_size[0]), int(cfg.grid_size[1])
    idx = np.floor((pts[:, :3] - lo) / vs).astype(np.int64)
    ok = (idx[:, 0] >= 0) & (idx[:, 0] < gx) & (idx[:, 1] >= 0) & (idx[:, 1] < gy) & (idx[:, 2] >= 0) \
        & (idx[:, 2] < int(cfg.grid_size[2]))
    occ = np.zeros((gy, gx), bool)
    occ[idx[ok, 1], idx[ok, 0]] = True
    for _ in range(3):                                 # k3 s2 pad 1: output o reads inputs 2o-1, 2o, 2o+1
        h, w = (occ.shape[0] + 1) // 2, (occ.shape[1] + 1) // 2
        pad = np.pad(occ, ((1, 2), (1, 2)))
        out = np.zeros((h, w), bool)
        for dy in range(3):
            for dx in range(3):
                out |= pad[dy:dy + 2 * h:2, dx:dx + 2 * w:2]
        occ = out
    return occ


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    cfg = config.get_config("car.fhd")
    occ = np.stack([bev_occupancy(cfg, s, 29000) for s in range(B)]).astype(np.uint8)
    _, H, W = occ.shape
    flags = strip_flags(occ, LAYERS, ROWS)
    computed = [float(f.mean()) for f in flags]
    band = [float(b.mean()) for b in strip_bands(flags, ROWS)]
    tiles = float(tail_tiles(flags[-1], ROWS).mean())
    map_bytes = B * H * W * PIXEL_BYTES
    mb = lambda x: "%.0f MB" % (x / 1e6)
    print("B = %d, BEV %d x %d, data pixels %.1f %%, one map %s" % (B, H, W, 100 * occ.mean(), mb(map_bytes)))
    print("computed share per layer:", " ".join("%.3f" % c for c in computed))
    print("band share per layer:    ", " ".join("%.3f" % b for b in band))
    print("tail tiles computed:      %.3f" % tiles)
    zero_now = (B * (H + 2) * (W + 2)) * PIXEL_BYTES
    zero_new = occ.sum() * PIXEL_BYTES + occ.size
    print("BEV zero-fill     %s -> %s" % (mb(zero_now), mb(zero_new)))
    fill_now = sum(1.0 - c for c in computed) * map_bytes
    fill_new = sum(band) * map_bytes
    print("3x3 fill stores   %s (%.3f maps) -> %s (%.3f maps)" % (mb(fill_now), fill_now / map_bytes, mb(fill_new),
                                                                 fill_new / map_bytes))
    tail_now, tail_new = map_bytes, tiles * map_bytes           # the tail reads whole 8 x 16 tiles (edges: zero fill)
    print("tail reads of x   %s -> %s" % (mb(tail_now), mb(tail_new)))
    print("removed per step  %s" % mb(zero_now - zero_new + fill_now - fill_new + tail_now - tail_new))


if __name__ == "__main__":
    main()
