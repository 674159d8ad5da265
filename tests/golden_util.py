"""helpers shared by the golden-fixture tests (CPU oracle path and GPU product path)."""
import glob
import hashlib
import os

import numpy as np

from b2second import config, synth

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def cases():
    """(config name, seed, num_points, fixture path); fixtures named <config>.seed<S>.n<P>[.mv<max_voxels>].npz"""
    import re
    out = []
    for p in sorted(glob.glob(os.path.join(GOLDEN_DIR, "*.npz"))):
        m = re.match(r"^(.*)\.seed(\d+)\.n(\d+)(?:\.mv(\d+))?$", os.path.basename(p)[:-4])
        out.append((m.group(1), int(m.group(2)), int(m.group(3)), p))
    return out


def max_voxels_of(fix, name):
    """the voxel cap the fixture was generated with (older fixtures: the config's own)."""
    return int(fix["max_voxels"]) if "max_voxels" in fix else config.get_config(name).max_voxels


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def make_cloud(name, seed, n):
    cfg = config.get_config(name)
    if "nuscenes" in name:
        return synth.nuscenes_cloud(seed, n)
    return synth.kitti_cloud(seed, n, cfg.point_cloud_range)


def border_cloud(cfg, F, seed, n=2000):
    """points on the first and last row and column of the voxel grid (hence of the BEV map), z mid-range"""
    rng = np.random.default_rng(seed)
    r, vs = np.asarray(cfg.point_cloud_range, np.float64), np.asarray(cfg.voxel_size, np.float64)
    pts = np.zeros((n, F), np.float32)
    side = np.arange(n) % 4
    t = rng.random(n)
    x = r[0] + t * (r[3] - r[0])
    y = r[1] + t * (r[4] - r[1])
    x = np.where(side == 0, r[0] + 0.25 * vs[0], np.where(side == 1, r[3] - 0.25 * vs[0], x))
    y = np.where(side == 2, r[1] + 0.25 * vs[1], np.where(side == 3, r[4] - 0.25 * vs[1], y))
    pts[:, 0], pts[:, 1] = x, y
    pts[:, 2] = 0.5 * (r[2] + r[5]) + 0.25 * (r[5] - r[2]) * (rng.random(n) - 0.5)
    pts[:, 3:] = rng.random((n, F - 3))
    return pts


def assert_detections_close(got, fix, box_tol=1e-4, score_tol=1e-5):
    gb = np.asarray(got["box3d_lidar"], dtype=np.float32)
    gs = np.asarray(got["scores"], dtype=np.float32)
    gl = np.asarray(got["label_preds"]).astype(np.int64)
    rb, rs, rl = fix["box3d_lidar"], fix["scores"], fix["label_preds"]
    assert gb.shape == rb.shape, "detection count differs: got %d, golden %d" % (gb.shape[0], rb.shape[0])
    np.testing.assert_allclose(gs, rs, rtol=0, atol=score_tol)
    # detections arrive in descending score order; among (numerically) EQUAL scores the order is whatever torch.topk /
    # the sort produced -- unspecified upstream -- so rows inside a run of tied scores are matched by nearest centre
    order = np.arange(len(rs))
    i = 0
    while i < len(rs):
        j = i + 1
        while j < len(rs) and abs(float(rs[j]) - float(rs[i])) <= 2 * score_tol:
            j += 1
        if j - i > 1:
            free = list(range(i, j))
            for a in range(i, j):
                k = min(free, key=lambda q: float(np.abs(gb[q, :3] - rb[a, :3]).sum()))
                free.remove(k)
                order[a] = k
        i = j
    gb, gs, gl = gb[order], gs[order], gl[order]
    # labels: argmax over class logits; only decided where the top-2 logit margin is above fp32 noise
    decided = np.asarray(fix["label_margin"]) > 1e-3 if "label_margin" in fix else np.ones(rl.shape, bool)
    np.testing.assert_array_equal(gl[decided], rl[decided])
    # The bar (BASELINE.json north_star) is 1e-4 on the box REGRESSION outputs.  The decode
    # (box_torch_ops.py:56-102) multiplies them by the anchor: x = xt*diag + xa, z = zt*h + za, w = exp(wt)*wa ...,
    # so a decoded coordinate may move by 1e-4 * max(1, diag, h) of its own box (NuScenes buses: diag ~ 12 m),
    # plus 2e-5 relative for fp32 rounding of the decoded magnitude (|x| ~ 70 m).
    scale = np.maximum(1.0, np.maximum(np.hypot(rb[:, 3], rb[:, 4]), rb[:, 5]))[:, None]
    err = np.abs(gb[:, :6] - rb[:, :6])
    bound = 2e-5 * np.abs(rb[:, :6]) + box_tol * scale
    bad = err > bound
    assert not bad.any(), "decoded boxes differ: %d elements, worst %g (bound %g)" % (
        int(bad.sum()), float((err - bound).max() + bound[np.unravel_index(np.argmax(err - bound), err.shape)]),
        float(bound[np.unravel_index(np.argmax(err - bound), err.shape)]))
    # angles are compared modulo 2*pi (direction fix-up adds multiples of the period)
    d = np.abs(gb[:, 6] - rb[:, 6])
    d = np.minimum(d, np.abs(d - 2 * np.pi))
    assert d.max(initial=0.0) < box_tol * 10, "yaw mismatch %g" % d.max()
