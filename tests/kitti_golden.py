"""Load the KITTI evaluation fixtures (tests/golden/kitti_eval, make_kitti_eval_golden.py and
make_kitti_edges_golden.py) back into anno dicts."""
import glob
import os

import numpy as np

import golden_util as gu

DIR = os.path.join(gu.GOLDEN_DIR, "kitti_eval")
EVAL_FIXTURES = sorted(glob.glob(os.path.join(DIR, "eval.*.npz")))
EVAL_IDS = [os.path.basename(p)[:-4] for p in EVAL_FIXTURES]
# scenes on the evaluation's decision edges (make_kitti_edges_golden.py)
EDGE_FIXTURES = sorted(glob.glob(os.path.join(DIR, "edges.*.npz")))
EDGE_IDS = [os.path.basename(p)[:-4] for p in EDGE_FIXTURES]
CONVERT_FIXTURE = os.path.join(DIR, "convert.car_fhd.npz")
KEYS = ("name", "bbox", "location", "dimensions", "rotation_y", "alpha", "truncated", "occluded", "score")


def annos(fix, prefix):
    off = fix[prefix + "offsets"]
    keys = [k for k in KEYS if prefix + k in fix.files]
    out = []
    for lo, hi in zip(off[:-1], off[1:]):
        a = {k: fix[prefix + k][lo:hi] for k in keys}
        a["occluded"] = a["occluded"].astype(np.int64)
        out.append(a)
    return out


def load(path):
    fix = np.load(path, allow_pickle=False)
    return fix, annos(fix, "gt_"), annos(fix, "dt_")
