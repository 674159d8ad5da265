"""Generate tests/golden/metrics/*.npz FROM THE UNMODIFIED REFERENCE (needs the reference tree; runs on the CPU).

    python tests/golden/make_metrics_golden.py [--force]

For car.fhd (one class) and nuscenes.all.pp.mhead (ten classes) the reference's own builders make the VoxelNet, its
metric buffers are preset near 2^24 (tests/metrics_ref.state0) and its unmodified ``update_metrics``
(second/pytorch/models/voxelnet.py:654-679) runs on the seeded steps of tests/metrics_ref.make_steps.  Each file holds,
per step s: the inputs (s_cls_preds, s_labels, s_cared, s_cls_loss, s_loc_loss), the running buffers after the step
(s_<buffer>, tests/metrics_ref.BUFFERS) and the returned dict (s_dict_json); and the preset state (init_<buffer>).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))
OUT = os.path.join(HERE, "metrics")

import metrics_ref as mr  # noqa: E402
from b2second import config, loader, refcompat  # noqa: E402

CASES = {"car.fhd": (11, 2, 512), "nuscenes.all.pp.mhead": (12, 2, 256)}     # name: (seed, batch, anchors)

_MAP = {"acc_total": ("rpn_acc", "total"), "acc_count": ("rpn_acc", "count"),
        "prec_total": ("rpn_metrics", "prec_total"), "prec_count": ("rpn_metrics", "prec_count"),
        "rec_total": ("rpn_metrics", "rec_total"), "rec_count": ("rpn_metrics", "rec_count"),
        "cls_total": ("rpn_cls_loss", "total"), "cls_count": ("rpn_cls_loss", "count"),
        "loc_total": ("rpn_loc_loss", "total"), "loc_count": ("rpn_loc_loss", "count")}


def buffers(net):
    """the reference network's running buffers under tests/metrics_ref.BUFFERS' names"""
    return {k: getattr(getattr(net, m), b) for k, (m, b) in _MAP.items()}


def reference_network(name):
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    return refcompat.build_network(refcompat.load_config(f).model.second).train()


def main():
    refcompat.install(loader.ORACLE_DIR)
    force = "--force" in sys.argv
    os.makedirs(OUT, exist_ok=True)
    for name, (seed, batch, anchors) in CASES.items():
        path = os.path.join(OUT, name + ".npz")
        if os.path.exists(path) and not force:
            continue
        net = reference_network(name)
        C = int(net._num_class)
        fix = {"name": name, "num_class": np.int32(C)}
        init = mr.state0(net.rpn_metrics.thresholds)
        with torch.no_grad():
            for k, t in buffers(net).items():
                t.copy_(torch.from_numpy(init[k]))
        for k, v in init.items():
            fix["init_" + k] = v
        steps = mr.make_steps(seed, batch, anchors, C)
        for s, st in enumerate(steps):
            for k, v in st.items():
                fix["%d_%s" % (s, k)] = np.asarray(v)
            d = net.update_metrics(*mr.to_torch(st))
            for k, t in buffers(net).items():
                fix["%d_%s" % (s, k)] = t.detach().numpy().copy()
            fix["%d_dict_json" % s] = json.dumps(d, sort_keys=True)
        fix["steps"] = np.int32(len(steps))
        np.savez_compressed(path, **fix)
        print("->", os.path.relpath(path, HERE), os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main()
