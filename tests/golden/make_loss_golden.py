"""Generate tests/golden/loss/*.npz FROM THE UNMODIFIED REFERENCE (needs the reference tree; runs on the CPU).

    python tests/golden/make_loss_golden.py [--force]

For each config the reference's own builders (b2second.refcompat.build_network) make the VoxelNet, and its unmodified
``loss`` (second/pytorch/models/voxelnet.py:239-312) runs in train() mode on the seeded synthetic batches of
tests/loss_ref.make_case (cases a-e, two frames each), followed by ``loss.backward()``.  The loss reads only the yaw of
the anchors, so no anchor map is built.  Each case runs twice: on the float32 inputs and on the same inputs as float64
(the reference's loss is dtype-generic, so that is a float64 oracle from the reference itself).

Inputs are regenerated from the seed; each file holds outputs only, per case c:
  ref32_c_scalars     float32 [6]: loss, cls_loss_reduced, loc_loss_reduced, dir_loss_reduced, cls_pos_loss, cls_neg_loss
  ref64_c_scalars     float64 [6]: the same in float64
  ref64_c_cls_loss, ref64_c_loc_loss, ref64_c_cared     the per-anchor outputs (float64, bool)
  ref64_c_grad_box_preds, ref64_c_grad_cls_preds, ref64_c_grad_dir_cls_preds     d loss / d preds (float64)
  ref32_c_dir_bins    int8 [B, A]: get_direction_target's float32 bins
and the loss settings b2second.loss.plan reads off the reference network (settings_json).
"""
import dataclasses
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))
OUT = os.path.join(HERE, "loss")

import loss_ref  # noqa: E402
from b2second import config, loader, loss, refcompat  # noqa: E402


def reference_network(name):
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    cfgp = refcompat.load_config(f)
    return refcompat.build_network(cfgp.model.second).train()


def run(net, example, preds, dtype):
    pr = {k: v.to(dtype).clone().requires_grad_() for k, v in preds.items()}
    ex = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in example.items()}
    r = net.loss(ex, pr)
    r["loss"].backward()
    return r, {k: pr[k].grad.detach().numpy() for k in pr}


def main():
    refcompat.install(loader.ORACLE_DIR)
    from second.pytorch.models.voxelnet import get_direction_target
    force = "--force" in sys.argv
    os.makedirs(OUT, exist_ok=True)
    for name in loss_ref.CONFIGS:
        path = os.path.join(OUT, name + ".npz")
        if os.path.exists(path) and not force:
            continue
        net = reference_network(name)
        s = loss.plan(net).settings
        fix = {"name": name, "settings_json": json.dumps(dataclasses.asdict(s), sort_keys=True)}
        for case in loss_ref.CASES:
            example, preds = loss_ref.case_inputs(name, case, s)
            r32, _ = run(net, example, preds, torch.float32)
            r64, g64 = run(net, example, preds, torch.float64)
            fix["ref32_%s_scalars" % case] = np.array([float(r32[k].detach()) for k in loss_ref.SCALARS], np.float32)
            fix["ref64_%s_scalars" % case] = np.array([float(r64[k].detach()) for k in loss_ref.SCALARS], np.float64)
            fix["ref64_%s_cls_loss" % case] = r64["cls_loss"].detach().numpy()
            fix["ref64_%s_loc_loss" % case] = r64["loc_loss"].detach().numpy()
            fix["ref64_%s_cared" % case] = r64["cared"].numpy()
            for k, g in g64.items():
                fix["ref64_%s_grad_%s" % (case, k)] = g
            bins = get_direction_target(example["anchors"], example["reg_targets"], dir_offset=net._dir_offset,
                                        num_bins=net._num_direction_bins).argmax(-1)
            fix["ref32_%s_dir_bins" % case] = bins.numpy().astype(np.int8)
            lab = example["labels"].numpy()
            print(name, case, "pos", int((lab > 0).sum()), "neg", int((lab == 0).sum()), "ignored",
                  int((lab < 0).sum()), "loss32 %.9g loss64 %.17g" % (fix["ref32_%s_scalars" % case][0],
                                                                       fix["ref64_%s_scalars" % case][0]), flush=True)
        np.savez_compressed(path, **fix)
        print("->", os.path.relpath(path, HERE), os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main()
