"""This repository against what the UNMODIFIED reference (second.pytorch) produced, stored under tests/golden/reference by
tests/golden/make_reference_golden.py:
  * the hand-written config dataclasses equal the parsed reference config files
  * the mirror network has the reference's state-dict keys/shapes and anchors bit for bit, and gives the reference's
    detections on the oracle
  * the fused engine plans the mirror exactly as it planned the reference network
  * the per-class NMS branch gives the reference's detections
"""
import dataclasses
import gzip
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from b2second import config, models, synth
from conftest import REPO

GOLDEN = os.path.join(REPO, "tests", "golden")


@pytest.fixture(scope="module")
def golden():
    with gzip.open(os.path.join(GOLDEN, "reference", "reference.json.gz"), "rt") as f:
        g = json.load(f)
    with np.load(os.path.join(GOLDEN, "reference", "reference.npz")) as z:
        g["arrays"] = {k: z[k] for k in z.files}
    return g


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("name", sorted(config.BUILTIN))
def test_builtin_config_equals_reference_file(golden, name):
    import sys
    sys.path.insert(0, GOLDEN)
    from make_reference_golden import as_json
    parsed = golden["configs"][name]
    builtin = config.get_config(name)
    assert set(parsed) == set(builtin.__dataclass_fields__)
    for f in builtin.__dataclass_fields__:
        assert as_json(getattr(builtin, f)) == parsed[f], f


@pytest.mark.parametrize("name", ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea"])
def test_mirror_equals_reference_network(golden, oracle, name):
    ref = golden["networks"][name]
    mine = models.build_network(name, oracle).eval()
    sd_r, sd_m = ref["state_dict"], mine.state_dict()
    assert set(sd_m) <= set(sd_r)
    assert all(k.split(".")[0].startswith("rpn_") for k in set(sd_r) - set(sd_m))   # training metric buffers only
    for k in sd_m:
        assert [list(sd_m[k].shape), str(sd_m[k].dtype)] == sd_r[k], k
    models.synthetic_weights_(mine, name)
    a = mine.anchors()
    assert [list(a.shape), str(a.dtype), sha256(a)] == ref["anchors"]
    if name != "car.fhd":
        return                                                   # forward equality: one config is enough here
    b = config.get_config(name)
    pts = synth.kitti_cloud(4, 12000, b.point_cloud_range)
    res = mine.voxel_generator.generate(pts, b.max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    ex = {"anchors": torch.from_numpy(a[None].copy()), "voxels": torch.from_numpy(res["voxels"]),
          "num_points": torch.from_numpy(res["num_points_per_voxel"]), "coordinates": torch.from_numpy(coords)}
    with torch.no_grad():
        o_m = mine(ex)[0]
    r_box = torch.from_numpy(golden["arrays"]["forward.car.fhd.box3d_lidar"])
    r_lab = torch.from_numpy(golden["arrays"]["forward.car.fhd.label_preds"])
    assert r_box.shape == o_m["box3d_lidar"].shape and r_box.shape[0] > 0
    assert torch.allclose(r_box, o_m["box3d_lidar"], atol=1e-6)
    assert torch.equal(r_lab, o_m["label_preds"])


@pytest.mark.parametrize("name", sorted(config.BUILTIN))
def test_engine_plan_from_reference_network_equals_plan_from_mirror(golden, oracle, name):
    """b2second.spec reads a network through the reference's attribute names only, so the fused engine plans the
    mirror exactly as it planned the UNMODIFIED reference VoxelNet (second_builder.build): same layer list, folded
    BN constants, NMS / direction parameters, RPN weights and anchors -- for all five BASELINE configs."""
    import sys
    from b2second import spec, tc
    sys.path.insert(0, GOLDEN)
    from make_reference_golden import plan_digest, signature_json
    ref = golden["spec"][name]
    mine = models.build_network(name, oracle).eval()
    models.synthetic_weights_(mine, name)
    cfg = config.get_config(name)
    s_mine = spec.spec_from_module(mine, max_voxels=cfg.max_voxels)
    a, b = ref["signature"], signature_json(s_mine)
    assert set(a) == set(b)
    for k in a:
        assert a[k] == b[k], "spec field %s differs between the reference network and the mirror" % k
    fm = cfg.feature_map_size
    assert ref["anchors"] == sha256(spec.anchors_for(s_mine, (fm[1], fm[2])))
    # the RPN launch program is planned from the module tree, too
    assert plan_digest(tc.plan_rpn(mine.rpn, 64, 48)) == ref["plan"]


@pytest.mark.parametrize("name,agnostic", [("all.fhd", False), ("nuscenes.all.pp.largea", True)])
def test_multiclass_nms_branch_mirror_equals_reference(golden, oracle, name, agnostic):
    """the per-class NMS branch of predict() (voxelnet.py:458-547; off in the five BASELINE configs, SURVEY §8(f)3):
    the mirror with use_multi_class_nms switched on vs the UNMODIFIED reference network, on the CPU oracle."""
    b = dataclasses.replace(config.get_config(name), use_multi_class_nms=True, nms_class_agnostic=agnostic)
    mine = models.build_network(b, oracle).eval()
    models.synthetic_weights_(mine, name)
    a = mine.anchors()
    pts = synth.nuscenes_cloud(1, 40000) if "nuscenes" in name else synth.kitti_cloud(4, 12000, b.point_cloud_range)
    res = mine.voxel_generator.generate(pts, b.max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    ex = {"anchors": torch.from_numpy(a[None].copy()), "voxels": torch.from_numpy(res["voxels"]),
          "num_points": torch.from_numpy(res["num_points_per_voxel"]), "coordinates": torch.from_numpy(coords)}
    with torch.no_grad():
        o_m = mine(ex)[0]
    key = "multiclass.%s.%d." % (name, int(agnostic))
    r_box, r_lab, r_sc = (torch.from_numpy(golden["arrays"][key + k]) for k in ("box3d_lidar", "label_preds", "scores"))
    assert r_box.shape == o_m["box3d_lidar"].shape and r_box.shape[0] > 0
    assert len(set(r_lab.tolist())) > 1                                  # more than one class produced detections
    assert torch.allclose(r_box, o_m["box3d_lidar"], atol=1e-6)
    assert torch.equal(r_lab, o_m["label_preds"]) and torch.allclose(r_sc, o_m["scores"])
