"""Anchor-area mask on the GPU (csrc/anchor_mask.cu through b2s_anchor_area_mask) against what the unmodified
reference's prep_pointcloud produced (tests/golden/anchor_mask, make_anchor_mask_golden.py): the mask bit for bit, and
the fused engine's detections with the mask computed inside its CUDA graph.  Bars: indices exact, boxes <=
1e-4 * max(1, diag, h), scores <= 1e-5 (golden_util.assert_detections_close)."""
import glob
import os
import re

import numpy as np
import pytest
import torch

import anchor_mask_ref
import golden_util as gu
from b2second import anchor_mask, config, fastpath, inputs, models, synth

pytestmark = pytest.mark.gpu
FIXTURES = sorted(glob.glob(os.path.join(gu.GOLDEN_DIR, "anchor_mask", "*.npz")))
IDS = [os.path.basename(p)[:-4] for p in FIXTURES]


@pytest.fixture(autouse=True)
def _fp32_convs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _case(path):
    m = re.match(r"^(.*)\.seed(\d+)\.n(\d+)(?:\.mv\d+)?\.npz$", os.path.basename(path))
    return m.group(1), int(m.group(2)), int(m.group(3))


def _cloud(name, seed, n):
    cfg = config.get_config(name)
    return synth.nuscenes_cloud(seed, n) if "nuscenes" in name else synth.kitti_cloud(seed, n, cfg.point_cloud_range)


def _net(name, product):
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    return net.cuda()


def _voxel_example(net, pts, max_voxels, batch_index=0):
    res = net.voxel_generator.generate(pts, max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)), constant_values=batch_index)
    return res, {"voxels": torch.from_numpy(res["voxels"]).cuda(),
                 "num_points": torch.from_numpy(res["num_points_per_voxel"]).cuda(),
                 "coordinates": torch.from_numpy(coords).cuda()}


def _fixture_mask(fix):
    return torch.from_numpy(np.unpackbits(fix["mask_packed"])[:int(fix["num_anchors"])].astype(bool))


def _dets(out):
    return {k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()}


def _nomask(fix):
    return {k: fix["nomask_" + k] for k in ("box3d_lidar", "scores", "label_preds", "label_margin")}


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_kernel_mask_bit_exact_single_frame(product, path):
    fix = np.load(path)
    name, seed, n = _case(path)
    cfg = config.get_config(name)
    net = _net(name, product)
    res, ex = _voxel_example(net, _cloud(name, seed, n), int(fix["max_voxels"]))
    assert res["voxel_num"] == int(fix["voxel_num"]) and gu.sha(res["coordinates"]) == str(fix["coords_sha1"])
    got = inputs.anchor_area_mask(ex["coordinates"], 1, net.anchors(), cfg.voxel_size, cfg.point_cloud_range,
                                  cfg.grid_size, float(fix["threshold"]))
    assert got.dtype == torch.bool and got.shape == (1, int(fix["num_anchors"]))
    assert torch.equal(got[0].cpu(), _fixture_mask(fix))


@pytest.mark.parametrize("name", ["pointpillars.car.xyres_16", "car.fhd", "nuscenes.all.pp.mhead"])
def test_kernel_mask_bit_exact_batch_of_four_with_empty_frame(product, name):
    """B = 4: two different fixture clouds, an empty frame, the first cloud again -- frames are independent"""
    paths = [p for p in FIXTURES if _case(p)[0] == name][:2]
    fixes = [np.load(p) for p in paths]
    cfg = config.get_config(name)
    net = _net(name, product)
    coords, want = [], []
    for b, (p, fix) in enumerate(zip(paths + [None, paths[0]], fixes + [None, fixes[0]])):
        if p is None:
            want.append(torch.zeros(int(fixes[0]["num_anchors"]), dtype=torch.bool))
            continue
        _, ex = _voxel_example(net, _cloud(*_case(p)), int(fix["max_voxels"]), batch_index=b)
        coords.append(ex["coordinates"])
        want.append(_fixture_mask(fix))
    thr = float(fixes[0]["threshold"])
    assert all(float(f["threshold"]) == thr for f in fixes)
    got = inputs.anchor_area_mask(torch.cat(coords, 0), 4, torch.from_numpy(net.anchors()).cuda(), cfg.voxel_size,
                                  cfg.point_cloud_range, cfg.grid_size, thr)
    assert torch.equal(got.cpu(), torch.stack(want, 0))
    assert not got[2].any()


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_engine_computes_the_mask_for_points_and_voxels(product, path):
    """net(example) with raw points, and with the voxel dict without a mask, matches the reference's masked
    detections; the engine's mask is the fixture's; graph replay is stable; status stays clean"""
    fix = np.load(path)
    name, seed, n = _case(path)
    pts = _cloud(name, seed, n)
    mv = int(fix["max_voxels"])
    net = fastpath.accelerate(_net(name, product), max_points=max(n, 1000), max_voxels=mv,
                              anchor_area_threshold=float(fix["threshold"]))
    anchors = torch.from_numpy(net.anchors()[None]).cuda()
    ex = {"points": [torch.from_numpy(pts).cuda()], "anchors": anchors}
    out = net(ex)[0]
    eng = net.b2s_fastpath.engines[1]
    assert torch.equal(eng.anchors_mask[0].cpu().bool(), _fixture_mask(fix))
    gu.assert_detections_close(_dets(out), fix)
    again = net(ex)[0]
    assert torch.equal(again["box3d_lidar"], out["box3d_lidar"]) and torch.equal(again["scores"], out["scores"])
    assert eng.check_status() & ~1 == 0
    # the reference's own dict without anchors_mask: the engine computes it from the caller's coordinates
    _, vex = _voxel_example(net, pts, mv)
    vex["anchors"] = anchors
    vout = net(vex)[0]
    assert torch.equal(eng.anchors_mask[0].cpu().bool(), _fixture_mask(fix))
    gu.assert_detections_close(_dets(vout), fix)
    assert eng.check_status() & ~1 == 0
    # the mask has teeth: without it the reference returns other detections, and so does an engine given all-ones
    nm = _nomask(fix)
    assert nm["box3d_lidar"].shape != fix["box3d_lidar"].shape or not np.array_equal(nm["box3d_lidar"], fix["box3d_lidar"])
    ones = dict(vex, anchors_mask=torch.ones(1, int(fix["num_anchors"]), dtype=torch.bool, device="cuda"))
    gu.assert_detections_close(_dets(net(ones)[0]), nm)
    # and back: the computed-mask graph is still there and still right
    gu.assert_detections_close(_dets(net(ex)[0]), fix)
    assert len(eng._graphs) == 3


def test_example_mask_overrides_the_computed_one(product):
    path = [p for p in FIXTURES if _case(p)[0] == "pointpillars.car.xyres_16"][0]
    fix = np.load(path)
    name, seed, n = _case(path)
    net = fastpath.accelerate(_net(name, product), max_points=n, anchor_area_threshold=1)
    anchors = torch.from_numpy(net.anchors()[None]).cuda()
    g = torch.Generator().manual_seed(5)
    given = (torch.rand(1, anchors.shape[1], generator=g) < 0.5).cuda()
    pts = [torch.from_numpy(_cloud(name, seed, n)).cuda()]
    out = net({"points": pts, "anchors": anchors, "anchors_mask": given})[0]
    eng = net.b2s_fastpath.engines[1]
    assert torch.equal(eng.anchors_mask.bool(), given)
    # the same result as an engine without the threshold given the same mask
    plain = fastpath.accelerate(_net(name, product), max_points=n)
    ref = plain({"points": pts, "anchors": anchors, "anchors_mask": given})[0]
    assert torch.equal(out["box3d_lidar"], ref["box3d_lidar"]) and torch.equal(out["scores"], ref["scores"])


@pytest.mark.parametrize("name", ["pointpillars.car.xyres_16", "car.fhd"])
def test_cropped_points_mask_equals_oracle_over_engine_coordinates(product, name):
    """points + crop_planes: the crop changes the cloud, so the check is the engine's mask against the oracle mask over
    the engine's own voxel coordinates of the cropped clouds (B = 2)"""
    from test_inputs import kitti_calib, raw_kitti_cloud
    cfg = config.get_config(name)
    P2, rect, Trv2c, shape = kitti_calib()
    planes = inputs.frustum_planes(rect, Trv2c, P2, shape)
    net = fastpath.accelerate(_net(name, product), max_points=60000, anchor_area_threshold=1)
    anchors = torch.from_numpy(net.anchors()[None]).cuda()
    clouds = [torch.from_numpy(raw_kitti_cloud(s, 12000)).cuda() for s in (4, 5)]
    net({"points": clouds, "crop_planes": planes, "anchors": anchors})
    eng = net.b2s_fastpath.engines[2]
    nv = int(eng.num_voxels[0].item())
    coors = eng.vox_coors[:nv].cpu().numpy()
    boxes = anchor_mask.anchor_boxes(net.anchors(), cfg.voxel_size, cfg.point_cloud_range, cfg.grid_size)
    want = anchor_mask_ref.anchor_area_mask_np(coors, 2, boxes, cfg.grid_size, 1.0)
    got = eng.anchors_mask.cpu().numpy().astype(bool)
    assert 0 < got.sum() < got.size and np.array_equal(got, want)
    assert eng.check_status() & ~1 == 0


@pytest.mark.parametrize("name", ["pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"])
def test_threshold_off_is_the_default_engine(product, name):
    from b2second.engine import InferenceEngine
    pts = _cloud(name, 0, 20000)
    net = _net(name, product)
    outs, launches = [], []
    for kw in ({}, {"anchor_area_threshold": None}, {"anchor_area_threshold": -1}):
        eng = InferenceEngine(net, batch_size=1, max_points=20000, **kw)
        eng.infer([torch.from_numpy(pts).cuda()])
        outs.append(eng.detections()[0])
        launches.append(eng.kernel_launches_per_step())
        assert eng.anchors_mask is None and not eng.use_mask
    assert launches[0] == launches[1] == launches[2]
    for o in outs[1:]:
        assert torch.equal(o["box3d_lidar"], outs[0]["box3d_lidar"]) and torch.equal(o["scores"], outs[0]["scores"])
    on = InferenceEngine(net, batch_size=1, max_points=20000, anchor_area_threshold=1)
    assert on.kernel_launches_per_step() == launches[0] + 4

