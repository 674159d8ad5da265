"""Anchor-area mask (second/data/preprocess.py:345-357), CPU side.

  * the float32 host boxes (b2second.anchor_mask) equal the reference's rbbox2d_to_near_bbox + fused_get_anchors_area
    arithmetic for every anchor of six configs (needs the reference tree; skipped without it);
  * the numpy oracle (tests/anchor_mask_ref.py) equals the reference's own numba functions on random coordinate sets,
    batch > 1 with an empty frame (needs the reference tree);
  * the oracle reproduces the mask of every fixture the reference's prep_pointcloud wrote (no reference needed).
"""
import glob
import os
import re

import numpy as np
import pytest

import anchor_mask_ref
import golden_util as gu
from b2second import anchor_mask, config, models, refcompat, synth

AM_DIR = os.path.join(gu.GOLDEN_DIR, "anchor_mask")
FIXTURES = sorted(glob.glob(os.path.join(AM_DIR, "*.npz")))
CONFIGS = ["pointpillars.car.xyres_16", "car.fhd", "car.lite", "all.fhd", "nuscenes.all.pp.largea",
           "nuscenes.all.pp.mhead"]
needs_reference = pytest.mark.skipif(not refcompat.reference_available(), reason="reference tree not present")


def _fixture_case(path):
    """<config>.seed<S>.n<P>[.mv<max_voxels>].npz -> (config, seed, num_points)"""
    m = re.match(r"^(.*)\.seed(\d+)\.n(\d+)(?:\.mv\d+)?\.npz$", os.path.basename(path))
    return m.group(1), int(m.group(2)), int(m.group(3))


def _fixture_name(path):
    return _fixture_case(path)[0]


def _reference_net(name):
    files = dict(config.REFERENCE_FILES, **getattr(config, "EXTRA_REFERENCE_FILES", {}))
    cfgp = refcompat.load_config(files[name])
    net = refcompat.build_network(cfgp.model.second).eval()
    return net, refcompat.generate_anchors(net, cfgp.model.second)


class _RecordingMap:
    """stands in for the dense map of fused_get_anchors_area's Python body: records the (row, col) of every read."""
    dtype = np.float32

    def __init__(self):
        self.reads = []

    def __getitem__(self, rc):
        self.reads.append((int(rc[0]), int(rc[1])))
        return np.float32(0)


def test_boxes_outside_the_grid_are_rejected():
    cfg = config.get_config("car.lite")
    a = np.zeros((2, 7), np.float32)
    a[:, 3:6] = 1.6, 3.9, 1.5
    a[1, 0] = -50.0                                   # left of point_cloud_range[0] = 0: x1 < 0 after the clamp
    with pytest.raises(ValueError, match="outside"):
        anchor_mask.anchor_boxes(a, cfg.voxel_size, cfg.point_cloud_range, cfg.grid_size)


@needs_reference
@pytest.mark.parametrize("name", CONFIGS)
def test_host_boxes_equal_reference_arithmetic(ref_env, name):
    from second.core import box_np_ops
    net, anchors = _reference_net(name)
    vg = net.voxel_generator
    bv_ref = box_np_ops.rbbox2d_to_near_bbox(anchors[:, [0, 1, 3, 4, 6]])
    bv = anchor_mask.near_bboxes(anchors)
    assert bv.dtype == bv_ref.dtype == np.float32 and np.array_equal(bv, bv_ref)
    rec = _RecordingMap()
    box_np_ops.fused_get_anchors_area.py_func(rec, bv_ref, vg.voxel_size, vg.point_cloud_range, vg.grid_size)
    r = np.array(rec.reads, np.int64).reshape(-1, 4, 2)   # per anchor: ID (y1,x1), IA (y0,x0), IB, IC
    ref_boxes = np.stack([r[:, 1, 1], r[:, 1, 0], r[:, 0, 1], r[:, 0, 0]], axis=1)
    got = anchor_mask.anchor_boxes(anchors, [float(x) for x in vg.voxel_size], [float(x) for x in vg.point_cloud_range],
                                   vg.grid_size)
    assert got.shape == (anchors.shape[0], 4)
    assert np.array_equal(got, ref_boxes), "%d of %d boxes differ" % (int((got != ref_boxes).any(1).sum()), got.shape[0])


def _random_coords(rng, grid, batch, n_per_frame, empty=()):
    """voxel coordinates (b, z, y, x), unique per frame, clustered so that anchor areas cover 0 .. dozens"""
    nx, ny, nz = grid
    out = []
    for b in range(batch):
        if b in empty:
            continue
        centres = rng.uniform([0, 0], [nx, ny], (12, 2))
        c = centres[rng.integers(0, 12, n_per_frame)] + rng.normal(0, [nx / 30, ny / 30], (n_per_frame, 2))
        x = np.clip(c[:, 0], 0, nx - 1).astype(np.int32)
        y = np.clip(c[:, 1], 0, ny - 1).astype(np.int32)
        z = rng.integers(0, nz, n_per_frame).astype(np.int32)
        f = np.unique(np.stack([np.full(n_per_frame, b, np.int32), z, y, x], 1), axis=0)
        out.append(f[rng.permutation(f.shape[0])])
    return np.concatenate(out, 0) if out else np.zeros((0, 4), np.int32)


@needs_reference
@pytest.mark.parametrize("name", ["pointpillars.car.xyres_16", "car.lite"])
def test_oracle_equals_reference_numba_functions(ref_env, name):
    from second.core import box_np_ops
    net, anchors = _reference_net(name)
    vg = net.voxel_generator
    grid = [int(g) for g in vg.grid_size]
    boxes = anchor_mask.anchor_boxes(anchors, vg.voxel_size, vg.point_cloud_range, grid)
    bv = box_np_ops.rbbox2d_to_near_bbox(anchors[:, [0, 1, 3, 4, 6]])
    rng = np.random.default_rng(7)
    B = 3
    coors = _random_coords(rng, grid, B, 6000, empty=(1,))
    for thr in (0.0, 1.0, 3.0):
        got = anchor_mask_ref.anchor_area_mask_np(coors, B, boxes, grid, thr)
        assert got.shape == (B, anchors.shape[0])
        for b in range(B):
            c = coors[coors[:, 0] == b][:, 1:]
            dense = box_np_ops.sparse_sum_for_anchors_mask(c, tuple(vg.grid_size[::-1][1:]))
            dense = dense.cumsum(0).cumsum(1)
            area = box_np_ops.fused_get_anchors_area(dense, bv, vg.voxel_size, vg.point_cloud_range, vg.grid_size)
            ref = area > thr
            assert np.array_equal(got[b], ref), (thr, b, int((got[b] != ref).sum()))
        assert not got[1].any()                       # the empty frame masks every anchor
        assert 0 < got[0].sum() < anchors.shape[0]


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[:-4] for p in FIXTURES])
def test_oracle_reproduces_fixture_masks(oracle, path):
    """the mirror network's anchors and the oracle voxelizer's coordinates are the reference's (sha1); the oracle mask
    over them is exactly the mask prep_pointcloud stored"""
    fix = np.load(path)
    name, seed, n = _fixture_case(path)
    cfg = config.get_config(name)
    net = models.build_network(cfg, oracle).eval()
    anchors = net.anchors()
    assert gu.sha(anchors) == str(fix["anchors_sha1"])
    pts = synth.nuscenes_cloud(seed, n) if "nuscenes" in name else synth.kitti_cloud(seed, n, cfg.point_cloud_range)
    assert gu.sha(pts) == str(fix["points_sha1"])
    res = net.voxel_generator.generate(pts, int(fix["max_voxels"]))
    assert res["voxel_num"] == int(fix["voxel_num"]) and gu.sha(res["coordinates"]) == str(fix["coords_sha1"])
    coors = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    boxes = anchor_mask.anchor_boxes(anchors, cfg.voxel_size, cfg.point_cloud_range, cfg.grid_size)
    got = anchor_mask_ref.anchor_area_mask_np(coors, 1, boxes, cfg.grid_size, float(fix["threshold"]))[0]
    want = np.unpackbits(fix["mask_packed"])[:anchors.shape[0]].astype(bool)
    assert int(want.sum()) == int(fix["num_masked_in"])
    assert np.array_equal(got, want), "%d anchors differ" % int((got != want).sum())


def test_fixtures_cover_the_issue_cases():
    names = {_fixture_name(p) for p in FIXTURES}
    assert names >= {"pointpillars.car.xyres_16", "car.fhd", "car.lite", "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"}
    assert any(".mv" in p for p in FIXTURES)
    for p in FIXTURES:
        assert os.path.getsize(p) < 64 * 1024


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[:-4] for p in FIXTURES])
def test_fixture_mask_changes_the_detections(path):
    """the stored with-mask and without-mask detections of the reference differ: the mask has teeth on every case"""
    fix = np.load(path)
    a, b = fix["box3d_lidar"], fix["nomask_box3d_lidar"]
    assert a.shape != b.shape or not np.array_equal(a, b) or not np.array_equal(fix["scores"], fix["nomask_scores"])
