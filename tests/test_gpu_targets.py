"""Target assignment on the GPU (csrc/targets.cu through b2second.targets) against the fixtures the unmodified
reference's TargetAssigner.assign produced (tests/golden/make_targets_golden.py) and against tests/targets_ref.py.
Labels, importance and the + - * / sqrt box-target components bit for bit, the log components within 4 float32 ulp."""
import numpy as np
import pytest
import torch

import targets_ref as tr
from b2second import inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _anchors_dict(plan):
    return {plan.classes[i]: {"anchors": plan.anchors[s.begin:s.end]} for i, s in enumerate(plan.segments)}


_check = tr.check_frame


def _pack(plan, frames, device=DEV):
    gts = [fr["gt_boxes"] for fr in frames]
    offs = np.concatenate([[0], np.cumsum([len(g) for g in gts])]).astype(np.int32)
    gt = torch.from_numpy(np.concatenate(gts)).to(device)
    cls = torch.from_numpy(np.concatenate([fr["gt_classes"] for fr in frames]).astype(np.int32)).to(device)
    imp = torch.from_numpy(np.concatenate([fr["importance"] for fr in frames]).astype(np.float32)).to(device)
    A = plan.num_anchors
    mask = torch.from_numpy(np.stack([fr["mask"] if fr["mask"] is not None else np.ones(A, bool)
                                      for fr in frames])).to(device)
    return gt, torch.from_numpy(offs).to(device), cls, imp, mask


@pytest.mark.parametrize("name", tr.CONFIGS)
def test_assign_equals_reference(name):
    _, frames = tr.load_fixture(name)
    plan = tr.mirror_plan(name)
    for fr in frames:
        r = plan.assign(plan.anchors, _anchors_dict(plan), fr["gt_boxes"], anchors_mask=fr["mask"],
                        gt_classes=fr["gt_classes"], gt_names=fr["gt_names"],
                        matched_thresholds=plan.matched_thresholds, unmatched_thresholds=plan.unmatched_thresholds,
                        importance=fr["importance"])
        assert r["labels"].is_cuda and r["labels"].dtype == torch.int32
        _check(r["labels"], r["bbox_targets"], r["importance"], fr)
        if "inds" in fr:
            np.testing.assert_array_equal(r["assigned_anchors_inds"].cpu().numpy(), fr["inds"])
            np.testing.assert_array_equal(r["positive_gt_id"].cpu().numpy(), fr["gt_id"])
            if len(fr["gt_boxes"]):
                np.testing.assert_array_equal(r["assigned_anchors_overlap"].cpu().numpy(), fr["overlap"])
            np.testing.assert_array_equal(r["bbox_outside_weights"].cpu().numpy(),
                                          (fr["labels"] > 0).astype(np.float32))


@pytest.mark.parametrize("name", tr.CONFIGS)
def test_assign_batch_equals_reference_and_per_frame(name):
    _, frames = tr.load_fixture(name)
    plan = tr.mirror_plan(name)
    gt, offs, cls, imp, mask = _pack(plan, frames)
    r = plan.assign_batch(gt, offs, cls, imp, mask)
    assert r["labels"].dtype == torch.int32 and r["reg_targets"].dtype == torch.float32
    assert int(plan.last_status.item()) == 0
    for f, fr in enumerate(frames):
        _check(r["labels"][f], r["reg_targets"][f], r["importance"][f], fr)
        one = plan.assign_batch(*_pack(plan, [fr]))
        for k in r:
            assert torch.equal(one[k][0], r[k][f]), (f, k)
    again = plan.assign_batch(gt, offs, cls, imp, mask)
    for k in r:
        assert torch.equal(again[k], r[k]), k


def test_cuda_graph_replay_equals_eager():
    _, frames = tr.load_fixture("all.fhd")
    plan = tr.mirror_plan("all.fhd")
    gt, offs, cls, imp, mask = _pack(plan, frames)
    eager = plan.assign_batch(gt, offs, cls, imp, mask)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.assign_batch(gt, offs, cls, imp, mask)                 # warm the device tables outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = plan.assign_batch(gt, offs, cls, imp, mask)
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


@pytest.mark.parametrize("name,dtype", [("car.fhd", np.float32), ("nuscenes.all.pp.largea", np.float64),
                                        ("nuscenes.all.pp.mhead", np.float64)])
def test_random_600_gt_frame_equals_restatement(name, dtype):
    plan = tr.mirror_plan(name)
    rng = np.random.default_rng(7)
    a = plan.anchors[rng.integers(0, plan.num_anchors, 600)].astype(np.float64)
    a[:, :2] += rng.uniform(-1.5, 1.5, (600, 2))
    a[:, 3:6] *= rng.uniform(0.8, 1.2, (600, 3))
    a[:, 6] = rng.uniform(-np.pi, np.pi, 600)
    gt = a.astype(dtype)
    ncls = len(plan.classes)
    cls = rng.integers(1, ncls + 1, 600).astype(np.int32)
    imp = rng.uniform(0.5, 2.0, 600).astype(np.float32)
    mask = rng.random(plan.num_anchors) < 0.8
    seg = (cls - 1) if plan.assign_per_class else np.zeros(600, np.int32)
    labels, tg, im, _, _ = tr.assign(plan, gt, seg, cls, imp, mask)
    r = plan.assign_batch(torch.from_numpy(gt).to(DEV), torch.tensor([0, 600], dtype=torch.int32, device=DEV),
                          torch.from_numpy(cls).to(DEV), torch.from_numpy(imp).to(DEV),
                          torch.from_numpy(mask[None]).to(DEV))
    pos = np.flatnonzero(labels > 0)
    _check(r["labels"][0], r["reg_targets"][0], r["importance"][0],
           {"labels": labels, "importance_out": im, "pos": pos, "targets": tg[pos]})


def test_class_with_every_anchor_pruned():
    """the documented divergence: the reference raises; here the class's anchors come out -1 / 0 / 0"""
    _, frames = tr.load_fixture("all.fhd")
    plan = tr.mirror_plan("all.fhd")
    fr = dict(frames[1])
    seg = plan.segments[plan.classes.index(fr["gt_names"][0])]
    mask = np.ones(plan.num_anchors, bool)
    mask[seg.begin:seg.end] = False
    fr["mask"] = mask
    r = plan.assign_batch(*_pack(plan, [fr]))
    lab = r["labels"][0].cpu().numpy()
    assert (lab[seg.begin:seg.end] == -1).all()
    assert not r["importance"][0][seg.begin:seg.end].any() and not r["reg_targets"][0][seg.begin:seg.end].any()
    labels, tg, im, _, _ = tr.assign(plan, fr["gt_boxes"], tr.segments_of(plan, fr["gt_names"]), fr["gt_classes"],
                                     fr["importance"], mask)
    pos = np.flatnonzero(labels > 0)
    _check(r["labels"][0], r["reg_targets"][0], r["importance"][0],
           {"labels": labels, "importance_out": im, "pos": pos, "targets": tg[pos]})


def test_xyres16_chain_anchor_area_mask_then_assign_batch():
    from b2second import config
    name = "pointpillars.car.xyres_16"
    z, frames = tr.load_fixture(name)
    plan = tr.mirror_plan(name)
    cfg = config.get_config(name)
    coors = torch.from_numpy(np.pad(z["cloud_coors"], ((0, 0), (1, 0)))).to(DEV)      # (b, z, y, x)
    B = len(frames) - 1
    coors = torch.cat([coors + torch.tensor([b, 0, 0, 0], dtype=coors.dtype, device=DEV) for b in range(B)])
    mask = inputs.anchor_area_mask(coors, B, plan.anchors, cfg.voxel_size, cfg.point_cloud_range, cfg.grid_size, 1.0)
    want = np.unpackbits(z["cloud_mask"])[:plan.num_anchors].astype(bool)
    for b in range(B):
        np.testing.assert_array_equal(mask[b].cpu().numpy(), want)
    gt, offs, cls, imp, _ = _pack(plan, frames[1:])
    r = plan.assign_batch(gt, offs, cls, imp, mask)
    for f, fr in enumerate(frames[1:]):
        _check(r["labels"][f], r["reg_targets"][f], r["importance"][f], fr)

