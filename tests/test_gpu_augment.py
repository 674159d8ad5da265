"""b2second.augment on the GPU against the reference's fixtures (tests/golden/make_augment_golden.py) and the numpy
restatement (tests/augment_ref.py)."""
import numpy as np
import pytest
import torch

import augment_ref as ar
from b2second import augment, config

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _plan(name):
    cfg = config.get_config(name)
    return cfg, augment.plan(cfg.augment, cfg.point_cloud_range, ar.class_names(name))


def _inputs(name, fr):
    pts, boxes, names = ar.frame(name, str(fr["kind"]), int(fr["seed"]))
    valid, cls = ar.class_mask(name, names)
    return pts, boxes, names, valid, cls


def _pack(frames_in):
    """[(pts, boxes, valid, cls)] -> device tensors of augment_batch"""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    pts = np.concatenate([f[0] for f in frames_in])
    boxes = np.concatenate([f[1] for f in frames_in])
    poff = np.cumsum([0] + [len(f[0]) for f in frames_in]).astype(np.int32)
    goff = np.cumsum([0] + [len(f[1]) for f in frames_in]).astype(np.int32)
    return (t(pts), t(poff), t(boxes), t(goff), t(np.concatenate([f[2] for f in frames_in])),
            t(np.concatenate([f[3] for f in frames_in])))


def _unpack(out, frames_in, d):
    """device outputs of augment_batch -> per-frame dicts of host arrays (the layout augment_ref.augment returns)"""
    h = {k: v.cpu().numpy() for k, v in out.items()}
    res = []
    p0 = g0 = 0
    for f, fi in enumerate(frames_in):
        n, g = len(fi[0]), len(fi[1])
        k0, k1 = h["gt_offsets"][f], h["gt_offsets"][f + 1]
        pb = h["point_box"][p0:p0 + n]
        res.append({"points": h["points"][p0:p0 + n], "point_box": np.where(pb >= 0, pb - g0, -1),
                    "selected": h["selected"][g0:g0 + g], "boxes": h["boxes"][k0:k1], "classes": h["classes"][k0:k1],
                    "importance": h["importance"][k0:k1], "src_row": h["src_row"][k0:k1] - g0})
        p0 += n
        g0 += g
    return res


def _batch(name, frames):
    cfg, plan = _plan(name)
    fin = []
    rs_list = []
    for fr in frames:
        pts, boxes, _, valid, cls = _inputs(name, fr)
        fin.append((pts, boxes, valid, cls))
        rs_list.append(int(fr["seed"]))
    # one draw per frame on its own seeded state, concatenated in frame order
    ds = [augment.draw(np.random.RandomState(s), cfg.augment, [len(fi[1])], [len(fi[0])]) for s, fi in
          zip(rs_list, fin)]
    d = augment.Draws(
        loc_noise=np.concatenate([x.loc_noise for x in ds]) if plan.object_noise else None,
        rot_noise=np.concatenate([x.rot_noise for x in ds]) if plan.object_noise else None,
        frame=np.concatenate([x.frame for x in ds]),
        perm=np.concatenate([x.perm for x in ds]) if cfg.augment.shuffle_points else None,
        num_gt=[len(fi[1]) for fi in fin], num_points=[len(fi[0]) for fi in fin])
    return plan, fin, d


@pytest.mark.parametrize("name", ar.CONFIGS)
def test_augment_frame_equals_reference(name):
    _, frames = ar.load_fixture(name)
    _, plan = _plan(name)
    for f, fr in enumerate(frames):
        pts, boxes, names, valid, cls = _inputs(name, fr)
        rs = np.random.RandomState(int(fr["seed"]))
        got_pts, gd = plan.augment_frame(pts, boxes, names, rs=rs, device=DEV, with_debug=True)
        assert ar.state_digest(rs) == str(fr["state"])
        got = {"points": got_pts, "point_box": gd["point_box"], "selected": gd["selected"], "boxes": gd["gt_boxes"],
               "classes": gd["gt_classes"], "importance": gd["gt_importance"].astype(np.float32),
               "src_row": gd["src_row"]}
        what = "%s frame %d (%s)" % (name, f, fr["kind"])
        ar.compare(got, fr, what)
        np.testing.assert_array_equal(gd["gt_names"], names[fr["src_row"]])
        assert gd["gt_importance"].dtype == boxes.dtype


@pytest.mark.parametrize("name", ar.CONFIGS)
def test_augment_batch_equals_reference_and_per_frame(name):
    _, frames = ar.load_fixture(name)
    plan, fin, d = _batch(name, frames)
    out = plan.augment_batch(*_pack(fin), None, d, with_debug=True)
    assert int(plan.last_status.item()) == 0
    for f, (got, fr) in enumerate(zip(_unpack(out, fin, d), frames)):
        ar.compare(got, fr, "%s batch frame %d (%s)" % (name, f, fr["kind"]))
    again = plan.augment_batch(*_pack(fin), None, d, with_debug=True)
    for k in out:
        assert torch.equal(again[k], out[k]), k


def test_cuda_graph_replay_equals_eager():
    _, frames = ar.load_fixture("car.fhd")
    plan, fin, d = _batch("car.fhd", frames)
    args = _pack(fin)
    eager = plan.augment_batch(*args, None, d, with_debug=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.augment_batch(*args, None, d, with_debug=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = plan.augment_batch(*args, None, d, with_debug=True)
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


@pytest.mark.parametrize("name,n", [("car.fhd", 300), ("car.fhd", 1000), ("pointpillars.car.xyres_16", 600),
                                    ("nuscenes.all.pp.largea", 700)])
def test_random_crowded_frames_equal_restatement(name, n):
    cfg, plan = _plan(name)
    rng = np.random.default_rng(n)
    r = np.asarray(cfg.point_cloud_range)
    b = np.zeros((n, 9 if ar.is_nuscenes(name) else 7))
    b[:, :2] = rng.uniform(r[:2], r[3:5], (n, 2))
    b[:, 2] = rng.uniform(-2, -1, n)
    b[:, 3:6] = rng.uniform([1.5, 3.5, 1.4], [2.0, 4.6, 1.8], (n, 3))
    b[:, 6] = rng.uniform(-np.pi, np.pi, n)
    if b.shape[1] == 9:
        b[:, 7:] = rng.normal(0, 3, (n, 2))
    boxes = b.astype(np.float64 if ar.is_nuscenes(name) else np.float32)
    valid = rng.random(n) < 0.8
    cls = np.where(valid, 1, 0).astype(np.int32)
    pts = np.concatenate([rng.uniform(r[:3], r[3:], (20000, 3)), rng.random((20000, 2 if b.shape[1] == 9 else 1))],
                         1).astype(np.float32)
    d = augment.draw(np.random.RandomState(n), cfg.augment, [n], [len(pts)])
    fin = [(pts, boxes, valid, cls)]
    out = plan.augment_batch(*_pack(fin), None, d, with_debug=True)
    assert int(plan.last_status.item()) == 0
    got = _unpack(out, fin, d)[0]
    want = ar.augment(plan, pts, boxes, valid, cls, None, d)
    assert (want["selected"] > 0).any() or not plan.object_noise
    ar.compare(got, want, "%s random %d GTs" % (name, n))


def test_box_cap_and_bad_offsets_raise_status():
    cfg, plan = _plan("car.fhd")
    n = augment.MAX_BOXES + 1
    rng = np.random.default_rng(1)
    boxes = np.zeros((n, 7), np.float32)
    boxes[:, :2] = rng.uniform([0, -40], [70, 40], (n, 2))
    boxes[:, 3:6] = [1.6, 3.9, 1.5]
    pts = rng.uniform([0, -40, -3, 0], [70, 40, 1, 1], (1000, 4)).astype(np.float32)
    valid = np.ones(n, bool)
    d = augment.draw(np.random.RandomState(0), cfg.augment, [n], [len(pts)])
    out = plan.augment_batch(*_pack([(pts, boxes, valid, np.ones(n, np.int32))]), None, d, with_debug=True)
    assert int(plan.last_status.item()) == 64
    assert (out["selected"].cpu().numpy() == augment.SEL_SKIPPED).all()
    assert (out["point_box"].cpu().numpy() == -1).all()
    # gt_offsets past num_gt
    small = boxes[:5]
    d = augment.draw(np.random.RandomState(0), cfg.augment, [5], [len(pts)])
    args = list(_pack([(pts, small, valid[:5], np.ones(5, np.int32))]))
    args[3] = torch.tensor([0, 9], dtype=torch.int32, device=DEV)
    plan.augment_batch(*args, None, d)
    assert int(plan.last_status.item()) & 32


def test_xyres16_chain_augment_voxelize_anchor_mask_assign():
    """augment_batch -> b2s_voxelize -> b2s_anchor_area_mask -> assign_batch without a host sync equals the same
    stages fed the restatement's output"""
    from b2second import anchor_mask, models, targets
    from spconv import _lib as L
    name = "pointpillars.car.xyres_16"
    _, frames = ar.load_fixture(name)
    cfg, plan = _plan(name)
    _, fin, d = _batch(name, frames[1:5])
    tplan = targets.plan(models.MirrorTargetAssigner(cfg), cfg.feature_map_size)
    lib = L.load()
    B = len(fin)
    P = sum(len(f[0]) for f in fin)
    cap, T = B * cfg.max_voxels, cfg.max_points_per_voxel
    hcap = lib.b2s_voxelize_hash_capacity(P)
    ny, nx = int(cfg.grid_size[1]), int(cfg.grid_size[0])
    aboxes = torch.from_numpy(anchor_mask.anchor_boxes(tplan.anchors, cfg.voxel_size, cfg.point_cloud_range,
                                                       cfg.grid_size)).to(DEV)
    A = int(aboxes.shape[0])
    args = _pack(fin)

    def stages(points, poff, boxes, goff, cls, imp):
        coors = torch.empty(cap, 4, dtype=torch.int32, device=DEV)
        npv = torch.empty(cap, dtype=torch.int32, device=DEV)
        slots = torch.empty(cap, T, dtype=torch.int32, device=DEV)
        nvox = torch.empty(1 + B, dtype=torch.int32, device=DEV)
        hk = torch.empty(hcap, dtype=torch.int64, device=DEV)
        hv = torch.empty(hcap, dtype=torch.int32, device=DEV)
        wsb = lib.b2s_voxelize_workspace_bytes(P, B, cfg.max_voxels, T)
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=DEV)
        st = torch.zeros(1, dtype=torch.int32, device=DEV)
        L.check(lib.b2s_voxelize(L.ptr(points), L.ptr(poff), P, int(points.shape[1]), B,
                                 L.f3(cfg.point_cloud_range[:3]), L.f3(cfg.voxel_size), L.i3(cfg.grid_size), T,
                                 cfg.max_voxels, L.ptr(coors), L.ptr(npv), L.ptr(slots), None, 0, 0, None,
                                 L.ptr(nvox), L.ptr(hk), L.ptr(hv), hcap, 0, L.ptr(ws), wsb, L.ptr(st), L.stream()),
                "b2s_voxelize")
        mws_b = lib.b2s_anchor_area_mask_workspace_bytes(B, ny, nx)
        mws = torch.empty(max(mws_b, 1), dtype=torch.uint8, device=DEV)
        mask = torch.empty(B, A, dtype=torch.uint8, device=DEV)
        L.check(lib.b2s_anchor_area_mask(L.ptr(coors), L.ptr(nvox), cap, B, ny, nx, L.ptr(aboxes), A, 1.0,
                                         L.ptr(mws), mws_b, L.ptr(mask), L.stream()), "b2s_anchor_area_mask")
        r = tplan.assign_batch(boxes, goff, cls, imp, mask.bool())
        return nvox, coors, mask, r

    out = plan.augment_batch(*args, None, d)
    stages(out["points"], args[1], out["boxes"], out["gt_offsets"], out["classes"], out["importance"])   # warm tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = plan.augment_batch(*args, None, d)
        got = stages(out["points"], args[1], out["boxes"], out["gt_offsets"], out["classes"], out["importance"])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = []
    g0 = 0
    for f, fi in enumerate(fin):
        want.append(ar.augment(plan, fi[0], fi[1], fi[2], fi[3], None, d, f, g0))
        g0 += len(fi[1])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    woff = np.cumsum([0] + [len(w["boxes"]) for w in want]).astype(np.int32)
    assert woff[-1] > 0
    np.testing.assert_array_equal(out["gt_offsets"].cpu().numpy(), woff)
    exp = stages(t(np.concatenate([w["points"] for w in want])), args[1], t(np.concatenate([w["boxes"] for w in want])),
                 t(woff), t(np.concatenate([w["classes"] for w in want])),
                 t(np.concatenate([w["importance"] for w in want])))
    nv = int(exp[0][0])
    assert torch.equal(got[0], exp[0])
    assert torch.equal(got[1][:nv], exp[1][:nv])
    assert torch.equal(got[2], exp[2])
    for k in got[3]:
        assert torch.equal(got[3][k], exp[3][k]), k
