"""b2second.dbsample on the GPU against the reference's fixtures (tests/golden/make_dbsample_golden.py)."""
import numpy as np
import pytest
import torch

import augment_ref as ar
import dbsample_ref as dr
from b2second import augment, config, dbsample

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sampler(name, tmp_path):
    z, frames = dr.load_fixture(name)
    db, uid2obj = dr.load_db(name, z, str(tmp_path), DEV)
    rs0 = np.random.RandomState(int(z["seed_init"]))
    ds = dbsample.DatabaseSampler(db, config.get_config(name).db_sampler, dr.class_names(name), rs0)
    assert ar.state_digest(rs0) == str(z["state_init"])
    return z, frames, ds, uid2obj


def _check_frame(got_pts, gd, fr, uid2obj, what):
    np.testing.assert_array_equal(got_pts, fr["out_points"], err_msg=what + " points")
    assert gd["gt_boxes"].dtype == fr["out_boxes"].dtype, what
    np.testing.assert_array_equal(gd["gt_boxes"], fr["out_boxes"], err_msg=what + " boxes")
    np.testing.assert_array_equal(gd["gt_names"], fr["out_names"], err_msg=what + " names")
    assert gd["gt_importance"].dtype == fr["out_importance"].dtype, what
    np.testing.assert_array_equal(gd["gt_importance"], fr["out_importance"], err_msg=what + " importance")
    np.testing.assert_array_equal(gd["gt_boxes_mask"], fr["out_mask"], err_msg=what + " mask")
    np.testing.assert_array_equal(gd["candidates"], [uid2obj[int(u)] for u in fr["cand"]], err_msg=what + " cand")
    acc = gd["candidates"][gd["accepted"]]
    np.testing.assert_array_equal(acc, [uid2obj[int(u)] for u in fr["acc"]], err_msg=what + " accepted")


@pytest.mark.parametrize("name", dr.CONFIGS)
def test_sample_frame_equals_reference(name, tmp_path):
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    for f, fr in enumerate(frames):
        pts, boxes, names = fr["in_points"], fr["in_boxes"], fr["in_names"]
        rs = np.random.RandomState(int(fr["seed"]))
        got_pts, gd = ds.sample_frame(pts, {"gt_boxes": boxes, "gt_names": names}, rs=rs, with_debug=True)
        what = "%s frame %d (%s)" % (name, f, fr["kind"])
        _check_frame(got_pts, gd, fr, uid2obj, what)
        if "chain_points" in fr:
            continue                                        # test_xyres16_chain_sample_then_augment
        assert ar.state_digest(rs) == str(fr["state"]), what
    assert int(ds.last_status.item()) == 0


@pytest.mark.parametrize("name", dr.CONFIGS)
def test_sample_all_equals_reference(name, tmp_path):
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    cfg = config.get_config(name)
    for f, fr in enumerate(frames):
        _, boxes, names = dr.frame_inputs(fr)
        rs = np.random.RandomState(int(fr["seed"]))
        got = ds.sample_all(str(tmp_path), boxes, names, cfg.num_point_features, rs=rs)
        what = "%s frame %d (%s)" % (name, f, fr["kind"])
        if bool(fr["sa_none"]):
            assert got is None, what
            continue
        for k in ("gt_names", "difficulty", "gt_boxes", "points", "gt_masks", "group_ids"):
            np.testing.assert_array_equal(got[k], fr["sa_" + k], err_msg="%s %s" % (what, k))
        assert got["gt_boxes"].dtype == fr["sa_gt_boxes"].dtype and got["points"].dtype == np.float32


def _pack(frames):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    ins = [dr.frame_inputs(fr) for fr in frames]
    pts = np.concatenate([i[0] for i in ins])
    boxes = np.concatenate([i[1] for i in ins])
    return ins, (t(pts), t(np.cumsum([0] + [len(i[0]) for i in ins]).astype(np.int32)), t(boxes),
                 t(np.cumsum([0] + [len(i[1]) for i in ins]).astype(np.int32)))


def _batch(name, ds, frames, z, uid2obj):
    classes = dr.class_names(name)
    ins, (pts, poff, boxes, goff) = _pack(frames)
    names = np.concatenate([i[2] for i in ins])
    valid = torch.from_numpy(np.array([n in classes for n in names], np.bool_)).to(DEV)
    cls = torch.from_numpy(np.array([classes.index(n) + 1 if n in classes else 0 for n in names], np.int32)).to(DEV)
    cand = dr.candidates(name, z, frames, uid2obj)
    return ds.sample_batch(pts, poff, boxes, goff, valid, cls, None, cand), cand


@pytest.mark.parametrize("name", dr.CONFIGS)
def test_sample_batch_equals_frames(name, tmp_path):
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    res, cand = _batch(name, ds, frames, z, uid2obj)
    n_b, n_p = res.counts()
    assert int(ds.last_status.item()) == 0
    h = {k: v.cpu().numpy() for k, v in res.items()}
    G = sum(len(dr.frame_inputs(fr)[1]) for fr in frames)
    for f, fr in enumerate(frames):
        what = "%s batch frame %d (%s)" % (name, f, fr["kind"])
        p0, p1 = h["point_offsets"][f], h["point_offsets"][f + 1]
        g0, g1 = h["gt_offsets"][f], h["gt_offsets"][f + 1]
        assert (n_b[f], n_p[f]) == (g1 - g0, p1 - p0)
        np.testing.assert_array_equal(h["points"][p0:p1], fr["out_points"], err_msg=what)
        np.testing.assert_array_equal(h["boxes"][g0:g1], fr["out_boxes"], err_msg=what)
        np.testing.assert_array_equal(h["gt_valid"][g0:g1], fr["out_mask"], err_msg=what)
        imp = fr["out_importance"].astype(np.float32)
        np.testing.assert_array_equal(h["importance"][g0:g1], imp, err_msg=what)
        n_own = len(dr.frame_inputs(fr)[1])
        np.testing.assert_array_equal(h["src_object"][g0:g0 + n_own], -1)
        np.testing.assert_array_equal(h["src_object"][g0 + n_own:g1], [uid2obj[int(u)] for u in fr["acc"]])
        cls = [dr.class_names(name).index(str(n)) + 1 if str(n) in dr.class_names(name) else 0
               for n in fr["out_names"]]
        np.testing.assert_array_equal(h["classes"][g0:g1], cls, err_msg=what)
    # rows past the packed ones are zeros
    assert (h["points"][h["point_offsets"][-1]:] == 0).all() and (h["boxes"][h["gt_offsets"][-1]:] == 0).all()
    assert (h["src_object"][h["gt_offsets"][-1]:] == -1).all() and len(h["boxes"]) == G + len(cand.objects)
    again, _ = _batch(name, ds, frames, z, uid2obj)
    for k in res:
        assert torch.equal(again[k], res[k]), k


def test_cuda_graph_replay_equals_eager(tmp_path):
    """a captured sample_batch reads its candidates from the caller's pinned staging buffer at every replay: refilled
    with other candidates of the same count and point total, the replay equals an eager call on those"""
    name = "car.fhd"
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    classes = dr.class_names(name)
    ins, (pts, poff, boxes, goff) = _pack(frames)
    names = np.concatenate([i[2] for i in ins])
    valid = torch.from_numpy(np.array([n in classes for n in names], np.bool_)).to(DEV)
    cls = torch.from_numpy(np.array([classes.index(n) + 1 if n in classes else 0 for n in names], np.int32)).to(DEV)
    cand = dr.candidates(name, z, frames, uid2obj)
    # the same candidates, each frame's in reverse order (one sample group): same count and point total
    rev = dbsample.Candidates(objects=np.concatenate([cand.objects[a:b][::-1] for a, b in
                                                      zip(cand.offsets[:-1], cand.offsets[1:])]).astype(np.int32),
                              group=cand.group.copy(), offsets=cand.offsets.copy())
    assert not np.array_equal(rev.objects, cand.objects)
    eager = ds.sample_batch(pts, poff, boxes, goff, valid, cls, None, cand)
    eager_rev = ds.sample_batch(pts, poff, boxes, goff, valid, cls, None, rev)
    host, _, _ = dbsample.pack_candidates(cand, ds.db)
    staging = torch.empty(len(host), dtype=torch.int32).pin_memory()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ds.sample_batch(pts, poff, boxes, goff, valid, cls, None, cand, staging=staging)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError):
        with torch.cuda.graph(g):
            ds.sample_batch(pts, poff, boxes, goff, valid, cls, None, cand)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ds.sample_batch(pts, poff, boxes, goff, valid, cls, None, cand, staging=staging)
    junk = [torch.full((len(host),), -7, dtype=torch.int32).pin_memory() for _ in range(4)]   # reuse of freed blocks
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k
    staging.copy_(torch.from_numpy(dbsample.pack_candidates(rev, ds.db)[0]))
    g.replay()
    torch.cuda.synchronize()
    for k in eager_rev:
        assert torch.equal(out[k], eager_rev[k]), k
    assert not torch.equal(eager_rev["boxes"], eager["boxes"])
    del junk


def _raw_call(ds, pts, poff, boxes, goff, cand_obj, cand_grp, cand_off, cand_pto, CP, guard=64):
    """b2s_db_sample through the C ABI with every output followed by a guard region of sentinels"""
    from spconv import _lib as L
    lib = L.load()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    P, F, B = len(pts), pts.shape[1], len(poff) - 1
    G, C = len(boxes), len(cand_obj)
    pts_out = torch.full(((P + CP + guard) * F,), 12345.0, device=DEV)
    boxes_out = torch.full(((G + C + guard) * 7,), 12345.0, device=DEV)
    small = {k: torch.full((G + C + guard,), 99, dtype=d, device=DEV)
             for k, d in (("valid", torch.uint8), ("cls", torch.int32), ("src", torch.int32))}
    imp_out = torch.full((G + C + guard,), 99.0, device=DEV)
    acc = torch.full((C + guard,), 99, dtype=torch.uint8, device=DEV)
    offs = torch.full((2 * (B + 1) + guard,), 99, dtype=torch.int32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    wsb = lib.b2s_db_sample_workspace_bytes(B, P, C)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    db = ds.db
    ins = [t(pts), t(np.asarray(poff, np.int32)), t(boxes), t(np.asarray(goff, np.int32)), t(np.ones(G, np.uint8)),
           t(np.ones(G, np.int32)), t(np.asarray(cand_obj, np.int32)), t(np.asarray(cand_grp, np.int32)),
           t(np.asarray(cand_off, np.int32)), t(np.asarray(cand_pto, np.int32))]
    L.check(lib.b2s_db_sample(
        L.ptr(ins[0]), P, F, L.ptr(ins[1]), B, L.ptr(ins[2]), 0, 7, G, L.ptr(ins[3]), L.ptr(ins[4]), L.ptr(ins[5]), None,
        L.ptr(ins[6]) if C else None, L.ptr(ins[7]) if C else None, L.ptr(ins[8]), L.ptr(ins[9]), C, CP,
        L.ptr(db.points), L.ptr(db.point_offsets), L.ptr(db.boxes), L.ptr(db.classes), db.num_objects, 1.0, 1,
        L.ptr(pts_out), L.ptr(offs), L.ptr(boxes_out), ctypes_off(offs, B + 1), L.ptr(small["valid"]),
        L.ptr(small["cls"]), L.ptr(imp_out), L.ptr(small["src"]), L.ptr(acc) if C else None, L.ptr(ws), wsb,
        L.ptr(status), L.stream()), "b2s_db_sample")
    torch.cuda.synchronize()
    n_out = {"points": (pts_out, (P + CP) * F, 12345.0), "boxes": (boxes_out, (G + C) * 7, 12345.0),
             "valid": (small["valid"], G + C, 99), "cls": (small["cls"], G + C, 99), "src": (small["src"], G + C, 99),
             "imp": (imp_out, G + C, 99.0), "acc": (acc, C, 99), "offs": (offs, 2 * (B + 1), 99)}
    for k, (buf, n, sentinel) in n_out.items():
        assert (buf[n:] == sentinel).all(), "write past the end of %s" % k
    po = offs[:B + 1].cpu().numpy()
    return int(status.item()), pts_out[:(P + CP) * F].view(-1, F), po, offs[B + 1:2 * (B + 1)].cpu().numpy()


def ctypes_off(t, elems):
    import ctypes
    return ctypes.c_void_p(t.data_ptr() + 4 * elems)


def test_overlapping_offsets_raise_status_and_stay_in_bounds(tmp_path):
    """a decreasing interior offset makes its neighbours' ranges overlap: every frame touching it is treated as
    empty, the status says so, and nothing is written past any output"""
    z, frames, ds, uid2obj = _sampler("car.fhd", tmp_path)
    rng = np.random.default_rng(5)
    pts = rng.uniform([0, -40, -3, 0], [70, 40, 1, 1], (20, 4)).astype(np.float32)
    boxes = np.zeros((0, 7), np.float32)
    st, out, po, go = _raw_call(ds, pts, [0, 10, 5, 20], boxes, [0, 0, 0, 0], [], [], [0, 0, 0, 0], [0], 0)
    assert st & 32
    assert po[-1] <= 20 and (np.diff(po) >= 0).all()
    # the usable ranges: none of [0, 10), [10, 5), [5, 20) lies before every later and after every earlier entry
    assert po[-1] == 0 and (out.cpu().numpy() == 0).all()
    # a valid batch next to it: frame 0 and 2 usable, frame 1 empty with a decreasing pair past it
    st, out, po, _ = _raw_call(ds, pts, [0, 10, 10, 20], boxes, [0, 0, 0, 0], [], [], [0, 0, 0, 0], [0], 0)
    assert st == 0 and list(po) == [0, 10, 10, 20]
    np.testing.assert_array_equal(out.cpu().numpy(), pts)
    # overlapping candidate ranges and a candidate point prefix that does not match the database
    cand = dbsample.draw(np.random.RandomState(0), ds.state, [[], []])
    C = len(cand.objects)
    npts = np.diff(ds.db.point_offsets_host)[cand.objects]
    cpo = np.concatenate([[0], np.cumsum(npts)])
    far = np.zeros((2, 7), np.float32)
    far[:, :2] = 500.0
    far[:, 3:6] = 1.0
    assert C >= 4
    bad_off = [0, C, C // 2, C]                              # frames 0 and 2 would share candidates C // 2 .. C
    st, out, po, go = _raw_call(ds, pts, [0, 10, 15, 20], far, [0, 1, 2, 2], cand.objects, cand.group, bad_off, cpo,
                                int(cpo[-1]))
    assert st & 32 and po[-1] <= 20 + cpo[-1] and go[-1] <= 2 + C
    short = cpo.copy()
    short[1:] = short[1:] // 2                               # steps disagree with the objects' point counts
    st, out, po, go = _raw_call(ds, pts, [0, 10, 20], far, [0, 1, 2], cand.objects, cand.group,
                                [0, C // 2, C], short, int(short[-1]))
    assert st & 32 and po[-1] <= 20 + short[-1]


def test_sample_frame_carries_other_gt_dict_keys(tmp_path):
    """keys beyond boxes, names and importance: per-box arrays lose their DontCare rows, group_ids gain the samples'
    ids (preprocess.py:239-242), the rest passes through"""
    name = "car.fhd"
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    fr = next(f for f in frames if "DontCare" in list(f["in_names"]))
    n = len(fr["in_names"])
    keep = fr["in_names"] != "DontCare"
    gids = np.arange(100, 100 + n)
    _, gd = ds.sample_frame(fr["in_points"], {"gt_boxes": fr["in_boxes"], "gt_names": fr["in_names"],
                                              "group_ids": gids, "difficulty": np.arange(n), "tag": "x"},
                            rs=np.random.RandomState(int(fr["seed"])))
    G, total = int(keep.sum()), len(gd["gt_boxes"])
    assert total > G
    np.testing.assert_array_equal(gd["group_ids"], np.concatenate([gids[keep], np.arange(G, total)]))
    np.testing.assert_array_equal(gd["difficulty"], np.arange(n)[keep])
    assert gd["tag"] == "x"


def test_box_cap_and_bad_offsets_raise_status(tmp_path):
    name = "car.fhd"
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    n = dbsample.MAX_BOXES - 2
    rng = np.random.default_rng(3)
    boxes = np.zeros((n, 7), np.float32)
    boxes[:, 0] = rng.uniform(200, 300, n)                  # far from every database box
    boxes[:, 1] = rng.uniform(200, 300, n)
    boxes[:, 3:6] = [1.6, 3.9, 1.5]
    pts = rng.uniform([0, -40, -3, 0], [70, 40, 1, 1], (500, 4)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    cand = dbsample.draw(np.random.RandomState(0), ds.state, [[]])
    assert len(cand.objects) == 15
    args = [t(pts), t(np.array([0, 500], np.int32)), t(boxes), t(np.array([0, n], np.int32)),
            t(np.ones(n, np.bool_)), t(np.ones(n, np.int32)), None, cand]
    res = ds.sample_batch(*args)
    assert int(ds.last_status.item()) == 128
    assert not res["accepted"].any()
    n_b, n_p = res.counts()
    assert n_b == [n] and n_p == [500]
    assert torch.equal(res["points"][:500], args[0])
    # under the cap, the same frame samples
    args[2], args[3] = t(boxes[:10]), t(np.array([0, 10], np.int32))
    args[4], args[5] = t(np.ones(10, np.bool_)), t(np.ones(10, np.int32))
    res = ds.sample_batch(*args)
    assert int(ds.last_status.item()) == 0 and res["accepted"].any()
    # gt_offsets past num_gt
    args[3] = t(np.array([0, 12], np.int32))
    ds.sample_batch(*args)
    assert int(ds.last_status.item()) & 32


def test_xyres16_chain_sample_then_augment(tmp_path):
    """sample_frame then augment_frame on one stream equals prep_pointcloud's training branch on the fixture frame"""
    name = "pointpillars.car.xyres_16"
    z, frames, ds, uid2obj = _sampler(name, tmp_path)
    cfg = config.get_config(name)
    plan = augment.plan(cfg.augment, cfg.point_cloud_range, dr.class_names(name))
    for f, fr in enumerate(frames):
        rs = np.random.RandomState(int(fr["seed"]))
        if "chain_points" not in fr:
            dbsample.draw(rs, ds.state, [dr.frame_inputs(fr)[2]])       # carry the samplers to the chain frame
            continue
        pts, gd = ds.sample_frame(fr["in_points"], {"gt_boxes": fr["in_boxes"], "gt_names": fr["in_names"]}, rs=rs)
        got_pts, ad = plan.augment_frame(pts, gd["gt_boxes"], gd["gt_names"], importance=gd["gt_importance"], rs=rs,
                                         device=DEV, with_debug=True)
        assert ar.state_digest(rs) == str(fr["state"])
        got = {"points": got_pts, "point_box": ad["point_box"], "selected": ad["selected"], "boxes": ad["gt_boxes"],
               "classes": ad["gt_classes"], "importance": ad["gt_importance"].astype(np.float32),
               "src_row": ad["src_row"]}
        want = {k[len("chain_"):]: v for k, v in fr.items() if k.startswith("chain_")}
        assert (want["src_row"] >= len(dr.frame_inputs(fr)[1])).any()      # sampled boxes reach the output
        ar.compare(got, want, "%s chain frame %d" % (name, f))
        return
    raise AssertionError("no chain frame in the fixture")
