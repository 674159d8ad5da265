"""The detection stage (csrc/detect.cu, csrc/geometry.cuh) against the fp64 reference of tests/detect_ref.py, on
boxes that look like detections: clusters of near-duplicates at rotation 0 and pi/2, near the origin and at KITTI /
NuScenes range, with exact duplicates, shared edges, nested boxes, slivers and tied scores.

* overlaps: element by element within the derived per-pair bounds; the corners-given error must not grow with the
  distance from the origin;
* NMS: every keep list must pass the certificate (pairs within the bound of the threshold may go either way; nothing
  is skipped);
* b2s_nms sweep: 32 frames per call with mixed counts around the 64-box mask tile and the 4096-key sort capacity,
  candidates above the cap, pre_max / post_max at their limits, code 7 and 9, direction fix-up on and off, range on
  and off; the ranked order exactly, kept rows bit-exact from their candidates, the yaw bit-exact;
* the per-class branch and the decode entry points against the fp64 decode and sigmoid."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import detect_ref as R
from b2second import box_ops

pytestmark = pytest.mark.gpu

THRESHOLDS = [0.01, 0.1, 0.5, 0.7]
_errors = {}                                       # measured max error / bound per path and position, for the report


@pytest.fixture(scope="module", autouse=True)
def _report(out_dir):
    yield
    with open(os.path.join(out_dir, "detect_fp64_errors.json"), "w") as f:
        json.dump(_errors, f, indent=1, sort_keys=True)


def _note(key, err, bound):
    e, b = _errors.get(key, (0.0, 0.0))
    _errors[key] = (max(e, float(err)), max(b, float(bound)))


def _corners32(b7):
    """host fp32 corners of (x, y, z, w, l, h, r) boxes, as second.pytorch's box_np_ops builds them."""
    b7 = np.asarray(b7, np.float32)
    return box_ops.corners_2d_np(b7[:, :2], b7[:, 3:5], b7[:, 6]).astype(np.float32)


def _b5(b7):
    return np.ascontiguousarray(np.asarray(b7, np.float32)[:, [0, 1, 3, 4, 6]])


# ------------------------------------------------------------------------------------------------ overlaps
@pytest.mark.parametrize("seed", [0, 1])
def test_rbbox_iou_and_intersection_within_clip_bound(product, seed):
    rng = np.random.default_rng(seed)
    b = R.clusters(rng, 700)
    c = _corners32(b)
    siou = box_ops.standup_iou_np(box_ops.standup_np(c), 0.0)
    ov = R.overlaps(c, c, gate=siou > 0)
    for fn, crit in (("rbbox_iou", -1), ("rbbox_intersection", 2)):
        got = getattr(product.utils, fn)(c, c, siou, 0.0).astype(np.float64)
        bound = np.where(siou > 0, R.clip_bound(c, c, ov, crit), 0.0)
        err = np.abs(got - ov[crit])
        i, j = np.unravel_index(np.argmax(err - bound), err.shape)
        assert (err <= bound).all(), "%s (%d, %d): %r vs %r, bound %.3g" % (fn, i, j, got[i, j], ov[crit][i, j],
                                                                             bound[i, j])
        _note("%s corners given" % fn, err.max(), bound[siou > 0].max())
    # boxes that only touch (shared edges at yaw 0 on a 2^-6 grid): the stand-up gate gives exactly 0, on the
    # corners-given and the box-parameter path
    sa = box_ops.standup_np(c)
    edge = np.zeros((len(c), len(c)), bool)
    for ax in (0, 1):
        edge |= (sa[:, None, 2 + ax] == sa[None, :, ax]) & (np.minimum(sa[:, None, 3 - ax], sa[None, :, 3 - ax]) >
                                                           np.maximum(sa[:, None, 1 - ax], sa[None, :, 1 - ax]))
    iou = product.utils.rbbox_iou(c, c, siou, 0.0)
    ev = product.utils.rotate_iou_eval(torch.from_numpy(_b5(b)).cuda(), torch.from_numpy(_b5(b)).cuda()).cpu().numpy()
    assert edge.sum() > 10 and (iou[edge] == 0).all() and (ev[edge] == 0).all()
    # the clip itself on every pair, touching and disjoint ones included (gate forced open)
    ov_all = R.overlaps(c, c, gate=np.ones_like(edge))
    forced = product.utils.rbbox_iou(c, c, np.ones_like(siou), 0.0).astype(np.float64)
    bound = R.clip_bound(c, c, ov_all)
    assert (np.abs(forced - ov_all[-1]) <= bound).all()
    same = (c[:, None] == c[None]).all((2, 3))
    assert same.sum() > len(c) + 20                                    # exact duplicates are present
    assert np.abs(iou[same] - 1.0).max() <= R.clip_bound(c, c, ov)[same].max()


def test_rotated_iou_error_is_independent_of_position(product):
    """The same clusters translated to each centre: the corners-given error must stay within the position-
    independent clip bound.  Raw-coordinate clipping grows ~ u * (|x| + |y|) * P / U and fails this at KITTI
    range."""
    rng = np.random.default_rng(11)
    base = np.concatenate([R.cluster(rng, 40, s, k) for s in (0.0, 1e-3, 0.05) for k in ("car", "ped", "cyc")
                           for _ in range(3)])
    # spread the clusters over a few metres so they do not all overlap each other
    base[:, 0] += np.repeat(np.arange(27) % 9 * 9.0, 40).astype(np.float32)
    base[:, 1] += np.repeat(np.arange(27) // 9 * 9.0, 40).astype(np.float32)
    base[:, :2] -= np.float32(36.0)
    fails = []
    for cx, cy in R.CENTRES + [(100.0, 50.0)]:
        b = base.copy()
        b[:, :2] += np.array([cx, cy], np.float32)
        c = _corners32(b)
        siou = box_ops.standup_iou_np(box_ops.standup_np(c), 0.0)
        ov = R.overlaps(c, c, gate=siou > 0)
        got = product.utils.rbbox_iou(c, c, siou, 0.0).astype(np.float64)
        bound = np.where(siou > 0, R.clip_bound(c, c, ov), 0.0)
        err = np.abs(got - ov[-1])
        _note("rbbox_iou at (%g, %g)" % (cx, cy), err.max(), bound[siou > 0].max())
        if not (err <= bound).all():
            fails.append("(%g, %g): max error %.3g, %d pairs over their bound (largest bound %.3g)"
                         % (cx, cy, err.max(), int((err > bound).sum()), bound.max()))
    assert not fails, "; ".join(fails)


def test_rotate_iou_eval_all_criteria_within_corner_bound(product):
    rng = np.random.default_rng(5)
    b5 = _b5(R.clusters(rng, 500))
    q5 = np.concatenate([b5[::3], _b5(R.clusters(rng, 130))])          # shares boxes with b5: IoU 1 pairs
    ca, cq = R.bev_corners(b5), R.bev_corners(q5)
    grow = np.array([-1e-3, -1e-3, 1e-3, 1e-3])                      # the fp32 gate may differ at the edges
    ov = R.overlaps(ca, cq, gate=R.standup_overlap(R.standup(ca) + grow, R.standup(cq)))
    bd, qd = torch.from_numpy(b5).cuda(), torch.from_numpy(q5).cuda()
    for crit in (-1, 0, 1, 2):
        got = product.utils.rotate_iou_eval(bd, qd, crit).cpu().numpy().astype(np.float64)
        bound = R.corner_bound(b5, q5, ov, crit)
        err = np.abs(got - ov[crit])
        assert (err <= bound).all(), (crit, float((err - bound).max()))
        _note("rotate_iou_eval criterion %d" % crit, err.max(), bound[ov["inter"] > 0].max())
    assert float(ov[-1].max()) > 0.99


# ------------------------------------------------------------------------------------------------ NMS certificates
def _rank_iou(c64_ranked, b5_ranked=None, rotated=True, eps=1.0, delta=None):
    """[n,n] IoU and bound of ranked boxes (row = earlier), upper triangle."""
    if rotated:
        ov = R.overlaps(c64_ranked, c64_ranked)
        bound = R.clip_bound(c64_ranked, c64_ranked, ov) if b5_ranked is None else \
            R.corner_bound(b5_ranked, b5_ranked, ov)
        return np.triu(ov[-1], 1), bound
    s = R.standup(c64_ranked)
    iou, _, _ = R.aligned_iou(s, s, eps)
    d = 0.0 if delta is None else delta
    return np.triu(iou, 1), R.aligned_bound(s, s, eps, d, d)


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_host_nms_certificates(product, thr):
    rng = np.random.default_rng(int(thr * 100))
    n = 1500
    b = R.clusters(rng, n)
    scores = R.scores_for(rng, n)
    order = np.lexsort((np.arange(n), -scores.astype(np.float64))).astype(np.int32)
    c = _corners32(b)
    siou = box_ops.standup_iou_np(box_ops.standup_np(c), 0.0)
    # rotate_non_max_suppression_cpu: corners given, IoU >= thr
    keep = product.utils.rotate_non_max_suppression_cpu(c, order, siou, thr)
    iou, bound = _rank_iou(c[order].astype(np.float64))
    assert R.nms_certificate(order, keep, iou, bound, thr, n, True) is None
    # the aligned functions on the stand-up boxes: non_max_suppression (+1, '>', sorted dets) and
    # non_max_suppression_cpu (eps, '>=', any order)
    st = box_ops.standup_np(c).astype(np.float32)
    dets = np.concatenate([st[order], scores[order, None]], 1).astype(np.float32)
    k = np.zeros(n, np.int32)
    nk = product.utils.non_max_suppression(dets, k, thr, 0)
    iou, _, _ = R.aligned_iou(dets[:, :4], dets[:, :4], 1.0)
    bd = R.aligned_bound(dets[:, :4], dets[:, :4], 1.0)
    assert R.nms_certificate(np.arange(n), k[:nk], np.triu(iou, 1), bd, thr, n, False) is None
    for eps in (0.0, 1.0):
        got = product.utils.non_max_suppression_cpu(np.concatenate([st, scores[:, None]], 1), order, thr, eps)
        iou, gate, _ = R.aligned_iou(st[order], st[order], eps)
        iou = np.where(gate, iou, 0.0)
        bd = R.aligned_bound(st[order], st[order], eps)
        assert R.nms_certificate(order, got, np.triu(iou, 1), bd, thr, n, True) is None, eps


class _Nms:
    """b2s_nms on [B, cap] candidate arrays (numpy in, numpy out)."""

    def __init__(self, product, box, score, label, dirs, anchor, count, cap):
        self.L = product._lib
        self.lib = self.L.load()
        self.B, self.cap, self.code = box.shape[0], cap, box.shape[2]
        self.d = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (box, score, label, dirs, anchor)]
        self.cnt = torch.tensor(count, dtype=torch.int32, device="cuda")

    def __call__(self, rotated, pre_max, post_max, thr, use_dir=0, dir_offset=0.0, dir_limit=0.0, bins=2,
                 rng6=None, extra=1):
        L, B, S = self.L, self.B, self.code + 2
        ws_bytes = self.lib.b2s_nms_workspace_bytes(B, self.cap, pre_max)
        ws = torch.zeros(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
        width = post_max * S + extra
        rec = torch.full((B, width), -7.0, device="cuda")
        det_count = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        self.last = (rec, det_count)
        L.check(self.lib.b2s_nms(*[L.ptr(t) for t in self.d], L.ptr(self.cnt), B, self.cap, self.code, rotated,
                                 pre_max, post_max, thr, use_dir, dir_offset, dir_limit, bins,
                                 None if rng6 is None else L.f6(rng6), L.ptr(rec), width, L.ptr(det_count), L.ptr(ws),
                                 ws_bytes, L.stream()), "b2s_nms")
        torch.cuda.synchronize()
        sorted_slot = ws[:4 * B * pre_max].view(torch.int32).view(B, pre_max).cpu().numpy()
        return rec.cpu().numpy(), det_count.cpu().numpy(), sorted_slot


def _frames(rng, counts, cap, code, edge_rows=True):
    """[B, cap] candidate arrays from detection clusters; cand_label holds the slot index so each output row names
    its candidate; a few yaws make val/period + offset an exact integer."""
    B = len(counts)
    box = np.zeros((B, cap, code), np.float32)
    score = np.zeros((B, cap), np.float32)
    label = np.zeros((B, cap), np.int32)
    dirs = np.zeros((B, cap), np.int32)
    anchor = np.zeros((B, cap), np.int32)
    for f, n in enumerate(counts):
        m = min(n, cap)
        if m == 0:
            continue
        b = R.clusters(rng, m)
        box[f, :m, :7] = b
        box[f, :m, 7:] = rng.uniform(-1, 1, (m, code - 7))
        if edge_rows and m > 8:                                         # integer points of the direction fix-up
            period = np.float32(np.pi)
            for i, k in enumerate((0, -2, -1, 1, 2)):
                box[f, i, 6] = np.float32(0.78) + (np.float32(k) + np.float32(0.5)) * period
        score[f, :m] = R.scores_for(rng, m)
        if edge_rows and m > 8:
            score[f, 0] = np.float32(0.999)                             # ranked first: always kept
        label[f, :m] = np.arange(m)
        dirs[f, :m] = rng.integers(0, 2, m)
        anchor[f, :m] = rng.permutation(max(2 * m, 70000))[:m]
    return box, score, label, dirs, anchor


def _check_frames(nms, arrays, counts, cap, rotated, pre_max, post_max, thr, use_dir, dir_offset=0.78, dir_limit=0.5,
                  rng6=None):
    box, score, label, dirs, anchor = arrays
    rec, det_count, sorted_slot = nms(rotated, pre_max, post_max, thr, use_dir, dir_offset, dir_limit, 2)
    S = box.shape[2] + 2
    code = box.shape[2]
    rows_all = []
    for f, n in enumerate(counts):
        order = R.topk_order(score[f], anchor[f], n, cap, pre_max)
        assert sorted_slot[f, :len(order)].tolist() == order.tolist(), "frame %d: ranked order differs" % f
        k = int(det_count[f])
        assert rec[f, -1] == float(k)                                   # the count rides at the record's end
        rows = rec[f, :post_max * S].reshape(post_max, S)[:k]
        slots = rows[:, code + 1].astype(np.int64)
        assert (rows[:, code + 1] == slots).all() and ((slots >= 0) & (slots < min(n, cap))).all()
        cb = box[f, slots]
        np.testing.assert_array_equal(rows[:, :6], cb[:, :6])
        np.testing.assert_array_equal(rows[:, 7:code], cb[:, 7:code])
        np.testing.assert_array_equal(rows[:, code], score[f, slots])
        want_r = R.dir_fixup_f32(cb[:, 6], dirs[f, slots], dir_offset, dir_limit, 2) if use_dir else cb[:, 6]
        np.testing.assert_array_equal(rows[:, 6], want_r)
        ranked = box[f, order]
        b5 = _b5(ranked)
        c64 = R.bev_corners(b5)
        if rotated:
            iou, bound = _rank_iou(c64, b5)
        else:
            iou, bound = _rank_iou(c64, rotated=False, eps=1.0, delta=R.corner_rounding(b5))
        err = R.nms_certificate(order, slots, iou, bound, thr, post_max, inclusive=bool(rotated))
        assert err is None, "frame %d (%d candidates): %s" % (f, n, err)
        rows_all.append(rows)
    if rng6 is not None:                                                # the range test filters the same rows
        rec2, cnt2, _ = nms(rotated, pre_max, post_max, thr, use_dir, dir_offset, dir_limit, 2, rng6=rng6)
        lo, hi = np.asarray(rng6[:3], np.float32), np.asarray(rng6[3:], np.float32)
        for f, rows in enumerate(rows_all):
            m = np.all(rows[:, :3] >= lo, 1) & np.all(rows[:, :3] <= hi, 1)
            assert int(cnt2[f]) == int(m.sum()) and rec2[f, -1] == float(m.sum())
            np.testing.assert_array_equal(rec2[f, :post_max * S].reshape(post_max, S)[:int(m.sum())], rows[m])
    return det_count


@pytest.mark.parametrize("rotated", [1, 0])
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_b2s_nms_certificate(product, rotated, thr):
    rng = np.random.default_rng(int(thr * 100) + 7 * rotated)
    counts, cap = [1200, 700, 300, 64, 1], 1200
    arrays = _frames(rng, counts, cap, 7)
    nms = _Nms(product, *arrays, counts, cap)
    kept = _check_frames(nms, arrays, counts, cap, rotated, 1000, 300, thr, 1)
    assert kept[0] > 10


SWEEP_COUNTS = [0, 1, 63, 64, 65, 128, 129, 999, 1000, 1001, 4095, 4096, 4097]
PRE_MAX_LIMIT = 1280                                # largest pre_max whose mask fits the 200 KB reduce


@pytest.mark.parametrize("rotated,code,pre_max,post_max,use_dir,thr", [
    (1, 7, PRE_MAX_LIMIT, 1024, 1, 0.5), (1, 9, 1000, 100, 0, 0.1), (0, 7, 65, 1, 1, 0.5), (0, 9, 64, 300, 1, 0.7),
    (1, 7, 1, 100, 0, 0.01), (1, 9, 1000, 1024, 1, 0.7)])
def test_b2s_nms_sweep(product, rotated, code, pre_max, post_max, use_dir, thr):
    rng = np.random.default_rng(pre_max + post_max + code)
    cap = 4200
    counts = SWEEP_COUNTS + [int(x) for x in rng.choice(SWEEP_COUNTS, 32 - len(SWEEP_COUNTS) - 2)] + [5000, 4300]
    arrays = _frames(rng, counts, cap, code)
    box = arrays[0]
    # boxes exactly on the range faces (inclusive)
    rng6 = [-60.0, -45.0, -1.25, 75.0, 45.0, 0.0]
    for f in range(len(counts)):
        m = min(counts[f], cap)
        for i in range(min(m, 6)):
            box[f, m - 1 - i, i % 3] = np.float32(rng6[i % 3 + 3 * (i // 3)])
    nms = _Nms(product, *arrays, counts, cap)
    kept = _check_frames(nms, arrays, counts, cap, rotated, pre_max, post_max, thr, use_dir, rng6=rng6)
    if 4 * post_max < pre_max:
        assert int(kept.max()) == post_max                               # more survivors than post_max


def test_b2s_nms_rejects_out_of_range_sizes(product):
    rng = np.random.default_rng(0)
    counts, cap = [10, 3], 16
    nms = _Nms(product, *_frames(rng, counts, cap, 7, edge_rows=False), counts, cap)
    for pre_max, post_max in ((0, 10), (2049, 10), (PRE_MAX_LIMIT + 1, 10), (100, 0), (100, 1025)):
        with pytest.raises(RuntimeError, match="b2s_nms"):
            nms(1, pre_max, post_max, 0.5)
        torch.cuda.synchronize()
        rec, det_count = nms.last                                       # nothing was launched
        assert bool((rec == -7.0).all()) and bool((det_count == -1).all())
    rec, cnt, _ = nms(1, PRE_MAX_LIMIT, 1024, 0.5)                      # the limits themselves are accepted
    assert 1 <= cnt[0] <= 10 and 1 <= cnt[1] <= 3 and rec[0, -1] == float(cnt[0])


# ------------------------------------------------------------------------------------------------ decode
def _heads(rng, B, a_loc, H, W, code, ncls, nb):
    box = rng.normal(0, 0.4, (B, a_loc * code, H, W)).astype(np.float32)
    cls = rng.normal(-1.5, 2.0, (B, a_loc * ncls, H, W)).astype(np.float32)
    dirp = rng.normal(0, 1, (B, a_loc * nb, H, W)).astype(np.float32)
    A = a_loc * H * W
    anchors = np.zeros((A, code), np.float32)
    anchors[:, 0] = rng.uniform(0, 70.4, A)
    anchors[:, 1] = rng.uniform(-40, 40, A)
    anchors[:, 2] = -1.0
    anchors[:, 3:6] = [1.6, 3.9, 1.56]
    anchors[:, 6] = np.where(np.arange(A) // (H * W) % 2, np.float32(np.pi / 2), 0).astype(np.float32)
    # saturated logits (classes tie at 1.0: the first wins) and equal direction logits (bin 0)
    sat = [20.0, 90.0, 104.0]
    cls4 = cls.reshape(B, a_loc, ncls, H * W)
    for k in range(6):
        cls4[:, k % a_loc, :, k] = sat[k % 3] if ncls == 1 else np.roll(sat * ncls, k)[:ncls]
        cls4[:, (k + 1) % a_loc, :, 50 + k] = -np.array(sat)[k % 3]
    dirp.reshape(B, a_loc, nb, H * W)[:, :, 1, :40] = dirp.reshape(B, a_loc, nb, H * W)[:, :, 0, :40]
    return box, cls, dirp, anchors


def _decode_expect(box, cls, dirp, anchors, b, a_loc, H, W, code, ncls, nb, thr, mask=None):
    """fp64 reference of one frame: per anchor, the per-class sigmoid and its bound, decoded box and bound, dir."""
    HW = H * W
    A = a_loc * HW
    t = box[b].reshape(a_loc, code, HW).transpose(0, 2, 1).reshape(A, code)
    x = cls[b].reshape(a_loc, ncls, HW).transpose(0, 2, 1).reshape(A, ncls)
    d = dirp[b].reshape(a_loc, nb, HW).transpose(0, 2, 1).reshape(A, nb)
    s64, sb = R.sigmoid64(x), R.sigmoid_bound(x)
    top = s64.max(1)
    o = R.decode64(t, anchors)
    ob = R.decode_bound(t, anchors, o)
    return dict(s64=s64, sb=sb, top=top, o=o, ob=ob, dir=d.argmax(1), mask=mask)


def _check_candidates(ref, thr, got_anchor, got_score, got_box, got_label, got_dir, n_anchors):
    s64, sb, top = ref["s64"], ref["sb"], ref["top"]
    topb = sb[np.arange(len(top)), s64.argmax(1)]
    eligible = np.ones(n_anchors, bool) if ref["mask"] is None else ref["mask"].astype(bool)
    sure_in = eligible & (top - topb >= thr)
    maybe = eligible & (np.abs(top - thr) < topb)
    got = dict(zip(got_anchor.tolist(), range(len(got_anchor))))
    assert len(got) == len(got_anchor), "an anchor appears twice"
    assert set(np.nonzero(sure_in)[0]) <= set(got)
    assert set(got) <= set(np.nonzero(sure_in | maybe)[0])
    a = np.array(sorted(got))
    i = np.array([got[v] for v in a])
    assert (got_score[i] >= np.float32(thr)).all()                      # a near-threshold anchor joins iff its score does
    err = np.abs(got_score[i].astype(np.float64) - top[a])
    assert (err <= topb[a]).all(), float((err - topb[a]).max())
    # label: the first class among those whose fp32 score equals the max; fp64 near-ties may go either way
    lab = got_label[i]
    near_max = s64[a] + sb[a] >= (top[a] - topb[a])[:, None]
    assert near_max[np.arange(len(a)), lab].all()
    assert ((lab == s64[a].argmax(1)) | (near_max.sum(1) > 1)).all()
    np.testing.assert_array_equal(got_dir[i], ref["dir"][a])
    err = np.abs(got_box[i].astype(np.float64) - ref["o"][a])
    assert (err <= ref["ob"][a]).all(), float((err / ref["ob"][a]).max())
    return a, i


def _alloc(B, cap, code):
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
    return dict(box=z(B, cap, code), score=z(B, cap), label=z(B, cap, dt=torch.int32), dir=z(B, cap, dt=torch.int32),
                anchor=z(B, cap, dt=torch.int32), count=z(B, dt=torch.int32), status=z(1, dt=torch.int32))


def _cand_args(L, c, cap):
    return [L.ptr(c["box"]), L.ptr(c["score"]), L.ptr(c["label"]), L.ptr(c["dir"]), L.ptr(c["anchor"]),
            L.ptr(c["count"]), cap, L.ptr(c["status"]), L.stream()]


def _check_all(ref_of, c, B, thr, code):
    for b in range(B):
        n = int(c["count"][b])
        ref = ref_of(b)
        a, i = _check_candidates(ref, thr, c["anchor"][b, :n].cpu().numpy(), c["score"][b, :n].cpu().numpy(),
                                 c["box"][b, :n].cpu().numpy(), c["label"][b, :n].cpu().numpy(),
                                 c["dir"][b, :n].cpu().numpy(), len(ref["top"]))
        sat = (ref["top"][a] == 1.0)
        assert sat.sum() > 0 and (c["label"][b, :n].cpu().numpy()[i][sat] == 0).all()
        assert (c["score"][b, :n].cpu().numpy()[i][sat] == 1.0).all()


@pytest.mark.parametrize("ncls", [1, 3])
def test_decode_filter_nchw_and_strided(product, ncls):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(ncls)
    B, a_loc, H, W, code, nb, thr = 2, 4, 20, 24, 7, 2, 0.3
    A = a_loc * H * W
    box, cls, dirp, anchors = _heads(rng, B, a_loc, H, W, code, ncls, nb)
    t = {k: torch.from_numpy(v).cuda() for k, v in dict(box=box, cls=cls, dir=dirp, an=anchors).items()}
    c = _alloc(B, A, code)
    L.check(lib.b2s_decode_filter(L.ptr(t["box"]), L.ptr(t["cls"]), L.ptr(t["dir"]), L.ptr(t["an"]), None, B, a_loc, H,
                                  W, code, ncls, nb, thr, *_cand_args(L, c, A)), "b2s_decode_filter")
    torch.cuda.synchronize()
    assert int(c["status"]) == 0
    _check_all(lambda b: _decode_expect(box, cls, dirp, anchors, b, a_loc, H, W, code, ncls, nb, thr), c, B, thr, code)
    # the same heads as one packed NHWC record per pixel, with and without an anchors mask
    S = a_loc * (code + ncls + nb) + 3
    rec = np.zeros((B, H, W, S), np.float32)
    rec[..., :a_loc * code] = box.transpose(0, 2, 3, 1)
    rec[..., a_loc * code:a_loc * (code + ncls)] = cls.transpose(0, 2, 3, 1)
    rec[..., a_loc * (code + ncls):a_loc * (code + ncls + nb)] = dirp.transpose(0, 2, 3, 1)
    rd = torch.from_numpy(rec).cuda()
    sat_anchors = [(k % a_loc) * H * W + k for k in range(6)]
    for use_mask in (False, True):
        mask = (rng.random((B, A)) < 0.6).astype(np.uint8) if use_mask else None
        if use_mask:
            mask[:, sat_anchors] = 1                                    # keep the saturated anchors visible
        md = torch.from_numpy(mask).cuda() if use_mask else None
        c = _alloc(B, A, code)
        p = rd.data_ptr()
        L.check(lib.b2s_decode_filter_strided(ctypes.c_void_p(p), ctypes.c_void_p(p + 4 * a_loc * code),
                                              ctypes.c_void_p(p + 4 * a_loc * (code + ncls)), H * W * S, H * W * S,
                                              H * W * S, 1, S, L.ptr(t["an"]), L.ptr(md), B, a_loc, H, W, code, ncls,
                                              nb, thr, *_cand_args(L, c, A)), "b2s_decode_filter_strided")
        torch.cuda.synchronize()

        def ref_of(b):
            r = _decode_expect(box, cls, dirp, anchors, b, a_loc, H, W, code, ncls, nb, thr)
            r["mask"] = None if mask is None else mask[b]
            return r
        _check_all(ref_of, c, B, thr, code)


def test_decode_filter_segments_with_a_gap(product):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(9)
    B, code, ncls, nb, thr = 2, 9, 2, 2, 0.25
    shapes = [(2, 16, 20), (4, 8, 10)]
    gap = 37
    heads = [_heads(rng, B, a, H, W, code, ncls, nb) for a, H, W in shapes]
    bases = [0, shapes[0][0] * shapes[0][1] * shapes[0][2] + gap]
    A = bases[1] + shapes[1][0] * shapes[1][1] * shapes[1][2]
    anchors = np.zeros((A, code), np.float32)
    for (a, H, W), base, h in zip(shapes, bases, heads):
        anchors[base:base + a * H * W] = h[3]
    keep = [tuple(torch.from_numpy(x).cuda() for x in h[:3]) for h in heads]
    segs = []
    for (a, H, W), base, (bx, cl, dr) in zip(shapes, bases, keep):
        segs.append(dict(box=bx.data_ptr(), cls=cl.data_ptr(), dir=dr.data_ptr(), box_batch_stride=a * code * H * W,
                         cls_batch_stride=a * ncls * H * W, dir_batch_stride=a * nb * H * W, ch_stride=H * W,
                         pix_stride=1, a_loc=a, H=H, W=W, anchor_base=base))
    arr = L.head_segments(segs)
    ad = torch.from_numpy(anchors).cuda()
    c = _alloc(B, A, code)
    L.check(lib.b2s_decode_filter_segments(arr, 2, L.ptr(ad), None, A, B, code, ncls, nb, thr, *_cand_args(L, c, A)),
            "b2s_decode_filter_segments")
    torch.cuda.synchronize()
    for b in range(B):
        n = int(c["count"][b])
        got_a = c["anchor"][b, :n].cpu().numpy()
        assert not ((got_a >= bases[0] + shapes[0][0] * shapes[0][1] * shapes[0][2]) & (got_a < bases[1])).any()
        for (a, H, W), base, h in zip(shapes, bases, heads):
            sel = (got_a >= base) & (got_a < base + a * H * W)
            ref = _decode_expect(h[0], h[1], h[2], anchors[base:base + a * H * W], b, a, H, W, code, ncls, nb, thr)
            _check_candidates(ref, thr, got_a[sel] - base, c["score"][b, :n].cpu().numpy()[sel],
                              c["box"][b, :n].cpu().numpy()[sel], c["label"][b, :n].cpu().numpy()[sel],
                              c["dir"][b, :n].cpu().numpy()[sel], a * H * W)


# ------------------------------------------------------------------------------------------------ per-class branch
@pytest.mark.parametrize("agnostic", [False, True])
def test_multiclass_decode_nms_concat(product, agnostic):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(21 + agnostic)
    B, a_loc, H, W, code, ncls, nb = 3, 6, 24, 20, 7, 3, 2
    A = a_loc * H * W
    box, cls, dirp, anchors = _heads(rng, B, a_loc, H, W, code, ncls, nb)
    # dense clusters: neighbouring anchors share their centre so the NMS has work
    anchors[:, :2] = np.round(anchors[:, :2] / 4) * 4
    lo, hi = [0, 2, 4], [2, 4, 6]
    thr = np.array([0.3, 0.4, 0.35], np.float32)
    t = {k: torch.from_numpy(v).cuda() for k, v in dict(box=box, cls=cls, dir=dirp, an=anchors).items()}
    V, cap = ncls * B, A
    c = _alloc(V, cap, code)
    ilo, ihi = (ctypes.c_int * 3)(*lo), (ctypes.c_int * 3)(*hi)
    L.check(lib.b2s_decode_filter_multiclass(
        L.ptr(t["box"]), L.ptr(t["cls"]), L.ptr(t["dir"]), a_loc * code * H * W, a_loc * ncls * H * W,
        a_loc * nb * H * W, H * W, 1, L.ptr(t["an"]), B, a_loc, H, W, code, ncls, nb, None if agnostic else ilo,
        None if agnostic else ihi, thr.ctypes.data_as(ctypes.c_void_p), *_cand_args(L, c, cap)),
        "b2s_decode_filter_multiclass")
    torch.cuda.synchronize()
    assert int(c["status"]) == 0
    HW = H * W
    for cl in range(ncls):
        for b in range(B):
            v = cl * B + b
            n = int(c["count"][v])
            ref = _decode_expect(box, cls, dirp, anchors, b, a_loc, H, W, code, ncls, nb, float(thr[cl]))
            # one class at a time: the class's own score, the anchor range unless class-agnostic
            ref["s64"], ref["sb"] = ref["s64"][:, cl:cl + 1], ref["sb"][:, cl:cl + 1]
            ref["top"] = ref["s64"][:, 0]
            if not agnostic:
                ref["mask"] = ((np.arange(A) // HW >= lo[cl]) & (np.arange(A) // HW < hi[cl])).astype(np.uint8)
            lab = c["label"][v, :n].cpu().numpy()
            assert (lab == cl).all()
            _check_candidates(ref, float(thr[cl]), c["anchor"][v, :n].cpu().numpy(), c["score"][v, :n].cpu().numpy(),
                              c["box"][v, :n].cpu().numpy(), np.zeros(n, np.int64), c["dir"][v, :n].cpu().numpy(), A)
    # per-class NMS over the ncls*B virtual frames, then the class-order concat
    post, pre = 8, 500
    cand = [c[k].cpu().numpy() for k in ("box", "score", "label", "dir", "anchor")]
    counts = c["count"].cpu().tolist()
    nms = _Nms(product, *cand, counts, cap)
    rec, cnt, _ = nms(1, pre, post, 0.1, 1, 0.78, 0.5, 2, extra=0)
    S = code + 2
    assert int(cnt.max()) == post                                         # more survivors than the per-class post
    for v in range(V):
        order = R.topk_order(cand[1][v], cand[4][v], counts[v], cap, pre)
        rows = rec[v].reshape(post, S)[:int(cnt[v])]
        # rows -> candidate slots by their (box, score) bits
        key = {cand[0][v, s, :6].tobytes() + cand[1][v, s].tobytes(): s for s in order}
        slots = np.array([key[r[:6].tobytes() + r[code:code + 1].tobytes()] for r in rows], np.int64)
        b5 = _b5(cand[0][v, order])
        iou, bound = _rank_iou(R.bev_corners(b5), b5)
        assert R.nms_certificate(order, slots, iou, bound, 0.1, post, True) is None
    det = torch.full((B, ncls * post * S + 1), -3.0, device="cuda")
    det_count = torch.zeros(B, dtype=torch.int32, device="cuda")
    mc = torch.from_numpy(rec).cuda()
    cd = torch.from_numpy(cnt.astype(np.int32)).cuda()
    L.check(lib.b2s_concat_class_detections(L.ptr(mc), L.ptr(cd), B, ncls, post, code, L.ptr(det), det.shape[1],
                                            L.ptr(det_count), L.stream()), "b2s_concat_class_detections")
    torch.cuda.synchronize()
    det = det.cpu().numpy()
    for b in range(B):
        want = np.concatenate([rec[cl * B + b].reshape(post, S)[:int(cnt[cl * B + b])] for cl in range(ncls)])
        assert int(det_count[b]) == len(want) and det[b, -1] == float(len(want))
        np.testing.assert_array_equal(det[b, :len(want) * S].reshape(-1, S), want)
        assert np.array_equal(want[:, code + 1], np.sort(want[:, code + 1], kind="stable"))   # class order
