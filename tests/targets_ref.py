"""numpy restatement of csrc/targets.cu's two-pass target assignment, for one frame of a b2second.targets.TargetPlan.

Pass 1 takes each GT's maximum similarity over the unpruned anchors of its segment, GTs in chunks of CHUNK; pass 2
recomputes the same float32 similarities, the anchors' max / first argmax and the forced flag, then writes labels,
importance and box targets.  The dtypes follow the reference's: float32 anchors, GT of its own dtype, float64 where
iou_jit's eps or distance_similarity's dist_norm enter, float32 storage.
"""
import numpy as np

CHUNK = 128


def near_bbox(boxes):
    """rbbox2d_to_near_bbox of [N, >=7] boxes in their own dtype (numpy's promotion with weak Python floats)."""
    rots = boxes[:, 6]
    rp = np.abs(rots - np.floor(rots / np.pi + 0.5) * np.pi)
    swap = rp > np.pi / 4
    dx = np.where(swap, boxes[:, 4], boxes[:, 3])
    dy = np.where(swap, boxes[:, 3], boxes[:, 4])
    return np.stack([boxes[:, 0] - dx / 2, boxes[:, 1] - dy / 2, boxes[:, 0] + dx / 2, boxes[:, 1] + dy / 2], 1)


def similarity(kind, dn, asim, q):
    """asim float32 [n, 4] (plan.anchor_sim rows), q [k, 4] in the GT dtype -> float32 [n, k]"""
    T = q.dtype.type
    if kind == 0:
        a = asim
        a_area = (a[:, 2] - a[:, 0]).astype(np.float64) * (a[:, 3] - a[:, 1]).astype(np.float64)
        q_area = (q[:, 2] - q[:, 0]).astype(np.float64) * (q[:, 3] - q[:, 1]).astype(np.float64)
        iw = (np.minimum(a[:, None, 2].astype(T), q[None, :, 2]) - np.maximum(a[:, None, 0].astype(T), q[None, :, 0]))
        ih = (np.minimum(a[:, None, 3].astype(T), q[None, :, 3]) - np.maximum(a[:, None, 1].astype(T), q[None, :, 1]))
        iw, ih = iw.astype(np.float64), ih.astype(np.float64)
        inter = iw * ih
        ua = (a_area[:, None] + q_area[None, :]) - inter
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (inter / ua).astype(np.float32)
        return np.where((iw > 0) & (ih > 0), s, np.float32(0))
    dx = asim[:, None, 0].astype(T) - q[None, :, 0]
    dy = asim[:, None, 1].astype(T) - q[None, :, 1]
    near = (np.abs(dx).astype(np.float64) <= dn) & (np.abs(dy).astype(np.float64) <= dn)
    dist = (dx * dx + dy * dy).astype(np.float64)
    s = (1.0 - np.minimum(dist / dn, dn)).astype(np.float32)
    return np.where(near, s, np.float32(0))


def encode(g, a, linear_dim=False, vec_encode=False):
    """GroundBox3dCoder.encode of GT rows g (own dtype) against float32 anchors a, stored as float32"""
    diag = np.sqrt(a[:, 4] * a[:, 4] + a[:, 3] * a[:, 3])
    out = [(g[:, 0] - a[:, 0]) / diag, (g[:, 1] - a[:, 1]) / diag, (g[:, 2] - a[:, 2]) / a[:, 5]]
    for k in (3, 4, 5):
        r = g[:, k] / a[:, k]
        out.append(r - 1 if linear_dim else np.log(r))
    if vec_encode:
        out += [np.cos(g[:, 6]) - np.cos(a[:, 6]), np.sin(g[:, 6]) - np.sin(a[:, 6])]
    else:
        out.append(g[:, 6] - a[:, 6])
    out += [g[:, k] - a[:, k] for k in range(7, a.shape[1])]
    return np.stack([o.astype(np.float32) for o in out], 1)


def assign(plan, gt_boxes, gt_seg, gt_class, importance=None, mask=None):
    """one frame: gt_boxes [G, ndim] float32/float64, gt_seg [G] segment of each GT (-1: none), gt_class [G] label
    values, importance [G] or None, mask [A] bool or None.
    -> labels int32 [A], targets float32 [A, code], importance float32 [A], gt_id int32 [A], overlap float32 [A]"""
    A = plan.num_anchors
    labels = np.full(A, -1, np.int32)
    targets = np.zeros((A, plan.code_size), np.float32)
    imp_out = np.zeros(A, np.float32)
    gt_id = np.full(A, -1, np.int32)
    overlap = np.zeros(A, np.float32)
    mask = np.ones(A, bool) if mask is None else np.asarray(mask, bool)
    imp = np.ones(len(gt_boxes), np.float32) if importance is None else np.asarray(importance, np.float32)
    for s, seg in enumerate(plan.segments):
        idx = np.flatnonzero(mask[seg.begin:seg.end]) + seg.begin
        gts = np.flatnonzero(np.asarray(gt_seg) == s)
        if len(idx) == 0:
            continue                                               # every anchor pruned: -1 / 0 / 0
        if len(gts) == 0:
            labels[idx] = 0
            imp_out[idx] = 1
            continue
        gb = gt_boxes[gts]
        q = np.stack([gb[:, 0], gb[:, 1], np.zeros_like(gb[:, 0]), np.zeros_like(gb[:, 0])], 1) \
            if seg.kind == 1 else near_bbox(gb)
        asim = plan.anchor_sim[idx]
        gmax = np.empty(len(gts), np.float32)
        for c0 in range(0, len(gts), CHUNK):                        # pass 1
            gmax[c0:c0 + CHUNK] = similarity(seg.kind, seg.distance_norm, asim, q[c0:c0 + CHUNK]).max(0)
        gmax[gmax == 0] = -1
        best = np.full(len(idx), -np.inf, np.float32)
        arg = np.zeros(len(idx), np.int64)
        forced = np.zeros(len(idx), bool)
        for c0 in range(0, len(gts), CHUNK):                        # pass 2
            sm = similarity(seg.kind, seg.distance_norm, asim, q[c0:c0 + CHUNK])
            cm, ca = sm.max(1), sm.argmax(1)
            better = cm > best
            best = np.where(better, cm, best)
            arg = np.where(better, ca + c0, arg)
            forced |= (sm == gmax[None, c0:c0 + CHUNK]).any(1)
        cls = np.asarray(gt_class)[gts][arg]
        pos = best >= plan.matched_thresholds[idx]
        lab = np.where(forced, cls, np.where(best < plan.unmatched_thresholds[idx], 0, np.where(pos, cls, -1)))
        labels[idx] = lab
        imp_out[idx] = np.where(pos, imp[arg], np.float32(1))
        fg = (forced | pos) & (cls > 0)
        if fg.any():
            targets[idx[fg]] = encode(gb[arg[fg]], plan.anchors[idx[fg]], plan.linear_dim, plan.vec_encode)
            gt_id[idx[fg]] = arg[fg]
            overlap[idx[fg]] = best[fg]
    return labels, targets, imp_out, gt_id, overlap


# ------------------------------------------------------------------------------------------------ fixtures
LOG_COLUMNS = (3, 4, 5)          # np.log in GroundBox3dCoder.encode (without linear_dim): libm-dependent last bits
CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"]


def sha1(a):
    import hashlib
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixture_path(name):
    import os
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "targets", name + ".npz")


def mirror_plan(name):
    from b2second import config, models, targets
    cfg = config.get_config(name)
    return targets.plan(models.MirrorTargetAssigner(cfg), cfg.feature_map_size)


def load_fixture(name):
    """-> (npz dict, list of frames: dict gt_boxes, gt_names, gt_classes, importance, mask, labels, importance_out,
    pos, targets[, overlap, gt_id, inds])"""
    z = dict(np.load(fixture_path(name), allow_pickle=False))
    A = int(z["num_anchors"])
    frames = []
    for f in range(int(z["num_frames"])):
        fr = {k: z["%s_%d" % (k, f)] for k in ("gt_boxes", "gt_names", "gt_classes", "importance", "labels",
                                                "importance_out", "pos", "targets", "overlap", "gt_id", "inds")
              if "%s_%d" % (k, f) in z}
        fr["labels"] = fr["labels"].astype(np.int32)
        fr["mask"] = np.unpackbits(z["mask_%d" % f])[:A].astype(bool) if "mask_%d" % f in z else None
        frames.append(fr)
    return z, frames


def segments_of(plan, gt_names):
    """per-class mode: the segment of each GT by name (-1: no class of that name); assign_all: 0"""
    if not plan.assign_per_class:
        return np.zeros(len(gt_names), np.int32)
    return np.array([plan.classes.index(n) if n in plan.classes else -1 for n in gt_names], np.int32)


def ulp_diff(a, b):
    """elementwise distance in float32 units in the last place"""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(ordered(a) - ordered(b))


def assert_targets_match(got, want, log_ulp=4):
    """box targets: every column but the log ones bit-equal, the log ones within log_ulp float32 ulp"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (got.shape, want.shape)
    exact = [c for c in range(want.shape[1]) if c not in LOG_COLUMNS]
    np.testing.assert_array_equal(got[:, exact], want[:, exact])
    if len(want):
        d = ulp_diff(got[:, list(LOG_COLUMNS)], want[:, list(LOG_COLUMNS)])
        assert d.max() <= log_ulp, "log components differ by %d ulp" % d.max()


def check_frame(labels, tg, imp, fr):
    """one frame's CUDA labels, box targets and importance against the expected ones of `fr` (labels,
    importance_out, pos, targets): equal, the log components of the targets within assert_targets_match's ulp"""
    labels, tg, imp = (x.cpu().numpy() for x in (labels, tg, imp))
    np.testing.assert_array_equal(labels, fr["labels"])
    np.testing.assert_array_equal(imp, fr["importance_out"])
    np.testing.assert_array_equal(np.flatnonzero(labels > 0), fr["pos"])
    assert_targets_match(tg[fr["pos"]], fr["targets"])
    assert not tg[labels <= 0].any()
