"""Numpy restatement of csrc/augment.cu (b2second.augment) and the synthetic frames of the augmentation fixtures.

``augment(plan, points, boxes, valid, draws_frame...)`` repeats the kernels' arithmetic step by step in the same dtypes
(float32 points, box dtype T, float64 draws): the pose selection of noise_per_box with box_collision_test's predicates,
the first-containing-box point transform, box3d_transform_, the flips, global rotation, scaling, translation, the
range filter and limit_period.  ``frame(name, kind, seed)`` regenerates the fixture frames' inputs from their seeds.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "second.pytorch_b200"))

from b2second import augment as aug, config  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "augment")
CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"]
KINDS = ["empty", "one", "crowd", "overlap", "many", "outside"]
OTHER_NAMES = ["Truck", "Misc"]          # names outside every class list: obstacles that drop


def is_nuscenes(name):
    return name.startswith("nuscenes")


def class_names(name):
    return [c.class_name for c in config.get_config(name).classes]


# ------------------------------------------------------------------------------------------------ synthetic frames
def frame(name, kind, seed):
    """-> (points float32 [N, F], boxes [G, 7 or 9] (float32 KITTI, float64 NuScenes), names [G]) of a fixture frame.
    Points concentrate in and around the boxes, plus a sparse background over the point cloud range."""
    cfg = config.get_config(name)
    rng = np.random.default_rng(seed)
    r = np.asarray(cfg.point_cloud_range, np.float64)
    classes = class_names(name)
    nus = is_nuscenes(name)

    def rand_boxes(n, lo=None, hi=None):
        lo = r[:2] + 2.0 if lo is None else np.asarray(lo, np.float64)
        hi = r[3:5] - 2.0 if hi is None else np.asarray(hi, np.float64)
        b = np.zeros((n, 7))
        b[:, :2] = rng.uniform(lo, hi, (n, 2))
        b[:, 2] = rng.uniform(-1.9, -1.2, n)
        b[:, 3] = rng.uniform(1.5, 2.0, n)
        b[:, 4] = rng.uniform(3.5, 4.6, n)
        b[:, 5] = rng.uniform(1.4, 1.8, n)
        b[:, 6] = rng.uniform(-np.pi, np.pi, n)
        return b

    if kind == "empty":
        b = np.zeros((0, 7))
    elif kind == "one":
        b = rand_boxes(1, r[:2] + 10, r[3:5] - 10)
    elif kind == "crowd":
        # a 4 x 4 block of cars with 0.3 m gaps (inner ones cannot move) and a pair of heavily overlapping boxes
        c0 = rng.uniform(r[:2] + 15, r[3:5] - 15)
        gx, gy = np.meshgrid(np.arange(4) * 2.1, np.arange(4) * 4.5)
        b = np.zeros((16, 7))
        b[:, 0] = c0[0] + gx.ravel()
        b[:, 1] = c0[1] + gy.ravel()
        b[:, 2] = -1.6
        b[:, 3:6] = [1.8, 4.2, 1.5]
        b[:, 6] = rng.uniform(-0.01, 0.01, 16)
        pair = rand_boxes(1, r[:2] + 10, r[3:5] - 10)
        twin = pair.copy()
        twin[0, :2] += rng.uniform(-0.2, 0.2, 2)
        b = np.concatenate([b, pair, twin, rand_boxes(4)])
    elif kind == "overlap":
        a = rand_boxes(4, r[:2] + 8, r[3:5] - 8)
        inner = a.copy()
        inner[:, 3:5] *= 0.4                 # fully inside its partner: only the containment test sees it
        inner[:, 6] += 0.3
        b = np.concatenate([a, inner, rand_boxes(6)])
    elif kind == "many":
        b = rand_boxes(210)
    elif kind == "outside":
        b = rand_boxes(12)
        # centres within a metre of the range's x / y edges: flips, rotation and noise push some out
        b[:6, 0] = np.where(rng.random(6) < 0.5, r[0] + rng.uniform(0.2, 1.0, 6), r[3] - rng.uniform(0.2, 1.0, 6))
        b[6:, 1] = np.where(rng.random(6) < 0.5, r[1] + rng.uniform(0.2, 1.0, 6), r[4] - rng.uniform(0.2, 1.0, 6))
    else:
        raise KeyError(kind)
    n = len(b)
    pool = classes + OTHER_NAMES
    names = np.array([pool[i] for i in rng.integers(0, len(pool), n)] if n else [], dtype="<U20")
    if n:
        names[0] = classes[0]
    if nus:
        b = np.concatenate([b, rng.normal(0, 3.0, (n, 2))], axis=1)
        boxes = b.astype(np.float64)
    else:
        boxes = b.astype(np.float32)
    # points: per box a cloud over the box grown by 40 %, then background
    per_box = max(6, min(60, 2400 // max(n, 1)))
    pts = []
    for i in range(n):
        bx = b[i]
        loc = rng.uniform(-0.7, 0.7, (per_box, 3)) * bx[3:6]
        c, s = np.cos(bx[6]), np.sin(bx[6])
        wx = loc[:, 0] * c - loc[:, 1] * s
        wy = loc[:, 0] * s + loc[:, 1] * c
        pts.append(np.stack([wx + bx[0], wy + bx[1], loc[:, 2] + bx[2]], 1))
    bg = rng.uniform(r[:3], r[3:], (400, 3))
    xyz = np.concatenate(pts + [bg]) if pts else bg
    nf = 5 if nus else 4
    extra = rng.uniform(0, 1, (len(xyz), nf - 3))
    return np.concatenate([xyz, extra], 1).astype(np.float32), boxes, names


def class_mask(name, names):
    classes = class_names(name)
    valid = np.array([n in classes for n in names], np.bool_)
    cls = np.array([classes.index(n) + 1 if v else 0 for n, v in zip(names, valid)], np.int32)
    return valid, cls


# ------------------------------------------------------------------------------------------------ restatement
def _f(T, v):
    return np.asarray(v, dtype=T)[()]


def _trig(T, a):
    a = np.asarray(a, np.float64)
    return np.cos(a).astype(T), np.sin(a).astype(T)


def _rot(x, y, c, s):
    """(x, y) @ [[c, -s], [s, c]], each product rounded in the operands' dtype, then the sum"""
    return x * c + y * s, x * (-s) + y * c


def corners2d(b):
    T = b.dtype.type
    c, s = _trig(T, b[:, 6])
    nx = np.array([-0.5, -0.5, 0.5, 0.5], T)
    ny = np.array([-0.5, 0.5, 0.5, -0.5], T)
    px = b[:, 3:4] * nx
    py = b[:, 4:5] * ny
    x, y = _rot(px, py, c[:, None], s[:, None])
    return np.stack([x + b[:, 0:1], y + b[:, 1:2]], -1)          # [N, 4, 2]


def standup(cor):
    return np.concatenate([cor.min(1), cor.max(1)], -1)          # [N, 4]: x0 y0 x1 y1


def _contains(a, q):
    """[..., 4, 2] pairs: every corner of q strictly inside clockwise a"""
    ok = np.ones(np.broadcast_shapes(a.shape[:-2], q.shape[:-2]), bool)
    for l in range(4):
        for k in range(4):
            k1 = (k + 1) % 4
            v0 = -(a[..., k, 0] - a[..., k1, 0])
            v1 = -(a[..., k, 1] - a[..., k1, 1])
            cross = v1 * (a[..., k, 0] - q[..., l, 0])
            cross = cross - v0 * (a[..., k, 1] - q[..., l, 1])
            ok &= ~(cross >= 0)
    return ok


def collide(a, asu, q, qsu):
    """box_collision_test's decision for broadcast pairs a [..., 4, 2] / q [..., 4, 2]"""
    iw = np.minimum(asu[..., 2], qsu[..., 2]) - np.maximum(asu[..., 0], qsu[..., 0])
    ih = np.minimum(asu[..., 3], qsu[..., 3]) - np.maximum(asu[..., 1], qsu[..., 1])
    near = (iw > 0) & (ih > 0)
    hit = np.zeros(near.shape, bool)
    for k in range(4):
        A0, A1 = a[..., k, 0], a[..., k, 1]
        B0, B1 = a[..., (k + 1) % 4, 0], a[..., (k + 1) % 4, 1]
        for l in range(4):
            C0, C1 = q[..., l, 0], q[..., l, 1]
            D0, D1 = q[..., (l + 1) % 4, 0], q[..., (l + 1) % 4, 1]
            acd = (D1 - A1) * (C0 - A0) > (C1 - A1) * (D0 - A0)
            bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0)
            abc = (C1 - A1) * (B0 - A0) > (B1 - A1) * (C0 - A0)
            abd = (D1 - A1) * (B0 - A0) > (B1 - A1) * (D0 - A0)
            hit |= (acd != bcd) & (abc != abd)
    return near & (hit | _contains(a, q) | _contains(q, a))


def select_tries(boxes, valid, loc, rot):
    """noise_per_box: the first collision-free try of each valid box in order (-1: none)"""
    T = boxes.dtype.type
    n = len(boxes)
    cor = corners2d(boxes)
    su = standup(cor)
    sel = np.full(n, -1, np.int32)
    for i in range(n):
        if not valid[i]:
            continue
        c, s = _trig(T, rot[i])                                  # [M]
        x = cor[i, None, :, 0] - boxes[i, 0]
        y = cor[i, None, :, 1] - boxes[i, 1]
        x, y = _rot(x, y, c[:, None], s[:, None])                # [M, 4]
        ox = boxes[i, 0].astype(np.float64) + loc[i, :, 0]
        oy = boxes[i, 1].astype(np.float64) + loc[i, :, 1]
        tc = np.stack([(x.astype(np.float64) + ox[:, None]).astype(T),
                       (y.astype(np.float64) + oy[:, None]).astype(T)], -1)   # [M, 4, 2]
        tsu = standup(tc)
        # only boxes whose standup box meets the tries' combined standup box can collide (iw > 0 and ih > 0)
        lo, hi = tsu[:, :2].min(0), tsu[:, 2:].max(0)
        near = (np.minimum(su[:, 2], hi[0]) - np.maximum(su[:, 0], lo[0]) > 0) & \
               (np.minimum(su[:, 3], hi[1]) - np.maximum(su[:, 1], lo[1]) > 0)
        near[i] = False
        others = np.flatnonzero(near)
        if len(others):
            hit = collide(tc[:, None], tsu[:, None], cor[None, others], su[None, others]).any(1)
        else:
            hit = np.zeros(len(tc), bool)
        free = np.flatnonzero(~hit)
        if len(free):
            j = int(free[0])
            sel[i] = j
            cor[i] = tc[j]
            su[i] = tsu[j]
    return sel


def planes(boxes):
    """[N, 6, 4]: inward normals and d of center_to_corner_box3d(origin 0.5) surfaces, in the box dtype"""
    T = boxes.dtype.type
    c, s = _trig(T, boxes[:, 6])
    cx = np.array([0, 0, 0, 0, 1, 1, 1, 1])
    cy = np.array([0, 0, 1, 1, 0, 0, 1, 1])
    cz = np.array([0, 1, 1, 0, 0, 1, 1, 0])
    h = lambda bits: np.where(bits == 1, T(0.5), T(-0.5)).astype(T)   # noqa: E731
    x = boxes[:, 3:4] * h(cx)
    y = boxes[:, 4:5] * h(cy)
    z = boxes[:, 5:6] * h(cz)
    x, y = _rot(x, y, c[:, None], s[:, None])
    cr = np.stack([x + boxes[:, 0:1], y + boxes[:, 1:2], z + boxes[:, 2:3]], -1)   # [N, 8, 3]
    idx = [(0, 1, 2), (7, 6, 5), (0, 3, 7), (1, 5, 6), (0, 4, 5), (3, 2, 6)]
    out = np.zeros((len(boxes), 6, 4), T)
    for j, (i0, i1, i2) in enumerate(idx):
        s0, s1, s2 = cr[:, i0], cr[:, i1], cr[:, i2]
        a = s0 - s1
        b = s1 - s2
        n0 = a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1]
        n1 = a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2]
        n2 = a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]
        out[:, j] = np.stack([n0, n1, n2, (-s0[:, 0]) * n0 - s0[:, 1] * n1 - s0[:, 2] * n2], -1)
    return out


def first_box(points, boxes, valid):
    """index of the first valid box whose 3-D box holds each point (-1 none)"""
    T = boxes.dtype.type
    pl = planes(boxes)
    p = points[:, :3].astype(T)
    out = np.full(len(points), -1, np.int32)
    for g in range(len(boxes)):
        if not valid[g]:
            continue
        sign = p[:, 0] * pl[g, :, 0][:, None] + p[:, 1] * pl[g, :, 1][:, None]
        sign = sign + p[:, 2] * pl[g, :, 2][:, None]
        sign = sign + pl[g, :, 3][:, None]                         # [6, N]
        inside = (sign < 0).all(0) & (out < 0)
        out[inside] = g
    return out


def _pt(p, c, op):
    """float32 point op box value in the promoted dtype, stored as float32"""
    if np.asarray(c).dtype == np.float64:
        return op(p.astype(np.float64), c).astype(np.float32)
    return op(p, c)


def augment(plan, points, boxes, valid, classes, importance, d, f=0, g0=0):
    """frame f of draws ``d`` (its boxes start at row g0 of d.loc_noise) -> dict of host arrays:
    points (float32, permuted), point_box, selected, boxes (kept, input dtype), classes, importance, src_row."""
    T = boxes.dtype.type
    n = len(boxes)
    pts = points.copy()
    if plan.object_noise and n:
        loc = d.loc_noise[g0:g0 + n]
        rot = d.rot_noise[g0:g0 + n]
        if n > aug.MAX_BOXES:
            sel = np.full(n, aug.SEL_SKIPPED, np.int32)
        else:
            sel = select_tries(boxes, valid, loc, rot)
        fb = first_box(pts, boxes, valid) if n <= aug.MAX_BOXES else np.full(len(pts), -1, np.int32)
        lt = np.zeros((n, 3))
        rt = np.zeros(n)
        ok = sel >= 0
        lt[ok] = loc[ok, sel[ok]]
        rt[ok] = rot[ok, sel[ok]]
        m = fb >= 0
        g = fb[m]
        c32, s32 = _trig(np.float32, rt[g])
        ctr = boxes[g, :3]
        x = _pt(pts[m, 0], ctr[:, 0], np.subtract)
        y = _pt(pts[m, 1], ctr[:, 1], np.subtract)
        z = _pt(pts[m, 2], ctr[:, 2], np.subtract)
        x, y = _rot(x, y, c32, s32)
        x, y, z = (_pt(x, ctr[:, 0], np.add), _pt(y, ctr[:, 1], np.add), _pt(z, ctr[:, 2], np.add))
        pts[m, 0] = _pt(x, lt[g, 0], np.add)
        pts[m, 1] = _pt(y, lt[g, 1], np.add)
        pts[m, 2] = _pt(z, lt[g, 2], np.add)
        b = boxes.copy()
        b[:, :3] = (b[:, :3].astype(np.float64) + lt).astype(T)
        b[:, 6] = (b[:, 6].astype(np.float64) + rt).astype(T)
        if n > aug.MAX_BOXES:
            b = boxes.copy()
    else:
        sel = np.full(n, aug.SEL_SKIPPED if plan.object_noise else aug.SEL_NONE, np.int32)
        if plan.object_noise and n == 0:
            sel = np.zeros(0, np.int32)
        fb = np.full(len(pts), -1, np.int32)
        b = boxes.copy()
    flip_y, flip_x, translate, angle, scale = d.frame[f, :5]
    t = d.frame[f, 5:8]
    vel = b.shape[1] == 9
    if flip_y:
        b[:, 1] = -b[:, 1]
        b[:, 6] = -b[:, 6] + T(np.pi)
        if vel:
            b[:, 8] = -b[:, 8]
        pts[:, 1] = -pts[:, 1]
    if flip_x:
        b[:, 0] = -b[:, 0]
        b[:, 6] = -b[:, 6]
        if vel:
            b[:, 7] = -b[:, 7]
        pts[:, 0] = -pts[:, 0]
    c32, s32 = _trig(np.float32, angle)
    pts[:, 0], pts[:, 1] = _rot(pts[:, 0], pts[:, 1], c32, s32)
    cT, sT = _trig(T, angle)
    b[:, 0], b[:, 1] = _rot(b[:, 0], b[:, 1], cT, sT)
    b[:, 6] = b[:, 6] + T(angle)
    if vel:
        b[:, 7], b[:, 8] = _rot(b[:, 7], b[:, 8], T(c32), T(s32))
    pts[:, :3] *= np.float32(scale)
    b[:, :6] *= T(scale)
    if vel:
        b[:, 7:] *= T(scale)
    if translate:
        pts[:, :3] = (pts[:, :3].astype(np.float64) + t).astype(np.float32)
        b[:, :3] = (b[:, :3].astype(np.float64) + t).astype(T)
    rx0, ry0, rx1, ry1 = plan.bv_range
    dx, dy = np.float32(rx1 - rx0), np.float32(ry1 - ry0)
    poly = np.array([[rx0, ry0], [rx0, ry0 + dy], [rx0 + dx, ry0 + dy], [rx0 + dx, ry0]], np.float32)
    inr = np.ones(n, bool)
    for k in range(4):
        kp = (k + 3) % 4
        v0, v1 = poly[k, 0] - poly[kp, 0], poly[k, 1] - poly[kp, 1]
        cross = T(v1) * (T(poly[k, 0]) - b[:, 0])
        cross = cross - T(v0) * (T(poly[k, 1]) - b[:, 1])
        inr &= ~(cross >= 0)
    kept = valid & inr
    period = T(2 * np.pi)
    b[:, 6] = b[:, 6] - np.floor(b[:, 6] / period + T(0.5)) * period
    order = np.arange(len(pts))
    if d.perm is not None:
        p0 = sum(d.num_points[:f])
        order = d.perm[p0:p0 + len(pts)].astype(np.int64)
    imp = np.ones(n, np.float32) if importance is None else np.asarray(importance, np.float32)
    src = np.flatnonzero(kept).astype(np.int32)
    return {"points": pts[order], "point_box": fb[order], "selected": sel, "boxes": b[src], "classes": classes[src],
            "importance": imp[src], "src_row": src}


# ------------------------------------------------------------------------------------------------ fixtures
def fixture_path(name):
    return os.path.join(GOLDEN, name + ".npz")


def load_fixture(name):
    z = np.load(fixture_path(name), allow_pickle=False)
    frames = []
    for f in range(int(z["num_frames"])):
        fr = {k[:-len("_%d" % f)]: z[k] for k in z.files if k.endswith("_%d" % f)}
        frames.append(fr)
    return z, frames


def state_digest(rs):
    """sha1 of a RandomState's full state (key, position, cached gaussian)"""
    st = rs.get_state() if hasattr(rs, "get_state") else np.random.get_state()
    h = hashlib.sha1()
    h.update(np.asarray(st[1]).tobytes())
    h.update(np.array([st[2], st[3]], np.float64).tobytes())
    h.update(np.float64(st[4]).tobytes())
    return h.hexdigest()


def ulp32(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def assert_close_rows(got, want, cols, what):
    """values of ``cols`` within 4 float32 ulp of each row's largest |coordinate| of ``cols``, and within 4 ulp of the
    value itself at float64"""
    got = np.asarray(got)
    want = np.asarray(want)
    if got.shape != want.shape:
        raise AssertionError("%s: shape %s != %s" % (what, got.shape, want.shape))
    if not len(got):
        return
    g = got[:, cols].astype(np.float64)
    w = want[:, cols].astype(np.float64)
    if want.dtype == np.float64:
        tol = 4 * np.maximum(np.spacing(np.abs(w)), ulp32(np.abs(w).max(1, keepdims=True)))
    else:
        tol = 4 * ulp32(np.abs(w).max(1, keepdims=True))
    bad = np.abs(g - w) > tol
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError("%s: row %d col %d: %r vs %r (tol %r), %d bad" % (
            what, i[0], cols[i[1]], g[tuple(i)], w[tuple(i)], tol[tuple(i)], int(bad.sum())))


def compare(got, fr, what):
    """augmentation outputs (dict of host arrays) against a fixture frame: the decisions, order and the element-wise
    values exactly; rotated values (x, y of points and boxes, box velocity) within assert_close_rows's bound"""
    np.testing.assert_array_equal(got["selected"], fr["selected"], err_msg=what + " selected")
    np.testing.assert_array_equal(got["point_box"], fr["point_box"], err_msg=what + " point_box")
    np.testing.assert_array_equal(got["src_row"], fr["src_row"], err_msg=what + " src_row")
    np.testing.assert_array_equal(got["classes"], fr["classes"], err_msg=what + " classes")
    np.testing.assert_array_equal(got["importance"], fr["importance"], err_msg=what + " importance")
    gp, wp = got["points"], fr["points"]
    assert gp.dtype == np.float32 and gp.shape == wp.shape, (what, gp.shape, wp.shape)
    np.testing.assert_array_equal(gp[:, 3:], wp[:, 3:], err_msg=what + " point features")
    assert_close_rows(gp, wp, [0, 1, 2], what + " points xyz")
    gb, wb = got["boxes"], fr["boxes"]
    assert gb.dtype == wb.dtype and gb.shape == wb.shape, (what, gb.dtype, wb.dtype, gb.shape, wb.shape)
    np.testing.assert_array_equal(gb[:, 3:6], wb[:, 3:6], err_msg=what + " box dims")
    assert_close_rows(gb, wb, [0, 1, 2], what + " box xyz")
    np.testing.assert_array_equal(gb[:, 6], wb[:, 6], err_msg=what + " box yaw")
    if gb.shape[1] == 9:
        assert_close_rows(gb, wb, [7, 8], what + " box velocity")
