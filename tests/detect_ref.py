"""Plain fp64 reference of the detection stage (csrc/detect.cu, csrc/geometry.cuh), vectorised numpy.

* `inter_area`: intersection area of convex quads, by a different algorithm from the kernel's Sutherland-Hodgman
  clip: collect the corners of each quad that lie in the other (closed) quad and every edge-edge crossing, sort them
  by angle about their mean, shoelace.  Every point lies on the boundary of the convex intersection, so shared and
  collinear edges, identical and nested quads need no special case.  The orientation predicate is exact for float32
  corners: differences of float32 values and their products fit a float64 mantissa.
* `overlaps` (IoU and criteria 0, 1, 2 of `rotate_iou_gpu_eval`), `bev_corners` in fp64 from float32 boxes.
* per-pair error bounds of the fp32 kernels (`clip_bound`, `corner_bound`, `aligned_bound`), derived below.
* `nms_certificate`: accepts exactly the keep lists greedy NMS can produce when pairs within the bound of the
  threshold may go either way.
* `topk_order`, `decode64`, `sigmoid64` and the fp32 direction fix-up `dir_fixup_f32`.
* generators of detection-like box clusters (`clusters`).
"""
import numpy as np

U = 2.0 ** -24                                  # unit roundoff of float32
C_CLIP = 8.0                                    # constant of the clip bound (see clip_bound)

# cluster centres: near the origin, and at KITTI / NuScenes range
CENTRES = [(0.0, 0.0), (70.4, 40.0), (70.4, -40.0), (51.2, 51.2), (-51.2, 51.2), (51.2, -51.2), (-51.2, -51.2)]


# ------------------------------------------------------------------------------------------------ geometry
def bev_corners(boxes5):
    """float32 (x, y, w, l, r) [N,5] -> exact-math corners [N,4,2] in float64, in the kernel's order (clockwise from
    the min corner, rotated clockwise for positive r; geometry.cuh bev_corners)."""
    b = np.asarray(boxes5, np.float32).astype(np.float64).reshape(-1, 5)
    x, y, w, l, r = b.T
    s, c = np.sin(r)[:, None], np.cos(r)[:, None]
    px = w[:, None] * np.array([-0.5, -0.5, 0.5, 0.5])
    py = l[:, None] * np.array([-0.5, 0.5, 0.5, -0.5])
    return np.stack([px * c + py * s + x[:, None], -px * s + py * c + y[:, None]], -1)


def quad_area(q):
    """|shoelace| of quads [M,4,2] (float64)."""
    q = np.asarray(q, np.float64)
    x, y = q[..., 0], q[..., 1]
    return 0.5 * np.abs((x * np.roll(y, -1, -1) - np.roll(x, -1, -1) * y).sum(-1))


def _inside(p, q):
    """points p [M,K,2] in the closed convex quads q [M,4,2] (either orientation) -> [M,K] bool."""
    a, b = q, np.roll(q, -1, 1)
    e = (b - a)[:, None]                                                  # [M,1,4,2]
    d = p[:, :, None, :] - a[:, None]                                     # [M,K,4,2]
    cr = e[..., 0] * d[..., 1] - e[..., 1] * d[..., 0]                    # [M,K,4]
    return (cr >= 0).all(-1) | (cr <= 0).all(-1)


def _inter_chunk(a, b):
    M = a.shape[0]
    pa, pb = _inside(a, b), _inside(b, a)
    # edge-edge crossings: edge i of a against edge j of b
    a1, a2 = a[:, :, None], np.roll(a, -1, 1)[:, :, None]
    b1, b2 = b[:, None], np.roll(b, -1, 1)[:, None]
    d1, d2 = a2 - a1, b2 - b1
    den = d1[..., 0] * d2[..., 1] - d1[..., 1] * d2[..., 0]
    w = b1 - a1
    ok = den != 0
    sden = np.where(ok, den, 1.0)
    t = (w[..., 0] * d2[..., 1] - w[..., 1] * d2[..., 0]) / sden
    s = (w[..., 0] * d1[..., 1] - w[..., 1] * d1[..., 0]) / sden
    ok &= (t >= 0) & (t <= 1) & (s >= 0) & (s <= 1)
    x = (a1 + t[..., None] * d1).reshape(M, 16, 2)
    pts = np.concatenate([a, b, x], 1)                                    # [M,24,2]
    valid = np.concatenate([pa, pb, ok.reshape(M, 16)], 1)
    nv = valid.sum(1)
    cen = (pts * valid[..., None]).sum(1) / np.maximum(nv, 1)[:, None]
    ang = np.arctan2(pts[..., 1] - cen[:, None, 1], pts[..., 0] - cen[:, None, 0])
    ang = np.where(valid, ang, 10.0)                                      # invalid points sort last
    o = np.argsort(ang, 1, kind="stable")
    sp = np.take_along_axis(pts, o[..., None], 1)
    sv = np.take_along_axis(valid, o, 1)
    sp = np.where(sv[..., None], sp, sp[:, :1])                           # invalid -> the first point: no area
    # shoelace about the mean point: products of small numbers, no cancellation of raw coordinates
    sp = sp - cen[:, None]
    xs, ys = sp[..., 0], sp[..., 1]
    area = 0.5 * np.abs((xs * np.roll(ys, -1, 1) - np.roll(xs, -1, 1) * ys).sum(1))
    return np.where(nv >= 3, area, 0.0)


def inter_area(a, b, chunk=50000):
    """intersection area of convex quads a[i], b[i] ([M,4,2] each) in float64."""
    a = np.asarray(a, np.float64).reshape(-1, 4, 2)
    b = np.asarray(b, np.float64).reshape(-1, 4, 2)
    out = np.zeros(a.shape[0])
    for s in range(0, a.shape[0], chunk):
        out[s:s + chunk] = _inter_chunk(a[s:s + chunk], b[s:s + chunk])
    return out


def standup(c):
    c = np.asarray(c, np.float64)
    return np.concatenate([c.min(1), c.max(1)], 1)


def standup_overlap(sa, sb):
    """[N,4],[K,4] stand-up boxes -> [N,K] bool: both overlaps strictly positive (iou_jit(eps=0) > 0)."""
    iw = np.minimum(sa[:, None, 2], sb[None, :, 2]) - np.maximum(sa[:, None, 0], sb[None, :, 0])
    ih = np.minimum(sa[:, None, 3], sb[None, :, 3]) - np.maximum(sa[:, None, 1], sb[None, :, 1])
    return (iw > 0) & (ih > 0)


def overlaps(ca, cb, gate=None):
    """all pairs of corner sets ca [N,4,2], cb [K,4,2] -> dict of [N,K] float64 matrices: inter, area_a, area_b,
    union, and the criteria iou (-1), 0 (inter/area_a), 1 (inter/area_b), 2 (inter).  Pairs outside `gate` (default:
    stand-up boxes overlap) are 0, as in the kernels."""
    ca, cb = np.asarray(ca, np.float64), np.asarray(cb, np.float64)
    N, K = ca.shape[0], cb.shape[0]
    if gate is None:
        gate = standup_overlap(standup(ca), standup(cb))
    ii, jj = np.nonzero(gate)
    inter = np.zeros((N, K))
    inter[ii, jj] = inter_area(ca[ii], cb[jj])
    aa, ab = quad_area(ca)[:, None] + 0 * inter, quad_area(cb)[None, :] + 0 * inter
    union = aa + ab - inter
    return {"inter": inter, "area_a": aa, "area_b": ab, "union": union, -1: inter / union, 0: inter / aa,
            1: inter / ab, 2: inter}


# ------------------------------------------------------------------------------------------------ error bounds
def _perimeter(c):
    return np.linalg.norm(c - np.roll(c, -1, -2), axis=-1).sum(-1)


def _pair_diameter(ca, cb):
    """[N,4,2],[K,4,2] -> [N,K] diameter of the 8 corners of each pair (the extent of the pair's union)."""
    ext_lo = np.minimum(ca.min(1)[:, None], cb.min(1)[None])            # [N,K,2]
    ext_hi = np.maximum(ca.max(1)[:, None], cb.max(1)[None])
    return np.linalg.norm(ext_hi - ext_lo, axis=-1)                      # bounding-box diagonal >= diameter


def clip_bound(ca, cb, ov, criterion=-1):
    """|overlap_fp32 - overlap_fp64| for the corners-given paths (rbbox_iou / rbbox_intersection, the rotated NMS of
    given corners), where the kernel and the reference see the same float32 corners.

    Derivation.  The kernel subtracts a corner of the pair from all eight corners; for a far pair the subtraction is
    exact (Sterbenz), near the origin it costs u*D.  All later coordinates are bounded by the pair's diameter D.
    * A shoelace term x_i*y_j - x_j*y_i has rounding <= 2u*D*|edge| after bounding |x|,|y| by D and pairing
      |y_j - y_i| with the edge; summed over a polygon this is u*D*P (P the perimeter), plus u*|area| per addition.
    * A Sutherland-Hodgman vertex p + t*(q - p) moves along the edge pq; an error in t (from the rounded signed
      distances sp, sq <= 2u*D*|e_B|) moves it by at most err/|sp - sq| * |pq| along pq, which changes the area by at
      most 2u*D*|pq| because |sp|, |sq| <= |sp - sq| when they differ in sign.  A rounded inside/outside decision
      moves a vertex at distance <= 2u*D from the line: the same order.  The clipped polygon's perimeter is at most
      P_A + P_B, so |dI| <= c*u*D*(P_A + P_B), and |dA| <= c*u*D*P_A, |dB| <= c*u*D*P_B.
    * IoU = I/(A + B - I): |dIoU| <= (|dI| + IoU*(|dA| + |dB| + |dI|)) / U <= 2c*u*D*(P_A + P_B) / U.
    The constant C_CLIP = 8 covers c (about 4) and the factor 2.  The bound depends on box size only, not on where
    the pair lies.  Criteria 0 / 1 divide by A / B instead of U; criterion 2 is the absolute area error."""
    ca, cb = np.asarray(ca, np.float64), np.asarray(cb, np.float64)
    P = _perimeter(ca)[:, None] + _perimeter(cb)[None, :]
    e = C_CLIP * U * P * _pair_diameter(ca, cb)
    den = {-1: ov["union"], 0: ov["area_a"], 1: ov["area_b"], 2: 1.0}[criterion]
    return e / den + 2 * U * np.abs(ov[criterion])


def corner_rounding(boxes5):
    """max |fp32 corner - exact corner| of geometry.cuh bev_corners per box [N]: the products px*cos, py*sin with
    sincosf's 2 ulp (4u relative, CUDA Programming Guide, table of single-precision functions) and one rounding each,
    one rounding of their sum and one of the final + x: u*(|x| + |y|) + 7u*(w + l)/2, doubled for both axes."""
    b = np.asarray(boxes5, np.float32).astype(np.float64).reshape(-1, 5)
    return U * (np.abs(b[:, 0]) + np.abs(b[:, 1]) + 4.0 * (b[:, 2] + b[:, 3])) * 2.0


def corner_bound(ba, bb, ov, criterion=-1):
    """the box-parameter paths (b2s_nms rotated, b2s_rotate_iou_eval, KITTI): clip_bound plus the rounding of the
    float32 corners.  Moving every corner of A by <= d_A changes A, and the part of I near A's boundary, by
    <= d_A*P_A; so |dIoU| <= 3*(d_A*P_A + d_B*P_B) / U on top of the clip error.  This part grows with |x| + |y|:
    it is the ulp of the box position, inherent in fp32 corners."""
    ca, cb = bev_corners(ba), bev_corners(bb)
    da, db = corner_rounding(ba), corner_rounding(bb)
    e = 3.0 * (da[:, None] * _perimeter(ca)[:, None] + db[None, :] * _perimeter(cb)[None, :])
    den = {-1: ov["union"], 0: ov["area_a"], 1: ov["area_b"], 2: 1.0}[criterion]
    return clip_bound(ca, cb, ov, criterion) + e / den


def aligned_iou(sa, sb, eps):
    """stand-up IoU with `eps` added to widths (+1 convention of nms_gpu.py / nms_cpu.py), float64, [N,K]; also the
    inclusive path's gate (width > 0 and height > 0)."""
    sa, sb = np.asarray(sa, np.float64), np.asarray(sb, np.float64)
    w = np.minimum(sa[:, None, 2], sb[None, :, 2]) - np.maximum(sa[:, None, 0], sb[None, :, 0]) + eps
    h = np.minimum(sa[:, None, 3], sb[None, :, 3]) - np.maximum(sa[:, None, 1], sb[None, :, 1]) + eps
    gate = (w > 0) & (h > 0)
    inter = np.maximum(w, 0) * np.maximum(h, 0)
    area = lambda s: (s[:, 2] - s[:, 0] + eps) * (s[:, 3] - s[:, 1] + eps)
    union = area(sa)[:, None] + area(sb)[None, :] - inter
    return inter / union, gate, union


def aligned_bound(sa, sb, eps, delta_a=0.0, delta_b=0.0):
    """|IoU_fp32 - IoU_fp64| of the aligned NMS.  Each length right - left + eps carries <= 2u*(M + eps) from two
    roundings (M the largest coordinate magnitude of the pair) plus 2*delta when the stand-up coordinates are
    themselves uncertain by delta (the rotated boxes' fp32 corners in b2s_nms).  Then |dI| <= e*(w + h) + u*I, the
    same for each area, and |dIoU| <= (2|dI| + |dSa| + |dSb|) / U + 2u; doubled."""
    sa, sb = np.asarray(sa, np.float64), np.asarray(sb, np.float64)
    iou, _, union = aligned_iou(sa, sb, eps)
    M = np.maximum(np.abs(sa).max(1)[:, None], np.abs(sb).max(1)[None, :])
    d = np.maximum(np.broadcast_to(np.asarray(delta_a, np.float64), sa.shape[:1])[:, None],
                   np.broadcast_to(np.asarray(delta_b, np.float64), sb.shape[:1])[None, :])
    e = 2 * U * (M + abs(eps)) + 2 * d
    wa, ha = sa[:, 2] - sa[:, 0] + eps, sa[:, 3] - sa[:, 1] + eps
    wb, hb = sb[:, 2] - sb[:, 0] + eps, sb[:, 3] - sb[:, 1] + eps
    wmax = np.maximum(wa[:, None], wb[None, :])
    hmax = np.maximum(ha[:, None], hb[None, :])
    dI = e * (wmax + hmax) + U * wmax * hmax
    dSa = e * (wa + ha)[:, None] + (U * wa * ha)[:, None]
    dSb = e * (wb + hb)[None, :] + (U * wb * hb)[None, :]
    return 2.0 * ((2 * dI + dSa + dSb) / union + 2 * U)


# ------------------------------------------------------------------------------------------------ NMS certificate
def nms_certificate(order, keep, iou64, bound, thr, post_max, inclusive):
    """Is `keep` a keep list greedy NMS may produce on the ranked boxes `order` when every pair whose fp64 IoU lies
    within `bound` of `thr` may go either way?  iou64 / bound: [n, n] indexed by rank (row = earlier box); keep: box
    ids from `order`.  Suppression: IoU >= thr (inclusive) or IoU > thr.  Returns an error string, or None.
      * kept boxes come in rank order;
      * no kept box is clearly suppressed by an earlier kept box;
      * every dropped box ranked before the stop point is possibly suppressed by an earlier kept box;
      * the list stops at post_max, or when the ranked boxes run out."""
    order = np.asarray(order)
    n = len(order)
    pos = {int(b): i for i, b in enumerate(order)}
    if any(int(k) not in pos for k in keep):
        return "kept box not among the ranked candidates"
    r = np.array([pos[int(k)] for k in keep], np.int64)
    if len(r) > post_max:
        return "%d kept > post_max %d" % (len(r), post_max)
    if len(r) > 1 and not (np.diff(r) > 0).all():
        return "kept boxes out of rank order"
    iou64, bound = np.asarray(iou64, np.float64), np.asarray(bound, np.float64)
    if inclusive:
        clearly, possibly = iou64 - bound >= thr, iou64 + bound >= thr
    else:
        clearly, possibly = iou64 - bound > thr, iou64 + bound > thr
    if len(r):
        sub = clearly[np.ix_(r, r)]
        bad = np.triu(sub, 1)
        if bad.any():
            i, j = np.argwhere(bad)[0]
            return "kept rank %d is clearly suppressed by kept rank %d (IoU %.9f, bound %.2e)" % (
                r[j], r[i], iou64[r[i], r[j]], bound[r[i], r[j]])
    stop = n if len(r) < post_max else (int(r[-1]) + 1 if len(r) else 0)
    kept = np.zeros(n, bool)
    kept[r] = True
    dropped = np.nonzero(~kept[:stop])[0]
    if len(dropped):
        if not len(r):
            return "no box kept although %d are ranked" % stop
        sup = possibly[np.ix_(r, dropped)] & (r[:, None] < dropped[None, :])
        lost = dropped[~sup.any(0)]
        if len(lost):
            return "rank %d dropped although no earlier kept box can suppress it" % lost[0]
    return None


# ------------------------------------------------------------------------------------------------ top-k, decode
def topk_order(scores, anchors, count, cap, pre_max):
    """candidate slots in b2s_nms's rank order: score desc, anchor asc, over the first min(count, cap) slots."""
    n = min(int(count), int(cap))
    s = np.asarray(scores, np.float32)[:n].astype(np.float64)
    return np.lexsort((np.asarray(anchors)[:n], -s))[:pre_max]


def sigmoid64(x):
    x = np.asarray(x, np.float64)
    return 1.0 / (1.0 + np.exp(-x))


def sigmoid_bound(x):
    """|fp32 1/(1+expf(-x)) - sigmoid64(x)|: expf is 2 ulp (<= 4u relative), the add and the division one rounding
    each.  With e = exp(-x): |ds| <= s * ((4u*e + u*(1 + e)) / (1 + e) + u), i.e. about 3 ulp of s."""
    x = np.asarray(x, np.float64)
    e = np.exp(-x)
    s = 1.0 / (1.0 + e)
    with np.errstate(invalid="ignore"):
        rel = np.where(np.isinf(e), 0.0, (4 * U * e + U * (1 + e)) / (1 + e))
    return s * (rel + U) + 1e-45


def decode64(t, anchors):
    """second_box_decode in float64 on float32 inputs: [n, code] -> [n, code]."""
    t, a = np.asarray(t, np.float32).astype(np.float64), np.asarray(anchors, np.float32).astype(np.float64)
    diag = np.sqrt(a[:, 4] ** 2 + a[:, 3] ** 2)
    o = np.empty_like(t)
    o[:, 0] = t[:, 0] * diag + a[:, 0]
    o[:, 1] = t[:, 1] * diag + a[:, 1]
    o[:, 2] = t[:, 2] * a[:, 5] + a[:, 2]
    o[:, 3] = np.exp(t[:, 3]) * a[:, 3]
    o[:, 4] = np.exp(t[:, 4]) * a[:, 4]
    o[:, 5] = np.exp(t[:, 5]) * a[:, 5]
    o[:, 6:] = t[:, 6:] + a[:, 6:]
    return o


def decode_bound(t, anchors, o):
    """|fp32 decode - decode64| per element: x, y: the diagonal (two products, a sum, sqrtf: <= 3u relative) and the
    product with t (u) on |t*diag|, plus u on the sum; z: u on |t*h| + u; w, l, h: expf 2 ulp + the product = 5u
    relative; the additive components one rounding; all doubled."""
    t, a = np.asarray(t, np.float32).astype(np.float64), np.asarray(anchors, np.float32).astype(np.float64)
    diag = np.sqrt(a[:, 4] ** 2 + a[:, 3] ** 2)
    b = U * np.abs(o)
    b[:, 0] += 4 * U * np.abs(t[:, 0] * diag)
    b[:, 1] += 4 * U * np.abs(t[:, 1] * diag)
    b[:, 2] += U * np.abs(t[:, 2] * a[:, 5])
    b[:, 3:6] += 4 * U * np.abs(o[:, 3:6])
    return 2.0 * b + 1e-45


def dir_fixup_f32(r, dir_label, dir_offset, dir_limit_offset, bins):
    """voxelnet.py:598-607 as detect.cu evaluates it, float32 round-to-nearest at every step."""
    f = np.float32
    period = f(2.0 * np.pi / bins)
    val = (np.asarray(r, f) - f(dir_offset)).astype(f)
    fl = np.floor((val / period).astype(f) + f(dir_limit_offset)).astype(f)
    dir_rot = (val - (fl * period).astype(f)).astype(f)
    return ((dir_rot + f(dir_offset)).astype(f) + (period * np.asarray(dir_label).astype(f)).astype(f)).astype(f)


# ------------------------------------------------------------------------------------------------ generators
SCORE_SET = np.array([0.3, 0.41, 0.55, 0.62, 0.7, 0.85, 0.93], np.float32)


def cluster(rng, n, sigma, kind="car"):
    """n boxes (x, y, z, w, l, h, r) float32 around the origin that look like decoded neighbouring anchors: rotation
    0 or pi/2 plus N(0, sigma), centre jitter up to 0.3 * size, size jitter +-5 %, exact duplicates, pi/2-rotated
    copies with w and l swapped, neighbours one width away (a shared edge), nested boxes."""
    if kind == "car":
        w0, l0, h0 = 1.6, 3.9, 1.56
    elif kind == "ped":
        w0, l0, h0 = rng.uniform(0.05, 0.6), rng.uniform(0.5, 0.9), 1.73
    else:
        w0, l0, h0 = 0.6, 1.76, 1.73
    q = lambda v: np.round(np.asarray(v) * 64) / 64       # 2^-6 grid: sums and halves stay exact in float32
    base = np.zeros(7)
    base[3:6] = [q(w0), q(l0), h0]
    base[2] = -1.0
    base[6] = 0.0 if rng.random() < 0.6 else np.pi / 2
    out = [base.copy()]
    while len(out) < n:
        p = out[rng.integers(len(out))].copy()
        k = rng.random()
        if k < 0.45:                                        # neighbouring anchor
            b = base.copy()
            b[0:2] = rng.uniform(-0.3, 0.3, 2) * np.array([base[3], base[4]])
            b[3:6] = base[3:6] * (1 + rng.uniform(-0.05, 0.05, 3))
            b[6] = base[6] + (rng.normal(0, sigma) if sigma > 0 else 0.0)
        elif k < 0.55:                                      # exact duplicate
            b = p
        elif k < 0.65:                                      # same footprint, rotated by pi/2 with w and l swapped
            b = p.copy()
            b[3], b[4] = p[4], p[3]
            b[6] = p[6] + np.pi / 2
        elif k < 0.8:                                       # shared edge: a pair one width apart at yaw 0 (exact corners)
            b = base.copy()
            b[6] = 0.0
            b[0], b[1] = q(p[0]), q(p[1])
            out.append(b.copy())
            b[0] += base[3] * rng.choice([-1, 1])
        else:                                               # nested
            b = p.copy()
            b[3:5] = p[3:5] * 0.5
        out.append(b)
    return np.array(out[:n], np.float32)


def clusters(rng, n, centres=CENTRES, sigmas=(0.0, 1e-3, 0.05), spread=12.0, max_size=40):
    """n boxes [n,7] in clusters of 1..max_size around the given centres (a cluster is placed at centre + U(+-spread)
    on a 2^-6 grid), with a mix of cars, pedestrian slivers and cyclists."""
    out = []
    while sum(len(c) for c in out) < n:
        m = int(rng.integers(1, max_size + 1))
        kind = rng.choice(["car", "car", "ped", "cyc"])
        c = cluster(rng, m, float(rng.choice(sigmas)), kind)
        cx, cy = centres[rng.integers(len(centres))]
        off = np.round((np.array([cx, cy]) + rng.uniform(-spread, spread, 2)) * 64) / 64
        c[:, :2] += off.astype(np.float32)
        out.append(c)
    return np.concatenate(out)[:n]


def scores_for(rng, n):
    """fp32 scores from a small set (ties are common) plus one-ulp neighbours."""
    s = rng.choice(SCORE_SET, n)
    bump = rng.random(n)
    s = np.where(bump < 0.15, np.nextafter(s, np.float32(1)), s)
    s = np.where(bump > 0.85, np.nextafter(s, np.float32(0)), s)
    return s.astype(np.float32)
