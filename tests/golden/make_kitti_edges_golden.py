"""Generate tests/golden/kitti_eval/edges.*.npz from the UNMODIFIED reference (needs the reference tree; runs on the CPU).

    python tests/golden/make_kitti_edges_golden.py

make_kitti_eval_golden.py keeps its random scenes away from every decision the evaluation takes.  These scenes sit on
those decisions instead, one small case per frame:

  limits      ground-truth heights at exactly 40 / 25 px and one ulp above (clean_data ignores height <= MIN_HEIGHT),
              detection heights at exactly 40 / 25 px and one ulp below (height < MIN_HEIGHT), truncation at
              0.15 / 0.3 / 0.5 and one ulp above, occlusion 0..3
  limits32    the same decisions on float32 annotations whose y1 lies near the image top, where the float32 height
              y2 - y1 (what the reference computes) differs from the float64 one; limits32as64 is the same scene widened
              to float64 first
  overlap     bbox IoU of exactly 0.7 / 0.5 / 0.25 (dyadic coordinates) and one ulp above; axis-aligned BEV / 3D boxes
              whose exact IoU (fractions.Fraction) is the float32 value at each min_overlap or the nearest one above it
              that the reference's float32 clip reproduces exactly; DontCare regions covering a detection by exactly 0.7 / 0.5;
              a detection whose best match is an ignored ground truth; Van / Person_sitting, unknown and mixed-case
              names
  overlap_lidar  the overlap scene with lidar boxes (z_axis 2, z_center 0.5)
  counts      score ties within and across frames, one at a recall sample point of get_thresholds; a class without a
              valid ground truth at the easy difficulty; frames with only DontCare, frames without detections, a class
              without detections; alpha differences of +-pi and 2 pi

Every case that sits on a decision carries a nudge: the same scene with that case moved one ulp (or one occlusion step)
across the decision.  The generator evaluates each nudged scene and fails unless the reference's output changes -- an
ignore flag, a count (precision or thresholds) or a printed digit -- so every such case is an edge.  The name cases and
the AOS angles are not decisions of a compared value and have no nudge.

Each fixture holds the scene, get_official_eval_result's and get_coco_eval_result's strings, the eval_class_v3 arrays
of those calls, and clean_data's ignored_gt / ignored_dt for every (class, difficulty), concatenated over the frames.
"""
import os
import sys
from fractions import Fraction

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
OUT = os.path.join(HERE, "kitti_eval")

from b2second import loader, refcompat  # noqa: E402

refcompat.install(loader.ORACLE_DIR)
_linspace = np.linspace


def _linspace_float_num(start, stop, num=50, *a, **k):
    # do_coco_style_eval passes num as a float64 (eval.py:704), which numpy >= 1.18 rejects
    return _linspace(start, stop, int(num) if float(num).is_integer() else num, *a, **k)


np.linspace = _linspace_float_num
from second.utils import eval as E  # noqa: E402

KEYS = ("bbox", "location", "dimensions", "rotation_y", "alpha", "truncated", "occluded")
N_FRAMES = 50                      # the reference splits the frames into 50 parts: it needs at least 50
F32_07 = float(np.float32(0.7))


def up(x, ft):
    return ft(np.nextafter(ft(x), ft(np.inf)))


def down(x, ft):
    return ft(np.nextafter(ft(x), ft(-np.inf)))


# ------------------------------------------------------------------------------------------------ scene building
class Box:
    """one annotation: bbox, a 3D box given by its BEV centre / extents and height, and the difficulty fields."""

    def __init__(self, name, bbox, bev=(0.0, 0.0, 4.0, 4.0), height=2.0, alpha=0.0, trunc=0.0, occ=0, score=None):
        self.name, self.bbox, self.bev, self.height = name, list(bbox), list(bev), height
        self.alpha, self.trunc, self.occ, self.score = alpha, trunc, occ, score

    def fields(self, lidar):
        x, z, l, w = self.bev
        if lidar:
            loc, dims = [x, z, 1.0], [l, w, self.height]
        else:
            loc, dims = [x, 1.5, z], [l, self.height, w]
        return dict(bbox=self.bbox, location=loc, dimensions=dims, rotation_y=0.0, alpha=self.alpha,
                    truncated=self.trunc, occluded=self.occ)


class Case:
    """frames(nudged) -> [(gt boxes, dt boxes)]; nudge False when the case has no decision to cross."""

    def __init__(self, tag, frames, nudge=True):
        self.tag, self.frames, self.nudge = tag, frames, nudge


def stack(boxes, lidar, ft, with_score):
    a = {"name": np.array([b.name for b in boxes], dtype="<U16")}
    width = {"bbox": 4, "location": 3, "dimensions": 3}
    for k in KEYS:
        dt = np.int64 if k == "occluded" else ft
        vals = [b.fields(lidar)[k] for b in boxes]
        a[k] = np.array(vals, dtype=dt).reshape((len(boxes), width[k]) if k in width else (len(boxes),))
    if with_score:
        a["score"] = np.array([b.score for b in boxes], dtype=np.float32)
    return a


def build(cases, nudged, lidar, ft):
    """the scene's frames as anno lists; cases[nudged] (an index, or None) is the nudged one."""
    frames = []
    for i, c in enumerate(cases):
        frames += c.frames(i == nudged)
    frames += [([], [])] * max(0, N_FRAMES - len(frames))
    score = iter(np.float32(1.0 - k / 1024.0) for k in range(1, 1024))
    gts, dts = [], []
    for g, d in frames:
        for b in d:
            if b.score is None:
                b.score = next(score)
        gts.append(stack(g, lidar, ft, False))
        dts.append(stack(d, lidar, ft, True))
    return gts, dts


def pair(name, bbox, ft, **gt_kw):
    """a ground truth and the detection of the same box"""
    return [Box(name, bbox, **gt_kw)], [Box(name, list(bbox))]


# ------------------------------------------------------------------------------------------------ limits
NAMES = ["Car", "Pedestrian", "Cyclist"]


def f32_top_y1(rng, h, wider):
    """a float32 y1 in [0, 8) with y2 = fl32(y1 + h) whose float32 height y2 - y1 is exactly h while the exact
    (float64) height is above h (wider) or below it"""
    while True:
        y1 = np.float32(rng.uniform(0, 8))
        y2 = np.float32(y1 + np.float32(h))
        if np.float32(y2 - y1) == h and ((float(y2) - float(y1) > h) if wider else (float(y2) - float(y1) < h)):
            return float(y1)


def limits_cases(ft):
    rng = np.random.default_rng(40)
    cases = []
    for k, h in enumerate((40.0, 25.0)):
        name = NAMES[k]
        # ground truth: exactly h is ignored (height <= h), one ulp above is not
        for above in (False, True):
            y1 = f32_top_y1(rng, h, wider=True) if ft is np.float32 else 100.0 + 8 * k
            y2 = ft(ft(y1) + ft(h))
            y2 = up(y2, ft) if above else y2

            def frames(nudged, y1=y1, y2=y2, above=above, name=name):
                gy2 = (down(y2, ft) if above else up(y2, ft)) if nudged else y2
                return [([Box(name, [10.0, y1, 74.0, gy2])], [Box(name, [10.0, y1, 74.0, y2])])]
            cases.append(Case("gt_height_%g%s" % (h, "+" if above else ""), frames))
        # detection: exactly h is kept (height < h is ignored), one ulp below is not
        for below in (False, True):
            y1 = f32_top_y1(rng, h, wider=False) if ft is np.float32 else 100.0 + 8 * k
            y2 = ft(ft(y1) + ft(h))
            y2 = down(y2, ft) if below else y2

            def frames(nudged, y1=y1, y2=y2, below=below, name=name):
                dy2 = (up(y2, ft) if below else down(y2, ft)) if nudged else y2
                return [([Box(name, [10.0, y1, 74.0, float(y1) + 44.0])], [Box(name, [10.0, y1, 74.0, dy2])])]
            cases.append(Case("dt_height_%g%s" % (h, "-" if below else ""), frames))
    for k, t in enumerate((0.15, 0.3, 0.5)):
        for above in (False, True):
            tv = up(t, ft) if above else ft(t)

            def frames(nudged, tv=tv, above=above, name=NAMES[k]):
                tt = (down(tv, ft) if above else up(tv, ft)) if nudged else tv
                return [pair(name, [10.0, 100.0, 74.0, 160.0], ft, trunc=tt)]
            cases.append(Case("truncation_%g%s" % (t, "+" if above else ""), frames))
    for occ in range(4):
        def frames(nudged, occ=occ):
            o = (occ + 1 if occ < 3 else occ - 1) if nudged else occ
            return [pair(NAMES[occ % 3], [10.0, 100.0, 74.0, 160.0], ft, occ=o)]
        cases.append(Case("occlusion_%d" % occ, frames))
    return cases


# ------------------------------------------------------------------------------------------------ overlap
def exact_iou(gl, gw, dl, dw):
    """IoU of two axis-aligned boxes sharing a centre, the detection inside the ground truth"""
    g, d = (Fraction(float(gl)) * Fraction(float(gw)), Fraction(float(dl)) * Fraction(float(dw)))
    return d / (g + d - d)


def rotated_exact(gt, dt, lidar):
    """whether the reference's float32 BEV and 3D overlaps of these two boxes both equal the exact IoU"""
    z_axis, z_center = (2, 0.5) if lidar else (1, 1.0)
    g, d = gt.fields(lidar), dt.fields(lidar)
    bev_ax = [0, 1] if lidar else [0, 2]
    bev = lambda b: np.array([[*np.take(b["location"], bev_ax), *np.take(b["dimensions"], bev_ax), 0.0]])
    box = lambda b: np.array([[*b["location"], *b["dimensions"], 0.0]])
    want = exact_iou(gt.bev[2], gt.bev[3], dt.bev[2], dt.bev[3])
    got_bev = E.bev_box_overlap(bev(g), bev(d)).astype(np.float64)[0, 0]
    got_3d = E.box3d_overlap(box(g), box(d), z_axis=z_axis, z_center=z_center).astype(np.float64)[0, 0]
    return Fraction(float(got_bev)) == want and Fraction(float(got_3d)) == want


# a 4 x 4 ground truth with a corner at the origin and a 4 x 4v detection inside it on the same corner: every corner
# coordinate is exact in float32, whether taken as it is or relative to a box's first corner
GT_BEV = (2.0, 2.0, 4.0, 4.0)


def dt_bev(v):
    return (2.0, 2.0 * float(v), 4.0, 4.0 * float(v))


def rotated_iou_values(iou, name, lidar):
    """(float32 IoU at the min_overlap, the nearest float32 IoU above it) that the reference's clip reproduces
    exactly for the GT_BEV / dt_bev(v) pair"""
    exact = lambda v: rotated_exact(Box(name, [0, 0, 1, 1], bev=GT_BEV), Box(name, [0, 0, 1, 1], bev=dt_bev(v)), lidar)
    at = np.float32(iou)
    assert exact(at), (name, iou)
    above = up(at, np.float32)
    while not exact(above):
        above = up(above, np.float32)
    return at, above


def overlap_cases(lidar):
    ft = np.float64
    cases = []
    # bbox: ground truth 64 x 200, detection 64 x h inside it: IoU = h / 200 exactly as a rational
    for name, ious in (("Car", (0.7, 0.5)), ("Pedestrian", (0.5, 0.25))):
        for iou in ious:
            for above in (False, True):
                y2 = 100.0 + 200.0 * iou
                y2 = up(y2, ft) if above else y2
                assert Fraction(y2 - 100.0) / 200 == Fraction(iou).limit_denominator(100) or above

                def frames(nudged, y2=y2, above=above, name=name):
                    dy2 = (down(y2, ft) if above else up(y2, ft)) if nudged else y2
                    return [([Box(name, [10.0, 100.0, 74.0, 300.0])], [Box(name, [10.0, 100.0, 74.0, dy2])])]
                cases.append(Case("bbox_%s_%g%s" % (name, iou, "+" if above else ""), frames))
    # BEV / 3D: ground truth 4 x 4, detection 4 x 4v inside it on one corner, same height: IoU = v in both metrics
    for name, ious in (("Car", (F32_07, 0.5)), ("Pedestrian", (0.5, 0.25))):
        for iou in ious:
            at, above_v = rotated_iou_values(iou, name, lidar)
            # one ulp above 0.25 the float32 clip's last bit differs between implementations (0.25 against
            # 0.2500000298), which puts that case on the wrong side of the threshold: it is only the nudge target
            for above in (False,) if iou == 0.25 else (False, True):
                # nudged: the other one of the two (at most a few ulps apart)
                v = above_v if above else at

                def frames(nudged, v=v, other=(at if above else above_v), name=name):
                    dv = other if nudged else v
                    bb = [10.0, 100.0, 74.0, 160.0]
                    return [([Box(name, bb, bev=GT_BEV)], [Box(name, list(bb), bev=dt_bev(dv))])]
                cases.append(Case("rotated_%s_%.8g%s" % (name, iou, "+" if above else ""), frames))
    # DontCare: a second detection whose area a DontCare box covers by exactly min_overlap (criterion 0) stays a false
    # positive; one ulp more coverage takes it off the false positives (bbox metric)
    for name, cover in (("Car", 0.7), ("Pedestrian", 0.5)):
        def frames(nudged, name=name, cover=cover):
            y2 = 100.0 + 100.0 * cover
            y2 = up(y2, ft) if nudged else y2
            g = [Box(name, [10.0, 100.0, 74.0, 160.0]), Box("DontCare", [200.0, 100.0, 264.0, y2], occ=-1, trunc=-1)]
            d = [Box(name, [10.0, 100.0, 74.0, 160.0]), Box(name, [200.0, 100.0, 264.0, 200.0], bev=(50.0, 0.0, 4, 4))]
            return [(g, d)]
        cases.append(Case("dontcare_%s_%g" % (name, cover), frames))

    # the detection's best match is an ignored ground truth (height exactly 40: ignored when easy) listed first; the
    # valid one behind it overlaps at 0.8 and goes unmatched.  Nudged: the first is valid and takes the detection.
    def frames(nudged):
        y2 = up(140.0, ft) if nudged else 140.0
        g = [Box("Car", [10.0, 100.0, 74.0, y2]), Box("Car", [10.0, 100.0, 74.0, 150.0], bev=(0.0, 0.0, 4.0, 4.5))]
        return [(g, [Box("Car", [10.0, 100.0, 74.0, 140.0])])]
    cases.append(Case("ignored_gt_first", frames))

    # Van / Person_sitting matched by a Car / Pedestrian detection count as neither hit nor miss; an unknown name
    # in their place makes the detection a false positive
    for gname, dname in (("Van", "Car"), ("Person_sitting", "Pedestrian")):
        def frames(nudged, gname=gname, dname=dname):
            return [([Box("Truck" if nudged else gname, [10.0, 100.0, 74.0, 160.0])],
                     [Box(dname, [10.0, 100.0, 74.0, 160.0])])]
        cases.append(Case("alternate_%s" % gname, frames))

    # names: lower-cased for the class, but only exactly "DontCare" is a don't-care region
    def frames(nudged):
        g = [Box("car", [10.0, 100.0, 74.0, 160.0]), Box("CAR", [100.0, 100.0, 164.0, 170.0], bev=(20.0, 0.0, 4, 4)),
             Box("dontcare", [200.0, 100.0, 264.0, 200.0]), Box("Truck", [300.0, 100.0, 364.0, 180.0]),
             Box("pedestrian", [400.0, 100.0, 420.0, 160.0], bev=(40.0, 0.0, 1.0, 1.0))]
        d = [Box("cAr", [10.0, 100.0, 74.0, 160.0]), Box("Car", [100.0, 100.0, 164.0, 170.0], bev=(20.0, 0.0, 4, 4)),
             Box("Car", [200.0, 100.0, 264.0, 200.0], bev=(60.0, 0.0, 4, 4)), Box("Truck", [300.0, 100.0, 364.0, 180.0]),
             Box("Misc", [500.0, 100.0, 564.0, 180.0]), Box("PEDESTRIAN", [400.0, 100.0, 420.0, 160.0],
                                                             bev=(40.0, 0.0, 1.0, 1.0))]
        return [(g, d)]
    cases.append(Case("names", frames, nudge=False))
    return cases


# ------------------------------------------------------------------------------------------------ counts
def counts_cases():
    cases = []
    bb = lambda k: [10.0 + 100 * k, 100.0, 74.0 + 100 * k, 160.0]
    tied = np.float32(0.75)

    # across frames: four true positives share one score
    def frames(nudged):
        out = [pair("Car", bb(0), np.float64) for _ in range(4)]
        for k, (_, d) in enumerate(out):
            d[0].score = down(tied, np.float32) if (nudged and k == 3) else tied
        return out
    cases.append(Case("tie_across_frames", frames))

    # within a frame: two true positives and a false positive share one score; with 40 valid cars every true positive
    # score is a threshold, so the false positive counts at that threshold
    def frames(nudged):
        g = [Box("Car", bb(0)), Box("Car", bb(1), bev=(20.0, 0.0, 4, 4))]
        d = [Box("Car", bb(0), score=np.float32(0.5)), Box("Car", bb(1), bev=(20.0, 0.0, 4, 4), score=np.float32(0.5)),
             Box("Car", bb(3), bev=(60.0, 0.0, 4, 4), score=down(0.5, np.float32) if nudged else np.float32(0.5))]
        return [(g, d)]
    cases.append(Case("tie_within_frame_and_fp", frames))

    # Cyclists all between 25 and 40 px: no valid one when easy; nudged, one is 40 px plus one ulp
    def frames(nudged):
        out = []
        for k in range(3):
            y2 = up(140.0, np.float64) if (nudged and k == 0) else 130.0 + k
            out.append(pair("Cyclist", [10.0, 100.0, 40.0, y2], np.float64))
        return out
    cases.append(Case("no_valid_easy_cyclist", frames))

    # Pedestrians without any Pedestrian detection
    def frames(nudged):
        return [([Box("Pedestrian", [10.0, 100.0, 30.0, 170.0], bev=(0.0, 0.0, 1.0, 1.0))], [])]
    cases.append(Case("pedestrian_without_detections", frames, nudge=False))
    cases.append(Case("only_dontcare", lambda nudged: [([Box("DontCare", [0.0, 0.0, 50.0, 50.0])], [])], nudge=False))
    cases.append(Case("no_detections", lambda nudged: [([Box("Car", bb(0))], [])], nudge=False))

    # AOS: alpha differences of pi, -pi and 2 pi
    def frames(nudged):
        out = []
        for ga, da in ((np.pi / 2, -np.pi / 2), (-np.pi / 2, np.pi / 2), (np.pi, -np.pi), (-3.0, 3.0)):
            g, d = pair("Car", bb(0), np.float64, alpha=ga)
            d[0].alpha = da
            out.append((g, d))
        return out
    cases.append(Case("aos_wrap", frames, nudge=False))
    # 40 valid cars, each detected, so get_thresholds samples every true positive
    for k in range(34):
        cases.append(Case("car_%d" % k, lambda nudged: [pair("Car", bb(0), np.float64)], nudge=False))
    return cases


# ------------------------------------------------------------------------------------------------ evaluation
class _Recorder:
    """wraps the reference's eval_class_v3 to keep what it returned (code unchanged)."""

    def __init__(self):
        self.evals, self._ev = [], E.eval_class_v3

        def ev(gt, dt, classes, diffs, metric, min_overlaps, compute_aos=False, **kw):
            r = self._ev(gt, dt, classes, diffs, metric, min_overlaps, compute_aos, **kw)
            self.evals.append((metric, compute_aos, r))
            return r
        E.eval_class_v3 = ev

    def close(self):
        E.eval_class_v3 = self._ev


def evaluate(gts, dts, classes, lidar):
    z = dict(z_axis=2, z_center=0.5) if lidar else dict(z_axis=1, z_center=1.0)
    rec = _Recorder()
    try:
        off = E.get_official_eval_result(gts, dts, classes, **z)
        n_off = len(rec.evals)
        coco = E.get_coco_eval_result(gts, dts, classes, **z)
    finally:
        rec.close()
    out = {"classes": np.array(classes, dtype=np.int64), "z_axis": np.int64(z["z_axis"]),
           "z_center": np.float64(z["z_center"]), "official_result": np.array(off["result"]),
           "coco_result": np.array(coco["result"])}
    for i, (metric, aos, r) in enumerate(rec.evals):
        tag = "official" if i < n_off else "coco"
        for k in ("precision", "orientation", "thresholds"):
            out["%s_m%d_%s" % (tag, metric, k)] = r[k]
        out["%s_m%d_aos" % (tag, metric)] = np.bool_(aos)
    ig = np.zeros((len(classes), 3, sum(len(a["name"]) for a in gts)), np.int8)
    idt = np.zeros((len(classes), 3, sum(len(a["name"]) for a in dts)), np.int8)
    for m, c in enumerate(classes):
        for d in range(3):
            r = E._prepare_data(gts, dts, c, d)
            ig[m, d] = np.concatenate(r[2]) if ig.shape[2] else ig[m, d]
            idt[m, d] = np.concatenate(r[3]) if idt.shape[2] else idt[m, d]
    out["ignored_gt"], out["ignored_dt"] = ig, idt
    return out


def signature(out):
    return {k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in out.items()}


def flatten(prefix, annos):
    out = {prefix + "offsets": np.concatenate([[0], np.cumsum([len(a["name"]) for a in annos])]).astype(np.int64)}
    for k in ("name",) + KEYS + (("score",) if "score" in annos[0] else ()):
        out[prefix + k] = np.concatenate([a[k] for a in annos])
    return out


def run_scene(name, cases, classes, lidar=False, ft=np.float64, widen=None):
    """evaluate the scene, check every case's nudge, write edges.<name>.npz (and edges.<widen>.npz: the same scene
    widened to float64)."""
    gts, dts = build(cases, None, lidar, ft)
    base = evaluate(gts, dts, classes, lidar)
    sig = signature(base)
    for i, c in enumerate(cases):
        if not c.nudge:
            continue
        ng, nd = build(cases, i, lidar, ft)
        moved = signature(evaluate(ng, nd, classes, lidar))
        changed = sorted(k for k in sig if sig[k] != moved[k])
        assert changed, "%s/%s: the nudged scene evaluates the same; the case is not an edge" % (name, c.tag)
        print("  %-28s nudge changes %s" % (c.tag, ", ".join(changed[:4]) + (" ..." if len(changed) > 4 else "")))
    write(name, base, gts, dts)
    if widen:
        wide = lambda annos: [{k: (v.astype(np.float64) if v.dtype == ft else v) for k, v in a.items()} for a in annos]
        gts, dts = wide(gts), wide(dts)
        write(widen, evaluate(gts, dts, classes, lidar), gts, dts)


def write(name, out, gts, dts):
    out = dict(out)
    out.update(flatten("gt_", gts))
    out.update(flatten("dt_", dts))
    path = os.path.join(OUT, "edges.%s.npz" % name)
    np.savez_compressed(path, **out)
    print("edges.%s written (%d bytes)" % (name, os.path.getsize(path)))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    which = sys.argv[1:] or ["limits", "limits32", "overlap", "overlap_lidar", "counts"]
    if "limits" in which:
        run_scene("limits", limits_cases(np.float64), [0, 1, 2])
    if "limits32" in which:
        run_scene("limits32", limits_cases(np.float32), [0, 1, 2], ft=np.float32, widen="limits32as64")
    if "overlap" in which:
        run_scene("overlap", overlap_cases(False), [0, 1])
    if "overlap_lidar" in which:
        run_scene("overlap_lidar", overlap_cases(True), [0, 1], lidar=True)
    if "counts" in which:
        run_scene("counts", counts_cases(), [0, 1, 2])
