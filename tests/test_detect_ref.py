"""The fp64 detection reference (tests/detect_ref.py) pinned on the CPU: known answers, agreement with the
independent corner/edge restatement of test_oracle_nms, certificate mutations, and the size of the bound."""
import numpy as np
import pytest

import detect_ref as R
from test_oracle_nms import independent_inter_area


def _quad(x, y, w, l, r):
    return R.bev_corners(np.array([[x, y, w, l, r]], np.float32))[0]


def test_known_answers():
    a = _quad(3.0, -2.0, 1.5, 4.0, 0.3)
    assert np.isclose(R.inter_area(a[None], a[None])[0], 6.0, rtol=1e-12)              # identical
    b = _quad(10.0, 5.0, 2.0, 4.0, 0.0)
    c = _quad(12.0, 5.0, 2.0, 4.0, 0.0)                                                 # shares the edge x = 11
    assert R.inter_area(b[None], c[None])[0] == 0.0
    assert R.inter_area(b[None], b[None])[0] == 8.0
    d = _quad(10.25, 5.5, 1.0, 2.0, 0.0)                                                # nested in b
    assert R.inter_area(b[None], d[None])[0] == 2.0 and R.inter_area(d[None], b[None])[0] == 2.0
    s = _quad(0.0, 0.0, 2.0, 2.0, 0.0)
    t = np.array([[0.0, -np.sqrt(2)], [-np.sqrt(2), 0.0], [0.0, np.sqrt(2)], [np.sqrt(2), 0.0]])   # s turned 45 deg
    assert np.isclose(R.inter_area(s[None], t[None])[0], 8 * (np.sqrt(2) - 1), rtol=1e-14)          # regular octagon
    ov = R.overlaps(np.stack([s, b]), np.stack([s, c]))
    assert ov[-1][0, 0] == 1.0 and ov[-1][1, 1] == 0.0 and ov[2][0, 1] == 0.0
    # the criteria
    e = _quad(0.5, 0.0, 2.0, 2.0, 0.0)
    ov = R.overlaps(s[None], e[None])
    assert np.isclose(ov[2][0, 0], 3.0) and np.isclose(ov[-1][0, 0], 3.0 / 5.0)
    assert np.isclose(ov[0][0, 0], 0.75) and np.isclose(ov[1][0, 0], 0.75)


def test_agrees_with_independent_restatement():
    rng = np.random.default_rng(3)
    boxes = np.concatenate([R.clusters(rng, 120, centres=[(0.0, 0.0), (70.4, 40.0)], spread=3.0),
                            np.concatenate([rng.uniform(0, 8, (60, 2)), rng.uniform(-1, 0, (60, 1)),
                                            rng.uniform(0.5, 5, (60, 3)), rng.uniform(-np.pi, np.pi, (60, 1))], 1)])
    c = R.bev_corners(boxes[:, [0, 1, 3, 4, 6]].astype(np.float32)).astype(np.float32)
    ov = R.overlaps(c, c)
    ii, jj = np.nonzero(ov["inter"] > 0)
    pick = rng.choice(len(ii), 400, replace=False)
    worst = max(abs(ov["inter"][i, j] - independent_inter_area(c[i], c[j])) for i, j in zip(ii[pick], jj[pick]))
    assert worst < 1e-9
    assert len(ii) > 1000


def _greedy(iou, thr, post_max, inclusive):
    n = iou.shape[0]
    sup, keep = np.zeros(n, bool), []
    for i in range(n):
        if sup[i]:
            continue
        keep.append(i)
        if len(keep) == post_max:
            break
        sup |= (iou[i] >= thr) if inclusive else (iou[i] > thr)
    return keep


@pytest.mark.parametrize("thr,inclusive", [(0.1, True), (0.5, True), (0.5, False)])
def test_certificate_accepts_greedy_and_rejects_mutations(thr, inclusive):
    rng = np.random.default_rng(int(thr * 10) + inclusive)
    boxes = R.clusters(rng, 300, centres=[(0.0, 0.0)], spread=15.0)
    c = R.bev_corners(boxes[:, [0, 1, 3, 4, 6]])
    order = rng.permutation(300)                                       # box ids in rank order
    ov = R.overlaps(c[order], c[order])
    iou = np.triu(ov[-1], 1)
    bound = R.clip_bound(c[order], c[order], ov)
    keep_r = _greedy(iou, thr, 10 ** 6, inclusive)
    keep = order[keep_r]
    cert = lambda k, pm=10 ** 6: R.nms_certificate(order, k, iou, bound, thr, pm, inclusive)
    assert cert(keep) is None
    assert 10 < len(keep) < 250
    assert cert(keep[:7], 7) is None                                   # stops at post_max
    clearly = (iou - bound >= thr) if inclusive else (iou - bound > thr)
    possibly = (iou + bound >= thr) if inclusive else (iou + bound > thr)
    kr = np.array(keep_r)
    # drop a kept box that no earlier kept box could suppress
    free = [q for q in range(1, len(kr)) if not possibly[kr[:q], kr[q]].any()]
    assert free
    assert cert(np.delete(keep, free[0])) is not None
    # swap two kept boxes
    k2 = keep.copy()
    k2[[3, 4]] = k2[[4, 3]]
    assert "order" in cert(k2)
    # add a box that an earlier kept box clearly suppresses, at its rank position
    dropped = [d for d in range(len(order)) if d not in set(keep_r) and clearly[kr[kr < d], d].any()]
    assert dropped
    d = dropped[0]
    k3 = order[sorted(keep_r + [d])]
    assert "clearly suppressed" in cert(k3)
    # stop one box early
    assert cert(keep[:-1], len(keep)) is not None
    if not possibly[kr[:-1], kr[-1]].any():
        assert cert(keep[:-1]) is not None


def test_certificate_tolerates_pairs_at_the_threshold():
    # two boxes whose IoU is the threshold to within the bound: keeping or dropping the second are both valid
    iou = np.array([[0.0, 0.5], [0.0, 0.0]])
    bound = np.full((2, 2), 1e-6)
    for keep in ([0], [0, 1]):
        assert R.nms_certificate([0, 1], keep, iou, bound, 0.5 + 5e-7, 100, True) is None
    assert R.nms_certificate([0, 1], [0], iou, bound, 0.51, 100, True) is not None


def test_bound_is_small_on_car_clusters_at_every_position():
    rng = np.random.default_rng(7)
    worst = 0.0
    for sigma in (0.0, 1e-3, 0.05):
        base = R.cluster(rng, 40, sigma, "car")
        for cx, cy in R.CENTRES:
            b = base.copy()
            b[:, :2] += np.array([cx, cy], np.float32)
            c = R.bev_corners(b[:, [0, 1, 3, 4, 6]]).astype(np.float32)
            ov = R.overlaps(c, c)
            bd = R.clip_bound(c, c, ov)
            worst = max(worst, float(bd[ov["inter"] > 0].max()))
    assert 1e-7 < worst < 1e-5


def test_direction_fixup_and_topk():
    # val/period + offset an exact integer: floor must not move it
    period = np.float32(np.pi)
    r = np.array([np.float32(0.78) + np.float32(0.5) * period, 0.1, -3.0], np.float32)
    val = r - np.float32(0.78)
    x = (val / period).astype(np.float32) + np.float32(0.5)
    assert x[0] == np.floor(x[0])
    got = R.dir_fixup_f32(r, np.array([1, 0, 1]), 0.78, 0.5, 2)
    assert got.dtype == np.float32 and abs(float(got[1]) - 0.1) < 1e-6
    s = np.array([0.5, 0.7, 0.7, 0.2, 0.9], np.float32)
    a = np.array([4, 9, 2, 0, 1])
    assert R.topk_order(s, a, 5, 5, 3).tolist() == [4, 2, 1]
    assert R.topk_order(s, a, 9, 4, 10).tolist() == [2, 1, 0, 3]       # count above the cap: the first cap slots
