"""GPU parity of the numpy-facing spconv.utils NMS functions: keep lists identical to the oracle's; rotated: when
a pair lies within the fp32 clip's error bound of the threshold, the keep list must pass the fp64 certificate of
tests/detect_ref.py instead."""
import numpy as np
import pytest

import detect_ref as R
from b2second import box_ops

pytestmark = pytest.mark.gpu


def random_rboxes(rng, n, spread):
    xy = rng.uniform(0, spread, (n, 2))
    wl = rng.uniform(1.0, 5.0, (n, 2))
    r = rng.uniform(-np.pi, np.pi, (n, 1))
    return np.concatenate([xy, wl, r], 1).astype(np.float32)


@pytest.mark.parametrize("n,spread,thresh", [(100, 20, 0.01), (1000, 70, 0.01), (1000, 40, 0.1), (300, 15, 0.5),
                                             (1, 5, 0.1), (65, 10, 0.3)])
def test_rotate_nms_matches_oracle(product, oracle, n, spread, thresh):
    rng = np.random.default_rng(n + int(thresh * 1000))
    rb = random_rboxes(rng, n, spread)
    scores = rng.uniform(0, 1, n).astype(np.float32)
    order = np.argsort(-scores, kind="stable").astype(np.int32)
    corners = box_ops.corners_2d_np(rb[:, :2], rb[:, 2:4], rb[:, 4])
    siou = box_ops.standup_iou_np(box_ops.standup_np(corners), 0.0)
    ref = oracle.utils.rotate_non_max_suppression_cpu(corners, order, siou, thresh)
    got = product.utils.rotate_non_max_suppression_cpu(corners, order, siou, thresh)
    c = corners[order].astype(np.float64)
    ov = R.overlaps(c, c, gate=siou[np.ix_(order, order)] > 0)
    iou, bound = np.triu(ov[-1], 1), R.clip_bound(c, c, ov)
    assert R.nms_certificate(order, got, iou, bound, thresh, n, True) is None
    near = int(np.triu(np.abs(iou - thresh) <= bound, 1)[iou > 0].sum())
    if near == 0:                     # no decision the fp32 clip may flip: the same list as the oracle's
        assert got == ref


@pytest.mark.parametrize("n,thresh", [(1000, 0.5), (200, 0.1), (64, 0.7), (1, 0.5)])
def test_aligned_nms_matches_oracle(product, oracle, n, thresh):
    rng = np.random.default_rng(n)
    xy = rng.uniform(0, 40, (n, 2))
    wh = rng.uniform(0.5, 6, (n, 2))
    scores = np.sort(rng.uniform(0, 1, n))[::-1]
    dets = np.concatenate([xy, xy + wh, scores[:, None]], 1).astype(np.float32)
    ka, kb = np.zeros(n, np.int32), np.zeros(n, np.int32)
    na = product.utils.non_max_suppression(dets, ka, thresh, 0)
    nb = oracle.utils.non_max_suppression(dets, kb, thresh, 0)
    assert na == nb and ka[:na].tolist() == kb[:nb].tolist()
    order = rng.permutation(n).astype(np.int32)
    assert product.utils.non_max_suppression_cpu(dets, order, thresh, 0.0) == \
        oracle.utils.non_max_suppression_cpu(dets, order, thresh, 0.0)
    assert product.utils.non_max_suppression_cpu(dets, order, thresh, 1.0) == \
        oracle.utils.non_max_suppression_cpu(dets, order, thresh, 1.0)


def test_empty(product):
    assert product.utils.rotate_non_max_suppression_cpu(np.zeros((0, 4, 2), np.float32), np.zeros(0, np.int32),
                                                        np.zeros((0, 0), np.float32), 0.1) == []
    assert product.utils.non_max_suppression(np.zeros((0, 5), np.float32), np.zeros(0, np.int32), 0.5, 0) == 0
