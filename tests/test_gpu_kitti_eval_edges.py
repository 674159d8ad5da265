"""KITTI evaluation on the GPU at its decision edges (tests/golden/kitti_eval/edges.*, make_kitti_edges_golden.py):
difficulty limits hit exactly in float64 and float32 annotations, overlaps equal to min_overlap, DontCare and
ignored boxes, score ties and empty classes, against the unmodified reference.  Bars as test_gpu_kitti_eval.py:
result strings identical, precision and thresholds bit-equal, orientation within 1e-12 relative; and clean_data's
ignore flags equal to the reference's."""
import numpy as np
import pytest

import kitti_golden as kg
from b2second import kitti_eval as ke

pytestmark = pytest.mark.gpu


def _z(fix):
    return dict(z_axis=int(fix["z_axis"]), z_center=float(fix["z_center"]))


def _check(got, fix, tag, metric):
    assert np.array_equal(got["precision"], fix["%s_m%d_precision" % (tag, metric)], equal_nan=True)
    assert np.array_equal(got["thresholds"], fix["%s_m%d_thresholds" % (tag, metric)])
    want = fix["%s_m%d_orientation" % (tag, metric)]
    assert np.allclose(got["orientation"], want, rtol=1e-12, atol=0, equal_nan=True)


@pytest.mark.parametrize("path", kg.EDGE_FIXTURES, ids=kg.EDGE_IDS)
def test_edge_results_match_reference(product, path):
    fix, gts, dts = kg.load(path)
    classes = fix["classes"].tolist()
    assert ke.get_official_eval_result(gts, dts, classes, **_z(fix))["result"] == str(fix["official_result"])
    assert ke.get_coco_eval_result(gts, dts, classes, **_z(fix))["result"] == str(fix["coco_result"])
    for tag, mo in (("official", ke.official_min_overlaps(classes)), ("coco", ke.coco_min_overlaps(classes))):
        for metric in range(3):
            aos = bool(fix["%s_m%d_aos" % (tag, metric)])
            _check(ke.eval_class(gts, dts, classes, [0, 1, 2], metric, mo, aos, **_z(fix)), fix, tag, metric)


@pytest.mark.parametrize("path", kg.EDGE_FIXTURES, ids=kg.EDGE_IDS)
def test_edge_ignore_flags_match_reference(product, path):
    fix, gts, dts = kg.load(path)
    classes = fix["classes"].tolist()
    mo = ke.official_min_overlaps(classes)
    for metric in range(3):
        got = ke.eval_class(gts, dts, classes, [0, 1, 2], metric, mo, False, ignored=True, **_z(fix))
        for k in range(mo.shape[0]):            # every min_overlap of a (class, difficulty) shares its flags
            assert np.array_equal(got["ignored_gt"][:, :, k], fix["ignored_gt"]), (metric, k)
            assert np.array_equal(got["ignored_dt"][:, :, k], fix["ignored_dt"]), (metric, k)


def test_float32_limits_follow_the_annotation_dtype(product):
    """the same float32 scene, evaluated as given and widened to float64 first, gives each the reference's own result"""
    f32, gts, dts = kg.load(kg.EDGE_FIXTURES[kg.EDGE_IDS.index("edges.limits32")])
    f64, gts64, dts64 = kg.load(kg.EDGE_FIXTURES[kg.EDGE_IDS.index("edges.limits32as64")])
    assert gts[0]["bbox"].dtype == np.float32 and gts64[0]["bbox"].dtype == np.float64
    mo = ke.official_min_overlaps([0, 1, 2])
    for fix, g, d in ((f32, gts, dts), (f64, gts64, dts64)):
        got = ke.eval_class(g, d, [0, 1, 2], [0, 1, 2], 0, mo, True, ignored=True)
        assert np.array_equal(got["ignored_gt"][:, :, 0], fix["ignored_gt"])
        assert np.array_equal(got["ignored_dt"][:, :, 0], fix["ignored_dt"])
        _check(got, fix, "official", 0)
        assert ke.get_official_eval_result(g, d, [0, 1, 2])["result"] == str(fix["official_result"])
    assert not np.array_equal(f32["ignored_gt"], f64["ignored_gt"])
