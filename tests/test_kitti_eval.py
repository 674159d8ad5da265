"""Host side of the KITTI evaluation (b2second.kitti_eval): annotation packing, name encoding, the task table and the
result formatter, which must print the reference's strings from the reference's own precision arrays
(tests/golden/kitti_eval, make_kitti_eval_golden.py).  No GPU needed."""
import numpy as np
import pytest

import kitti_golden as kg
from b2second import kitti_eval as ke


def test_fixtures_present_and_small():
    import os
    assert len(kg.EVAL_FIXTURES) >= 3 and os.path.exists(kg.CONVERT_FIXTURE)
    assert sum(os.path.getsize(p) for p in kg.EVAL_FIXTURES + [kg.CONVERT_FIXTURE]) < 1 << 20


def test_edge_fixtures_present_and_small():
    import os
    names = {os.path.basename(p) for p in kg.EDGE_FIXTURES}
    assert {"edges.limits.npz", "edges.limits32.npz", "edges.limits32as64.npz", "edges.overlap.npz",
            "edges.overlap_lidar.npz", "edges.counts.npz"} <= names
    assert sum(os.path.getsize(p) for p in kg.EDGE_FIXTURES) < 300 << 10
    for p in kg.EDGE_FIXTURES:
        fix, gts, dts = kg.load(p)
        assert len(gts) == len(dts) >= 50
        assert fix["ignored_gt"].shape == (len(fix["classes"]), 3, sum(len(a["name"]) for a in gts))
        assert fix["ignored_dt"].shape == (len(fix["classes"]), 3, sum(len(a["name"]) for a in dts))


def test_float32_scene_keeps_its_dtype_and_differs_from_float64():
    """the float32 limits scene reaches the evaluation as float32, and widening it to float64 first changes what
    clean_data ignores -- so the two fixtures pin the annotation-dtype arithmetic"""
    f32, gts, dts = kg.load(kg.EDGE_FIXTURES[kg.EDGE_IDS.index("edges.limits32")])
    f64, gts64, _ = kg.load(kg.EDGE_FIXTURES[kg.EDGE_IDS.index("edges.limits32as64")])
    assert gts[0]["bbox"].dtype == np.float32 and dts[0]["truncated"].dtype == np.float32
    assert gts64[0]["bbox"].dtype == np.float64
    assert not np.array_equal(f32["ignored_gt"], f64["ignored_gt"])
    assert not np.array_equal(f32["ignored_dt"], f64["ignored_dt"])


@pytest.mark.parametrize("path", kg.EDGE_FIXTURES, ids=kg.EDGE_IDS)
def test_difficulty_limits_match_clean_data(path):
    """pack_limits' bits against the reference's ignore flags: a detection is ignored (1) exactly when its bit is
    set, whatever its class; a ground truth of the evaluated class is ignored exactly when its bit is set"""
    fix, gts, dts = kg.load(path)
    gl, dl = ke.pack_limits(gts, is_gt=True), ke.pack_limits(dts, is_gt=False)
    gnames = np.char.lower(np.concatenate([a["name"] for a in gts]).astype(str))
    for m, c in enumerate(fix["classes"].tolist()):
        own = gnames == ke.CLASS_NAMES[c]
        for d in range(3):
            assert np.array_equal(fix["ignored_dt"][m, d] == 1, (dl >> d) & 1 == 1), (c, d)
            assert np.array_equal(fix["ignored_gt"][m, d][own] == 1, (gl[own] >> d) & 1 == 1), (c, d)


@pytest.mark.parametrize("path", kg.EDGE_FIXTURES, ids=kg.EDGE_IDS)
def test_formatter_reproduces_the_edge_strings(path):
    fix, _, dts = kg.load(path)
    classes = fix["classes"].tolist()
    aos = ke.compute_aos_of(dts)
    off = ke.format_official(classes, ke.official_min_overlaps(classes),
                             *[fix["official_m%d_precision" % m] for m in range(3)],
                             fix["official_m0_orientation"] if aos else None)
    assert off["result"] == str(fix["official_result"])
    coco = ke.format_coco(classes, *[fix["coco_m%d_precision" % m] for m in range(3)],
                          fix["coco_m0_orientation"] if aos else None)
    assert coco["result"] == str(fix["coco_result"])


def test_name_encoding():
    names = ["Car", "car", "CAR", "Van", "Pedestrian", "Person_sitting", "Cyclist", "DontCare", "dontcare", "Truck",
             "Tractor", "Misc"]
    got = ke.encode_names(names).tolist()
    assert got == [0, 0, 0, 3, 1, 4, 2, ke.DONTCARE, -1, -1, 6, -1]
    assert ke.encode_names([]).shape == (0,)


def test_pack_annos_rows_and_offsets():
    fix, gts, dts = kg.load(kg.EVAL_FIXTURES[0])
    rows, codes, off = ke.pack_annos(dts, with_score=True)
    assert off.dtype == np.int32 and off[0] == 0 and off[-1] == rows.shape[0] == codes.shape[0]
    assert rows.shape[1] == ke.ROW and rows.dtype == np.float64
    assert np.array_equal(np.diff(off), [len(a["name"]) for a in dts])
    assert any(len(a["name"]) == 0 for a in dts) and any(len(a["name"]) == 0 for a in gts)
    width = {"bbox": 4, "location": 3, "dimensions": 3}
    cat = lambda k: np.concatenate([np.asarray(a[k], dtype=np.float64).reshape(len(a["name"]), width.get(k, 1))
                                    for a in dts])
    assert np.array_equal(rows[:, 0:4], cat("bbox")) and np.array_equal(rows[:, 4:7], cat("location"))
    assert np.array_equal(rows[:, 7:10], cat("dimensions")) and np.array_equal(rows[:, 10], cat("rotation_y")[:, 0])
    assert np.array_equal(rows[:, 11], cat("alpha")[:, 0]) and np.array_equal(rows[:, 12], cat("score")[:, 0])
    grows, gcodes, _ = ke.pack_annos(gts, with_score=False)
    assert (grows[:, 12] == 0).all() and (gcodes == ke.DONTCARE).any()
    assert np.array_equal(grows[:, 13], np.concatenate([a["truncated"] for a in gts]))


def test_task_table_order_and_alternates():
    mo = ke.official_min_overlaps([0, 1, 2])
    info, m = ke.task_table([0, 1, 2], [0, 1, 2], mo, 1)
    assert info.shape == (18, 3) and m.shape == (18,)
    # class-major, then difficulty, then overlap (eval_class_v3's precision layout)
    assert info[:6, 0].tolist() == [0] * 6 and info[:6, 2].tolist() == [0, 0, 1, 1, 2, 2]
    assert info[0, 1] == ke.vocab_id("van") and info[6, 1] == ke.vocab_id("person_sitting") and info[12, 1] == ke.NO_ALT
    assert m[:2].tolist() == [0.7, 0.5] and m[6:8].tolist() == [0.5, 0.25]


def test_official_and_coco_min_overlaps():
    c = ke.coco_min_overlaps([0, 2])
    assert c.shape == (10, 3, 2) and np.allclose(c[:, 0, 0], np.linspace(0.5, 0.95, 10))
    assert np.allclose(c[:, 2, 1], np.linspace(0.25, 0.7, 10))


@pytest.mark.parametrize("path", kg.EVAL_FIXTURES, ids=kg.EVAL_IDS)
def test_formatter_reproduces_the_reference_strings(path):
    fix, _, dts = kg.load(path)
    classes = fix["classes"].tolist()
    aos = ke.compute_aos_of(dts)
    assert aos == bool(fix["official_m0_aos"])
    off = ke.format_official(classes, ke.official_min_overlaps(classes),
                             *[fix["official_m%d_precision" % m] for m in range(3)],
                             fix["official_m0_orientation"] if aos else None)
    assert off["result"] == str(fix["official_result"])
    coco = ke.format_coco(classes, *[fix["coco_m%d_precision" % m] for m in range(3)],
                          fix["coco_m0_orientation"] if aos else None)
    assert coco["result"] == str(fix["coco_result"])


def test_entry_points_reject_bad_arguments_and_missing_limit_bits_without_a_gpu():
    import ctypes
    from spconv import _lib
    lib = _lib.load()
    assert lib.b2s_kitti_overlaps(3, None, None, None, None, 1, None, 1, 1.0, None, None) == -2
    assert lib.b2s_kitti_overlaps(0, None, None, None, None, 1, None, 0, 1.0, None, None) == -2
    args = [0, None, None, None, None, 0, None, None, None, None, 0, 1, 4096, None, None, None, None, 1, 0, None, None,
            None, None, 0, None]
    assert lib.b2s_kitti_eval(*args) == -2 and b"4096 detections" in lib.b2s_last_error()
    # boxes need their difficulty limit bits: gt_limits (argument 3) for num_gt (5) > 0, dt_limits (8) for num_dt (10)
    dummy = ctypes.c_void_p(256)                      # never dereferenced: no tasks, so no kernel runs
    a = list(args)
    a[5], a[10], a[12], a[17] = 4, 4, 16, 0
    for gl, dl in ((None, dummy), (dummy, None)):
        a[3], a[8] = gl, dl
        assert lib.b2s_kitti_eval(*a) == -2 and b"limit bits" in lib.b2s_last_error()
    a[3], a[8] = dummy, dummy
    assert lib.b2s_kitti_eval(*a) == 0
    assert lib.b2s_kitti_eval_workspace_bytes(10, 80, 500, 18) > 0
    assert lib.b2s_kitti_convert(None, 8, 7, None, 1, None, None, None, None, None) == -2
