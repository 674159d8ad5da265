"""KITTI formatting and evaluation on the GPU (csrc/kitti_eval.cu through b2second.kitti_eval) against what the
unmodified reference computed (tests/golden/kitti_eval, make_kitti_eval_golden.py).  Bars: result strings identical,
precision and thresholds bit-equal, orientation within 1e-12 relative; converted annos in the same set and order,
values within 1e-9 relative."""
import numpy as np
import pytest
import torch

import kitti_golden as kg
from b2second import kitti_eval as ke

pytestmark = pytest.mark.gpu


def _check_arrays(got, fix, tag, metric):
    assert np.array_equal(got["precision"], fix["%s_m%d_precision" % (tag, metric)], equal_nan=True)
    assert np.array_equal(got["thresholds"], fix["%s_m%d_thresholds" % (tag, metric)])
    want = fix["%s_m%d_orientation" % (tag, metric)]
    assert np.allclose(got["orientation"], want, rtol=1e-12, atol=0, equal_nan=True)


@pytest.mark.parametrize("path", kg.EVAL_FIXTURES, ids=kg.EVAL_IDS)
def test_official_result_matches_reference(product, path):
    fix, gts, dts = kg.load(path)
    classes, z = fix["classes"].tolist(), dict(z_axis=int(fix["z_axis"]), z_center=float(fix["z_center"]))
    res = ke.get_official_eval_result(gts, dts, classes, **z)
    assert res["result"] == str(fix["official_result"])
    mo = ke.official_min_overlaps(classes)
    for metric in range(3):
        got = ke.eval_class(gts, dts, classes, [0, 1, 2], metric, mo, bool(fix["official_m%d_aos" % metric]), **z)
        _check_arrays(got, fix, "official", metric)


@pytest.mark.parametrize("path", kg.EVAL_FIXTURES, ids=kg.EVAL_IDS)
def test_coco_result_matches_reference(product, path):
    fix, gts, dts = kg.load(path)
    classes, z = fix["classes"].tolist(), dict(z_axis=int(fix["z_axis"]), z_center=float(fix["z_center"]))
    res = ke.get_coco_eval_result(gts, dts, classes, **z)
    assert res["result"] == str(fix["coco_result"])
    mo = ke.coco_min_overlaps(classes)
    for metric in range(3):
        got = ke.eval_class(gts, dts, classes, [0, 1, 2], metric, mo, bool(fix["coco_m%d_aos" % metric]), **z)
        _check_arrays(got, fix, "coco", metric)


def test_inputs_are_not_modified_and_runs_are_bit_identical(product):
    fix, gts, dts = kg.load(kg.EVAL_FIXTURES[0])
    before = [{k: v.copy() for k, v in a.items()} for a in dts]
    mo = ke.official_min_overlaps([0, 1, 2])
    runs = [ke.eval_class(gts, dts, [0, 1, 2], [0, 1, 2], 2, mo, True) for _ in range(2)]
    for k in ("precision", "orientation", "thresholds"):
        assert runs[0][k].tobytes() == runs[1][k].tobytes()
    for a, b in zip(before, dts):
        assert all(np.array_equal(a[k], b[k]) for k in a)


def test_any_frame_count_and_empty_frames(product):
    """below the reference's 50-frame floor: one frame, and frames without ground truth or detections"""
    fix, gts, dts = kg.load(kg.EVAL_FIXTURES[0])
    one = ke.get_official_eval_result(gts[:1], dts[:1], [0, 1, 2])
    assert one["result"].count("AP") >= 9
    empty_gt = [a for a in gts if len(a["name"]) == 0][0]
    empty_dt = [a for a in dts if len(a["name"]) == 0][0]
    res = ke.get_official_eval_result([empty_gt, gts[1]], [dts[1], empty_dt], ["Car"])
    assert "Car AP" in res["result"]
    res = ke.get_coco_eval_result([empty_gt], [empty_dt], ["Car"])
    assert "bbox AP:0.00, 0.00, 0.00" in res["result"]


def _perfect_set(seed, n_frames=60):
    rng = np.random.default_rng(seed)
    gts = []
    for f in range(n_frames):
        names = rng.choice(["Car", "Pedestrian", "Cyclist", "Van", "DontCare"], 8)
        x = rng.uniform(-20, 20, 8) + np.arange(8) * 50           # boxes far apart: no cross matches
        z = rng.uniform(5, 40, 8)
        loc = np.stack([x, rng.uniform(1.5, 1.8, 8), z], 1)
        dims = np.stack([rng.uniform(0.6, 4, 8), rng.uniform(1.4, 1.8, 8), rng.uniform(0.5, 1.8, 8)], 1)
        u = rng.uniform(0, 1000, 8) + np.arange(8) * 1500
        bbox = np.stack([u, np.full(8, 150.0), u + rng.uniform(30, 80, 8), 150 + rng.uniform(45, 90, 8)], 1)
        gts.append({"name": names, "bbox": bbox, "location": loc, "dimensions": dims,
                    "rotation_y": rng.uniform(-3, 3, 8), "alpha": rng.uniform(-3, 3, 8), "truncated": np.zeros(8),
                    "occluded": np.zeros(8, dtype=np.int64)})
    scores = rng.permutation(np.linspace(0.01, 0.99, 8 * n_frames)).reshape(n_frames, 8)
    dts = [dict(g, score=s.astype(np.float32)) for g, s in zip(gts, scores)]
    return gts, dts


def test_detections_equal_to_ground_truth_give_100(product):
    gts, dts = _perfect_set(7)
    res = ke.get_official_eval_result(gts, dts, [0, 1, 2])
    for cls, d in res["detail"].items():
        for key, aps in d.items():
            assert aps == [100.0, 100.0, 100.0], (cls, key, aps)
    coco = ke.get_coco_eval_result(gts, dts, [0, 1, 2])
    for cls, d in coco["detail"].items():
        for key, aps in d.items():
            assert np.allclose(aps, 100.0, rtol=0, atol=1e-9), (cls, key, aps)


def _convert_inputs(fix, device):
    off = fix["det_offsets"]
    dets, infos = [], []
    for i, (lo, hi) in enumerate(zip(off[:-1], off[1:])):
        dets.append({"box3d_lidar": torch.from_numpy(fix["det_box3d_lidar"][lo:hi].copy()).to(device),
                     "scores": torch.from_numpy(fix["det_scores"][lo:hi].copy()).to(device),
                     "label_preds": torch.from_numpy(fix["det_label_preds"][lo:hi].copy()).to(device),
                     "metadata": {"image_idx": i}})
        c = fix["calib"][i]
        infos.append({"calib": {"R0_rect": c[0], "Tr_velo_to_cam": c[1], "P2": c[2]},
                      "image": {"image_idx": i, "image_shape": fix["image_shape"][i]}})
    return dets, infos


def _assert_annos_close(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert list(g["name"]) == list(w["name"])
        assert np.array_equal(g["score"], w["score"])          # same boxes, same order
        for k in ("bbox", "location", "dimensions", "rotation_y"):
            assert np.allclose(g[k], w[k], rtol=1e-9, atol=1e-9), k
        # alpha = -arctan2(-y, x) + ry: the reference evaluates the arctan2 in float32, whose last bits depend on
        # numpy's vectorised float32 arctan2 -- compare at a few float32 ulps
        assert np.allclose(g["alpha"], w["alpha"], rtol=0, atol=2e-6)
        assert (g["truncated"] == 0).all() and (g["occluded"] == 0).all()


@pytest.mark.parametrize("where", ["cuda", "cpu"])
def test_conversion_matches_reference(product, where):
    fix = np.load(kg.CONVERT_FIXTURE, allow_pickle=False)
    dets, infos = _convert_inputs(fix, where)
    before = [{k: v.clone() for k, v in d.items() if torch.is_tensor(v)} for d in dets]
    got = ke.convert_detection_to_kitti_annos(dets, infos, fix["class_names"].tolist())
    want = kg.annos(fix, "anno_")
    _assert_annos_close(got, want)
    assert [a["metadata"]["image_idx"] for a in got] == list(range(len(dets)))
    for b, d in zip(before, dets):
        assert all(torch.equal(v, d[k]) for k, v in b.items())


def test_end_to_end_engine_then_conversion_then_eval(product):
    from b2second import config, fastpath, models, synth
    name = "car.fhd"
    cfg = config.get_config(name)
    conv = np.load(kg.CONVERT_FIXTURE, allow_pickle=False)
    _, infos = _convert_inputs(conv, "cpu")
    clouds = [synth.kitti_cloud(s, 20000, cfg.point_cloud_range) for s in (0, 1)]
    outs = {}
    for output in ("device", "host"):
        net = models.build_network(cfg, product).eval()
        models.synthetic_weights_(net, name, seed=0)
        net = fastpath.accelerate(net.cuda(), max_points=20000, output=output)
        anchors = torch.from_numpy(net.anchors()[None]).cuda()
        dets = []
        for pts in clouds:
            dets += net({"points": [torch.from_numpy(pts).cuda()], "anchors": anchors,
                         "metadata": [{"image_idx": len(dets)}]})
        assert dets[0]["box3d_lidar"].is_cuda == (output == "device")
        outs[output] = ke.convert_detection_to_kitti_annos(dets, infos[:2], ["Car"])
    for a, b in zip(outs["device"], outs["host"]):
        assert a.keys() == b.keys()
        for k in a:
            if k != "metadata":
                assert np.array_equal(a[k], b[k]), k
    assert sum(len(a["name"]) for a in outs["device"]) > 0
    res = ke.get_official_eval_result(outs["device"], outs["host"], ["Car"])
    assert res["result"].startswith("Car AP(Average Precision)@0.70, 0.70, 0.70:")
