"""The NuScenes multi-head network (VoxelNetNuscenesMultiHead, nuscenes/all.pp.mhead) on the CPU: the mirror on the
oracle reproduces the fixtures generated from the unmodified reference (tests/golden/make_mhead_golden.py), the
mirror and the reference network have the same structure, spec and launch plan, and the launch plan -- interpreted
with torch.conv2d -- computes what the torch modules of both heads compute."""
import glob
import json
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from b2second import config, loader, models, spec, tc

NAME = "nuscenes.all.pp.mhead"
MHEAD_DIR = os.path.join(gu.GOLDEN_DIR, "mhead")


def mhead_cases():
    """(seed, num_points, fixture path) of every fixture under golden/mhead"""
    out = []
    for p in sorted(glob.glob(os.path.join(MHEAD_DIR, "*.npz"))):
        m = re.match(r"^(.*)\.seed(\d+)\.n(\d+)(?:\.mv(\d+))?$", os.path.basename(p)[:-4])
        assert m.group(1) == NAME
        out.append((int(m.group(2)), int(m.group(3)), p))
    return out


CASES = mhead_cases()
IDS = ["s%d-n%d%s" % (c[0], c[1], "-mv" if ".mv" in c[2] else "") for c in CASES]


def build(backend):
    net = models.build_network(config.get_config(NAME), backend).eval()
    models.synthetic_weights_(net, NAME, seed=0)
    return net


def test_config_is_known_but_not_a_baseline_config():
    cfg = config.get_config(NAME)
    assert isinstance(cfg, config.MultiHeadModelConfig) and NAME not in config.BUILTIN
    assert cfg.num_anchors_per_loc == 20 and len(cfg.class_feature_map_sizes) == 10
    assert len(CASES) == 4


@pytest.mark.parametrize("seed,n,path", CASES, ids=IDS)
def test_mirror_on_oracle_reproduces_reference_golden(oracle, seed, n, path):
    fix = np.load(path)
    pts = gu.make_cloud(NAME, seed, n)
    assert gu.sha(pts) == str(fix["points_sha1"]), "synthetic cloud generator drifted"
    net = build(oracle)
    anchors = net.anchors()
    assert anchors.shape[0] == int(fix["num_anchors"]) == 324800 and gu.sha(anchors) == str(fix["anchors_sha1"])
    res = net.voxel_generator.generate(pts, int(fix["max_voxels"]))
    assert res["voxel_num"] == int(fix["voxel_num"])
    assert gu.sha(res["coordinates"]) == str(fix["coords_sha1"]) and gu.sha(res["voxels"]) == str(fix["voxels_sha1"])
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    ex = {"anchors": torch.from_numpy(anchors[None]), "voxels": torch.from_numpy(res["voxels"]),
          "num_points": torch.from_numpy(res["num_points_per_voxel"]), "coordinates": torch.from_numpy(coords)}
    with torch.no_grad():
        vf = net.voxel_feature_extractor(ex["voxels"], ex["num_points"], ex["coordinates"])
        pd = net.network_forward(ex["voxels"], ex["num_points"], ex["coordinates"], 1)
        out = net(ex)[0]
    np.testing.assert_allclose(vf.flatten()[fix["vfe_sel_idx"]].numpy(), fix["vfe_sel_val"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(pd["box_preds"].flatten()[fix["box_sel_idx"]].numpy(), fix["box_sel_val"], atol=1e-5)
    np.testing.assert_allclose(pd["cls_preds"].flatten()[fix["cls_sel_idx"]].numpy(), fix["cls_sel_val"], atol=1e-5)
    gu.assert_detections_close({k: (v.numpy() if hasattr(v, "numpy") else v) for k, v in out.items()}, fix)
    assert out["box3d_lidar"].shape[0] > 0


def _structure():
    with open(os.path.join(gu.GOLDEN_DIR, "reference", "mhead.json")) as f:
        return json.load(f)


def test_mirror_has_the_reference_structure(oracle):
    import importlib.util
    # the JSON digests are those the generator wrote (tests/golden/make_reference_golden.py)
    sp_ = importlib.util.spec_from_file_location("make_reference_golden",
                                                 os.path.join(gu.GOLDEN_DIR, "make_reference_golden.py"))
    mrg = importlib.util.module_from_spec(sp_)
    sp_.loader.exec_module(mrg)
    ref = _structure()
    cfg = config.get_config(NAME)
    assert ref["config"]["class"] == "MultiHeadModelConfig"
    assert {f: mrg.as_json(getattr(cfg, f)) for f in cfg.__dataclass_fields__} == ref["config"]["fields"]
    net = build(oracle)
    sd = {k: [list(v.shape), str(v.dtype)] for k, v in net.state_dict().items()}
    want = {k: v for k, v in ref["state_dict"].items() if k.split(".")[0] not in (
        "rpn_acc", "rpn_precision", "rpn_recall", "rpn_metrics", "rpn_cls_loss", "rpn_loc_loss", "rpn_total_loss")}
    assert sd == want
    a = net.anchors()
    assert [list(a.shape), str(a.dtype), mrg.sha256(a)] == ref["anchors"]
    s = spec.spec_from_module(net)
    assert mrg.signature_json(s) == ref["spec"]
    assert s.pfn_decoration == 1 and s.num_point_features == 4 and s.head_feature_map_sizes == [[100, 100], [160, 160]]
    H, W = int(cfg.grid_size[1]), int(cfg.grid_size[0])
    assert mrg.plan_digest(tc.plan_rpn_multihead(net.rpn, dict(s.heads), H, W)) == ref["plan"]
    assert tc.supported(net.rpn, s.heads) and not tc.supported(net.rpn)


def interpret(plan, x):
    """x [B, C, H, W] fp32 -> {segment name: packed heads [B, S, Hh, Wh]}, executing the ops with plain torch (the crop
    op: the interior window, then the zero padding of the next conv)."""
    B = x.shape[0]
    bufs = {"in": x}
    for name, (h, w, c) in plan["buffers"].items():
        bufs[name] = torch.zeros(B, c, h, w)
    for sg in plan["segments"]:
        bufs[sg["buffer"]] = torch.zeros(B, sg["stride"], sg["H"], sg["W"])
    for op in plan["ops"]:
        src = bufs[op["src"]]
        assert src.shape[1] == op["cin"] and tuple(src.shape[2:]) == (op["Hin"], op["Win"])
        if op["kind"] == "crop":
            c = op["crop"]
            bufs[op["dst"]] = src[:, :, c:op["Hin"] - c, c:op["Win"] - c].clone()
            continue
        w = (op["w_hi"].float() + op["w_lo"].float())[:, :op["cout"]]
        w = w.reshape(op["kh"], op["kw"], op["cout"], op["cin"]).permute(2, 3, 0, 1)
        y = F.conv2d(src, w, stride=op["stride"], padding=op["pad"])
        y = y * op["scale"].view(1, -1, 1, 1)
        if op["shift"] is not None:
            y = y + op["shift"].view(1, -1, 1, 1)
        if op["relu"]:
            y = torch.relu(y)
        c0 = op["dst_coff"]
        bufs[op["dst"]][:, c0:c0 + op["cout"], op["off_h"]::op["out_mul"], op["off_w"]::op["out_mul"]] = y
    return {sg["name"]: bufs[sg["buffer"]] for sg in plan["segments"]}


def test_multihead_program_semantics_on_cpu(oracle):
    net = build(oracle)
    s = spec.spec_from_module(net)
    H, W = 80, 96
    torch.manual_seed(1)
    x = torch.relu(torch.randn(2, 64, H, W)) * (torch.rand(2, 1, H, W) < 0.2)
    with torch.no_grad():
        ro = net.rpn(x)
        c = int(np.round(ro["stage0"].shape[2] * 0.1))
        small_in = net.small_head.net(ro["stage0"][:, :, c:-c, c:-c])
        refs = {}
        for name, m, feat in (("large", net.large_head, ro["out"]), ("small", net.small_head, small_in)):
            refs[name] = torch.cat([m.conv_box(feat), m.conv_cls(feat), m.conv_dir_cls(feat)], 1)
        plan = tc.plan_rpn_multihead(net.rpn, dict(s.heads), H, W)
        got = interpret(plan, x)
    assert [sg["name"] for sg in plan["segments"]] == ["large", "small"] and plan["crop"] == c == 4
    for sg in plan["segments"]:
        ref, g = refs[sg["name"]], got[sg["name"]]
        n = ref.shape[1]
        assert n == sg["offsets"][-1] and n in (228, 152) and tuple(g.shape[2:]) == tuple(ref.shape[2:])
        # wider than one 128-channel launch: two head ops with channel offsets 0 and 128
        assert [op["dst_coff"] for op in plan["ops"] if op["dst"] == sg["buffer"]] == [0, 128]
        err = float((g[:, :n] - ref).abs().max())
        assert err <= 2e-5 * max(1.0, float(ref.abs().max())), (sg["name"], err)


@pytest.mark.parametrize("vfe_name", ["PillarFeatureNetRadiusHeight", "PillarFeatureNetOld"])
def test_other_pillar_decorations_are_rejected(oracle, vfe_name):
    """same attributes as PillarFeatureNet(Radius), other decorations: the engine must not take them"""
    net = build(oracle)
    cls = type(vfe_name, (models.PillarFeatureNetRadius,), {})
    old = net.voxel_feature_extractor
    net.voxel_feature_extractor = cls(num_input_features=4, num_filters=[64], voxel_size=[0.25, 0.25, 8],
                                      pc_range=[-50, -50, -5, 50, 50, 3])
    net.voxel_feature_extractor.load_state_dict(old.state_dict())
    with pytest.raises(spec.UnsupportedNetwork, match=vfe_name):
        spec.spec_from_module(net)


def test_multihead_with_per_class_nms_is_rejected(oracle):
    net = build(oracle)
    net._multiclass_nms = True
    with pytest.raises(spec.UnsupportedNetwork, match="per-class NMS"):
        spec.spec_from_module(net)


def test_pillar_configs_keep_the_plain_decoration():
    sp = loader.oracle_spconv()
    for name in ("pointpillars.car.xyres_16", "nuscenes.all.pp.largea"):
        s = spec.spec_from_module(models.build_network(config.get_config(name), sp).eval())
        assert s.pfn_decoration == 0 and s.heads is None and "pfn_decoration" not in s.signature()
