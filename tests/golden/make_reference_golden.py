"""Generate reference/reference.json.gz and reference/reference.npz FROM THE UNMODIFIED REFERENCE.

Needs a checkout of the original second.pytorch (B2S_REFERENCE_ROOT, see b2second/refcompat.py) on the CPU oracle
``spconv`` package.  Stores what tests/test_reference_dropin.py and tests/test_inputs.py compare against, so those
tests run without the reference:
  * every field of the five BASELINE config files as parsed by config.ModelConfig.from_file
  * the reference network's state-dict keys / shapes / dtypes and the sha256 of its anchors
  * the engine spec signature and the RPN launch plan of the reference network (sha1 of every tensor)
  * the reference's detections for the car.fhd forward and the two multi-class NMS cases
  * the reference's KITTI FOV crop (which rows it keeps) and NuScenes sweep merge
Usage:  python tests/golden/make_reference_golden.py
"""
import dataclasses
import gzip
import hashlib
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))

import torch  # noqa: E402

from b2second import config, loader, models, refcompat, synth, spec, tc  # noqa: E402

MIRROR_CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea"]
MULTICLASS = [("all.fhd", False), ("nuscenes.all.pp.largea", True)]


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def plain(v):
    """numpy scalars / arrays / dataclasses as the Python numbers / lists / dicts they compare equal to, recursively"""
    if isinstance(v, np.generic):
        return v.item()
    if isinstance(v, np.ndarray):
        return v.tolist()
    if isinstance(v, (tuple, list)):
        return type(v)(plain(x) for x in v)
    if isinstance(v, dict):
        return {k: plain(x) for k, x in v.items()}
    if dataclasses.is_dataclass(v) and not isinstance(v, type):
        return {"__dataclass__": type(v).__name__, **{f: plain(getattr(v, f)) for f in v.__dataclass_fields__}}
    return v


def as_json(v):
    return json.loads(json.dumps(plain(v), default=repr))


def signature_json(s):
    return as_json(s.signature())


def plan_digest(plan):
    """the RPN launch plan as JSON-able data: tensors by sha1 + shape + dtype, everything else by repr"""
    def d(v):
        if isinstance(v, torch.Tensor):
            t = v.detach().cpu().contiguous()
            return ["tensor", list(t.shape), str(t.dtype), hashlib.sha1(t.numpy().tobytes()).hexdigest()]
        return repr(plain(v))
    return {"buffers": repr(plain(plan["buffers"])), "ops": [{k: d(v) for k, v in op.items()} for op in plan["ops"]]}


def example(net, anchors, pts, max_voxels):
    res = net.voxel_generator.generate(pts, max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    return {"anchors": torch.from_numpy(anchors[None].copy()), "voxels": torch.from_numpy(res["voxels"]),
            "num_points": torch.from_numpy(res["num_points_per_voxel"]), "coordinates": torch.from_numpy(coords)}


def main():
    refcompat.install(loader.ORACLE_DIR)
    import spconv
    assert getattr(spconv, "__oracle__", False)
    out, arrays = {}, {}
    # config files
    out["configs"] = {}
    for name in sorted(config.BUILTIN):
        path = os.path.join(refcompat.REFERENCE_ROOT, "second", "configs", config.REFERENCE_FILES[name])
        parsed = config.ModelConfig.from_file(path, name)
        out["configs"][name] = {f: as_json(getattr(parsed, f)) for f in parsed.__dataclass_fields__}
    # network structure, anchors, car.fhd forward
    out["networks"] = {}
    for name in MIRROR_CONFIGS:
        cfgp = refcompat.load_config(config.REFERENCE_FILES[name])
        ref = refcompat.build_network(cfgp.model.second).eval()
        models.synthetic_weights_(ref, name)
        a_ref = refcompat.generate_anchors(ref, cfgp.model.second)
        out["networks"][name] = {
            "state_dict": {k: [list(v.shape), str(v.dtype)] for k, v in ref.state_dict().items()},
            "anchors": [list(a_ref.shape), str(a_ref.dtype), sha256(a_ref)]}
        if name == "car.fhd":
            b = config.get_config(name)
            with torch.no_grad():
                o = ref(example(ref, a_ref, synth.kitti_cloud(4, 12000, b.point_cloud_range), b.max_voxels))[0]
            for k in ("box3d_lidar", "scores", "label_preds"):
                arrays["forward.car.fhd." + k] = o[k].numpy()
    # engine spec + RPN plan of the reference network
    out["spec"] = {}
    for name in sorted(config.BUILTIN):
        cfgp = refcompat.load_config(config.REFERENCE_FILES[name])
        ref = refcompat.build_network(cfgp.model.second).eval()
        models.synthetic_weights_(ref, name)
        cfg = config.get_config(name)
        s_ref = spec.spec_from_module(ref, max_voxels=cfg.max_voxels)
        fm = cfg.feature_map_size
        out["spec"][name] = {"signature": signature_json(s_ref),
                             "anchors": sha256(spec.anchors_for(s_ref, (fm[1], fm[2]))),
                             "plan": plan_digest(tc.plan_rpn(ref.rpn, 64, 48))}
    # multi-class NMS branch
    for name, agnostic in MULTICLASS:
        cfgp = refcompat.load_config(config.REFERENCE_FILES[name])
        for cs in cfgp.model.second.target_assigner.class_settings:
            cs.use_multi_class_nms = True
        cfgp.model.second.nms_class_agnostic = agnostic
        ref = refcompat.build_network(cfgp.model.second).eval()
        assert ref._multiclass_nms and ref._nms_class_agnostic == agnostic
        b = dataclasses.replace(config.get_config(name), use_multi_class_nms=True, nms_class_agnostic=agnostic)
        models.synthetic_weights_(ref, name)
        a_ref = refcompat.generate_anchors(ref, cfgp.model.second)
        pts = synth.nuscenes_cloud(1, 40000) if "nuscenes" in name else synth.kitti_cloud(4, 12000, b.point_cloud_range)
        with torch.no_grad():
            o = ref(example(ref, a_ref, pts, b.max_voxels))[0]
        for k in ("box3d_lidar", "scores", "label_preds"):
            arrays["multiclass.%s.%d.%s" % (name, int(agnostic), k)] = o[k].numpy()
    # input path: FOV crop and sweep merge (test_inputs.py builds the same inputs)
    import test_inputs as ti
    from second.core import box_np_ops
    P2, rect, Trv2c, shape = ti.kitti_calib()
    pts = ti.raw_kitti_cloud(0, 20000)
    kept = box_np_ops.remove_outside_points(pts, rect, Trv2c, P2, shape)
    rows = {r.tobytes(): i for i, r in enumerate(pts)}
    idx = np.array([rows[r.tobytes()] for r in kept], dtype=np.int64)
    assert np.all(np.diff(idx) > 0) and np.array_equal(pts[idx], kept)
    mask = np.zeros(pts.shape[0], dtype=bool)
    mask[idx] = True
    arrays["crop.kitti.seed0.n20000.keep"] = np.packbits(mask)
    # modules the dataset file imports at top level but this code path never uses: scikit-image and fire
    for name in ("skimage", "skimage.io", "fire"):
        if name not in sys.modules:
            try:
                __import__(name)
            except ImportError:
                sys.modules[name] = types.ModuleType(name)
    if not hasattr(sys.modules["skimage"], "io"):
        sys.modules["skimage"].io = sys.modules["skimage.io"]
    from second.data.nuscenes_dataset import NuScenesDataset
    sweeps, rots, trans, lags = ti.sweep_case(1)
    ts = 1.5e15
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i, p in enumerate(sweeps):
            f = os.path.join(tmp, "s%d.bin" % i)
            p.tofile(f)
            paths.append(f)
        info = {"token": "t", "lidar_path": paths[0], "timestamp": ts,
                "sweeps": [{"lidar_path": paths[i], "timestamp": ts - lags[i] * 1e6, "sweep2lidar_rotation": rots[i],
                            "sweep2lidar_translation": trans[i]} for i in range(1, len(sweeps))]}
        ds = object.__new__(NuScenesDataset)
        ds._nusc_infos = [info]
        arrays["sweeps.seed1.points"] = ds.get_sensor_data(0)["lidar"]["points"].astype(np.float32)
    os.makedirs(os.path.join(HERE, "reference"), exist_ok=True)
    with gzip.open(os.path.join(HERE, "reference", "reference.json.gz"), "wt") as f:
        json.dump(out, f, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, "reference", "reference.npz"), **arrays)
    print("wrote reference.json.gz, reference.npz:", sorted(arrays))


if __name__ == "__main__":
    main()
