"""Generate the anchor-area mask fixtures FROM THE UNMODIFIED REFERENCE.

For each case the reference's own eval preprocessing, ``second.data.preprocess.prep_pointcloud({"lidar": {"points":
pts}}, ..., training=False, max_voxels=..., anchor_area_threshold=...)``, voxelises the seeded synthetic cloud of
``b2second.synth`` and builds ``anchors_mask`` (preprocess.py:345-357).  The reference's own network (built by its own
``second_builder`` from its config, on the CPU oracle ``spconv`` with the seeded synthetic weights of
``b2second.models.synthetic_weights_``) then runs on that example with the mask, and its ``predict`` runs a second
time on the same head outputs without the mask.  The threshold is the config's own ``eval_input_reader`` value, or 1
where a config has it off (-1) and the case forces it on.
Writes anchor_mask/<config>.seed<S>.n<P>[.mv<max_voxels>].npz:
  mask_packed (np.packbits of the bool [A] mask), threshold, voxel_num, max_voxels, coords_sha1, anchors_sha1,
  num_anchors, and the detections in the fields of the single-head fixtures (make_golden.py) -- with the mask as
  box3d_lidar / scores / label_preds / label_margin, without it under the same names prefixed ``nomask_``.
Usage:  python tests/golden/make_anchor_mask_golden.py [--force]
"""
import hashlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))

from b2second import config, loader, models, refcompat, synth  # noqa: E402

CASES = [  # (config name, cloud kind, seed, num_points, force the threshold to 1[, max_voxels override])
    ("pointpillars.car.xyres_16", "kitti", 0, 20000, False),
    ("pointpillars.car.xyres_16", "kitti", 1, 6000, False),
    # more pillars than max_voxels: only the first 3000 count in the map
    ("pointpillars.car.xyres_16", "kitti", 3, 20000, False, 3000),
    ("car.fhd", "kitti", 0, 20000, True),                   # 3-D voxels: a column counts every voxel in it
    ("car.fhd", "kitti", 1, 6000, True),
    ("car.lite", "kitti", 0, 20000, True),
    ("car.lite", "kitti", 2, 3000, True),
    ("nuscenes.all.pp.largea", "nuscenes", 0, 60000, True),  # negative range origin, 360-degree anchors
    ("nuscenes.all.pp.largea", "nuscenes", 1, 20000, True),
    ("nuscenes.all.pp.mhead", "nuscenes", 0, 60000, True),   # two heads, global anchor ids
    ("nuscenes.all.pp.mhead", "nuscenes", 1, 20000, True),
]
OUT_DIR = os.path.join(HERE, "anchor_mask")


def reference_file(name):
    return config.REFERENCE_FILES[name] if name in config.REFERENCE_FILES else config.EXTRA_REFERENCE_FILES[name]


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def margins_of(cls_preds, num_class, scores):
    """per detection: margin between the best and second-best class logit of its anchor (label ties)"""
    import torch
    cl = cls_preds.reshape(-1, num_class)
    top = torch.sigmoid(cl).max(1)[0]
    out = []
    for sc in scores:
        a = int(torch.argmin((top - sc).abs()))
        v = torch.sort(cl[a], descending=True)[0]
        out.append(float(v[0] - v[1]) if v.numel() > 1 else 1e9)
    return np.array(out, np.float32)


def main():
    import torch
    refcompat.install(loader.ORACLE_DIR)
    import spconv
    assert getattr(spconv, "__oracle__", False)
    # modules second.data imports at top level but prep_pointcloud never calls (image I/O, plotting, CLI): empty stand-ins
    for mod in ("skimage", "skimage.io", "fire", "cv2", "seaborn", "matplotlib", "matplotlib.pyplot"):
        if mod not in sys.modules:
            try:
                __import__(mod)
            except ImportError:
                sys.modules[mod] = types.ModuleType(mod)
                if "." in mod:
                    parent, child = mod.rsplit(".", 1)
                    setattr(sys.modules[parent], child, sys.modules[mod])
    from second.data.preprocess import prep_pointcloud
    from second.utils.config_tool import get_downsample_factor
    torch.set_num_threads(8)
    force = "--force" in sys.argv
    os.makedirs(OUT_DIR, exist_ok=True)
    for case in CASES:
        name, kind, seed, npts, force_on = case[:5]
        max_voxels = case[5] if len(case) > 5 else None
        path = os.path.join(OUT_DIR, "%s.seed%d.n%d%s.npz" % (name, seed, npts, ".mv%d" % max_voxels if max_voxels else ""))
        if os.path.exists(path) and not force:
            continue
        cfgp = refcompat.load_config(reference_file(name))
        mcfg = cfgp.model.second
        native = float(cfgp.eval_input_reader.preprocess.anchor_area_threshold)
        threshold = 1.0 if force_on else native
        assert threshold >= 0, "%s: the mask is off in this config (%g)" % (name, native)
        net = refcompat.build_network(mcfg).eval()
        models.synthetic_weights_(net, name, seed=0)
        b = config.get_config(name)
        pts = synth.nuscenes_cloud(seed, npts) if kind == "nuscenes" else synth.kitti_cloud(seed, npts, b.point_cloud_range)
        mv = int(max_voxels or b.max_voxels)
        ex = prep_pointcloud({"lidar": {"points": pts}}, None, net.voxel_generator, net.target_assigner,
                             max_voxels=mv, training=False, create_targets=False,
                             num_point_features=int(pts.shape[1]), anchor_area_threshold=threshold,
                             out_size_factor=get_downsample_factor(mcfg))
        mask = np.asarray(ex["anchors_mask"], bool)
        anchors = np.asarray(ex["anchors"], np.float32)
        assert sha(anchors) == sha(refcompat.generate_anchors(net, mcfg))
        coords = np.pad(ex["coordinates"], ((0, 0), (1, 0)))
        tex = {"anchors": torch.from_numpy(anchors[None]), "voxels": torch.from_numpy(ex["voxels"]),
               "num_points": torch.from_numpy(ex["num_points"]), "coordinates": torch.from_numpy(coords),
               "anchors_mask": torch.from_numpy(mask[None])}
        with torch.no_grad():
            pd = net.network_forward(tex["voxels"], tex["num_points"], tex["coordinates"], 1)
            out = net.predict(tex, pd)[0]
            nomask = net.predict({k: v for k, v in tex.items() if k != "anchors_mask"}, pd)[0]
        fix = {
            "points_sha1": sha(pts), "num_points": pts.shape[0], "voxel_num": int(ex["voxels"].shape[0]),
            "max_voxels": mv, "threshold": threshold, "coords_sha1": sha(ex["coordinates"]),
            "anchors_sha1": sha(anchors), "num_anchors": anchors.shape[0], "mask_packed": np.packbits(mask),
            "num_masked_in": int(mask.sum()),
        }
        for prefix, o in (("", out), ("nomask_", nomask)):
            fix[prefix + "box3d_lidar"] = o["box3d_lidar"].numpy()
            fix[prefix + "scores"] = o["scores"].numpy()
            fix[prefix + "label_preds"] = o["label_preds"].numpy()
            fix[prefix + "label_margin"] = margins_of(pd["cls_preds"], b.num_class, o["scores"])
        np.savez_compressed(path, **fix)
        print(name, seed, npts, "thr", threshold, "voxels", fix["voxel_num"], "anchors kept", fix["num_masked_in"], "of",
              anchors.shape[0], "dets", out["box3d_lidar"].shape[0], "nomask", nomask["box3d_lidar"].shape[0], "->",
              os.path.relpath(path, HERE), os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main()
