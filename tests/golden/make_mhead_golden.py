"""Generate the multi-head network's fixtures FROM THE UNMODIFIED REFERENCE.

The reference's own ``VoxelNetNuscenesMultiHead`` (second/pytorch/models/net_multi_head.py, built by its own
``second_builder`` from second/configs/nuscenes/all.pp.mhead.config) runs on the CPU oracle ``spconv`` package with the
seeded synthetic weights of ``b2second.models.synthetic_weights_`` and the seeded NuScenes clouds of ``b2second.synth``.
Writes
  * mhead/nuscenes.all.pp.mhead.seed<S>.n<P>[.mv<max_voxels>].npz -- the fields of the single-head fixtures
    (make_golden.py); the head samples index the concatenated ``box_preds`` / ``cls_preds`` [B, A, k] of
    ``network_forward`` (large head's anchors first, then the small head's);
  * reference/mhead.json -- parsed config, state-dict shapes, anchor sha256, engine spec signature and the launch plan
    of the reference network.
Existing fixtures are left alone (a separate directory and file: the single-head suites glob golden/*.npz).
Usage:  python tests/golden/make_mhead_golden.py [--force]
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_reference_golden as mrg  # noqa: E402  (sets up sys.path, shares the JSON digests)
import torch  # noqa: E402

from b2second import config, loader, models, refcompat, spec, synth, tc  # noqa: E402

NAME = "nuscenes.all.pp.mhead"
CASES = [  # (seed, num_points[, max_voxels override])
    (0, 60000),
    (1, 120000),
    (2, 300000),
    # more pillars than max_voxels: the extra ones are dropped in first-come order
    (1, 120000, 12000),
]
OUT_DIR = os.path.join(HERE, "mhead")


def sha(a):
    return mrg.hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixtures(ref, anchors, force):
    os.makedirs(OUT_DIR, exist_ok=True)
    b = config.get_config(NAME)
    for case in CASES:
        seed, npts = case[:2]
        max_voxels = case[2] if len(case) > 2 else None
        path = os.path.join(OUT_DIR, "%s.seed%d.n%d%s.npz" % (NAME, seed, npts, ".mv%d" % max_voxels if max_voxels else ""))
        if os.path.exists(path) and not force:
            continue
        pts = synth.nuscenes_cloud(seed, npts)
        res = ref.voxel_generator.generate(pts, max_voxels or b.max_voxels)
        coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
        ex = {"anchors": torch.from_numpy(anchors[None]), "voxels": torch.from_numpy(res["voxels"]),
              "num_points": torch.from_numpy(res["num_points_per_voxel"]), "coordinates": torch.from_numpy(coords)}
        with torch.no_grad():
            vf = ref.voxel_feature_extractor(ex["voxels"], ex["num_points"], ex["coordinates"])
            sf = ref.middle_feature_extractor(vf, ex["coordinates"], 1)
            pd = ref.network_forward(ex["voxels"], ex["num_points"], ex["coordinates"], 1)
            out = ref(ex)[0]
        cl = pd["cls_preds"].reshape(-1, b.num_class)
        top = torch.sigmoid(cl).max(1)[0]
        margins = []
        for sc in out["scores"]:
            a = int(torch.argmin((top - sc).abs()))
            v = torch.sort(cl[a], descending=True)[0]
            margins.append(float(v[0] - v[1]))
        # head samples: half anywhere, half among the small head's anchors (the tail of the concatenation)
        n_large = 12 * 100 * 100
        rng = np.random.default_rng(0)
        box_n, cls_n = pd["box_preds"].numel(), pd["cls_preds"].numel()
        box_sel = np.concatenate([rng.choice(box_n, 256, replace=False),
                                  n_large * b.box_code_size + rng.choice(box_n - n_large * b.box_code_size, 256, replace=False)])
        cls_sel = np.concatenate([rng.choice(cls_n, 256, replace=False),
                                  n_large * b.num_class + rng.choice(cls_n - n_large * b.num_class, 256, replace=False)])
        nz = torch.nonzero(sf.flatten()).flatten().numpy()
        sel_nz = nz[np.random.default_rng(1).choice(nz.size, min(256, nz.size), replace=False)]
        fix = {
            "points_sha1": sha(pts), "num_points": pts.shape[0], "voxel_num": res["voxel_num"],
            "max_voxels": int(max_voxels or b.max_voxels),
            "coords_sha1": sha(res["coordinates"]), "num_points_per_voxel_sha1": sha(res["num_points_per_voxel"]),
            "voxels_sha1": sha(res["voxels"]), "coords_head": res["coordinates"][:64],
            "vfe_sum": float(vf.double().sum()), "vfe_abs": float(vf.double().abs().sum()),
            "vfe_sel_idx": np.arange(0, vf.numel(), max(1, vf.numel() // 256))[:256],
            "vfe_sel_val": vf.flatten()[np.arange(0, vf.numel(), max(1, vf.numel() // 256))[:256]].numpy(),
            "bev_shape": np.array(sf.shape), "bev_nonzero": int((sf != 0).sum()),
            "bev_sum": float(sf.double().sum()), "bev_abs": float(sf.double().abs().sum()),
            "bev_sel_idx": sel_nz, "bev_sel_val": sf.flatten()[sel_nz].numpy(),
            "box_abs": float(pd["box_preds"].double().abs().sum()), "cls_abs": float(pd["cls_preds"].double().abs().sum()),
            "box_sel_idx": box_sel, "box_sel_val": pd["box_preds"].flatten()[box_sel].numpy(),
            "cls_sel_idx": cls_sel, "cls_sel_val": pd["cls_preds"].flatten()[cls_sel].numpy(),
            "anchors_sha1": sha(anchors), "num_anchors": anchors.shape[0],
            "box3d_lidar": out["box3d_lidar"].numpy(), "scores": out["scores"].numpy(),
            "label_preds": out["label_preds"].numpy(), "label_margin": np.array(margins, np.float32),
            "num_pass_threshold": int((top >= b.nms_score_threshold).sum()),
        }
        np.savez_compressed(path, **fix)
        print(NAME, seed, npts, "voxels", res["voxel_num"], "pass", fix["num_pass_threshold"], "dets",
              out["box3d_lidar"].shape[0], "->", os.path.relpath(path, HERE), os.path.getsize(path), "bytes")


def structure(ref, anchors, force):
    path = os.path.join(HERE, "reference", "mhead.json")
    if os.path.exists(path) and not force:
        return
    cfg_path = os.path.join(refcompat.REFERENCE_ROOT, "second", "configs", config.EXTRA_REFERENCE_FILES[NAME])
    parsed = config.ModelConfig.from_file(cfg_path, NAME)
    s = spec.spec_from_module(ref)
    b = config.get_config(NAME)
    H, W = b.grid_size[1], b.grid_size[0]
    out = {
        "config": {"class": type(parsed).__name__,
                   "fields": {f: mrg.as_json(getattr(parsed, f)) for f in parsed.__dataclass_fields__}},
        "state_dict": {k: [list(v.shape), str(v.dtype)] for k, v in ref.state_dict().items()},
        "anchors": [list(anchors.shape), str(anchors.dtype), mrg.sha256(anchors)],
        "spec": mrg.signature_json(s),
        "plan": mrg.plan_digest(tc.plan_rpn_multihead(ref.rpn, dict(s.heads), int(H), int(W))),
    }
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("->", os.path.relpath(path, HERE), os.path.getsize(path), "bytes")


def main():
    refcompat.install(loader.ORACLE_DIR)
    import spconv
    assert getattr(spconv, "__oracle__", False)
    torch.set_num_threads(8)
    force = "--force" in sys.argv
    cfgp = refcompat.load_config(config.EXTRA_REFERENCE_FILES[NAME])
    ref = refcompat.build_network(cfgp.model.second).eval()
    assert type(ref).__name__ == "VoxelNetNuscenesMultiHead"
    models.synthetic_weights_(ref, NAME, seed=0)
    anchors = refcompat.generate_anchors(ref, cfgp.model.second)
    structure(ref, anchors, force)
    fixtures(ref, anchors, force)


if __name__ == "__main__":
    main()
