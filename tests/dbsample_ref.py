"""The database-sampling fixtures (tests/golden/make_dbsample_golden.py): loading, the synthetic database they record
rebuilt as a db_infos dict with its ``.bin`` files, and the mapping from the fixtures' info ids to b2second.dbsample's
object ids."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "second.pytorch_b200"))

from b2second import config, dbsample  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "dbsample")
CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"]


def class_names(name):
    return [c.class_name for c in config.get_config(name).classes]


def load_fixture(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    frames = []
    for f in range(int(z["num_frames"])):
        frames.append({k[:-len("_%d" % f)]: z[k] for k in z.files if k.endswith("_%d" % f)})
    return z, frames


def db_infos(z):
    """the recorded database as the reference's db_infos dict (keys in the recorded order)"""
    infos = {str(k): [] for k in z["db_keys"]}
    for uid in range(len(z["db_key"])):
        infos[str(z["db_key"][uid])].append({
            "name": str(z["db_name"][uid]), "path": str(z["db_path"][uid]), "box3d_lidar": z["db_box"][uid].copy(),
            "difficulty": int(z["db_difficulty"][uid]), "num_points_in_gt": int(z["db_npig"][uid]), "uid": uid})
    return infos


def write_bins(z, root):
    off = z["db_point_off"]
    for uid, path in enumerate(z["db_path"]):
        z["db_points"][off[uid]:off[uid + 1]].tofile(os.path.join(root, str(path)))


def load_db(name, z, root, device):
    """-> (Database, uid -> object id)"""
    write_bins(z, root)
    cfg = config.get_config(name)
    db = dbsample.load(cfg.db_sampler, db_infos(z), root, cfg.num_point_features, class_names(name), device)
    by_path = {p: i for i, p in enumerate(db.paths)}
    return db, {uid: by_path[str(p)] for uid, p in enumerate(z["db_path"]) if str(p) in by_path}


def frame_inputs(fr):
    """the frame as sample_all sees it: DontCare rows dropped (preprocess.py:191)"""
    names = fr["in_names"]
    keep = names != "DontCare"
    return fr["in_points"], np.ascontiguousarray(fr["in_boxes"][keep]), names[keep]


def candidates(name, z, frames, uid2obj):
    """the recorded candidates of ``frames`` as a dbsample.Candidates batch"""
    groups = [n for n, _ in dbsample.sampled_classes(config.get_config(name).db_sampler)]
    objs, grp, offs = [], [], [0]
    for fr in frames:
        for u in fr["cand"]:
            objs.append(uid2obj[int(u)])
            grp.append(groups.index(str(z["db_key"][int(u)])))
        offs.append(len(objs))
    return dbsample.Candidates(objects=np.array(objs, np.int32), group=np.array(grp, np.int32),
                               offsets=np.array(offs, np.int32))
