"""Ground-truth database sampling on the host: the parsed settings against the builtins, the prep filters and the
sampler bookkeeping of b2second.dbsample against the fixtures the unmodified reference produced
(tests/golden/make_dbsample_golden.py), the stream order of the batch path, and the settings it refuses."""
import copy
import os

import numpy as np
import pytest

import augment_ref as ar
import dbsample_ref as dr
from b2second import augment, config, dbsample, refcompat, spec


@pytest.mark.skipif(not refcompat.reference_available(), reason="needs the reference's config files")
@pytest.mark.parametrize("name", sorted(config.DB_SAMPLERS))
def test_parsed_settings_equal_builtins(name):
    rel = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    cfg = config.ModelConfig.from_file(os.path.join(refcompat.REFERENCE_ROOT, "second", "configs", rel))
    assert cfg.db_sampler == config.get_config(name).db_sampler


def test_settings_parse_from_prototxt():
    text = """
    model { second { voxel_generator { point_cloud_range: [0, -40, -3, 70.4, 40, 1] voxel_size: [0.05, 0.05, 0.1]
      max_number_of_points_per_voxel: 5 } voxel_feature_extractor { module_class_name: "SimpleVoxel" }
      middle_feature_extractor { module_class_name: "SpMiddleFHD" }
      rpn { module_class_name: "RPNV2" layer_nums: [5] layer_strides: [1] num_filters: [128] upsample_strides: [1]
            num_upsample_filters: [128] num_input_features: 128 }
      target_assigner { class_settings { class_name: "Car" anchor_generator_range { sizes: [1.6, 3.9, 1.56]
        rotations: [0, 1.57] anchor_ranges: [0, -40, -1, 70.4, 40, -1] } matched_threshold: 0.6
        unmatched_threshold: 0.45 } } } }
    train_input_reader { preprocess {
      remove_points_after_sample: true
      sample_importance: 0.5
      database_sampler {
        database_info_path: "/data/dbinfos.pkl"
        sample_groups { name_to_max_num { key: "Car" value: 12 } }
        sample_groups { name_to_max_num { key: "Van" value: 3 } }
        database_prep_steps { filter_by_difficulty { removed_difficulties: [-1, 3] } }
        database_prep_steps { filter_by_min_num_points { min_num_point_pairs { key: "Car" value: 5 }
                                                         min_num_point_pairs { key: "Van" value: 0 } } }
        global_random_rotation_range_per_object: [0, 0]
        rate: 0.7
      } } }
    """
    s = config.ModelConfig.from_prototxt(text).db_sampler
    assert s.sample_groups == [{"Car": 12}, {"Van": 3}]
    assert s.database_prep_steps == [("filter_by_difficulty", [-1, 3]),
                                     ("filter_by_min_num_points", [("Car", 5), ("Van", 0)])]
    assert s.rate == float(np.float32(0.7)) and s.sample_importance == 0.5
    assert s.remove_points_after_sample and s.database_info_path == "/data/dbinfos.pkl"
    assert s.global_random_rotation_range_per_object == [0.0, 0.0]
    assert config.ModelConfig.from_prototxt(text.replace("database_sampler", "unused_block")).db_sampler is None


@pytest.mark.parametrize("name", dr.CONFIGS)
def test_prep_filters_equal_reference(name):
    z, _ = dr.load_fixture(name)
    infos = dr.db_infos(z)
    before = copy.deepcopy(infos)
    got = dbsample.prep_infos(config.get_config(name).db_sampler, infos)
    assert list(got) == [str(k) for k in z["db_keys"]]
    off = z["filt_off"]
    for k, key in enumerate(got):
        np.testing.assert_array_equal([i["uid"] for i in got[key]], z["filt_uid"][off[k]:off[k + 1]], err_msg=key)
    assert [len(v) for v in infos.values()] == [len(v) for v in before.values()]     # the caller's dict is untouched
    steps = config.get_config(name).db_sampler.database_prep_steps
    assert 0 < len(z["filt_uid"]) and (len(z["filt_uid"]) < len(z["db_key"])) == bool(steps)


def _cpu_db(name, z, tmp_path):
    return dr.load_db(name, z, str(tmp_path), "cpu")


@pytest.mark.parametrize("name", dr.CONFIGS)
def test_host_sampler_equals_reference(name, tmp_path):
    """the samplers' construction and every frame's candidates, index for index, and the stream after each frame"""
    z, frames = dr.load_fixture(name)
    cfg = config.get_config(name)
    db, uid2obj = _cpu_db(name, z, tmp_path)
    rs0 = np.random.RandomState(int(z["seed_init"]))
    state = dbsample.SamplerState(rs0, db, cfg.db_sampler)
    assert ar.state_digest(rs0) == str(z["state_init"])
    assert list(state.indices) == [str(k) for k in z["db_keys"]]
    wrapped = False
    for f, fr in enumerate(frames):
        _, boxes, names = dr.frame_inputs(fr)
        rs = np.random.RandomState(int(fr["seed"]))
        idx_before = dict(state.idx)
        want_req = [n for n in dbsample.sample_counts(state, names) if n > 0]
        cand = dbsample.draw(rs, state, [names])
        np.testing.assert_array_equal(cand.objects, [uid2obj[int(u)] for u in fr["cand"]], err_msg="frame %d" % f)
        np.testing.assert_array_equal(want_req, fr["requested"])
        wrapped |= any(state.idx[k] < idx_before[k] or (state.idx[k] == 0 and idx_before[k] == 0 and want_req)
                       for k in state.idx)
        if "chain_points" in fr:
            augment.draw(rs, cfg.augment, [len(fr["out_boxes"])], [len(fr["out_points"])])
        assert ar.state_digest(rs) == str(fr["state"]), "frame %d (%s)" % (f, fr["kind"])
    assert wrapped


@pytest.mark.parametrize("name", dr.CONFIGS)
def test_sample_counts_round_half_even(name, tmp_path):
    z, _ = dr.load_fixture(name)
    db, _ = _cpu_db(name, z, tmp_path)
    s = copy.deepcopy(config.get_config(name).db_sampler)
    first = next(iter(s.sample_groups[0]))
    rows = z["rate_table"]
    assert (np.abs(np.remainder(rows[:, 0] * (s.sample_groups[0][first] - rows[:, 1]), 1) - 0.5) < 1e-9).any()
    for rate, k, req in rows:
        s.rate = float(rate)
        state = dbsample.SamplerState(np.random.RandomState(0), db, s)
        assert max(dbsample.sample_counts(state, [first] * int(k))[0], 0) == int(req), (rate, k)


def _pair_draws(name, db, names_pair, interleaved):
    """sampler and augmentation draws of two frames on one state, frame by frame or the batch path's order"""
    cfg = config.get_config(name)
    rs = np.random.RandomState(5)
    state = dbsample.SamplerState(rs, db, cfg.db_sampler)
    n_pts = [100, 120]
    if interleaved:
        cands, augs = [], []
        for names, npts in zip(names_pair, n_pts):
            cands.append(dbsample.draw(rs, state, [names]).objects)
            augs.append(augment.draw(rs, cfg.augment, [len(names) + len(cands[-1])], [npts]).frame)
        return list(np.concatenate(cands)), np.concatenate(augs), state
    c = dbsample.draw(rs, state, names_pair)
    n_c = np.diff(c.offsets)
    return list(c.objects), augment.draw(rs, cfg.augment, [len(n) + k for n, k in zip(names_pair, n_c)], n_pts).frame, \
        state


def test_batch_stream_order_equals_reference_without_a_later_wrap(tmp_path):
    name = "car.fhd"
    z, _ = dr.load_fixture(name)
    db, _ = _cpu_db(name, z, tmp_path)
    pair = [["Car"] * 14, ["Car"] * 13]                     # one and two candidates: no sampler wraps
    c0, a0, s0 = _pair_draws(name, db, pair, True)
    c1, a1, s1 = _pair_draws(name, db, pair, False)
    assert c0 == c1
    np.testing.assert_array_equal(a0, a1)
    assert all(np.array_equal(s0.indices[k], s1.indices[k]) for k in s0.indices)


def test_batch_stream_order_differs_after_a_wrap_in_a_later_frame(tmp_path):
    """the second frame's sampler wraps: its reshuffle comes before the first frame's augmentation draws"""
    name = "car.fhd"
    z, _ = dr.load_fixture(name)
    db, _ = _cpu_db(name, z, tmp_path)
    assert 15 < db.counts["Car"] <= 30
    pair = [[], []]                                         # fifteen candidates each: the second one wraps
    c0, a0, s0 = _pair_draws(name, db, pair, True)
    c1, a1, s1 = _pair_draws(name, db, pair, False)
    assert c0 == c1                                         # the wrap returns the remainder drawn before it
    assert s0.idx["Car"] == 0 and s1.idx["Car"] == 0
    assert not np.array_equal(a0, a1)
    assert not np.array_equal(s0.indices["Car"], s1.indices["Car"])


def _settings(edit):
    s = copy.deepcopy(config.get_config("all.fhd").db_sampler)
    edit(s)
    return s


@pytest.mark.parametrize("edit,what", [
    (lambda s: setattr(s, "sample_groups", [{"Car": 10, "Van": 2}]), "group sampling"),
    (lambda s: setattr(s, "global_random_rotation_range_per_object", [0.78, 2.35]), "per-object rotation"),
    (lambda s: setattr(s, "sample_groups", [{"Car": 10}, {"Truck": 2}]), "class outside class_names"),
])
def test_unsupported_settings_are_refused(edit, what, tmp_path):
    z, _ = dr.load_fixture("all.fhd")
    db, _ = _cpu_db("all.fhd", z, tmp_path)
    with pytest.raises(spec.UnsupportedNetwork):
        dbsample.DatabaseSampler(db, _settings(edit), dr.class_names("all.fhd"))


def test_random_crop_is_refused(tmp_path):
    z, _ = dr.load_fixture("car.fhd")
    db, _ = _cpu_db("car.fhd", z, tmp_path)
    ds = dbsample.DatabaseSampler(db, config.get_config("car.fhd").db_sampler, ["Car"], np.random.RandomState(0))
    with pytest.raises(spec.UnsupportedNetwork):
        ds.sample_all(str(tmp_path), np.zeros((0, 7), np.float32), [], 4, random_crop=True)


def test_narrow_per_object_rotation_range_is_accepted(tmp_path):
    z, _ = dr.load_fixture("all.fhd")
    db, _ = _cpu_db("all.fhd", z, tmp_path)
    dbsample.DatabaseSampler(db, _settings(lambda s: setattr(s, "global_random_rotation_range_per_object",
                                                             [0.5, 0.5005])), dr.class_names("all.fhd"))


def test_database_load_reads_sampled_classes_once(tmp_path):
    z, _ = dr.load_fixture("nuscenes.all.pp.mhead")
    db, uid2obj = _cpu_db("nuscenes.all.pp.mhead", z, tmp_path)
    assert sorted(db.objects) == ["bus", "trailer", "truck"]
    assert db.num_objects == sum(db.counts[k] for k in ("bus", "trailer", "truck"))
    assert db.boxes.dtype == __import__("torch").float64 and db.boxes.shape[1] == 9
    off = z["db_point_off"]
    for uid, obj in uid2obj.items():
        o0, o1 = db.point_offsets_host[obj], db.point_offsets_host[obj + 1]
        np.testing.assert_array_equal(db.points[o0:o1].numpy(), z["db_points"][off[uid]:off[uid + 1]])
        np.testing.assert_array_equal(db.boxes_host[obj], z["db_box"][uid])
    assert db.nbytes == db.points.numel() * 4 + db.point_offsets.numel() * 8 + db.boxes.numel() * 8 + \
        db.classes.numel() * 4 + db.difficulty.numel() * 4
