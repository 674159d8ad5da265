"""Training augmentation on the host: tests/augment_ref.py (a numpy restatement of csrc/augment.cu) against the fixtures
the unmodified reference produced (tests/golden/make_augment_golden.py), b2second.augment.draw against the reference's
use of the random stream, the parsed settings against the builtins, and the settings b2second.augment refuses."""
import copy
import os

import numpy as np
import pytest

import augment_ref as ar
from b2second import augment, config, refcompat, spec


def _frame_inputs(name, fr):
    pts, boxes, names = ar.frame(name, str(fr["kind"]), int(fr["seed"]))
    valid, cls = ar.class_mask(name, names)
    return pts, boxes, names, valid, cls


@pytest.mark.parametrize("name", ar.CONFIGS)
def test_restatement_equals_reference(name):
    _, frames = ar.load_fixture(name)
    cfg = config.get_config(name)
    plan = augment.plan(cfg.augment, cfg.point_cloud_range, ar.class_names(name))
    for f, fr in enumerate(frames):
        pts, boxes, names, valid, cls = _frame_inputs(name, fr)
        rs = np.random.RandomState(int(fr["seed"]))
        d = augment.draw(rs, cfg.augment, [len(boxes)], [len(pts)])
        got = ar.augment(plan, pts, boxes, valid, cls, None, d)
        ar.compare(got, fr, "%s frame %d (%s)" % (name, f, fr["kind"]))


@pytest.mark.parametrize("name", ar.CONFIGS)
def test_draw_consumes_the_stream_as_the_reference(name):
    _, frames = ar.load_fixture(name)
    cfg = config.get_config(name)
    for fr in frames:
        pts, boxes, _, _, _ = _frame_inputs(name, fr)
        rs = np.random.RandomState(int(fr["seed"]))
        augment.draw(rs, cfg.augment, [len(boxes)], [len(pts)])
        assert ar.state_digest(rs) == str(fr["state"]), fr["kind"]


def test_draw_arrays_follow_the_reference_calls():
    """the same arrays the reference's np.random calls give, frame after frame on one state"""
    s = config.get_config("pointpillars.car.xyres_16").augment
    d = augment.draw(np.random.RandomState(11), s, [3, 0, 2], [5, 4, 6])
    rs = np.random.RandomState(11)
    for f, (n, npts) in enumerate([(3, 5), (0, 4), (2, 6)]):
        g0 = [0, 3, 3][f]
        np.testing.assert_array_equal(rs.normal(scale=np.array(s.groundtruth_localization_noise_std, np.float32),
                                                size=[n, 100, 3]), d.loc_noise[g0:g0 + n])
        np.testing.assert_array_equal(rs.uniform(*s.groundtruth_rotation_uniform_noise, size=[n, 100]),
                                      d.rot_noise[g0:g0 + n])
        rs.uniform(0, 0, size=[n, 100])
        fx = rs.choice([False, True], replace=False, p=[0.5, 0.5])
        fy = rs.choice([False, True], replace=False, p=[0.5, 0.5])
        assert d.frame[f, 0] == float(fy) and d.frame[f, 1] == 0.0        # random_flip_x is false for xyres_16
        assert fx in (False, True)
        assert d.frame[f, 3] == rs.uniform(*s.global_rotation_uniform_noise)
        assert d.frame[f, 4] == rs.uniform(*s.global_scaling_uniform_noise)
        ts = s.global_translate_noise_std          # z uses std[0], as global_translate_ does
        t = [rs.normal(0, ts[0], 1)[0], rs.normal(0, ts[1], 1)[0], rs.normal(0, ts[0], 1)[0]]
        np.testing.assert_array_equal(d.frame[f, 5:8], t)
        p = np.arange(npts)
        rs.shuffle(p)
        p0 = [0, 5, 9][f]
        np.testing.assert_array_equal(d.perm[p0:p0 + npts], p)


def test_early_return_draws_no_object_noise():
    s = config.get_config("nuscenes.all.pp.largea").augment
    assert not augment.object_noise_enabled(s)
    d = augment.draw(np.random.RandomState(3), s, [4], [10])
    assert d.loc_noise is None and d.rot_noise is None and d.perm is None
    rs = np.random.RandomState(3)
    rs.choice([False, True], replace=False, p=[0.5, 0.5])
    rs.choice([False, True], replace=False, p=[0.5, 0.5])
    rs.uniform(0, 0)
    rs.uniform(1, 1)
    r2 = np.random.RandomState(3)
    augment.draw(r2, s, [4], [10])
    assert ar.state_digest(r2) == ar.state_digest(rs)


@pytest.mark.skipif(not refcompat.reference_available(), reason="needs the reference's config files")
@pytest.mark.parametrize("name", sorted(config.AUGMENTS))
def test_parsed_settings_equal_builtins(name):
    rel = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    cfg = config.ModelConfig.from_file(os.path.join(refcompat.REFERENCE_ROOT, "second", "configs", rel))
    assert cfg.augment == config.get_config(name).augment


def _settings(edit):
    s = copy.deepcopy(config.get_config("car.fhd").augment)
    edit(s)
    return s


@pytest.mark.parametrize("edit,what", [
    (lambda s: setattr(s, "global_random_rotation_range_per_object", [0.78, 2.35]), "per-object global rotation"),
    (lambda s: setattr(s, "use_group_id", True), "use_group_id"),
])
def test_unsupported_settings_are_refused(edit, what):
    cfg = config.get_config("car.fhd")
    with pytest.raises(spec.UnsupportedNetwork):
        augment.plan(_settings(edit), cfg.point_cloud_range, ["Car"])


def test_narrow_per_object_rotation_range_is_accepted():
    """noise_per_object_v3_ only enables the per-object rotation from a width of 1e-3"""
    cfg = config.get_config("car.fhd")
    augment.plan(_settings(lambda s: setattr(s, "global_random_rotation_range_per_object", [0.5, 0.5005])),
                 cfg.point_cloud_range, ["Car"])
