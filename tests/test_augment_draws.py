"""Device draws of the training augmentation on the host: tests/augment_draws_ref.py (the generator contract restated in
numpy) against numpy.random.Philox, its keyed permutation, and b2second.augment.DeviceDrawer's settings vocabulary and
refusals against ``draw``'s."""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch

import augment_draws_ref as dr
from b2second import augment, config, spec

M64 = 2 ** 64 - 1
CONFIGS = ("car.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea")


@pytest.mark.parametrize("seed,step,counter", [
    (0, 0, (0, 0, 0, 0)), (123, 7, (5, 2, 300, 0)), (M64, M64, (M64, M64, M64, M64)),
    (1, 2, (0, 1, 0, 0)),                                 # counter - 1 borrows from word 1 into word 0
    (9, 1, (0, 0, 1, 0)), (2 ** 63, 3, (M64, 0, 0, 5)), (5, 0, (7, 3, 4095, 255))])
def test_philox_equals_numpy(seed, step, counter):
    c = sum(w << (64 * i) for i, w in enumerate(counter))
    bg = np.random.Philox(key=seed | step << 64, counter=(c - 1) % 2 ** 256)   # numpy increments before each block
    raw = bg.random_raw(8)
    first = np.array([w[0] for w in dr.philox((seed, step), counter)], dtype=np.uint64)
    np.testing.assert_array_equal(first, raw[:4])
    nxt = sum(w << (64 * i) for i, w in enumerate(counter)) + 1
    words = [(nxt >> (64 * i)) & M64 for i in range(4)]                   # the next counter, with its carries
    np.testing.assert_array_equal(np.array([w[0] for w in dr.philox((seed, step), words)], dtype=np.uint64), raw[4:])


def test_philox_broadcasts_over_indices():
    idx = np.arange(50, dtype=np.uint64)
    w = dr.philox((3, 4), (1, 0, idx, 0))
    for i in (0, 17, 49):
        np.testing.assert_array_equal([v[i] for v in w], [v[0] for v in dr.philox((3, 4), (1, 0, i, 0))])


def test_uniform_and_normal_mappings():
    w = np.array([0, 2 ** 11 - 1, 2 ** 11, M64], dtype=np.uint64)
    np.testing.assert_array_equal(dr.uniform01(w), [0.0, 0.0, 2.0 ** -53, 1.0 - 2.0 ** -53])
    bg = np.random.Generator(np.random.Philox(key=5))
    raw = np.random.Philox(key=5).random_raw(4)
    np.testing.assert_array_equal(dr.uniform01(raw), bg.random(4))               # numpy's 53-bit doubles
    n0, n1 = dr.box_muller(np.array([M64 >> 1], np.uint64), np.array([M64 >> 2], np.uint64))
    r = np.sqrt(-2.0 * np.log(1.0 - dr.uniform01(np.uint64(M64 >> 1))))
    t = 2 * np.pi * dr.uniform01(np.uint64(M64 >> 2))
    assert n0[0] == r * np.cos(t) and n1[0] == r * np.sin(t)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5, 15, 16, 17, 1000, 4097, 30000])
def test_permutation_is_a_bijection(n):
    p = dr.permutation((11, 2), 3, n)
    assert p.dtype == np.int32 and p.shape == (n,)
    np.testing.assert_array_equal(np.sort(p), np.arange(n))
    if n <= 1:
        np.testing.assert_array_equal(p, np.arange(n))
    assert 4 ** dr.feistel_bits(n) >= n and (dr.feistel_bits(n) == 1 or 4 ** (dr.feistel_bits(n) - 1) < n)


def test_permutation_depends_on_key_and_frame():
    base = dr.permutation((1, 0), 0, 1000)
    assert not np.array_equal(base, dr.permutation((1, 1), 0, 1000))
    assert not np.array_equal(base, dr.permutation((2, 0), 0, 1000))
    assert not np.array_equal(base, dr.permutation((1, 0), 1, 1000))
    np.testing.assert_array_equal(base, dr.permutation((1, 0), 0, 1000))


def _settings(name, **kw):
    return dataclasses.replace(config.get_config(name).augment, **kw)


VARIANTS = [(name, {}) for name in CONFIGS] + [
    ("car.fhd", {"shuffle_points": False}),
    ("car.fhd", {"global_translate_noise_std": [0.0, 0.3, 0.0]}),
    ("car.fhd", {"global_translate_noise_std": []}),
    ("pointpillars.car.xyres_16", {"groundtruth_localization_noise_std": [0.0, 0.0, 0.0],
                                   "groundtruth_rotation_uniform_noise": [0.0, 0.0]}),
    ("nuscenes.all.pp.largea", {"groundtruth_rotation_uniform_noise": [-0.1, 0.1], "random_flip_x": False})]


@pytest.mark.parametrize("name,kw", VARIANTS)
def test_vocabulary_matches_draw(name, kw):
    """the restated device draws hold what ``draw`` holds: no loc_noise with the object noise off, no perm without
    shuffle_points, the translate flag 0 with zero std, flips only where the settings allow them, the same shapes"""
    s = _settings(name, **kw)
    counts, npts = [3, 0, 2], [5, 1, 7]
    host = augment.draw(np.random.RandomState(0), s, counts, npts)
    dev = dr.draws(s, 7, 3, counts, npts)
    p = augment.draw_params(s)
    for k in ("loc_noise", "rot_noise", "perm"):
        a, b = getattr(host, k), getattr(dev, k)
        assert (a is None) == (b is None), k
        if a is not None:
            assert a.shape == b.shape and a.dtype == b.dtype, k
    assert bool(p.object_noise) == (host.loc_noise is not None)
    assert host.frame.shape == dev.frame.shape
    np.testing.assert_array_equal(dev.frame[:, 2], host.frame[:, 2])
    if not s.random_flip_x:
        assert not dev.frame[:, 1].any()
    if not s.random_flip_y:
        assert not dev.frame[:, 0].any()
    if not dev.frame[0, 2]:
        assert not dev.frame[:, 5:].any()
    lo, hi = s.global_scaling_uniform_noise
    assert ((dev.frame[:, 4] >= lo) & (dev.frame[:, 4] <= hi)).all()


@pytest.mark.parametrize("kw", [{"groundtruth_localization_noise_std": [1.0, -0.5, 0.5]},
                                {"global_translate_noise_std": [0.2, -0.2, 0.2]},
                                {"global_translate_noise_std": [-0.2, 0.2, 0.2]}])
def test_negative_std_refused_like_draw(kw):
    s = _settings("pointpillars.car.xyres_16", **kw)
    with pytest.raises(ValueError):
        augment.draw(np.random.RandomState(0), s, [2], [3])
    with pytest.raises(ValueError, match=">= 0"):
        augment.draw_params(s)


def test_unused_translate_z_std_accepted_like_draw():
    """global_translate_ draws z with std[0]: std[2] only turns the translation on, for ``draw`` and the device"""
    s = _settings("pointpillars.car.xyres_16", global_translate_noise_std=[0.2, 0.2, -0.2])
    host = augment.draw(np.random.RandomState(0), s, [2], [3])
    assert augment.draw_params(s).translate_std[2] == -0.2
    assert host.frame[0, 2] == 1.0 and dr.draws(s, 1, 0, [2], [3]).frame[0, 2] == 1.0


@pytest.mark.parametrize("kw,err", [
    ({"global_random_rotation_range_per_object": [0.0, 0.5]}, spec.UnsupportedNetwork),
    ({"use_group_id": True}, spec.UnsupportedNetwork),
    ({"groundtruth_localization_noise_std": [1.0, 1.0]}, ValueError),
    ({"global_scaling_uniform_noise": [0.95, float("inf")]}, ValueError)])
def test_settings_refused_like_plan(kw, err):
    s = _settings("car.fhd", **kw)
    with pytest.raises(err):
        augment.draw_params(s)


def test_drawer_arguments_refused_without_a_device():
    with pytest.raises(ValueError, match="CUDA device"):
        augment.DeviceDrawer(0, "cpu")
    with pytest.raises(ValueError, match="seed"):
        augment.DeviceDrawer(-1, "cuda:0")
    with pytest.raises(ValueError, match="seed"):
        augment.DeviceDrawer(2 ** 64, "cuda:0")


def test_select_refuses_device_draws():
    d = augment.Draws(loc_noise=None, rot_noise=None, frame=torch.zeros(2, 8, dtype=torch.float64), perm=None,
                      num_gt=None, num_points=None)
    with pytest.raises(ValueError, match="frame_base"):
        augment.select(d, 0, 1)


def test_abi_argument_checks_run_before_any_cuda_call():
    from spconv import _lib
    lib = _lib.load()
    dummy = ctypes.c_void_p(256)                      # never dereferenced: every call below fails its argument check
    p = augment.draw_params(config.get_config("car.fhd").augment)

    def call(batch=2, G=4, P=10, loc=dummy, frame=dummy, base=0):
        return lib.b2s_augment_draws(1, dummy, base, batch, dummy, G, dummy, P, ctypes.byref(p), loc, dummy, frame,
                                     dummy, None)
    assert call(batch=0) == -2 and b"batch" in lib.b2s_last_error()
    assert call(G=-1) == -2
    assert call(loc=None) == -2 and b"loc_noise" in lib.b2s_last_error()
    assert call(frame=None) == -2
    assert call(base=M64) == -2 and b"frame_base" in lib.b2s_last_error()
