"""b2second.augment.DeviceDrawer on the GPU (csrc/augment_draws.cu): against the numpy restatement of the generator
contract (tests/augment_draws_ref.py), independent of how frames are split over calls, keyed by the device step
counter (also inside a CUDA graph), distributed as stated, read by augment_batch exactly as host draws are, and drawn
without a host sync."""
import dataclasses

import numpy as np
import pytest
import torch
from scipy import stats

import augment_draws_ref as dr
from b2second import augment, config

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
CONFIGS = ("car.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea")
# normals pass through log, sin and cos, CUDA's against libm's: a relative bound of a few ulp.  Everything else
# (uniforms, flips, scalars, the permutation) is bit-equal.
NORMAL_RTOL = 16 * 2.0 ** -52


def _offsets(counts):
    return torch.tensor(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32), device=DEV)


def _draw(dd, s, gts, pts, frame_base=0):
    return dd.draw(s, _offsets(gts), _offsets(pts), int(sum(gts)), int(sum(pts)), frame_base=frame_base)


def _host(d):
    """device Draws -> host Draws (numpy arrays)"""
    c = lambda t: None if t is None else t.cpu().numpy()   # noqa: E731
    return augment.Draws(c(d.loc_noise), c(d.rot_noise), c(d.frame), c(d.perm), None, None)


def _assert_normals(got, ref, what):
    assert got.shape == ref.shape, what
    err = np.abs(got - ref)
    bad = err > NORMAL_RTOL * np.abs(ref)
    assert not bad.any(), "%s: %d values over %.1e relative, worst %r vs %r" % (
        what, int(bad.sum()), NORMAL_RTOL, got[bad][:3], ref[bad][:3])


def _assert_draws_equal(a, b):
    for k in ("loc_noise", "rot_noise", "frame", "perm"):
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None) == (y is None), k
        if x is not None:
            np.testing.assert_array_equal(x, y, err_msg=k)


@pytest.mark.parametrize("name", CONFIGS)
def test_equals_restatement(name):
    s = config.get_config(name).augment
    gts, pts = [3, 0, 7, 40, 1], [1000, 1, 0, 30000, 17]
    dd = augment.DeviceDrawer(2 ** 63 + 12345, DEV)
    dd.step = 2 ** 40 + 3
    got = _host(_draw(dd, s, gts, pts, frame_base=2 ** 33))
    ref = dr.draws(s, 2 ** 63 + 12345, 2 ** 40 + 3, gts, pts, frame_base=2 ** 33)
    assert dd.step == 2 ** 40 + 4
    for k in ("loc_noise", "rot_noise", "perm"):
        assert (getattr(got, k) is None) == (getattr(ref, k) is None), k
    if ref.loc_noise is not None:
        _assert_normals(got.loc_noise, ref.loc_noise, name + " loc_noise")
        np.testing.assert_array_equal(got.rot_noise, ref.rot_noise)
    np.testing.assert_array_equal(got.frame[:, :5], ref.frame[:, :5])
    _assert_normals(got.frame[:, 5:], ref.frame[:, 5:], name + " translation")
    if ref.perm is not None:
        np.testing.assert_array_equal(got.perm, ref.perm)


def test_translation_equals_restatement():
    """xyres_16 translates; a zero x std with nonzero y keeps the flag and z's use of std[0]"""
    s = dataclasses.replace(config.get_config("pointpillars.car.xyres_16").augment,
                            global_translate_noise_std=[0.0, 0.3, 0.1])
    dd = augment.DeviceDrawer(4, DEV)
    got = _host(_draw(dd, s, [1] * 64, [2] * 64))
    ref = dr.draws(s, 4, 0, [1] * 64, [2] * 64)
    np.testing.assert_array_equal(got.frame[:, :5], ref.frame[:, :5])
    assert (got.frame[:, 2] == 1).all() and not got.frame[:, 5].any() and not got.frame[:, 7].any()
    _assert_normals(got.frame[:, 5:], ref.frame[:, 5:], "translation")


@pytest.mark.parametrize("name", ("car.fhd", "pointpillars.car.xyres_16"))
def test_partition_invariance(name):
    s = config.get_config(name).augment
    gts, pts = [4, 0, 9, 2, 6, 1], [300, 0, 4097, 5, 1000, 16]
    dd = augment.DeviceDrawer(99, DEV)
    dd.step = 7
    whole = _host(_draw(dd, s, gts, pts))
    parts = []
    for base in (0, 3):
        dd.step = 7
        parts.append(_host(_draw(dd, s, gts[base:base + 3], pts[base:base + 3], frame_base=base)))
    joined = augment.Draws(*[None if getattr(parts[0], k) is None else
                             np.concatenate([getattr(p, k) for p in parts])
                             for k in ("loc_noise", "rot_noise", "frame", "perm")], None, None)
    _assert_draws_equal(whole, joined)


def test_step_counter():
    s = config.get_config("car.fhd").augment
    gts, pts = [5, 3], [2000, 700]
    dd = augment.DeviceDrawer(1, DEV)
    a, b = _host(_draw(dd, s, gts, pts)), _host(_draw(dd, s, gts, pts))
    assert dd.step == 2
    for k in ("loc_noise", "rot_noise", "frame", "perm"):
        assert not np.array_equal(getattr(a, k), getattr(b, k)), k
    dd.step = 0
    _assert_draws_equal(a, _host(_draw(dd, s, gts, pts)))
    other = augment.DeviceDrawer(2, DEV)
    assert not np.array_equal(_host(_draw(other, s, gts, pts)).perm, a.perm)


def _batch(name, gts, pts, seed=0):
    """synthetic frames in the config's range: boxes, and half of each frame's points in and around them"""
    cfg = config.get_config(name)
    rng = np.random.default_rng(seed)
    r = np.asarray(cfg.point_cloud_range)
    nus = name.startswith("nuscenes")
    P, Bx = [], []
    for G, n in zip(gts, pts):
        b = np.zeros((G, 9 if nus else 7))
        b[:, :2] = rng.uniform(r[:2] + 2, r[3:5] - 2, (G, 2))
        b[:, 2] = rng.uniform(-2, -1, G)
        b[:, 3:6] = rng.uniform([1.5, 3.5, 1.4], [2.0, 4.6, 1.8], (G, 3))
        b[:, 6] = rng.uniform(-np.pi, np.pi, G)
        if nus:
            b[:, 7:] = rng.normal(0, 3, (G, 2))
        near = b[rng.integers(0, max(G, 1), n // 2)] if G else np.zeros((n // 2, b.shape[1]))
        xyz = np.concatenate([near[:, :3] + rng.uniform(-0.7, 0.7, (n // 2, 3)) * near[:, 3:6],
                              rng.uniform(r[:3], r[3:], (n - n // 2, 3))])
        P.append(np.concatenate([xyz, rng.random((n, cfg.num_point_features - 3))], 1).astype(np.float32))
        Bx.append(b.astype(np.float64 if nus else np.float32))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    G = int(sum(gts))
    plan = augment.plan(cfg.augment, cfg.point_cloud_range, [c.class_name for c in cfg.classes])
    valid = rng.random(G) < 0.9
    args = (t(np.concatenate(P)), _offsets(pts), t(np.concatenate(Bx)), _offsets(gts), t(valid),
            t(rng.integers(1, 3, G).astype(np.int32)), t(rng.random(G).astype(np.float32)))
    return cfg, plan, args


@pytest.mark.parametrize("name", CONFIGS)
def test_augment_batch_reads_device_draws_as_host_draws(name):
    gts, pts = [12, 0, 30, 5], [20000, 10, 25000, 3000]
    cfg, plan, args = _batch(name, gts, pts)
    dd = augment.DeviceDrawer(3, DEV)
    d = _draw(dd, cfg.augment, gts, pts)
    h = _host(d)
    host = augment.Draws(h.loc_noise, h.rot_noise, h.frame, h.perm, gts, pts)
    a = plan.augment_batch(*args, d, with_debug=True)
    b = plan.augment_batch(*args, host, with_debug=True)
    assert int(plan.last_status.item()) == 0
    assert set(a) == set(b) and {"selected", "point_box"} <= set(a)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    if plan.object_noise:
        assert (a["selected"][a["selected"] >= 0]).numel() > 0      # some box moved: the noise was read


def test_cuda_graph_replays_draw_and_augment():
    name, gts, pts, k = "car.fhd", [8, 3, 15], [9000, 400, 12000], 4
    cfg, plan, args = _batch(name, gts, pts, seed=1)
    dd = augment.DeviceDrawer(17, DEV)
    G, P = int(sum(gts)), int(sum(pts))

    def step():
        d = dd.draw(cfg.augment, args[3], args[1], G, P)
        return plan.augment_batch(*args, d, with_debug=True)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    dd.step = 50
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    assert dd.step == 50                                    # capture runs nothing
    replays = []
    for _ in range(k):
        g.replay()
        replays.append({key: v.clone() for key, v in out.items()})
    assert dd.step == 50 + k
    dd.step = 50
    for i in range(k):
        eager = step()
        for key in eager:
            assert torch.equal(eager[key], replays[i][key]), (i, key)
    assert not torch.equal(replays[0]["points"], replays[1]["points"])


def test_distribution():
    """at a fixed seed: normals and uniforms over 10^6 samples each, the flips and the frame uniforms over 50000
    frames, and the shuffle's positions for small frames over many steps"""
    s = dataclasses.replace(config.get_config("car.fhd").augment, groundtruth_localization_noise_std=[1.0, 1.0, 1.0],
                            groundtruth_rotation_uniform_noise=[-0.7, 0.9], global_translate_noise_std=[1.0, 1.0, 0.0],
                            random_flip_x=True, shuffle_points=False)
    dd = augment.DeviceDrawer(20261019, DEV)
    d = _host(_draw(dd, s, [2500] * 4, [0] * 4))
    for c in range(3):
        x = d.loc_noise[..., c].ravel()
        assert x.size >= 10 ** 6
        assert abs(x.mean()) < 5 / np.sqrt(x.size) and abs(x.std() - 1) < 5 / np.sqrt(2 * x.size), c
        assert stats.kstest(x, "norm").pvalue > 1e-3, c
    u = d.rot_noise.ravel()
    assert u.size >= 10 ** 6 and u.min() >= -0.7 and u.max() < 0.9
    assert stats.kstest(u, stats.uniform(-0.7, 1.6).cdf).pvalue > 1e-3

    B = 50000
    f = _host(_draw(dd, s, [0] * B, [0] * B)).frame
    for c in (0, 1):
        assert abs(f[:, c].mean() - 0.5) < 5 * 0.5 / np.sqrt(B), c
    assert abs(np.corrcoef(f[:, 0], f[:, 1])[0, 1]) < 5 / np.sqrt(B)
    lo, hi = s.global_rotation_uniform_noise
    assert stats.kstest(f[:, 3], stats.uniform(lo, hi - lo).cdf).pvalue > 1e-3
    lo, hi = s.global_scaling_uniform_noise
    assert stats.kstest(f[:, 4], stats.uniform(lo, hi - lo).cdf).pvalue > 1e-3
    for c in (5, 6, 7):
        assert stats.kstest(f[:, c], "norm").pvalue > 1e-3, c            # z uses std[0] = 1

    # positions of the shuffle at the frame sizes whose Feistel domain 4^k is the frame itself (no cycle walking).
    # Cycle-walked small frames are not uniform under the 4-round contract (n = 3: 5/16 to 11/32 per position even
    # with ideal round functions; DESIGN section 5), so they are not tested for it here.
    s = dataclasses.replace(s, shuffle_points=True)
    for n in (2, 4, 16):
        frames = 2000
        counts = np.zeros((n, n), np.int64)                                # counts[i, j]: perm[i] == j
        for _ in range(10):
            p = _host(_draw(dd, s, [0] * frames, [n] * frames)).perm.reshape(frames, n)
            np.add.at(counts, (np.broadcast_to(np.arange(n), p.shape), p), 1)
        assert (counts.sum(0) == 10 * frames).all() and (counts.sum(1) == 10 * frames).all()
        # a uniform permutation matrix's cells covary as P (x) P / (n - 1), P = I - J / n: Pearson's statistic over
        # the n x n table is n / (n - 1) times a chi-square of (n - 1)^2 degrees of freedom
        stat = stats.chisquare(counts.ravel()).statistic * (n - 1) / n
        assert stats.chi2.sf(stat, (n - 1) ** 2) > 1e-3, n


def test_draw_makes_no_host_sync():
    s = config.get_config("car.fhd").augment
    gts, pts = [6, 2], [5000, 800]
    goff, poff = _offsets(gts), _offsets(pts)
    dd = augment.DeviceDrawer(8, DEV)
    dd.draw(s, goff, poff, 8, 5800)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            dd.draw(s, goff, poff, 8, 5800, frame_base=5)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert dd.step == 4


def test_refusals_launch_nothing():
    s = config.get_config("car.fhd").augment
    dd = augment.DeviceDrawer(8, DEV)
    dd.step = 5
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        dd.draw(s, torch.tensor([0, 3], dtype=torch.int32), _offsets([10]), 3, 10)
    with pytest.raises(ValueError):
        dd.draw(s, _offsets([3]), _offsets([10, 2]), 3, 12)
    with pytest.raises(ValueError):
        dd.draw(s, _offsets([3]), _offsets([10]), 3, 10, frame_base=-1)
    with pytest.raises(ValueError):
        dd.draw(dataclasses.replace(s, groundtruth_localization_noise_std=[1.0, -1.0, 0.5]), _offsets([3]),
                _offsets([10]), 3, 10)
    assert dd.step == 5
    with pytest.raises(ValueError):
        dd.step = -1
