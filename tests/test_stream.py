"""FastPath.stream on the CPU: what it refuses, it refuses before any engine is built or anything is enqueued."""
import numpy as np
import pytest
import torch

import golden_util as gu
from b2second import config, fastpath, models

NAME = "car.fhd"


@pytest.fixture(scope="module")
def fast(oracle):
    net = models.build_network(config.get_config(NAME), oracle).eval()
    models.synthetic_weights_(net, NAME, seed=0)
    return fastpath.FastPath(net)


def _points_example(net, seed=0):
    return {"points": [torch.from_numpy(gu.make_cloud(NAME, seed, 2000))],
            "anchors": torch.from_numpy(net.anchors()[None]), "metadata": [{"token": "f%d" % seed}]}


def _voxels_example(net):
    res = net.voxel_generator.generate(gu.make_cloud(NAME, 0, 2000), 20000)
    return {"anchors": torch.from_numpy(net.anchors()[None]), "voxels": torch.from_numpy(res["voxels"]),
            "num_points": torch.from_numpy(res["num_points_per_voxel"]),
            "coordinates": torch.from_numpy(np.pad(res["coordinates"], ((0, 0), (1, 0))))}


def _refused(net):
    pts = _points_example(net)
    sweeps = {"sweeps": [{"sweeps": pts["points"], "rotations": [np.eye(3)], "translations": [np.zeros(3)],
                          "time_lags": [0.0]}], "anchors": pts["anchors"]}
    cropped = dict(pts, crop_planes=np.zeros((4, 4)))
    return {"voxels": _voxels_example(net), "sweeps": sweeps, "crop_planes": cropped,
            "no points": {"anchors": pts["anchors"]}}


@pytest.mark.parametrize("kind", ["voxels", "sweeps", "crop_planes", "no points"])
def test_stream_refuses_other_inputs_before_building_an_engine(fast, kind):
    ex = _refused(fast.net)[kind]
    gen = fast.stream([ex])
    with pytest.raises(ValueError, match="'points'"):
        next(gen)
    assert fast.engines == {}
    with pytest.raises(StopIteration):     # the generator has finished
        next(gen)


def test_stream_refuses_a_network_in_train_mode(fast):
    fast.net.train()
    try:
        with pytest.raises(RuntimeError, match="eval"):
            next(fast.stream([_points_example(fast.net)]))
    finally:
        fast.net.eval()
    assert fast.engines == {}


def test_stream_is_lazy(fast):
    """nothing is taken from the iterable, checked or built before the first result is asked for"""
    taken = []

    def examples():
        taken.append(1)
        yield _refused(fast.net)["voxels"]

    gen = fast.stream(examples())
    assert taken == [] and fast.engines == {}
    with pytest.raises(ValueError):
        next(gen)
    assert taken == [1]
