"""FastPath staleness on the CPU: eval() / train(False) and load_state_dict mark the fast path stale, a plain call does
no refresh work, the modes train() / eval() set on the network's children are those of an unaccelerated network, and a
refresh refuses a network whose structure or device changed.  No engine is built: the fast path's engines are stand-ins
that record what they are asked to do."""
import pytest
import torch
from torch import nn

import golden_util as gu
from b2second import config, fastpath, models, spec

NAMES = ["car.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"]
B = 2


class _Engine:
    """records what the fast path asks of an engine"""

    def __init__(self):
        self.calls = []

    def set_anchors(self, anchors):
        pass

    def set_anchors_mask(self, mask):
        pass

    def infer(self, frames):
        self.calls.append("infer")

    def detections(self, metadata=None, output="device"):
        return [{} for _ in range(B)]

    def refresh(self):
        self.calls.append("refresh")


def _net(oracle, name, seed=0):
    net = models.build_network(config.get_config(name), oracle).eval()
    return models.synthetic_weights_(net, name, seed=seed)


def _accelerated(oracle, name):
    net = fastpath.accelerate(_net(oracle, name))
    eng = _Engine()
    net.b2s_fastpath.engines[B] = eng
    return net, net.b2s_fastpath, eng


def _example(net, name):
    return {"points": [torch.from_numpy(gu.make_cloud(name, s, 1000)) for s in range(B)],
            "anchors": torch.from_numpy(net.anchors()[None])}


@pytest.mark.parametrize("name", NAMES)
def test_eval_and_load_state_dict_mark_stale(oracle, name):
    net, fast, eng = _accelerated(oracle, name)
    assert not fast.stale and fast.refreshes == 0
    net.train()
    assert not fast.stale, "train(True) does not mark"
    assert net.eval() is net
    assert fast.stale
    net(_example(net, name))
    assert not fast.stale and fast.refreshes == 1 and eng.calls == ["refresh", "infer"]
    net.train(False)
    assert fast.stale
    fast.refresh()
    assert not fast.stale and fast.refreshes == 2
    net.load_state_dict(_net(oracle, name, seed=1).state_dict())
    assert fast.stale
    fast.refresh()
    assert fast.refreshes == 3 and eng.calls == ["refresh", "infer", "refresh", "refresh"]


def test_refresh_re_reads_the_weights(oracle):
    """the spec holds what a newly read spec of the loaded network holds"""
    name = "car.fhd"
    net, fast, _ = _accelerated(oracle, name)
    other = _net(oracle, name, seed=1)
    before = fast.spec.signature()
    net.load_state_dict(other.state_dict())
    fast.refresh()
    after = fast.spec.signature()
    assert after != before
    assert after == spec.spec_from_module(other).signature()


@pytest.mark.parametrize("name", NAMES)
def test_a_plain_call_does_no_refresh_work(oracle, name, monkeypatch):
    net, fast, eng = _accelerated(oracle, name)
    monkeypatch.setattr(spec, "refresh", lambda *a: pytest.fail("refresh on a call that is not stale"))
    ex = _example(net, name)
    for _ in range(3):
        net(ex)
    assert not fast.stale and fast.refreshes == 0 and eng.calls == ["infer"] * 3


def _modes(net):
    return [(n, m.training) for n, m in net.named_modules()]


def test_child_modes_are_those_of_an_unaccelerated_network(oracle):
    name = "car.fhd"
    plain = _net(oracle, name)
    net = fastpath.accelerate(_net(oracle, name))
    steps = [lambda n: n.train(), lambda n: n.rpn.eval(), lambda n: n.train(False), lambda n: n.middle_feature_extractor.train(),
             lambda n: n.eval(), lambda n: n.train(True), lambda n: n.rpn.blocks[0].train(False)]
    for k, step in enumerate(steps):
        assert step(plain) is not None and step(net) is not None
        assert _modes(net) == _modes(plain), "step %d" % k
    assert all(m.training for n, m in net.named_modules() if not n.startswith("rpn.blocks.0"))


def test_accelerate_stays_idempotent(oracle):
    net = fastpath.accelerate(_net(oracle, "car.fhd"))
    fast, train = net.b2s_fastpath, net.train
    assert fastpath.accelerate(net) is net and net.b2s_fastpath is fast and net.train is train
    net.eval()
    assert fast.stale




@pytest.mark.parametrize("change", ["head", "sparse", "pfn", "small_head", "device"])
def test_refresh_refuses_a_changed_structure(oracle, change):
    name = {"sparse": "car.fhd", "pfn": "pointpillars.car.xyres_16", "small_head": "nuscenes.all.pp.mhead"}.get(
        change, "car.fhd")
    net, fast, eng = _accelerated(oracle, name)
    ex = _example(net, name)
    held = (fast.spec.layers, fast.spec.pfn, fast.spec.rpn, fast.spec.heads)
    if change == "head":
        old = net.rpn.conv_cls
        net.rpn.conv_cls = nn.Conv2d(old.in_channels, old.out_channels + 2, 1)
        match = "structure changed.*rpn"
    elif change == "sparse":
        conv = net.middle_feature_extractor.middle_conv[0]
        conv.weight = nn.Parameter(torch.zeros(*conv.weight.shape[:-1], conv.weight.shape[-1] * 2))
        conv.out_channels *= 2
        match = "structure changed.*layers"
    elif change == "pfn":
        lin = net.voxel_feature_extractor.pfn_layers[0].linear
        lin.weight = nn.Parameter(torch.zeros(lin.weight.shape[0], lin.weight.shape[1] + 1))
        match = "structure changed"
    elif change == "small_head":
        net.small_head.net = nn.Sequential(*list(net.small_head.net.children())[:3])
        match = "structure changed.*heads"
    else:
        bn = next(m for m in net.rpn.modules() if isinstance(m, nn.BatchNorm2d))
        bn.to("meta")
        match = "no longer on"
    net.eval()
    for _ in range(2):          # the fast path stays stale: every call raises, nothing is served
        with pytest.raises(spec.UnsupportedNetwork, match=match):
            net(ex)
        assert fast.stale
    with pytest.raises(spec.UnsupportedNetwork, match=match):
        fast.refresh()
    assert eng.calls == [] and fast.refreshes == 0
    assert (fast.spec.layers, fast.spec.pfn, fast.spec.rpn, fast.spec.heads) == held, "a refused refresh leaves the spec"


def test_engines_are_refreshed_in_place_of_a_rebuild(oracle):
    """refresh asks every engine built so far to refresh; none is rebuilt or dropped"""
    net, fast, eng = _accelerated(oracle, "car.fhd")
    other = _Engine()
    fast.engines[B + 2] = other
    net.eval()
    fast.refresh()
    assert fast.engines == {B: eng, B + 2: other}
    assert eng.calls == ["refresh"] and other.calls == ["refresh"]
    assert not fast.stale and fast.refreshes == 1
