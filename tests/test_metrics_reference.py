"""tests/metrics_ref.py against the reference tree itself (skipped where it is absent): the restatement gives the
reference's own torchplus.metrics buffers and update_metrics dict bit for bit over step sequences with a zero loss, a
step without positives, ignored anchors, int32 and int64 labels, and running sums past 2^24."""
import numpy as np
import pytest
import torch

import metrics_ref as mr
from b2second import config, refcompat

needs_reference = pytest.mark.skipif(not refcompat.reference_available(), reason="reference tree not present")
_MAP = {"acc_total": ("rpn_acc", "total"), "acc_count": ("rpn_acc", "count"),
        "prec_total": ("rpn_metrics", "prec_total"), "prec_count": ("rpn_metrics", "prec_count"),
        "rec_total": ("rpn_metrics", "rec_total"), "rec_count": ("rpn_metrics", "rec_count"),
        "cls_total": ("rpn_cls_loss", "total"), "cls_count": ("rpn_cls_loss", "count"),
        "loc_total": ("rpn_loc_loss", "total"), "loc_count": ("rpn_loc_loss", "count")}


def same_floats(a, b):
    """equal float32 bits, NaN equal to NaN (0/0 of a Scalar that never counted)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def same_dict(a, b):
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same_dict(a[k], b[k]) for k in a)
    return same_floats(a, b)


@needs_reference
@pytest.mark.parametrize("name,seed,preset", [("car.fhd", 1, False), ("car.fhd", 2, True),
                                              ("nuscenes.all.pp.mhead", 3, True)])
def test_restatement_equals_reference(ref_env, name, seed, preset):
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    net = refcompat.build_network(refcompat.load_config(f).model.second).train()
    C = int(net._num_class)
    ref = mr.MetricsRef(net.rpn_metrics.thresholds)
    bufs = {k: getattr(getattr(net, m), b) for k, (m, b) in _MAP.items()}
    if preset:
        init = mr.state0()
        ref.load(init)
        with torch.no_grad():
            for k, t in bufs.items():
                t.copy_(torch.from_numpy(init[k]))
    steps = mr.make_steps(seed, 2, 700, C, steps=7)
    if not preset:                          # the very first step with a zero loss: 0 / 0 in the dict
        steps[0]["cls_loss"] = np.float32(0.0)
    for s, st in enumerate(steps):
        want = net.update_metrics(*mr.to_torch(st))
        got = ref.update(*mr.to_torch(st), C)
        assert same_dict(got, want), (s, got, want)
        state = ref.state()
        for k, t in bufs.items():
            assert same_floats(state[k], t.detach().numpy()), (s, k, state[k], t)
    if preset:                              # the sums did round past 2^24
        assert float(bufs["acc_count"][0]) > 2 ** 24 and float(bufs["acc_count"][0]) % 2 == 0


@needs_reference
def test_mirror_takes_reference_metric_buffers(ref_env):
    """enable_gpu_metrics gives the mirror the reference's metric buffers (names, shapes, dtypes), and a reference
    checkpoint loads into it with their values"""
    from b2second import metrics, models
    name = "car.fhd"
    f = config.REFERENCE_FILES[name]
    ref = refcompat.build_network(refcompat.load_config(f).model.second)
    keys = [k for k in ref.state_dict() if k.split(".")[0] in metrics.METRIC_MODULES]
    assert len(keys) == 16
    mirror = metrics.enable_gpu_metrics(models.build_network(config.get_config(name), ref_env))
    own = mirror.state_dict()
    for k in keys:
        assert own[k].shape == ref.state_dict()[k].shape and own[k].dtype == ref.state_dict()[k].dtype, k
    with torch.no_grad():
        for i, k in enumerate(keys):
            ref.state_dict()[k].copy_(torch.arange(ref.state_dict()[k].numel(), dtype=torch.float32) + i)
    models.synthetic_weights_(ref, name, seed=0)
    mirror.load_reference_state_dict(ref.state_dict())
    for k in keys:
        assert torch.equal(mirror.state_dict()[k], ref.state_dict()[k]), k
    assert mirror.rpn_metrics.thresholds == ref.rpn_metrics.thresholds
