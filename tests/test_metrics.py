"""Host side of b2second.metrics (no GPU): plan and refusals, the mirror's metric buffers and checkpoints, the dict's
key names, clear_metrics, and tests/metrics_ref.py against the reference-made fixtures (tests/golden/metrics)."""
import glob
import json
import os

import numpy as np
import pytest
import torch

import metrics_ref as mr
from b2second import config, loader, metrics, models
from b2second.spec import UnsupportedNetwork
from conftest import REPO
from test_metrics_reference import same_dict, same_floats

GOLDEN = sorted(glob.glob(os.path.join(REPO, "tests", "golden", "metrics", "*.npz")))


def _mirror(name="car.fhd"):
    return metrics.enable_gpu_metrics(models.build_network(config.get_config(name), loader.oracle_spconv()))


def test_plan_reads_the_network():
    net = _mirror("nuscenes.all.pp.mhead")
    p = net.b2s_metrics
    assert p.thresholds == list(mr.THRESHOLDS) and p.num_class == 10
    params = p.params()
    assert params.num_thresholds == 7 and params.acc_threshold == 0.5
    assert params.thresholds[1] == float(np.float32(0.3))
    net.rpn_metrics._thresholds = [0.2, 0.6]
    assert metrics.plan(net).thresholds == [0.2, 0.6]


@pytest.mark.parametrize("what", ["softmax", "background", "acc_background", "nested", "too_many", "none"])
def test_plan_refuses_what_no_config_uses(what):
    net = _mirror()
    if what == "softmax":
        net.rpn_metrics._use_sigmoid_score = False
    elif what == "background":
        net.rpn_metrics._encode_background_as_zeros = False
    elif what == "acc_background":
        net.rpn_acc._encode_background_as_zeros = False
    elif what == "nested":
        net.rpn_metrics._thresholds = [[0.1, 0.5], [0.3]]
    elif what == "too_many":
        net.rpn_metrics._thresholds = [0.05 * i for i in range(1, 18)]
    else:
        net.rpn_metrics._thresholds = []
    with pytest.raises(UnsupportedNetwork):
        metrics.plan(net)


def test_mirror_gets_the_reference_buffers_and_methods():
    net = _mirror()
    sd = net.state_dict()
    want = {"rpn_acc.total": 1, "rpn_acc.count": 1, "rpn_precision.total": 1, "rpn_precision.count": 1,
            "rpn_recall.total": 1, "rpn_recall.count": 1, "rpn_metrics.prec_total": 7, "rpn_metrics.prec_count": 7,
            "rpn_metrics.rec_total": 7, "rpn_metrics.rec_count": 7, "rpn_cls_loss.total": 1, "rpn_cls_loss.count": 1,
            "rpn_loc_loss.total": 1, "rpn_loc_loss.count": 1, "rpn_total_loss.total": 1, "rpn_total_loss.count": 1}
    got = {k: v.numel() for k, v in sd.items() if k.split(".")[0] in metrics.METRIC_MODULES}
    assert got == want
    assert all(sd[k].dtype == torch.float32 for k in want)
    for m in ("update_metrics", "clear_metrics", "metrics_to_float", "update_global_step", "get_global_step"):
        assert callable(getattr(net, m)), m
    net.update_global_step()
    net.update_global_step()
    assert net.get_global_step() == 2
    net.clear_global_step()
    assert net.get_global_step() == 0
    net.metrics_to_float()
    assert net.rpn_acc.total.dtype == torch.float32


def test_mirror_loads_a_checkpoint_with_metric_buffers():
    """a reference checkpoint (the mirror's parameters plus the reference's metric buffers) loads them; before
    enable_gpu_metrics the same checkpoint loads with the buffers skipped"""
    plain = models.build_network(config.get_config("car.fhd"), loader.oracle_spconv())
    models.synthetic_weights_(plain, "car.fhd", seed=0)
    ck = dict(_mirror().state_dict())
    ck.update({k: v for k, v in plain.state_dict().items()})
    for i, k in enumerate(k for k in ck if k.split(".")[0] in metrics.METRIC_MODULES):
        ck[k] = torch.arange(ck[k].numel(), dtype=torch.float32) + 10 * i
    plain.load_reference_state_dict(ck)                      # skipped
    net = _mirror()
    net.load_reference_state_dict(ck)
    for k, v in net.state_dict().items():
        assert torch.equal(v, ck[k]), k


def test_dict_keys():
    assert int(0.3 * 100) == 29 + 1 and int(0.7 * 100) == 70 and int(0.95 * 100) == 95
    ref = mr.MetricsRef()
    st = mr.make_steps(0, 1, 64, 1, steps=1)[0]
    d = ref.update(*mr.to_torch(st), 1)
    assert set(d) == {"loss", "rpn_acc", "pr"}
    assert set(d["loss"]) == {"cls_loss", "cls_loss_rt", "loc_loss", "loc_loss_rt"}
    assert list(d["pr"]) == [f"{p}@{t}" for t in (10, 30, 50, 70, 80, 90, 95) for p in ("prec", "rec")]


def test_clear_metrics_zeroes_the_five_modules():
    """VoxelNet.clear_metrics: rpn_acc, rpn_metrics and the three Scalars go to zero; rpn_precision and rpn_recall,
    which the reference's clear_metrics does not touch, keep their values"""
    net = _mirror()
    with torch.no_grad():
        for k, v in net.state_dict().items():
            if k.split(".")[0] in metrics.METRIC_MODULES:
                v.fill_(3.0)
    net.clear_metrics()
    for k, v in net.state_dict().items():
        top = k.split(".")[0]
        if top in ("rpn_precision", "rpn_recall"):
            assert float(v.max()) == 3.0, k
        elif top in metrics.METRIC_MODULES:
            assert float(v.abs().max()) == 0.0, k


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_restatement_equals_reference_fixtures(path):
    """the restatement on the CPU gives the reference's buffers and dicts bit for bit at every step"""
    g = np.load(path)
    C = int(g["num_class"])
    ref = mr.MetricsRef()
    ref.load({k: g["init_" + k] for k in mr.BUFFERS})
    for s in range(int(g["steps"])):
        st = {k: g["%d_%s" % (s, k)] for k in ("cls_preds", "labels", "cared", "cls_loss", "loc_loss")}
        d = ref.update(*mr.to_torch(st), C)
        assert same_dict(d, json.loads(str(g["%d_dict_json" % s]))), s
        state = ref.state()
        for k in mr.BUFFERS:
            assert same_floats(state[k], g["%d_%s" % (s, k)]), (s, k)


def test_fixtures_cover_the_cases():
    assert len(GOLDEN) == 2
    for path in GOLDEN:
        g = np.load(path)
        dts = {g["%d_labels" % s].dtype for s in range(int(g["steps"]))}
        assert dts == {np.dtype(np.int32), np.dtype(np.int64)}
        assert any(float(g["%d_cls_loss" % s]) == 0.0 for s in range(int(g["steps"])))
        assert any(not (g["%d_labels" % s] > 0).any() for s in range(int(g["steps"])))
        assert all((g["%d_labels" % s] < 0).any() for s in range(int(g["steps"])))
        assert float(g["%d_acc_count" % (int(g["steps"]) - 1)][0]) > 2 ** 24
