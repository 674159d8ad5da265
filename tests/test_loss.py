"""The training loss on the host: tests/loss_ref.py (a torch restatement of VoxelNet.loss) against the float64 fixtures
the unmodified reference's ``loss`` produced (tests/golden/make_loss_golden.py), the loss settings the mirror and the
reference network expose, the parsed ``loss`` block, and what b2second.loss refuses."""
import copy
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import loss_ref as lr
from b2second import config, loader, loss, models, refcompat, spec


def _mirror(name, cfg=None):
    return models.build_network(cfg or config.get_config(name), loader.oracle_spconv())


@pytest.mark.parametrize("name", lr.CONFIGS)
def test_restatement_equals_reference_float64(name):
    z = lr.load_fixture(name)
    s = lr.mirror_settings(name)
    for case in lr.CASES:
        ex, pr = lr.case_inputs(name, case, s)
        out, grads = lr.reference_run(s, ex, pr, torch.float64)
        want = z["ref64_%s_scalars" % case]
        got = np.array([float(out[k]) for k in lr.SCALARS])
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300, err_msg=case)
        for k in ("cls_loss", "loc_loss"):
            np.testing.assert_allclose(out[k], z["ref64_%s_%s" % (case, k)], rtol=1e-12, atol=1e-300,
                                       err_msg="%s %s" % (case, k))
        np.testing.assert_array_equal(out["cared"], z["ref64_%s_cared" % case])
        for k, g in grads.items():
            ref = z["ref64_%s_grad_%s" % (case, k)]
            np.testing.assert_allclose(g, ref, rtol=1e-12, atol=1e-12 * max(np.abs(ref).max(), 1e-300),
                                       err_msg="%s grad %s" % (case, k))


@pytest.mark.parametrize("name", lr.CONFIGS)
def test_restatement_float32_bins_equal_reference(name):
    z = lr.load_fixture(name)
    s = lr.mirror_settings(name)
    ex, pr = lr.case_inputs(name, "e", s)
    out, _ = lr.reference_run(s, ex, pr, torch.float32)
    np.testing.assert_array_equal(out["dir_bins"], z["ref32_e_dir_bins"])


@pytest.mark.parametrize("name", lr.CONFIGS)
def test_mirror_plan_equals_fixture_plan(name):
    """the settings b2second.loss.plan read off the reference network when the fixtures were made"""
    z = lr.load_fixture(name)
    got = json.loads(json.dumps(dataclasses.asdict(lr.mirror_settings(name)), sort_keys=True))
    assert got == json.loads(str(z["settings_json"]))


def _edited(name, **kw):
    cfg = config.get_config(name)
    cfg.loss = dataclasses.replace(copy.deepcopy(cfg.loss), **kw)
    return _mirror(name, cfg)


@pytest.mark.parametrize("kw,what", [
    (dict(classification_loss="weighted_sigmoid"), "classification loss"),
    (dict(localization_loss="weighted_l2"), "localization loss"),
    (dict(loss_norm_type="NormByNumExamples"), "loss_norm_type"),
    (dict(encode_rad_error_by_sin=False), "encode_rad_error_by_sin"),
    (dict(code_weight=[1.0] * 8), "code_weight"),
])
def test_unsupported_loss_settings_are_refused(kw, what):
    with pytest.raises(spec.UnsupportedNetwork, match=what):
        loss.plan(_edited("car.fhd", **kw))


@pytest.mark.parametrize("attr,what", [("_encode_background_as_zeros", "encode_background_as_zeros"),
                                       ("_use_direction_classifier", "use_direction_classifier")])
def test_unsupported_network_settings_are_refused(attr, what):
    net = _mirror("car.fhd")
    setattr(net, attr, False)
    with pytest.raises(spec.UnsupportedNetwork, match=what):
        loss.plan(net)


def test_mirror_train_mode_without_gpu_loss_still_raises():
    net = _mirror("car.lite").train()
    assert not hasattr(net, "loss")
    anchors = torch.from_numpy(net.anchors()[None])
    A = anchors.shape[1]
    net.network_forward = lambda *a: {"box_preds": torch.zeros(1, A, 7), "cls_preds": torch.zeros(1, A, 1),
                                      "dir_cls_preds": torch.zeros(1, A, 2)}
    ex = {"voxels": torch.zeros(1, 5, 4), "num_points": torch.ones(1, dtype=torch.int32),
          "coordinates": torch.zeros(1, 4, dtype=torch.int32), "anchors": anchors}
    with pytest.raises(NotImplementedError):
        net(ex)


def test_cpu_preds_are_refused():
    lp = loss.plan(_mirror("car.fhd"))
    ex, pr = lr.case_inputs("car.fhd", "a", lp.settings)
    with pytest.raises(RuntimeError, match="CUDA"):
        lp.loss(ex, pr)


# last in the module: ref_env puts the CPU oracle under the name ``spconv`` until the module ends
@pytest.mark.skipif(not refcompat.reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("name", lr.CONFIGS)
def test_mirror_plan_equals_reference_plan(ref_env, name):
    f = config.REFERENCE_FILES.get(name) or config.EXTRA_REFERENCE_FILES[name]
    cfgp = refcompat.load_config(f)
    ref = refcompat.build_network(cfgp.model.second)
    assert loss.plan(ref).settings == loss.plan(_mirror(name)).settings
    parsed = config.ModelConfig.from_file(os.path.join(refcompat.REFERENCE_ROOT, "second", "configs", f))
    assert parsed.loss == config.get_config(name).loss
