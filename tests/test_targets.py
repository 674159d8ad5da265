"""Target assignment on the host: tests/targets_ref.py (a numpy restatement of the two passes of csrc/targets.cu)
against the fixtures the unmodified reference's TargetAssigner.assign produced (tests/golden/make_targets_golden.py),
the mirror's plan against the plan built from the reference's assigner, and the settings b2second.targets refuses."""
import copy

import numpy as np
import pytest

import targets_ref as tr
from b2second import config, models, spec, targets


@pytest.mark.parametrize("name", tr.CONFIGS)
def test_two_pass_restatement_equals_reference(name):
    z, frames = tr.load_fixture(name)
    plan = tr.mirror_plan(name)
    for f, fr in enumerate(frames):
        labels, tg, imp, gt_id, overlap = tr.assign(plan, fr["gt_boxes"], tr.segments_of(plan, fr["gt_names"]),
                                                    fr["gt_classes"], fr["importance"], fr["mask"])
        np.testing.assert_array_equal(labels, fr["labels"], err_msg="frame %d labels" % f)
        np.testing.assert_array_equal(imp, fr["importance_out"], err_msg="frame %d importance" % f)
        np.testing.assert_array_equal(np.flatnonzero(labels > 0), fr["pos"])
        tr.assert_targets_match(tg[fr["pos"]], fr["targets"])
        assert not tg[labels <= 0].any()
        if "inds" in fr:
            inds = np.flatnonzero(gt_id >= 0)
            np.testing.assert_array_equal(inds, fr["inds"])
            np.testing.assert_array_equal(gt_id[inds], fr["gt_id"])
            np.testing.assert_array_equal(overlap[inds], fr["overlap"])


@pytest.mark.parametrize("name", tr.CONFIGS)
def test_mirror_plan_equals_reference_plan(name):
    z, _ = tr.load_fixture(name)
    plan = tr.mirror_plan(name)
    assert plan.num_anchors == int(z["num_anchors"])
    for k, v in plan.params().items():
        assert tr.sha1(v) == str(z["plan_%s_sha1" % k]), k


def _mirror(name, edit):
    cfg = config.get_config(name)
    cfg.target_assigner = copy.deepcopy(cfg.target_assigner)
    edit(cfg.target_assigner)
    return models.MirrorTargetAssigner(cfg), cfg.feature_map_size


def _set_class(i, **kw):
    def edit(ta):
        for k, v in kw.items():
            setattr(ta.classes[i], k, v)
    return edit


@pytest.mark.parametrize("edit,what", [
    (lambda ta: setattr(ta, "sample_positive_fraction", 0.25), "sample_positive_fraction"),
    (_set_class(0, similarity="rotate_iou"), "RotateIouSimilarity"),
    (_set_class(0, similarity="distance", distance_norm=1.0, with_rotation=True), "with_rotation"),
    (lambda ta: setattr(ta, "box_coder", "bev"), "BevBoxCoder"),
])
def test_unsupported_settings_are_refused(edit, what):
    ta, fm = _mirror("car.fhd", edit)
    with pytest.raises(spec.UnsupportedNetwork, match=what):
        targets.plan(ta, fm)



def test_cpu_tensors_are_refused():
    import torch
    plan = tr.mirror_plan("car.fhd")
    with pytest.raises(RuntimeError, match="CUDA"):
        plan.assign_batch(torch.zeros(1, 7), torch.tensor([0, 1], dtype=torch.int32), torch.ones(1, dtype=torch.int32))
