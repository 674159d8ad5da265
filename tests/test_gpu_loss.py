"""The training loss on the GPU (csrc/loss.cu through b2second.loss) against the float64 fixtures the unmodified
reference's VoxelNet.loss produced (tests/golden/make_loss_golden.py) and against tests/loss_ref.py in float64.

Bounds.  The six scalars: 1e-5 relative to float64 (1e-7 absolute where the value is 0).  Every element of the
per-anchor outputs and of the gradients: |v - v64| <= C_REL eps32 |v64| + C_MAX eps32 max|v64|.  Each element is a
product of at most a dozen float32 roundings (the weight: one division and one product; the focal term: exp, log1p,
a reciprocal, the square, the alpha product, the CE sum; the smooth-L1: the difference, the code weight and the
square, and for the yaw sin of a rounded difference; the softmax: exp, sum, division), each contributing at most eps32
relative, so C_REL = 8 holds with room.  C_MAX covers the absolute error of the terms that cancel: the float32 inputs
of a sin-encoded yaw difference or of 1 - p near p = 1, whose rounding is eps32 of the larger operand; 1 suffices
because those terms are of order max|v64| or smaller."""
import dataclasses

import numpy as np
import pytest
import torch

import loss_ref as lr
from b2second import config, loader, loss, models, targets, training

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS32, C_REL, C_MAX = lr.EPS32, lr.C_REL, lr.C_MAX


def _plan(name):
    return loss.plan(models.build_network(config.get_config(name), loader.oracle_spconv()))


def _cuda(example, preds, labels32=False):
    ex = {k: v.to(DEV) for k, v in example.items()}
    if labels32:
        ex["labels"] = ex["labels"].to(torch.int32)
    return ex, {k: v.to(DEV).clone().requires_grad_() for k, v in preds.items()}


def _check_elem(got, want, what):
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.isfinite(got).all(), what
    bound = C_REL * EPS32 * np.abs(want) + C_MAX * EPS32 * (np.abs(want).max() if want.size else 0.0)
    err = np.abs(got - want)
    bad = err > bound
    assert not bad.any(), "%s: %d elements over the bound, worst err %g at bound %g" % (
        what, int(bad.sum()), float(err[bad].max()), float(bound[bad][np.argmax(err[bad])]))


_check_scalars = lr.check_scalars


def _scalars(r):
    return [float(r[k].detach()) for k in lr.SCALARS]


@pytest.mark.parametrize("name", lr.CONFIGS)
def test_loss_and_gradients_equal_reference(name):
    z = lr.load_fixture(name)
    lp = _plan(name)
    for case in lr.CASES:
        example, preds = lr.case_inputs(name, case, lp.settings)
        # the reference's own float32 values meet the scalar bound too (else the bound, not the kernel, is wrong)
        _check_scalars(z["ref32_%s_scalars" % case], z["ref64_%s_scalars" % case], "reference float32 " + case)
        for labels32 in (False, True):
            ex, pr = _cuda(example, preds, labels32)
            r = lp.loss(ex, pr)
            assert set(r) == {"loss", "cls_loss", "loc_loss", "cls_pos_loss", "cls_neg_loss", "cls_preds",
                              "cls_loss_reduced", "loc_loss_reduced", "cared", "dir_loss_reduced"}
            assert r["cls_preds"] is pr["cls_preds"]
            r["loss"].backward()
            torch.cuda.synchronize()
            assert int(lp.last_status.item()) == 0
            _check_scalars(_scalars(r), z["ref64_%s_scalars" % case], case)
            _check_elem(r["cls_loss"], z["ref64_%s_cls_loss" % case], case + " cls_loss")
            _check_elem(r["loc_loss"], z["ref64_%s_loc_loss" % case], case + " loc_loss")
            np.testing.assert_array_equal(r["cared"].cpu().numpy(), z["ref64_%s_cared" % case])
            for k in pr:
                _check_elem(pr[k].grad, z["ref64_%s_grad_%s" % (case, k)], "%s grad %s" % (case, k))
            if case == "e":
                # direction bins exact: dir logits are 0 there, so the target bin is the one negative gradient
                lab = ex["labels"].cpu().numpy()
                n = int((lab[0] > 0).sum())
                assert n > 0
                g = pr["dir_cls_preds"].grad.cpu().numpy()
                pos = lab > 0
                bins = np.argmin(g, -1)
                np.testing.assert_array_equal(bins[pos], z["ref32_e_dir_bins"][pos])
                assert (g[pos].min(-1) < 0).all()
            if case == "d":
                for k in pr:
                    assert torch.isfinite(pr[k].grad).all()


@pytest.mark.parametrize("name,B", [("car.fhd", 8), ("nuscenes.all.pp.mhead", 4)])
def test_full_size_batch_equals_restatement(name, B):
    lp = _plan(name)
    s = lp.settings
    A = int(models.build_network(config.get_config(name), loader.oracle_spconv()).anchors().shape[0])
    example, preds = lr.make_case("a", B, A, s.num_class, s.num_dir_bins, s.dir_offset, seed=31)
    out64, g64 = lr.reference_run(s, example, preds, torch.float64)
    ex, pr = _cuda(example, preds, labels32=True)
    r = lp.loss(ex, pr)
    r["loss"].backward()
    _check_scalars(_scalars(r), [float(out64[k]) for k in lr.SCALARS], name)
    _check_elem(r["cls_loss"], out64["cls_loss"], "cls_loss")
    _check_elem(r["loc_loss"], out64["loc_loss"], "loc_loss")
    for k in pr:
        _check_elem(pr[k].grad, g64[k], "grad " + k)


def _run(lp, ex, pr):
    for t in pr.values():
        t.grad = None
    r = lp.loss(ex, pr)
    r["loss"].backward()
    return [r[k] for k in lr.SCALARS] + [r["cls_loss"], r["loc_loss"], r["cared"]] + [pr[k].grad for k in pr]


def test_runs_and_cuda_graph_replay_are_bit_identical():
    lp = _plan("nuscenes.all.pp.mhead")
    s = lp.settings
    example, preds = lr.make_case("a", 4, 20000, s.num_class, s.num_dir_bins, s.dir_offset, seed=5)
    ex, pr = _cuda(example, preds)
    first = [t.clone() for t in _run(lp, ex, pr)]
    second = _run(lp, ex, pr)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    # leaves first used on a side stream (their gradient accumulators live there), warm-up there, then capture
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        pg = {k: v.detach().clone().requires_grad_() for k, v in pr.items()}
        for _ in range(3):
            _run(lp, ex, pg)
    torch.cuda.current_stream().wait_stream(st)
    for t in pg.values():
        t.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        r = lp.loss(ex, pg)
        r["loss"].backward()
    g.replay()
    torch.cuda.synchronize()
    got = [r[k] for k in lr.SCALARS] + [r["cls_loss"], r["loc_loss"], r["cared"]] + [pg[k].grad for k in pg]
    for a, b in zip(first, got):
        assert torch.equal(a, b)


def test_zero_weight_anchors_get_exactly_zero_gradient():
    lp = _plan("all.fhd")
    s = lp.settings
    example, preds = lr.make_case("d", 2, 3000, s.num_class, s.num_dir_bins, s.dir_offset, seed=8)
    ex, pr = _cuda(example, preds)
    lp.loss(ex, pr)["loss"].backward()
    lab = ex["labels"]
    ign, nonpos = lab < 0, lab <= 0
    assert ign.any() and (lab == 0).any()
    assert (pr["cls_preds"].grad[ign] == 0).all()
    assert (pr["box_preds"].grad[nonpos] == 0).all()
    assert (pr["dir_cls_preds"].grad[nonpos] == 0).all()
    # only the cls_loss_reduced gradient: box and direction gradients are exactly 0 everywhere
    for t in pr.values():
        t.grad = None
    r = lp.loss(ex, pr)
    r["cls_loss_reduced"].backward()
    assert not pr["box_preds"].grad.any() and not pr["dir_cls_preds"].grad.any()
    assert pr["cls_preds"].grad.any()


def test_out_of_range_label_raises_bad_input():
    from spconv import _lib
    lp = _plan("car.fhd")
    s = lp.settings
    example, preds = lr.make_case("a", 2, 1000, s.num_class, s.num_dir_bins, s.dir_offset, seed=9)
    example["labels"][0, 3] = 2                             # car.fhd has one class
    example["labels"][1, 7] = -5
    ex, pr = _cuda(example, preds)
    r = lp.loss(ex, pr)
    assert int(lp.last_status.item()) & 32
    assert "label" in _lib.status_message(int(lp.last_status.item()))
    assert not r["cared"][0, 3] and not r["cared"][1, 7]
    ok = example["labels"].clone()
    ok[0, 3] = -1
    ok[1, 7] = -1
    r2 = lp.loss(dict(ex, labels=ok.to(DEV)), pr)
    assert int(lp.last_status.item()) == 0
    for k in lr.SCALARS:
        assert torch.equal(r[k], r2[k]), k


def test_half_precision_preds_raise_type_error():
    lp = _plan("car.fhd")
    s = lp.settings
    example, preds = lr.make_case("a", 1, 500, s.num_class, s.num_dir_bins, s.dir_offset, seed=10)
    ex, pr = _cuda(example, preds)
    pr["cls_preds"] = pr["cls_preds"].detach().half()
    with pytest.raises(TypeError):
        lp.loss(ex, pr)


def test_non_contiguous_preds_are_accepted():
    lp = _plan("car.fhd")
    s = lp.settings
    example, preds = lr.make_case("a", 2, 1000, s.num_class, s.num_dir_bins, s.dir_offset, seed=11)
    ex, pr = _cuda(example, preds)
    ref = [float(v.detach()) for v in (lp.loss(ex, pr)[k] for k in lr.SCALARS)]
    box_t = pr["box_preds"].detach().transpose(0, 1).contiguous().transpose(0, 1)
    assert not box_t.is_contiguous()
    got = lp.loss(ex, dict(pr, box_preds=box_t))
    assert [float(got[k].detach()) for k in lr.SCALARS] == ref


def _car_lite_example(net, cfg):
    from b2second import synth
    onet = models.build_network(cfg, loader.oracle_spconv())
    res = onet.voxel_generator.generate(synth.kitti_cloud(2, 20000, cfg.point_cloud_range), cfg.max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    anchors = net.anchors()
    tp = targets.plan(net.target_assigner, cfg.feature_map_size)
    rng = np.random.default_rng(3)
    gt = anchors[rng.integers(0, len(anchors), 12)].astype(np.float32).copy()
    gt[:, :2] += rng.uniform(-0.5, 0.5, (12, 2)).astype(np.float32)
    gt[:, 6] = rng.uniform(-np.pi, np.pi, 12).astype(np.float32)
    tg = tp.assign_batch(torch.from_numpy(gt).to(DEV), torch.tensor([0, 12], dtype=torch.int32, device=DEV),
                         torch.ones(12, dtype=torch.int32, device=DEV))
    assert int((tg["labels"] > 0).sum()) > 0
    ex = {"voxels": torch.from_numpy(res["voxels"]).to(DEV),
          "num_points": torch.from_numpy(res["num_points_per_voxel"]).to(DEV),
          "coordinates": torch.from_numpy(coords).to(DEV), "anchors": torch.from_numpy(anchors[None]).to(DEV)}
    ex.update(tg)
    return ex


@pytest.fixture
def _fp32_torch():
    """cuDNN and matmul in fp32: with TF32, a 1e-6 difference in an incoming gradient can flip a 10-bit rounding"""
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


@pytest.mark.timeout(600)
def test_car_lite_train_step_matches_torch_loss(_fp32_torch):
    """mirror car.lite with enable_sparse_backward + enable_gpu_loss in train(): net(example) returns the reference's
    keys, and every parameter gradient of loss.backward() meets ||g - g_ref||_inf <= 2e-4 ||g_ref||_inf against the same
    network with the loss_ref torch chain (float32) as the loss"""
    name = "car.lite"
    cfg = config.get_config(name)
    sp = loader.product_spconv()
    net = models.build_network(cfg, sp)
    models.synthetic_weights_(net, name, seed=0)
    ref = models.build_network(cfg, sp)
    ref.load_state_dict(net.state_dict())
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV))).train()
    ref = training.enable_sparse_backward(ref.to(DEV)).train()
    ex = _car_lite_example(net, cfg)
    r = net(ex)
    assert {"loss", "cls_loss", "loc_loss", "cls_pos_loss", "cls_neg_loss", "cls_preds", "cls_loss_reduced",
            "loc_loss_reduced", "cared", "dir_loss_reduced"} <= set(r)
    r["loss"].backward()
    preds = ref.network_forward(ex["voxels"], ex["num_points"], ex["coordinates"], 1)
    r_ref = lr.loss(net.b2s_loss.settings, ex, preds)
    r_ref["loss"].backward()
    torch.cuda.synchronize()
    assert abs(float(r["loss"]) - float(r_ref["loss"])) <= 1e-5 * abs(float(r_ref["loss"]))
    errs = {}
    for (k, p), (_, p_ref) in zip(net.named_parameters(), ref.named_parameters()):
        if p_ref.grad is None:
            continue
        errs[k] = float((p.grad - p_ref.grad).abs().max()) / max(float(p_ref.grad.abs().max()), 1e-30)
    assert errs
    bad = {k: e for k, e in errs.items() if e > 2e-4}
    assert not bad, bad
