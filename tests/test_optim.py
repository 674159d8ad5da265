"""The optimizer step on the host: tests/optim_ref.py (the float64 restatement) against torch.optim.Adam with a literal
clip_grad_norm_ and decay loop, the tabulated schedules against closed forms, the parameter groups of the mirror
networks, the optimizer block as parsed from config text, what b2second.optim refuses, and checkpoints in
torch.optim.Adam's format.  test_optim_reference.py holds the comparisons with the reference tree."""
import dataclasses

import numpy as np
import pytest
import torch

import optim_ref as orf
from b2second import config, loader, models, optim, spec

OPTIMIZER_TEXT = """
train_config: {
  optimizer: {
    adam_optimizer: {
      learning_rate: { %s }
      weight_decay: %s
    }
    fixed_weight_decay: %s
    use_moving_average: false
  }
  steps: 23200
}
"""
ONE_CYCLE_TEXT = OPTIMIZER_TEXT % ("one_cycle: { lr_max: 2.25e-3 moms: [0.95, 0.85] div_factor: 10.0 pct_start: 0.4 }",
                                   "0.01", "true")
STAIRCASE_TEXT = OPTIMIZER_TEXT % ("exponential_decay: { initial_learning_rate: 0.0002 decay_length: 0.1 "
                                   "decay_factor: 0.8 staircase: True }", "0.0001", "false")


def _block(text):
    return config.parse_prototxt(text)["train_config"][-1]["optimizer"][-1]


@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_restatement_equals_torch_adam_float64(kind):
    """50 steps: optim_ref.ref_step on numpy float64 against torch.optim.Adam(foreach=False) on float64 tensors with
    clip_grad_norm_ and the per-parameter decay loop, the schedule's lr and beta1 set by hand each step"""
    s = orf.SETTINGS[kind]
    steps = 50
    case = orf.make_case("none_grad", seed=3, steps=steps)
    case["grads"][10] = [None if g is None else g * 0.01 for g in case["grads"][10]]      # one step under the clip
    net = case["module"].double()
    groups = optim.parameter_groups(net)
    params = [p for g in groups for p in g]
    p = [x.detach().numpy().copy() for x in params]
    start2 = p[2].copy()
    m, v = [np.zeros_like(x) for x in p], [np.zeros_like(x) for x in p]
    adam = orf.torch_adam(s, groups, foreach=False)
    lrs, moms = optim.schedule(s, steps)
    clipped = 0
    for i in range(steps):
        orf.set_grads(params, case["grads"][i])
        want_total = float(orf.torch_step(s, adam, lrs[i], moms[i]))
        total, _ = orf.ref_step(s, p, case["grads"][i], m, v, lrs[i], moms[i], i + 1)
        clipped += total > s.clip_norm
        assert total == pytest.approx(want_total, rel=1e-12)
    assert 0 < clipped < steps
    for k, x in enumerate(params):
        np.testing.assert_allclose(p[k], x.detach().numpy(), rtol=1e-10, atol=1e-14, err_msg="param %d" % k)
        if k != 2:
            np.testing.assert_allclose(m[k], adam.state[x]["exp_avg"].numpy(), rtol=1e-10, atol=1e-300)
            np.testing.assert_allclose(v[k], adam.state[x]["exp_avg_sq"].numpy(), rtol=1e-10, atol=1e-300)
    assert params[2] not in adam.state                               # never stepped; decayed in the decoupled form
    want = start2
    if s.decoupled:
        want = want * np.prod([1 - s.weight_decay * lr for lr in lrs])
    np.testing.assert_allclose(p[2], want, rtol=1e-12)


@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_float32_operation_order_stays_inside_the_stated_bounds(kind):
    """optim_ref.step_bounds, compounded over 50 steps, covers the float32 operation order of the kernel (emulated in
    numpy) against the float64 restatement: the bounds test_gpu_optim.py holds the GPU to are sound"""
    s = orf.SETTINGS[kind]
    steps = 50
    case = orf.make_case("above", seed=9, steps=steps)
    case["grads"][7] = [g * 0.01 for g in case["grads"][7]]
    p32 = [x.detach().numpy().copy() for x in case["params"]]
    m32, v32 = [np.zeros_like(x) for x in p32], [np.zeros_like(x) for x in p32]
    p = [x.astype(np.float64) for x in p32]
    m, v = [np.zeros_like(x) for x in p], [np.zeros_like(x) for x in p]
    lrs, moms = optim.schedule(s, steps)
    d = [(0.0, 0.0, 0.0)] * len(p)
    for i in range(steps):
        total, info = orf.ref_step(s, p, case["grads"][i], m, v, lrs[i], moms[i], i + 1)
        total32 = orf.f32_step(s, p32, case["grads"][i], m32, v32, lrs[i], moms[i], i + 1)
        assert abs(float(total32) - total) <= 1e-7 * total
        d = [orf.step_bounds(s, info[k], p[k], m[k], v[k], *d[k]) for k in range(len(p))]
    for k in range(len(p)):
        for got, want, bound, what in ((m32, m, d[k][0], "m"), (v32, v, d[k][1], "v"), (p32, p, d[k][2], "p")):
            worst = float((np.abs(got[k] - want[k]) / np.maximum(bound, 1e-300)).max())
            assert worst <= 1.0, "%s of parameter %d: %.3g of its bound" % (what, k, worst)
        # and the bounds are rounding-sized: a few float32 roundings of the values involved per step
        assert float((d[k][2] / (np.abs(p[k]) + sum(lrs))).max()) < steps * 40 * orf.EPS32


@pytest.mark.parametrize("s,total", [
    (orf.ONE_CYCLE, 23200), (orf.ONE_CYCLE, 50), (orf.STAIRCASE, 296960), (orf.STAIRCASE, 50),
    (dataclasses.replace(orf.STAIRCASE, staircase=False), 1000),
    (dataclasses.replace(orf.STAIRCASE, schedule="manual_stepping", boundaries=(0.8, 0.9),
                         rates=(1e-3, 1e-4, 5e-5)), 1000)], ids=lambda v: getattr(v, "schedule", str(v)))
def test_schedule_table_equals_closed_form(s, total):
    table = optim.schedule_table(s, total)
    assert table.shape == (total, len(optim.HYPER_COLS)) and table.dtype == np.float64
    lr, mom = orf.ref_schedule(s, total)
    t = np.arange(1, total + 1, dtype=np.float64)
    np.testing.assert_allclose(table[:, 0], lr, rtol=1e-12)
    np.testing.assert_allclose(table[:, 1], mom, rtol=1e-13)
    np.testing.assert_allclose(table[:, 2], 1 - mom ** t, rtol=1e-9, atol=0)
    np.testing.assert_allclose(table[:, 3], np.sqrt(1 - s.beta2 ** t), rtol=1e-12)
    np.testing.assert_allclose(table[:, 4], 1 - s.weight_decay * lr, rtol=1e-15)


def test_bad_schedules_raise():
    with pytest.raises(ValueError):
        optim.schedule(orf.ONE_CYCLE, 2)                             # the first phase would have no step
    with pytest.raises(ValueError):
        optim.schedule(orf.STAIRCASE, 5)                             # decay_length * total_step < 1
    with pytest.raises(ValueError):
        optim.schedule(orf.ONE_CYCLE, 0)


def _bn_and_other_parameters(net):
    bn = {id(p) for m in net.modules() if isinstance(m, optim._BN_TYPES) for p in m.parameters()}
    return bn


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"])
def test_parameter_groups_of_the_mirror(name):
    net = models.build_network(config.get_config(name), loader.oracle_spconv())
    first = next(net.parameters())
    first.requires_grad_(False)                                      # as freeze_params_v2 leaves it
    others, bns = optim.parameter_groups(net)
    bn = _bn_and_other_parameters(net)
    assert bns and all(id(p) in bn for p in bns) and not any(id(p) in bn for p in others)
    want = [p for p in net.parameters() if p.requires_grad]
    assert sorted(map(id, others + bns)) == sorted(map(id, want)) and len(set(map(id, others + bns))) == len(want)
    assert all(p is not first for p in others + bns)
    # module order within each group
    pos = {id(p): i for i, p in enumerate(net.parameters())}
    for g in (others, bns):
        assert [pos[id(p)] for p in g] == sorted(pos[id(p)] for p in g)


def test_settings_from_parsed_config_text():
    assert optim.settings(_block(ONE_CYCLE_TEXT)) == orf.ONE_CYCLE
    assert optim.settings(_block(STAIRCASE_TEXT)) == orf.STAIRCASE
    assert optim.settings(orf.ONE_CYCLE) is orf.ONE_CYCLE


@pytest.mark.parametrize("edit,word", [
    (lambda t: t.replace("adam_optimizer", "rms_prop_optimizer"), "rms_prop_optimizer"),
    (lambda t: t.replace("adam_optimizer", "momentum_optimizer"), "momentum_optimizer"),
    (lambda t: t.replace("weight_decay: 0.01", "weight_decay: 0.01 amsgrad: true"), "amsgrad"),
    (lambda t: t.replace("use_moving_average: false", "use_moving_average: true"), "use_moving_average"),
    (lambda t: t.replace("one_cycle", "multi_phase"), "multi_phase")])
def test_refused_optimizer_blocks(edit, word):
    with pytest.raises(spec.UnsupportedNetwork, match=word):
        optim.settings(_block(edit(ONE_CYCLE_TEXT)))


def test_refused_parameters():
    with pytest.raises(spec.UnsupportedNetwork, match="float32"):
        optim.plan(orf.ParamSet([(4,)]).half(), orf.ONE_CYCLE, 100)
    with pytest.raises(spec.UnsupportedNetwork, match="float32"):
        optim.plan(orf.ParamSet([(4,)]).double(), orf.ONE_CYCLE, 100)
    with pytest.raises(RuntimeError, match="CUDA"):
        if torch.cuda.is_available():
            raise RuntimeError("CUDA present: the CPU refusal cannot be shown")
        optim.plan(orf.ParamSet([(4,)]), orf.ONE_CYCLE, 100).step()


def test_plan_allocates_gradients_and_skips_frozen():
    case = orf.make_case("frozen")
    opt = optim.plan(case["module"], orf.ONE_CYCLE, 100)
    frozen = case["module"].w[3]
    assert frozen.grad is None and all(p is not frozen for p in opt.params)
    assert all(p.grad is not None and not p.grad.any() for p in opt.params)
    assert (opt.global_step, opt.lr, opt.mom) == (0, opt.table[0, 0], opt.table[0, 1])


@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_state_dict_round_trip_with_torch_adam(kind):
    """a torch.optim.Adam checkpoint (what the reference's OptimWrapper saves) loads into a plan, the plan's
    state_dict loads into a fresh torch.optim.Adam, and both carry the same moments and step"""
    s = orf.SETTINGS[kind]
    steps = 7
    case = orf.make_case("above", seed=5, steps=steps)
    groups = optim.parameter_groups(case["module"])
    adam = orf.torch_adam(s, groups)
    lrs, moms = optim.schedule(s, 100)
    for i in range(steps):
        orf.set_grads(case["params"], case["grads"][i])
        orf.torch_step(s, adam, lrs[i], moms[i])
    opt = optim.plan(case["module"], s, 100)
    opt.load_state_dict(adam.state_dict())
    assert opt.global_step == steps and opt.lr == lrs[steps] and opt.mom == moms[steps]
    for k, p in enumerate(opt.params):
        assert torch.equal(opt.exp_avg[k], adam.state[p]["exp_avg"])
        assert torch.equal(opt.exp_avg_sq[k], adam.state[p]["exp_avg_sq"])
    sd = opt.state_dict()
    assert [g["params"] for g in sd["param_groups"]] == [g["params"] for g in adam.state_dict()["param_groups"]]
    fresh = orf.torch_adam(s, groups)
    fresh.load_state_dict(sd)
    for p in opt.params:
        assert float(fresh.state[p]["step"]) == steps
        assert torch.equal(fresh.state[p]["exp_avg"], adam.state[p]["exp_avg"])
        assert torch.equal(fresh.state[p]["exp_avg_sq"], adam.state[p]["exp_avg_sq"])
    assert fresh.param_groups[0]["betas"] == (moms[steps], s.beta2)
    again = optim.plan(case["module"], s, 100)
    again.load_state_dict(sd)
    assert again.global_step == steps and torch.equal(again.exp_avg[0], opt.exp_avg[0])
    assert optim.plan(case["module"], s, 100).state_dict()["state"] == {}
    bad = adam.state_dict()
    bad["param_groups"][0]["params"] = bad["param_groups"][0]["params"][:-1]
    with pytest.raises(ValueError):
        opt.load_state_dict(bad)
