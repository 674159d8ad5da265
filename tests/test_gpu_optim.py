"""GPU tests of the optimizer step (b2second.optim over b2s_optim_step, csrc/optim.cu) against the float64 restatement
in tests/optim_ref.py with the per-element bounds of optim_ref.step_bounds, against torch's float32 Adam on the same
device, and for what the step promises beyond values: equal bits run to run and layout to layout, graph capture, no
stale weight caches in the drop-in after a step."""
import copy
import dataclasses

import numpy as np
import pytest
import torch

import optim_ref as orf
from b2second import models, optim, training

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _plan(case, s, total_step=100):
    """-> (a CUDA copy of the case's module, its plan)"""
    net = copy.deepcopy(case["module"]).to(DEV)
    return net, optim.plan(net, s, total_step)


def _state64(opt):
    return ([p.detach().cpu().numpy().astype(np.float64) for p in opt.params],
            [m.cpu().numpy().astype(np.float64) for m in opt.exp_avg],
            [v.cpu().numpy().astype(np.float64) for v in opt.exp_avg_sq])


def _bits(opt):
    return [t.detach().clone() for t in list(opt.params) + opt.exp_avg + opt.exp_avg_sq]


def _same_bits(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def _check(opt, p, m, v, d, what=""):
    got = _state64(opt)
    for name, g, want, col in (("m", got[1], m, 0), ("v", got[2], v, 1), ("p", got[0], p, 2)):
        for k in range(len(p)):
            worst = float((np.abs(g[k] - want[k]) / np.maximum(d[k][col], 1e-300)).max())
            assert worst <= 1.0, "%s %s of parameter %d: %.3g of its bound" % (what, name, k, worst)


@pytest.mark.parametrize("name", ["above", "below", "none_grad", "frozen"])
@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_one_step_from_float32_state_matches_float64(kind, name):
    """one step at t = 6 from random moments: m, v, p inside optim_ref.step_bounds (about 3 EPS32 (|m0| + |g|), 7 EPS32
    v, 1.5 EPS32 |p| + 4 EPS32 |update| + the moments' differences carried through), the norm within 1e-7 relative"""
    s = orf.SETTINGS[kind]
    case = orf.make_case(name, seed=1)
    net, opt = _plan(case, s)
    gen = torch.Generator().manual_seed(2)
    for m, v in zip(opt.exp_avg, opt.exp_avg_sq):
        m.copy_(torch.randn(m.shape, generator=gen) * 0.02)
        v.copy_((torch.randn(v.shape, generator=gen) * 0.02) ** 2)
    opt.global_step = 5
    grads = case["grads"][0]
    orf.set_grads(opt.params, grads)
    p, m, v = _state64(opt)
    total, info = orf.ref_step(s, p, grads, m, v, opt.table[5, 0], opt.table[5, 1], 6)
    got_total = opt.step()
    assert got_total.is_cuda and got_total.shape == ()
    assert abs(float(got_total) - total) <= 1e-7 * total
    assert (total > s.clip_norm) == (name != "below")
    assert opt.global_step == 6 and int(opt.status.item()) == 0
    d = [orf.step_bounds(s, info[k], p[k], m[k], v[k]) if info[k] is not None else (0.0, 0.0, 1.5 * orf.EPS32 * np.abs(p[k]))
         for k in range(len(p))]
    _check(opt, p, m, v, d)
    assert all(not g.grad.any() for g in opt.params if g.grad is not None)       # zeroed in place
    if name == "frozen":
        frozen = net.w[3]
        assert torch.equal(frozen.cpu(), case["module"].w[3]) and frozen.grad is None


@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_fifty_step_trajectory_matches_float64_and_torch_float32(kind):
    """50 steps with fresh gradients (one step under the clip norm): every m, v, p inside the one-step bounds
    compounded along the float64 trajectory, and within twice that of torch.optim.Adam in float32 on the same device
    driven by the literal sequence (clip_grad_norm_, decay loop, lr and betas set by hand), which meets the same bounds"""
    s = orf.SETTINGS[kind]
    steps = 50
    case = orf.make_case("above", seed=4, steps=steps)
    case["grads"][20] = [g * 0.01 for g in case["grads"][20]]
    net, opt = _plan(case, s, steps)
    twin = copy.deepcopy(case["module"]).to(DEV)
    twin_groups = optim.parameter_groups(twin)
    twin_params = [x for g in twin_groups for x in g]
    adam = orf.torch_adam(s, twin_groups)
    p, m, v = _state64(opt)
    d = [(0.0, 0.0, 0.0)] * len(p)
    for i in range(steps):
        orf.set_grads(opt.params, case["grads"][i])
        orf.set_grads(twin_params, case["grads"][i])
        total, info = orf.ref_step(s, p, case["grads"][i], m, v, opt.table[i, 0], opt.table[i, 1], i + 1)
        got = opt.step()
        want32 = orf.torch_step(s, adam, float(opt.table[i, 0]), float(opt.table[i, 1]))
        d = [orf.step_bounds(s, info[k], p[k], m[k], v[k], *d[k]) for k in range(len(p))]
        if i in (0, 20, steps - 1):
            assert abs(float(got) - total) <= 1e-7 * total
            assert abs(float(got) - float(want32)) <= 1e-6 * total
    assert opt.global_step == steps and opt.table_builds == 1 and int(opt.status.item()) == 0
    _check(opt, p, m, v, d, "float64:")
    for k, x in enumerate(twin_params):
        for name, got, want, col in (("p", opt.params[k], x, 2), ("m", opt.exp_avg[k], adam.state[x]["exp_avg"], 0),
                                     ("v", opt.exp_avg_sq[k], adam.state[x]["exp_avg_sq"], 1)):
            diff = (got.detach().double() - want.detach().double()).abs().cpu().numpy()
            worst = float((diff / np.maximum(2 * d[k][col], 1e-300)).max())
            assert worst <= 1.0, "torch float32: %s of parameter %d: %.3g of twice its bound" % (name, k, worst)


@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_two_runs_give_equal_bits(kind):
    s = orf.SETTINGS[kind]
    case = orf.make_case("above", seed=6, steps=3)
    runs = []
    for _ in range(2):
        net, opt = _plan(case, s)
        norms = []
        for i in range(3):
            orf.set_grads(opt.params, case["grads"][i])
            norms.append(opt.step().clone())
        runs.append(_bits(opt) + norms)
    assert _same_bits(*runs)


@pytest.mark.parametrize("name", ["above", "below"])
def test_result_does_not_depend_on_the_tensor_layout(name):
    """the same values as eleven tensors (sizes 1 .. 13824, most not multiples of 4) and as one flat tensor that starts
    4 bytes off a 16-byte boundary (so it takes the scalar path, the others the 16-byte one): equal bits of p, m, v
    after three steps, and the same norm.  The chunk partials of the norm add in a different order in the two
    layouts; their float64 sums differ by about 1e-16 relative, which rounds to the same float32 norm except on a
    rounding boundary."""
    s = orf.ONE_CYCLE
    case = orf.make_case(name, seed=7, steps=3)
    many = orf.ParamSet(orf.SHAPES)
    with torch.no_grad():
        for dst, src in zip(many.w, case["params"]):
            dst.copy_(src)
    n = len(orf.SHAPES)
    many, flat = many.to(DEV), orf.ParamSet([])
    total = sum(int(np.prod(sh)) for sh in orf.SHAPES)
    flat.w.append(torch.nn.Parameter(torch.zeros(total + 1, device=DEV)[1:]))
    with torch.no_grad():
        flat.w[0].copy_(torch.cat([x.detach().flatten() for x in many.w]))
    assert flat.w[0].data_ptr() % 16 == 4 and all(x.data_ptr() % 16 == 0 for x in many.w)
    a, b = optim.plan(many, s, 100), optim.plan(flat, s, 100)
    for i in range(3):
        gs = case["grads"][i][:n]
        orf.set_grads(a.params, gs)
        orf.set_grads(b.params, [np.concatenate([g.ravel() for g in gs])])
        ta, tb = a.step(), b.step()
        assert torch.equal(ta, tb)
    for xs, y in ((a.params, b.params[0]), (a.exp_avg, b.exp_avg[0]), (a.exp_avg_sq, b.exp_avg_sq[0])):
        assert _same_bits([torch.cat([x.detach().flatten() for x in xs])], [y.detach()])


@pytest.mark.parametrize("factor,clipped", [(1 - 1e-3, False), (1 + 1e-3, True)])
def test_clip_boundary(factor, clipped):
    """a gradient norm just under the clip norm leaves the step equal, bit for bit, to a step without clipping; just
    over it does not, and stays inside the float64 bounds"""
    s = orf.ONE_CYCLE
    case = orf.make_case("above", seed=8)
    g = case["grads"][0]
    norm = np.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in g))
    g = [(x * (s.clip_norm * factor / norm)).astype(np.float32) for x in g]
    _, opt = _plan(case, s)
    _, free = _plan(case, dataclasses.replace(s, clip_norm=1e30))
    p, m, v = _state64(opt)
    total, info = orf.ref_step(s, p, g, m, v, opt.table[0, 0], opt.table[0, 1], 1)
    assert (total > s.clip_norm) == clipped
    for o in (opt, free):
        orf.set_grads(o.params, g)
        o.step()
    assert _same_bits(_bits(opt), _bits(free)) == (not clipped)
    _check(opt, p, m, v, [orf.step_bounds(s, info[k], p[k], m[k], v[k]) for k in range(len(p))])


@pytest.mark.parametrize("kind", sorted(orf.SETTINGS))
def test_zero_gradients_and_set_to_none(kind):
    """all-zero gradients: the norm is 0, the moments stay 0, parameters only decay (decoupled form) or stay (L2: the
    decay enters Adam as a gradient).  set_to_none=True leaves grad None, and a step without gradients only decays."""
    s = orf.SETTINGS[kind]
    case = orf.make_case("zero", seed=9)
    _, opt = _plan(case, s)
    p0 = [x.detach().clone() for x in opt.params]
    total = opt.step(set_to_none=True)
    assert float(total) == 0.0 and all(x.grad is None for x in opt.params)
    decay = torch.tensor(1 - s.weight_decay * opt.table[0, 0], dtype=torch.float32, device=DEV)
    if s.decoupled:
        assert all(torch.equal(x.detach(), x0 * decay) for x, x0 in zip(opt.params, p0))
        assert all(not m.any() and not v.any() for m, v in zip(opt.exp_avg, opt.exp_avg_sq))
    p1 = [x.detach().clone() for x in opt.params]
    m1 = [m.clone() for m in opt.exp_avg]
    opt.step()                                                       # no gradient anywhere
    decay = torch.tensor(1 - s.weight_decay * opt.table[1, 0], dtype=torch.float32, device=DEV)
    for x, x1 in zip(opt.params, p1):
        assert torch.equal(x.detach(), x1 * decay if s.decoupled else x1)
    assert all(torch.equal(a, b) for a, b in zip(opt.exp_avg, m1))
    assert opt.global_step == 2 and opt.table_builds == 2


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_non_finite_gradient_propagates_as_in_torch(bad):
    """an input check: one inf or NaN gradient element makes the norm non-finite; the parameters turn NaN exactly where
    torch's sequence turns them NaN, and B2S_STATUS_OPT_NONFINITE is raised"""
    s = orf.ONE_CYCLE
    case = orf.make_case("above", seed=10)
    g = [x.copy() for x in case["grads"][0]]
    g[4][17] = bad
    net, opt = _plan(case, s)
    twin = copy.deepcopy(case["module"]).to(DEV)
    groups = optim.parameter_groups(twin)
    adam = orf.torch_adam(s, groups)
    orf.set_grads(opt.params, g)
    orf.set_grads([x for gr in groups for x in gr], g)
    total = opt.step()
    want = orf.torch_step(s, adam, float(opt.table[0, 0]), float(opt.table[0, 1]))
    assert not np.isfinite(float(total)) and (np.isnan(float(total)) == np.isnan(float(want)))
    assert int(opt.status.item()) & 256
    for x, y in zip(opt.params, [x for gr in groups for x in gr]):
        assert torch.equal(torch.isnan(x.detach()), torch.isnan(y.detach()))
    assert any(torch.isnan(x.detach()).any() for x in opt.params)


def test_captured_step_replays_along_the_schedule():
    """the step (with the copy that refills the persistent gradients) captured in a CUDA graph -- capture would raise
    on a host synchronisation -- and replayed 5 times equals 5 eager steps bit for bit: the schedule advances from the
    device counter and the tables are not rebuilt"""
    s = orf.ONE_CYCLE
    case = orf.make_case("above", seed=11, steps=2)
    runs = []
    for captured in (False, True):
        net, opt = _plan(case, s, 20)
        feed = [torch.from_numpy(g).to(DEV) for g in case["grads"][1]]
        orf.set_grads(opt.params, case["grads"][0])
        opt.step()                                                   # eager: builds the tables

        def one():
            for x, g in zip(opt.params, feed):
                x.grad.copy_(g)
            return opt.step()

        if captured:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                norm = one()
            assert opt.global_step == 1                              # capture ran nothing
            for _ in range(5):
                graph.replay()
        else:
            for _ in range(5):
                norm = one()
        torch.cuda.synchronize()
        assert opt.global_step == 6 and opt.table_builds == 1
        assert opt.lr == opt.table[6, 0] and opt.mom == opt.table[6, 1]
        runs.append(_bits(opt) + [norm.clone()])
    assert _same_bits(*runs)


@pytest.fixture(params=[True, False], ids=["tc", "fp32"])
def pipe(request, product, monkeypatch):
    monkeypatch.setattr(product, "USE_TENSOR_CORES", request.param)
    return request.param


def _lite_middle(product, oracle, n=12000):
    from test_gpu_sparse_backward import _middle_inputs, _smooth
    cfg, onet, vf, coords = _middle_inputs("car.lite", 1, n, oracle)

    def make(state):
        net = models.build_network(cfg, product)
        net.load_state_dict(onet.state_dict())
        mid = _smooth(training.enable_sparse_backward(net.middle_feature_extractor.to(DEV)).train())
        if state is not None:
            mid.load_state_dict(state)
        return mid
    return make, vf.to(DEV), coords.to(DEV)


@pytest.mark.timeout(600)
def test_forward_after_a_step_sees_the_new_weights(product, oracle, pipe):
    """forward -> backward -> opt.step() -> forward on car.lite's middle encoder on the drop-in: the second forward
    equals that of a fresh module loaded with the stepped weights (the packed fp16 weight planes and the folded batch
    norms are keyed on the parameters' versions, which step() bumps), in train() and, after it, in eval()"""
    make, vf, coords = _lite_middle(product, oracle)
    mid = make(None)
    opt = optim.plan(mid, dataclasses.replace(orf.ONE_CYCLE, lr_max=optim._f32(0.05)), 100)
    gen = torch.Generator().manual_seed(3)
    with torch.no_grad():
        mid.eval()
        before_eval = mid(vf, coords, 1).clone()                     # fills the eval-mode caches too
        mid.train()
    out = mid(vf, coords, 1)
    w = (torch.randn(out.shape, generator=gen) / out.numel() ** 0.5).to(DEV)
    (out * w).sum().backward()
    opt.step()
    fresh = make({k: v.clone() for k, v in mid.state_dict().items()})
    out2, want2 = mid(vf, coords, 1), fresh(vf, coords, 1)
    scale = float(want2.abs().max())
    assert float((out2 - out).abs().max()) > 1e-4 * scale            # the step moved the output
    assert float((out2 - want2).abs().max()) <= 1e-6 * scale
    with torch.no_grad():
        e, we = mid.eval()(vf, coords, 1), fresh.eval()(vf, coords, 1)
    assert float((e - before_eval).abs().max()) > 1e-4 * float(we.abs().max())
    assert float((e - we).abs().max()) <= 1e-6 * float(we.abs().max())


@pytest.mark.timeout(600)
def test_three_training_steps_match_the_torch_sequence(product, oracle):
    """twin car.lite middle encoders on the drop-in, same weights and inputs, loss = sum(dense_out * G): three steps
    with b2second.optim against three with clip_grad_norm_, the decay loop and torch.optim.Adam driven by the same
    schedule.  The first step's gradients are identical, so it differs by the optimizer's rounding alone; from the
    second on the twins' gradients differ by the rounding-sized difference of their weights, which Adam's g / sqrt(v)
    turns into a visible fraction of a step only where an element's gradient is itself rounding-sized.  So: 99% of
    all elements within 6 EPS32 |p| + 1% of the three steps' learning rates, and every element within the two full
    step lengths any two Adam runs stay within."""
    make, vf, coords = _lite_middle(product, oracle)
    s = orf.ONE_CYCLE
    a, b = make(None), make(None)
    p0 = [x.detach().clone() for x in a.parameters()]
    opt = optim.plan(a, s, 100)
    groups = optim.parameter_groups(b)
    adam = orf.torch_adam(s, groups)
    gen = torch.Generator().manual_seed(4)
    for i in range(3):
        outs = a(vf, coords, 1), b(vf, coords, 1)
        w = (torch.randn(outs[0].shape, generator=gen) * 30 / outs[0].numel() ** 0.5).to(DEV)
        for o in outs:
            (o * w).sum().backward()
        if i == 0:
            for x, y in zip(a.parameters(), b.parameters()):
                assert float((x.grad - y.grad).abs().max()) <= 1e-6 * float(y.grad.abs().max())
        got = opt.step()
        want = orf.torch_step(s, adam, float(opt.table[i, 0]), float(opt.table[i, 1]))
        assert abs(float(got) - float(want)) <= 1e-4 * float(want)
    lr_sum = float(opt.table[:3, 0].sum())
    named = dict(b.named_parameters())
    inside = []
    for (k, x), x0 in zip(a.named_parameters(), p0):
        diff = (x.detach() - named[k].detach()).abs()
        tight = 6 * orf.EPS32 * x.detach().abs() + 0.01 * lr_sum
        inside.append((diff <= tight).flatten())
        assert float(diff.max()) <= 2.2 * lr_sum + float(tight.max()), k
        assert float((x.detach() - x0).abs().max()) > 0.5 * float(opt.table[0, 0]), k
    assert float(torch.cat(inside).float().mean()) >= 0.99
