"""Train-mode BatchNorm + ReLU pairs on the H100 (b2s_bn_relu_train_forward / _backward through b2second.bn_train)
against the float64 reference of tests/bn_train_ref.py: y, the running buffers, num_batches_tracked, dX, dgamma and
dbeta within their bounds at car.fhd's RPN map (B = 8), xyres_16's maps (B = 2) in both layouts and at the edges; Inf
and NaN as torch carries them; bit-reproducible and capturable; every pair of a mirror car.fhd training step (the
middle encoder's row sets from bench-sized clouds, B = 8) checked from its own input; eval() unchanged."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import bn_train_ref as R
from b2second import bn_train, config, loader, loss, models, training

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MOM, EPS = 0.01, 1e-3
# momentum and eps as the kernels receive them (fp32), so the reference starts from the same numbers: with M = 2 the
# input gradient is proportional to eps / (var + eps), so even eps's fp32 rounding shows at the ulp level
MOM32, EPS32 = (float(np.float32(v)) for v in (MOM, EPS))


def _pair(C, dim, seed):
    torch.manual_seed(seed)
    bn = (nn.BatchNorm1d if dim == 2 else nn.BatchNorm2d)(C, eps=EPS, momentum=MOM)
    seq = nn.Sequential(bn, nn.ReLU()).to(DEV).train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
    return training.enable_bn_relu_training(seq)


def run(seq, x, dy):
    """forward and backward of the fused pair -> (y, dx, dgamma, dbeta, rm0, rv0) with the buffers before the step"""
    bn = seq[0]
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    bn.weight.grad = bn.bias.grad = None
    x = x.detach().clone().requires_grad_(True)
    y = seq(x)
    assert type(y.grad_fn).__name__ == "BNReLUTrainBackward", "the pair did not take the kernels"
    y.backward(dy)
    return y.detach(), x.grad, bn.weight.grad, bn.bias.grad, rm0, rv0


def check(bn, x, dy, out, limit=1.0):
    """every result of ``out`` (run()'s) within its bound of the float64 reference -> the worst ratio"""
    y, dx, dg, db, rm0, rv0 = out
    g, b = bn.weight.detach(), bn.bias.detach()
    xr = R.rows(x)
    fw = R.forward(xr, g, b, rm0, rv0, MOM32, EPS32)
    bw = R.backward(xr, R.rows(dy), R.rows(y), g, fw)
    ratios = {"y": R.ratio(R.rows(y), fw["y"], fw["y_bound"]),
              "running_mean": R.ratio(bn.running_mean, fw["running_mean"], fw["running_mean_bound"]),
              "running_var": R.ratio(bn.running_var, fw["running_var"], fw["running_var_bound"]),
              "dx": R.ratio(R.rows(dx), bw["dx"], bw["dx_bound"]),
              "dgamma": R.ratio(dg, bw["dgamma"], bw["dgamma_bound"]),
              "dbeta": R.ratio(db, bw["dbeta"], bw["dbeta_bound"])}
    for k, r in ratios.items():
        assert r <= limit, (k, r, ratios)
    assert y.stride() == x.stride() and dx.stride() == x.stride()
    return max(ratios.values())


def _map(B, C, H, W, cl, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, C, H, W, device=DEV, generator=gen) * 0.7 + 0.3
    dy = torch.randn(B, C, H, W, device=DEV, generator=gen)
    fmt = torch.channels_last if cl else torch.contiguous_format
    return x.contiguous(memory_format=fmt), dy.contiguous(memory_format=fmt)


def test_carfhd_rpn_map_b8():
    """rows 281,600 x 128: car.fhd's RPN map at B = 8 as Conv3x3TC returns it (channels_last)"""
    seq = _pair(128, 4, 0)
    x, dy = _map(8, 128, 200, 176, True, 1)
    check(seq[0], x, dy, run(seq, x, dy))
    assert int(seq[0].num_batches_tracked) == 1


@pytest.mark.parametrize("cl", [False, True])
@pytest.mark.parametrize("C,H,W", [(64, 248, 216), (128, 124, 108), (256, 62, 54)])
def test_xyres16_maps_b2(C, H, W, cl):
    seq = _pair(C, 4, C)
    x, dy = _map(2, C, H, W, cl, C + 1)
    check(seq[0], x, dy, run(seq, x, dy))


@pytest.mark.parametrize("layout", ["rows", "nchw", "nchw_odd"])
def test_edges(layout):
    """M = 2 (rows) / a small map; channel 0 constant (var = 0), channel 1 with |mean| / std = 1e4, channel 2 all
    negative after the shift (every gradient killed by the ReLU)"""
    C = 16
    gen = torch.Generator(device=DEV).manual_seed(5)
    if layout == "rows":
        x = torch.randn(2, C, device=DEV, generator=gen)
    else:
        x = torch.randn(3, C, 5, 7 if layout == "nchw_odd" else 8, device=DEV, generator=gen)   # HW odd: scalar path
    x[:, 0] = 3.0
    x[:, 1] = x[:, 1] * 1e-2 + 100.0
    dy = torch.randn(x.shape, device=DEV, generator=gen)
    seq = _pair(C, x.dim(), 7)
    with torch.no_grad():
        seq[0].bias[2] = -100.0
    out = run(seq, x, dy)
    check(seq[0], x, dy, out)
    y, dx, dg, db = out[:4]
    assert bool((R.rows(y)[:, 0] == max(float(seq[0].bias[0]), 0.0)).all())          # x - mean = 0 exactly
    assert bool((R.rows(y)[:, 2] == 0).all()) and float(dg[2]) == 0.0 and float(db[2]) == 0.0
    assert bool((R.rows(dx)[:, 2] == 0).all())


def test_nonfinite_as_torch():
    """NaN / Inf in x and NaN in dY give non-finite results exactly where torch's BatchNorm2d + ReLU give them"""
    C = 12
    gen = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(2, C, 6, 8, device=DEV, generator=gen)
    dy = torch.randn(x.shape, device=DEV, generator=gen)
    x[1, 3, 2, 2] = float("nan")
    x[0, 5, 1, 1] = float("inf")
    x[0, 7, 0, 0] = -float("inf")
    seq = _pair(C, 4, 11)
    with torch.no_grad():
        y_probe = torch.relu(torch.nn.functional.batch_norm(x, None, None, seq[0].weight, seq[0].bias, True, eps=EPS))
    dead = (y_probe[:, 8] == 0).nonzero()[0]
    dy[dead[0], 8, dead[1], dead[2]] = float("nan")            # masked by the ReLU: no effect
    live = (y_probe[:, 9] > 0).nonzero()[0]
    dy[live[0], 9, live[1], live[2]] = float("nan")            # passes the ReLU: channel 9's sums are NaN
    ref = nn.Sequential(nn.BatchNorm2d(C, eps=EPS, momentum=MOM), nn.ReLU()).to(DEV).train()
    ref.load_state_dict(seq.state_dict())
    y, dx, dg, db, _, _ = run(seq, x, dy)
    xt = x.clone().requires_grad_(True)
    yt = ref(xt)
    yt.backward(dy)
    for got, want in ((y, yt), (dx, xt.grad), (dg, ref[0].weight.grad), (db, ref[0].bias.grad),
                      (seq[0].running_mean, ref[0].running_mean), (seq[0].running_var, ref[0].running_var)):
        fin = torch.isfinite(want)
        assert torch.equal(torch.isfinite(got), fin)
        assert torch.allclose(got[fin], want[fin].detach(), rtol=1e-4, atol=1e-4)


def _abi_step(t, rm, rv, nbt, ws, outs, layout, B, C, S):
    L, lib = bn_train._lib()
    y, dx, dg, db = outs
    L.check(lib.b2s_bn_relu_train_forward(L.ptr(t["x"]), layout, B, C, S, L.ptr(t["g"]), L.ptr(t["b"]), L.ptr(rm),
                                          L.ptr(rv), L.ptr(nbt), MOM, EPS, L.ptr(y), L.ptr(ws), ws.numel(), L.stream()),
            "forward")
    L.check(lib.b2s_bn_relu_train_backward(L.ptr(t["x"]), L.ptr(t["dy"]), layout, B, C, S, L.ptr(t["g"]), L.ptr(ws),
                                           ws.numel(), L.ptr(dx), L.ptr(dg), L.ptr(db), L.stream()), "backward")


@pytest.mark.parametrize("layout", [0, 1])
def test_bit_reproducible_and_capturable(layout):
    """two runs and a CUDA-graph replay of forward + backward give the same bits (outputs and running buffers)"""
    L, lib = bn_train._lib()
    B, C, H, W = 4, 64, 100, 88
    x, dy = _map(B, C, H, W, layout == 1, 21)
    g = torch.rand(C, device=DEV) + 0.5
    b = torch.rand(C, device=DEV) - 0.5
    t = dict(x=x, dy=dy, g=g, b=b)
    S = H * W
    ws = torch.empty(int(lib.b2s_bn_relu_train_workspace_bytes(layout, B, C, S)), dtype=torch.uint8, device=DEV)
    rm, rv, nbt = torch.zeros(C, device=DEV), torch.ones(C, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    res = []
    outs = (torch.empty_like(x), torch.empty_like(x), torch.empty(C, device=DEV), torch.empty(C, device=DEV))
    for _ in range(2):
        rm.zero_(), rv.fill_(1.0), nbt.zero_()
        _abi_step(t, rm, rv, nbt, ws, outs, layout, B, C, S)
        torch.cuda.synchronize()
        res.append([o.clone() for o in outs] + [rm.clone(), rv.clone(), nbt.clone()])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _abi_step(t, rm, rv, nbt, ws, outs, layout, B, C, S)
    torch.cuda.current_stream().wait_stream(s)
    for o in outs:
        o.zero_()
    rm.zero_(), rv.fill_(1.0), nbt.zero_()
    graph.replay()
    torch.cuda.synchronize()
    res.append([o.clone() for o in outs] + [rm.clone(), rv.clone(), nbt.clone()])
    for a, c in zip(res[0], res[1]):
        assert torch.equal(a, c)
    for a, c in zip(res[0], res[2]):
        assert torch.equal(a, c)
    assert int(res[2][-1]) == 1


def _example(net, cfg, B):
    """B frames of bench-sized KITTI clouds (29 k points) through the CPU oracle's voxelizer, with GPU targets"""
    from b2second import synth, targets
    onet = models.build_network(cfg, loader.oracle_spconv())
    vox, num, coors = [], [], []
    for f in range(B):
        res = onet.voxel_generator.generate(synth.kitti_cloud(30 + f, 29000, cfg.point_cloud_range), cfg.max_voxels)
        vox.append(res["voxels"])
        num.append(res["num_points_per_voxel"])
        coors.append(np.pad(res["coordinates"], ((0, 0), (1, 0)), constant_values=f))
    anchors = net.anchors()
    tp = targets.plan(net.target_assigner, cfg.feature_map_size)
    rng = np.random.default_rng(3)
    gt = anchors[rng.integers(0, len(anchors), 6 * B)].astype(np.float32).copy()
    gt[:, :2] += rng.uniform(-0.5, 0.5, (6 * B, 2)).astype(np.float32)
    gt[:, 6] = rng.uniform(-np.pi, np.pi, 6 * B).astype(np.float32)
    tg = tp.assign_batch(torch.from_numpy(gt).to(DEV), torch.arange(0, 6 * B + 1, 6, dtype=torch.int32, device=DEV),
                         torch.ones(6 * B, dtype=torch.int32, device=DEV))
    ex = {"voxels": torch.from_numpy(np.concatenate(vox)).to(DEV),
          "num_points": torch.from_numpy(np.concatenate(num)).to(DEV),
          "coordinates": torch.from_numpy(np.concatenate(coors)).to(DEV),
          "anchors": torch.from_numpy(np.repeat(anchors[None], B, 0)).to(DEV)}
    ex.update(tg)
    return ex


def _net(name, fused):
    cfg = config.get_config(name)
    net = models.build_network(cfg, loader.product_spconv())
    models.synthetic_weights_(net, name, seed=0)
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV)))
    net = training.enable_rpn_training(net)
    if fused:
        net = training.enable_bn_relu_training(net)
    return net, cfg


@pytest.mark.timeout(900)
def test_carfhd_training_step_every_pair():
    """a mirror car.fhd training step at B = 8 with enable_sparse_backward + enable_rpn_training +
    enable_bn_relu_training: every one of the 21 pairs takes the kernels, and its y, running buffers, dX, dgamma and
    dbeta are within their bounds of the float64 reference from the pair's own input and upstream gradient"""
    net, cfg = _net("car.fhd", True)
    net.train()
    ex = _example(net, cfg, 8)
    pairs = bn_train.select(net)
    assert len(pairs) == 21
    seen = {}

    def pre(bn, inputs):
        x = inputs[0]
        rec = seen.setdefault(id(bn), {})
        rec.update(x=x.detach().clone(), rm0=bn.running_mean.clone(), rv0=bn.running_var.clone())
        if x.requires_grad:
            x.register_hook(lambda g: rec.__setitem__("dx", g.detach().clone()))

    def post(bn, inputs, y):
        rec = seen[id(bn)]
        rec.update(y=y.detach().clone(), fused=type(y.grad_fn).__name__ == "BNReLUTrainBackward")
        y.register_hook(lambda g: rec.__setitem__("dy", g.detach().clone()))
    hooks = [h for bn, _ in pairs for h in (bn.register_forward_pre_hook(pre), bn.register_forward_hook(post))]
    r = net(ex)
    r["loss"].backward()
    for h in hooks:
        h.remove()
    torch.cuda.synchronize()
    rows_seen = set()
    for bn, _ in pairs:
        rec = seen[id(bn)]
        assert rec["fused"], bn
        if rec["x"].dim() == 2:
            rows_seen.add(rec["x"].shape[0])
        check(bn, rec["x"], rec["dy"], (rec["y"], rec["dx"], bn.weight.grad, bn.bias.grad, rec["rm0"], rec["rv0"]))
        assert int(bn.num_batches_tracked) == 1
    assert len(rows_seen) >= 4 and min(rows_seen) > 1000, rows_seen      # the middle encoder's row sets


@pytest.mark.timeout(600)
def test_eval_unchanged_by_the_opt_in():
    """eval() outputs of car.fhd on the drop-in are bit-identical with and without enable_bn_relu_training"""
    outs = []
    ex = None
    for fused in (False, True):
        net, cfg = _net("car.fhd", fused)
        net.eval()
        ex = ex or _example(net, cfg, 2)
        with torch.no_grad():
            r = net({k: v for k, v in ex.items() if k in ("voxels", "num_points", "coordinates", "anchors")})
        outs.append(r if isinstance(r, list) else [r])
    assert len(outs[0]) == len(outs[1]) == 2
    for a, b in zip(outs[0], outs[1]):
        for k in a:
            if torch.is_tensor(a[k]):
                assert torch.equal(a[k], b[k]), k
