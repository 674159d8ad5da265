"""PointPillars' pillar feature net in training on the H100 (b2s_pfn_train_forward / b2s_pfn_train_backward through
b2second.pfn_train) against the float64 reference of tests/pfn_train_ref.py: the output, the BatchNorm1d buffers and
dW / dgamma / dbeta within their per-element bounds at both timing sizes and at the edges; simulated faults rejected;
bit-reproducible and capturable; a whole xyres_16 training step against the torch PFN and scatter."""
import numpy as np
import pytest
import torch

import fp32_ref as R
import pfn_train_ref as P
from b2second import config, loader, loss, models, pfn_train, training

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# the geometry as the kernels receive it (fp32), so the reference starts from the same numbers
GEOM = tuple(float(np.float32(v)) for v in (0.16, 0.16, 0.08, -39.6))
MOM, EPS = 0.01, 1e-3

# (seed, pillars, T, F, radius, frames): the xyres_16 training batch (2 x 12000 pillars, T = 100), the all.pp.mhead one
# (3 x 25000, T = 60, radius decoration), and a small batch with an empty frame (frame 1 holds no pillar)
CASES = {"xyres16_b2": (0, 24000, 100, 4, False, 2), "mhead_b3": (1, 75000, 60, 4, True, 3),
         "edges_empty_frame": (2, 700, 32, 5, False, 3)}


def run(vox, num, coors, w, g, b, rm, rv, dout, radius, graph=False):
    """one forward and one backward through the C ABI on fresh copies of the buffers -> dict of results"""
    L, lib = pfn_train._lib()
    N, T, F = vox.shape
    t = {k: v.to(DEV).contiguous() for k, v in dict(vox=vox, num=num, coors=coors, w=w, g=g, b=b, dout=dout).items()}
    rm, rv = rm.to(DEV).clone(), rv.to(DEV).clone()
    nbt = torch.zeros((), dtype=torch.int64, device=DEV)
    nbytes = int(lib.b2s_pfn_train_workspace_bytes(N))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = torch.empty(N, 64, device=DEV)
    arg = torch.empty(N, 64, dtype=torch.uint8, device=DEV)
    dw, dg, db = torch.empty_like(t["w"]), torch.empty(64, device=DEV), torch.empty(64, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    deco = 1 if radius else 0

    def calls():
        L.check(lib.b2s_pfn_train_forward(
            L.ptr(t["vox"]), N, T, F, L.ptr(t["num"]), L.ptr(t["coors"]), L.ptr(t["w"]), L.ptr(t["g"]), L.ptr(t["b"]),
            64, L.ptr(rm), L.ptr(rv), L.ptr(nbt), MOM, EPS, *GEOM, deco, L.ptr(out), L.ptr(arg), L.ptr(ws), nbytes,
            L.ptr(status), L.stream()), "b2s_pfn_train_forward")
        L.check(lib.b2s_pfn_train_backward(
            L.ptr(t["vox"]), N, T, F, L.ptr(t["num"]), L.ptr(t["coors"]), L.ptr(t["w"]), L.ptr(t["g"]), 64, *GEOM,
            deco, L.ptr(out), L.ptr(arg), L.ptr(t["dout"]), L.ptr(ws), nbytes, L.ptr(dw), L.ptr(dg), L.ptr(db),
            L.stream()), "b2s_pfn_train_backward")
    if graph:
        calls()                                    # warm-up, then reset the buffers and replay the captured pair
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            calls()
        rm.copy_(rv.new_tensor(P_RM[0]))
        rv.copy_(rv.new_tensor(P_RM[1]))
        nbt.zero_()
        gr.replay()
    else:
        calls()
    torch.cuda.synchronize()
    return dict(out=out, arg=arg, dW=dw, dgamma=dg, dbeta=db, running_mean=rm, running_var=rv, nbt=int(nbt),
                status=int(status))


P_RM = [None, None]


def _case(name):
    seed, n, T, F, radius, frames = CASES[name]
    c = list(P.case(seed, n, T, F, radius, batch=frames))
    if name == "edges_empty_frame":
        coors = c[2]
        coors[:, 0] = torch.where(coors[:, 0] == 1, torch.zeros_like(coors[:, 0]), coors[:, 0])
        assert not bool((coors[:, 0] == 1).any())
        assert bool((c[1] == T).any()) and bool((c[1] == 1).any())
        ys, xs = coors[:, 2], coors[:, 3]
        assert int(ys.min()) == 0 and int(xs.min()) == 0 and int(ys.max()) == 495 and int(xs.max()) == 431
    return c, radius


@pytest.fixture(scope="module", params=sorted(CASES))
def result(request):
    c, radius = _case(request.param)
    got = run(*c, radius)
    ref = P.reference(*[x.to(DEV) for x in c[:8]], MOM, EPS, *GEOM, radius, c[8].to(DEV))
    return request.param, c, radius, got, ref


KEYS = ("out", "running_mean", "running_var", "dW", "dgamma", "dbeta")


def test_against_float64(result):
    name, c, radius, got, ref = result
    assert got["status"] == 0 and got["nbt"] == 1
    ratios = {k: P.ratio(got[k], ref[k]) for k in KEYS}
    print(name, {k: "%.3g" % v for k, v in ratios.items()})
    for k in KEYS:
        assert ratios[k] <= 1.0, (name, k, ratios)
    assert bool((ref["raw"]["arg"] == c[0].shape[1]).any()), "some maximum is the padded value"
    R.assert_accurate(got["out"], ref["out_aggregate"], name)       # fp32_ref's per-element bound and RHO aggregate


@pytest.mark.parametrize("fault", P.FAULTS)
def test_faults_are_rejected(result, fault):
    name, c, radius, got, ref = result
    N, T = c[0].shape[:2]
    if fault == "biased_var" and N * T > 3_000_000:
        pytest.skip("M / (M - 1) - 1 = %.1e: below the fp32 rounding of running_var" % (1.0 / (N * T - 1)))
    bad = P.reference(*[x.to(DEV) for x in c[:8]], MOM, EPS, *GEOM, radius, c[8].to(DEV), fault=fault)
    ratios = {k: P.ratio(got[k].double() + (bad[k].y - ref[k].y), ref[k]) for k in KEYS}
    assert max(ratios.values()) > 1.0, (name, fault, ratios)


def test_bits_repeat_and_replay_from_a_graph():
    c, radius = _case("xyres16_b2")
    P_RM[0], P_RM[1] = c[6].tolist(), c[7].tolist()
    a, b = run(*c, radius), run(*c, radius)
    g = run(*c, radius, graph=True)
    for k in ("out", "arg", "dW", "dgamma", "dbeta", "running_mean", "running_var"):
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(a[k], g[k]), k
    assert a["nbt"] == b["nbt"] == g["nbt"] == 1


def test_bad_counts_raise_the_status():
    c, radius = _case("edges_empty_frame")
    c[1] = c[1].clone()
    c[1][5] = 0
    c[1][6] = c[0].shape[1] + 3
    assert run(*c, radius)["status"] == 32           # B2S_STATUS_BAD_INPUT


def _example(net, cfg, B=2):
    """B frames of bench-sized KITTI clouds through the CPU oracle's voxelizer, with GPU-assigned targets"""
    from b2second import synth, targets
    onet = models.build_network(cfg, loader.oracle_spconv())
    vox, num, coors = [], [], []
    for f in range(B):
        res = onet.voxel_generator.generate(synth.kitti_cloud(10 + f, 29000, cfg.point_cloud_range), cfg.max_voxels)
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


@pytest.fixture
def fp32_torch():
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


@pytest.mark.timeout(900)
def test_xyres16_training_step_against_torch_pfn(fp32_torch):
    """xyres_16 at B = 2 with enable_sparse_backward, enable_gpu_loss, enable_rpn_training and enable_pfn_training
    against the same step with the torch PFN and scatter, from the same weights: the loss scalars within 1e-5, the PFN
    parameter gradients within their bounds for the upstream gradient the step fed the PFN, the status word 0"""
    name = "pointpillars.car.xyres_16"
    cfg = config.get_config(name)
    sp = loader.product_spconv()
    runs = []
    ex = None
    for ours in (True, False):
        net = models.build_network(cfg, sp)
        models.synthetic_weights_(net, name, seed=0)
        net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV)))
        net = training.enable_rpn_training(net)
        if ours:
            net = training.enable_pfn_training(net)
        net.train()
        ex = ex or _example(net, cfg)
        bn = net.voxel_feature_extractor.pfn_layers[0].norm
        rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
        up = {}
        def grab(module, inputs, output):
            output.register_hook(lambda g: up.__setitem__("g", g.detach().clone()))
        h = net.voxel_feature_extractor.register_forward_hook(grab)
        r = net(ex)
        r["loss"].backward()
        h.remove()
        scalars = {k: float(v.detach()) for k, v in r.items() if torch.is_tensor(v) and v.numel() == 1
                   and v.is_floating_point()}
        runs.append((net, scalars, up["g"], rm0, rv0))
    (net, mine, g_up, rm0, rv0), (_, theirs, _, _, _) = runs
    assert mine.keys() == theirs.keys() and "loss" in mine
    for k in mine:
        assert abs(mine[k] - theirs[k]) <= 1e-5 * max(abs(theirs[k]), 1e-6), (k, mine[k], theirs[k])
    vfe = net.voxel_feature_extractor
    assert int(vfe._b2s_pfn_status) == 0
    lyr = vfe.pfn_layers[0]
    ref = P.reference(ex["voxels"], ex["num_points"], ex["coordinates"], lyr.linear.weight.detach(),
                      lyr.norm.weight.detach(), lyr.norm.bias.detach(), rm0, rv0, MOM, EPS,
                      *(float(np.float32(v)) for v in pfn_train.geometry(vfe)),
                      False, g_up)
    got = dict(dW=lyr.linear.weight.grad, dgamma=lyr.norm.weight.grad, dbeta=lyr.norm.bias.grad,
               running_mean=lyr.norm.running_mean, running_var=lyr.norm.running_var)
    for k, v in got.items():
        assert P.ratio(v, ref[k]) <= 1.0, k
