"""Data-parallel training on GPUs (b2second.dist.enable_data_parallel): the split metric entry points on one GPU, and
whole training steps on two or more NCCL ranks against a one-GPU emulation of torch.nn.DataParallel's step.

The emulation runs every rank's share on one GPU with the same parameters, accumulates ``(1/W) * loss_r`` into the
gradients, keeps the BatchNorm running buffers after share 0 (DataParallel's replica 0 is the module itself), adds the
shares' metric count records and takes one optimizer step.  For W = 2 the data-parallel step equals it bit for bit:
scaling by 1/2 is exact, the sum of two fp32 gradients is one rounding in either order, and every kernel on the path
is deterministic.  For W > 2 the summation order differs, so the ranks are compared with each other bit for bit and
with the emulation within a bound.

The NCCL tests need one device per rank and skip with a reason on fewer.  On one device, two gloo ranks share the GPU
(enable_data_parallel refuses gloo, so the test builds the handle itself and sums then halves the bucket where NCCL's
AVG would pre-multiply by 1/2 and sum: the same arithmetic for W = 2); that checks the bucket, the optimizer hook, the
metric count sum and the BatchNorm rule, not NCCL."""
import datetime
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import optim_ref as orf
import train_ref as tr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POINTS = 29000
STEPS = 3
CONFIGS = {"car.fhd": 2, "pointpillars.car.xyres_16": 2}       # name: frames per rank


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


# ---- the split metric entry points ------------------------------------------------------------------------------------
def _metric_batch(g, B, A, C):
    cls = torch.randn(B, A, C, device=DEV, generator=g) * 3
    labels = torch.randint(-1, C + 1, (B, A), device=DEV, generator=g)
    cared = torch.rand(B, A, device=DEV, generator=g) < 0.7
    # loc_loss elements on a coarse dyadic grid, so their float64 sums round to float32 the same per half and whole
    loc = torch.randint(0, 64, (B, A, 7), device=DEV, generator=g).float() / 64
    mask = torch.rand(B, A, device=DEV, generator=g) < 0.8
    return cls, labels, cared, loc, mask


def _scalars(vals):
    return [torch.tensor([v], dtype=torch.float32, device=DEV) for v in vals]


def test_count_then_finish_equals_the_one_call():
    """count on each half of a batch, add the two records, finish with loss_scale 1/2: the running buffers and the log
    record equal b2s_train_metrics on the whole batch bit for bit (per-half losses whose mean is exact)"""
    from b2second import config, loader, metrics, models
    import test_gpu_metrics as tgm
    name = "car.fhd"
    B, A, C = 4, 70400 * 2, 1
    one = metrics.enable_gpu_metrics(models.build_network(config.get_config(name), loader.product_spconv()).to(DEV))
    two = metrics.enable_gpu_metrics(models.build_network(config.get_config(name), loader.product_spconv()).to(DEV))
    g = torch.Generator(device=DEV).manual_seed(3)
    h = B // 2
    for step in range(3):
        cls, labels, cared, loc, mask = _metric_batch(g, B, A, C)
        # per-half losses (cls, loc, cls_pos, cls_neg, dir) and the whole batch's, their exact mean
        halves = [_scalars([0.75 + step, 0.5, 0.25, 1.5, 0.125]), _scalars([1.25 + step, 0.0, 0.75, 0.5, 0.375])]
        whole = _scalars([1.0 + step, 0.25, 0.5, 1.0, 0.25])

        def ret(s, sl):
            return {"loc_loss": loc[sl], "cls_pos_loss": s[2], "cls_neg_loss": s[3], "dir_loss_reduced": s[4]}

        want = one.b2s_metrics.update_metrics_async(whole[0], whole[1], cls, labels, cared, ret(whole, slice(None)),
                                                    mask)
        parts = []
        for k, sl in enumerate((slice(0, h), slice(h, B))):
            s = halves[k]
            parts.append(two.b2s_metrics.count(s[0], s[1], cls[sl], labels[sl], cared[sl], ret(s, sl), mask[sl],
                                               has_frame0=k == 0))
        got = two.b2s_metrics.finish(parts[0] + parts[1], 0.5)
        torch.cuda.synchronize()
        assert _same(got.record, want.record), (step, got.record, want.record)
        assert got.result() == want.result() and got.step_log() == want.step_log()
        s1, s2 = tgm._state(one), tgm._state(two)
        for k in s1:
            assert np.array_equal(s1[k].view(np.int32), s2[k].view(np.int32)), (step, k, s1[k], s2[k])
    # the frame-0 figures are the first frame's: a share without it adds zeros
    c = two.b2s_metrics.count(*_scalars([1.0, 1.0]), cls[h:], labels[h:], cared[h:], None, mask[h:], has_frame0=False)
    from spconv import _lib as L
    cnt = dict(zip(L.METRICS_CNT, c.cpu().tolist()))
    assert cnt["num_pos"] == cnt["num_neg"] == cnt["num_anchors"] == 0 and cnt["frames"] == B - h


# ---- training steps on several ranks ----------------------------------------------------------------------------------
def build(name, precision, seed=0, device=DEV):
    """the mirror network of `name` with every GPU training stage switched on, seeded synthetic weights, train()"""
    from b2second import config, loader, loss, metrics, models, training
    net = models.build_network(config.get_config(name), loader.product_spconv())
    models.synthetic_weights_(net, name, seed=seed)
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(device), precision=precision))
    net = training.enable_rpn_training(net, precision=precision)
    net = training.enable_bn_relu_training(training.enable_pfn_training(net))
    return metrics.enable_gpu_metrics(net).train()


def share(net, name, start, stop, device=DEV):
    """the example of global frames start .. stop - 1 of the seeded global batch: frame g's cloud has seed g and its
    ground truths come from rng(1000 + g), so a share does not depend on how the batch is split"""
    import bench
    from b2second import config, inputs, loader, targets
    cfg = config.get_config(name)
    B = stop - start
    plan = targets.plan(net.target_assigner, cfg.feature_map_size)
    clouds = bench.make_clouds(name, B, POINTS, seed0=start)
    gen = loader.product_spconv().utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range,
                                                        cfg.max_points_per_voxel, cfg.max_voxels)
    offs = np.cumsum([0] + [c.shape[0] for c in clouds]).astype(np.int32)
    pts = torch.from_numpy(np.concatenate(clouds, 0)).to(device)
    res = gen.generate_device(pts, cfg.max_voxels, frame_offsets=torch.from_numpy(offs).to(device), batch=B)
    n = int(res["num_voxels"][0].item())
    ex = {"voxels": res["voxels"][:n], "num_points": res["num_points_per_voxel"][:n],
          "coordinates": res["coordinates"][:n]}
    mask = None
    if cfg.anchor_area_threshold >= 0:
        mask = inputs.anchor_area_mask(ex["coordinates"], B, plan.anchors, cfg.voxel_size, cfg.point_cloud_range,
                                       cfg.grid_size, cfg.anchor_area_threshold)
    frames = [tr.gt_boxes(plan, np.random.default_rng(1000 + g), "ordinary") for g in range(start, stop)]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)   # noqa: E731
    ex.update(plan.assign_batch(t(np.concatenate([f[0] for f in frames])),
                                t(np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)),
                                t(np.concatenate([f[1] for f in frames])), t(np.concatenate([f[2] for f in frames])),
                                mask))
    ex["anchors"] = torch.from_numpy(net.anchors().reshape(-1, 7)).to(device)[None].repeat(B, 1, 1)
    return ex, mask


def _bn(net):
    from b2second import optim
    return [b for m in net.modules() if isinstance(m, optim._BN_TYPES) for b in m.buffers(recurse=False)]


def _metric_bufs(net):
    return [net.rpn_acc.total, net.rpn_acc.count, net.rpn_metrics.prec_total, net.rpn_metrics.prec_count,
            net.rpn_metrics.rec_total, net.rpn_metrics.rec_count, net.rpn_cls_loss.total, net.rpn_cls_loss.count,
            net.rpn_loc_loss.total, net.rpn_loc_loss.count]


def snapshot(net, opt, gnorm, record, grads):
    """the state after a step; grads: {"grad": the averaged gradient the optimizer stepped on, flat in parameter
    order, and on a data-parallel rank "local": the rank's own gradient before the all-reduce}"""
    c = lambda ts: [t.detach().cpu().clone() for t in ts]   # noqa: E731
    return {"params": c(opt.params), "exp_avg": c(opt.exp_avg), "exp_avg_sq": c(opt.exp_avg_sq),
            "gnorm": gnorm.detach().cpu().clone().view(1), "metrics": c(_metric_bufs(net)), "bn": c(_bn(net)),
            "record": record.detach().cpu().clone(), **grads}


def _record_gradients(dp):
    """make the handle keep the bucket before (this rank's gradient) and after its all-reduce; -> the dict it fills"""
    grads, reduce = {}, dp.all_reduce_grads

    def recording():
        grads["local"] = dp.bucket.detach().cpu().clone()
        reduce()
        grads["grad"] = dp.bucket.detach().cpu().clone()
    dp.all_reduce_grads = recording
    return grads


def _gloo_handle(net, world, rank):
    """what enable_data_parallel builds, over a gloo group whose ranks share one device (which it refuses): rank 0's
    state broadcast, the gradient bucket, and SUM then * 1/W in place of NCCL's AVG (the same arithmetic for W = 2)"""
    from b2second import dist as b2dist
    from b2second import optim
    state = list(net.parameters()) + list(net.buffers())
    with torch.no_grad():
        for t in state:
            dist.broadcast(t.data, 0)
    torch.autograd.graph.increment_version(state)
    params = [p for g in optim.parameter_groups(net) for p in g]
    dp = b2dist.DataParallel(net, params, b2dist.attach_grad_bucket(params), world, rank)

    def average():
        assert b2dist.grads_in_bucket(dp.params, dp.bucket)
        dist.all_reduce(dp.bucket)
        dp.bucket.mul_(1.0 / world)
    dp.all_reduce_grads = average
    net.b2s_data_parallel = dp
    return dp


def _metrics_args(ret, ex, mask):
    return (ret["cls_loss_reduced"], ret["loc_loss_reduced"], ret["cls_preds"], ex["labels"], ret["cared"], ret, mask)


def _deterministic():
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _worker(rank, world, port, name, precision, B, out_dir, q, backend):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dev = "cuda:%d" % (rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        timeout = datetime.timedelta(seconds=300)
        if backend == "nccl":
            dist.init_process_group("nccl", rank=rank, world_size=world, timeout=timeout, device_id=torch.device(dev))
        else:
            dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timeout)
        _deterministic()
        from b2second import dist as b2dist
        from b2second import optim, training
        net = build(name, precision, seed=rank, device=dev)          # rank 0's weights must win the broadcast
        if backend == "nccl":
            dp = training.enable_data_parallel(net)
        else:
            dp = _gloo_handle(net, world, rank)
        assert isinstance(dp, b2dist.DataParallel) and (dp.world, dp.rank) == (world, rank)
        grads = _record_gradients(dp)
        torch.save({"params": [p.detach().cpu() for p in net.parameters()],
                    "buffers": [b.detach().cpu() for b in net.buffers()]}, os.path.join(out_dir, "init%d.pt" % rank))
        opt = optim.plan(net, orf.ONE_CYCLE, STEPS, data_parallel=dp)
        ex, mask = share(net, name, rank * B, (rank + 1) * B, device=dev)
        snaps = []
        for _ in range(STEPS):
            ret = net(dict(ex))
            ret["loss"].backward()
            gnorm = opt.step()
            h = net.b2s_metrics.update_metrics_async(*_metrics_args(ret, ex, mask))
            snaps.append(snapshot(net, opt, gnorm, h.record, dict(grads)))
        torch.save(snaps, os.path.join(out_dir, "rank%d.pt" % rank))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:                                          # noqa: BLE001 -- reported to the parent
        q.put((rank, "%s: %s" % (type(e).__name__, e)))


def run_ranks(world, name, precision, B, out_dir, backend="nccl"):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, precision, B, str(out_dir), q, backend))
             for r in range(world)]
    for p in procs:
        p.start()
    res = []
    try:
        for _ in range(world):
            res.append(q.get(timeout=900))
            if res[-1][1] != "ok":
                break
    finally:
        for p in procs:
            p.join(60 if all(r[1] == "ok" for r in res) and len(res) == world else 1)
            if p.is_alive():
                p.kill()
                p.join(30)
    assert sorted(res) == [(r, "ok") for r in range(world)], res
    return [torch.load(os.path.join(out_dir, "rank%d.pt" % r)) for r in range(world)], \
        [torch.load(os.path.join(out_dir, "init%d.pt" % r)) for r in range(world)]


def emulate(world, name, precision, B):
    """torch.nn.DataParallel's step on one GPU: every share with the same parameters, (1/W) * loss_r accumulated into
    the gradients, the BatchNorm buffers kept after share 0, the count records added, one optimizer step"""
    from b2second import optim
    _deterministic()
    net = build(name, precision, seed=0)
    opt = optim.plan(net, orf.ONE_CYCLE, STEPS)
    shares = [share(net, name, r * B, (r + 1) * B) for r in range(world)]
    snaps = []
    for _ in range(STEPS):
        counts, bn0 = None, None
        for r, (ex, mask) in enumerate(shares):
            ret = net(dict(ex))
            (ret["loss"] * (1.0 / world)).backward()
            if r == 0:
                bn0 = [b.detach().clone() for b in _bn(net)]
            c = net.b2s_metrics.count(*_metrics_args(ret, ex, mask), has_frame0=r == 0)
            counts = c if counts is None else counts + c
        with torch.no_grad():
            for b, v in zip(_bn(net), bn0):
                b.copy_(v)
        grad = torch.cat([p.grad.reshape(-1) for p in opt.params]).cpu()
        gnorm = opt.step()
        h = net.b2s_metrics.finish(counts, 1.0 / world)
        snaps.append(snapshot(net, opt, gnorm, h.record, {"grad": grad}))
    return snaps, [p.detach().cpu() for p in net.parameters()], [b.detach().cpu() for b in net.buffers()]


def _need(n):
    have = torch.cuda.device_count()
    if have < n:
        pytest.skip("needs %d CUDA devices, %d visible" % (n, have))
    return have


def _check_init(inits, net_params, net_buffers):
    for r, init in enumerate(inits):
        assert all(_same(a, b) for a, b in zip(init["params"], net_params)), "rank %d: parameters not broadcast" % r
        assert all(_same(a, b) for a, b in zip(init["buffers"], net_buffers)), "rank %d: buffers not broadcast" % r


CASES = [("car.fhd", "fp32"), ("pointpillars.car.xyres_16", "fp32"), ("car.fhd", "f16")]


def _check_two_ranks(name, precision, tmp_path, backend):
    B = CONFIGS[name]
    ranks, inits = run_ranks(2, name, precision, B, tmp_path, backend)
    want, _, _ = emulate(2, name, precision, B)
    init_net = build(name, precision, seed=0)
    _check_init(inits, [p.detach().cpu() for p in init_net.parameters()],
                [b.detach().cpu() for b in init_net.buffers()])
    for s in range(STEPS):
        w = want[s]
        for r, snaps in enumerate(ranks):
            got = snaps[s]
            for key in ("params", "exp_avg", "exp_avg_sq", "metrics"):
                for i, (a, b) in enumerate(zip(got[key], w[key])):
                    assert _same(a, b), "%s %s step %d rank %d: %s[%d] differs" % (name, precision, s, r, key, i)
            assert _same(got["grad"], w["grad"]), (name, precision, s, r, "averaged gradient differs")
            assert _same(got["gnorm"], w["gnorm"]), (name, precision, s, r, got["gnorm"], w["gnorm"])
            assert _same(got["record"], w["record"]), (name, precision, s, r)
        for i, (a, b) in enumerate(zip(ranks[0][s]["bn"], w["bn"])):
            assert _same(a, b), "%s %s step %d: rank 0's BatchNorm buffer %d differs" % (name, precision, s, i)
    assert np.isfinite(float(want[-1]["gnorm"]))
    assert not _same(ranks[0][0]["local"], ranks[1][0]["local"])      # the two shares' gradients differ


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name,precision", CASES)
def test_two_ranks_equal_the_one_gpu_emulation(name, precision, tmp_path):
    """two NCCL ranks on devices 0 and 1, three steps: after the enable-time broadcast both ranks hold rank 0's
    parameters and buffers; after every step both ranks' averaged gradient, parameters, Adam moments, gradient norm and
    metric buffers, and rank 0's BatchNorm running buffers, equal the one-GPU emulation bit for bit"""
    _need(2)
    _check_two_ranks(name, precision, tmp_path, "nccl")


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name,precision", CASES)
def test_two_gloo_ranks_on_one_device_equal_the_emulation(name, precision, tmp_path):
    """the same comparison with two gloo ranks sharing device 0 (see the module docstring): everything but NCCL"""
    _check_two_ranks(name, precision, tmp_path, "gloo")


@pytest.mark.timeout(1800)
def test_all_visible_ranks_agree(tmp_path):
    """world = every visible device (4 to 8), car.fhd, three steps: the ranks' parameters are bit-identical to each
    other.  Against the one-GPU emulation (another summation order):
    - the averaged gradient, element by element, within 2 W 2^-24 S, where S = sum_r |g_r| / W from the ranks' own
      gradients: two orders of summing W terms differ by at most 2 (W - 1) roundings of their magnitude sum.  For W not
      a power of two 1/W is not exact, the emulation's backward of loss * fl(1/W) is not fl(g_r * fl(1/W)), and the
      bound widens to 1e-4 S;
    - the gradient norm to 1e-5 relative, the metric buffers to 1e-6 relative;
    - a parameter by at most 2 * (the learning rates of the steps so far) + 1e-6 |p|: an Adam step moves a parameter
      by at most about its learning rate, and a gradient component that is rounding noise can flip its sign."""
    have = _need(4)
    world = min(have, 8)
    name, B = "car.fhd", 1
    ranks, _ = run_ranks(world, name, "fp32", B, tmp_path)
    want, _, _ = emulate(world, name, "fp32", B)
    from b2second import optim
    lrs = optim.schedule_table(orf.ONE_CYCLE, STEPS)[:, 0]
    for s in range(STEPS):
        for r in range(1, world):
            for i, (a, b) in enumerate(zip(ranks[r][s]["params"], ranks[0][s]["params"])):
                assert _same(a, b), "step %d: rank %d parameter %d differs from rank 0's" % (s, r, i)
        got, w = ranks[0][s], want[s]
        S = sum(ranks[r][s]["local"].abs() for r in range(world)) / world
        rel = 2 * world * 2.0 ** -24 if world & (world - 1) == 0 else 1e-4
        err = (got["grad"] - w["grad"]).abs()
        assert torch.all(err <= rel * S), (s, float((err / S.clamp_min(1e-38)).max()))
        assert abs(float(got["gnorm"]) - float(w["gnorm"])) <= 1e-5 * abs(float(w["gnorm"])), (s, got["gnorm"],
                                                                                               w["gnorm"])
        bound = 2 * float(lrs[:s + 1].sum())
        for i, (a, b) in enumerate(zip(got["params"], w["params"])):
            assert torch.all((a - b).abs() <= bound + 1e-6 * b.abs()), (s, i, float((a - b).abs().max()))
        for i, (a, b) in enumerate(zip(got["metrics"], w["metrics"])):
            assert torch.allclose(a, b, rtol=1e-6, atol=0), (s, i, a, b)
