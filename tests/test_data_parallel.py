"""Data-parallel training on the host: the gradient bucket's layout and aliasing, and what enable_data_parallel and a
data-parallel optimizer step refuse (world 2 over gloo in spawned processes)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

import optim_ref as orf
from b2second import dist as b2dist
from b2second import augment, dbsample, optim


def _net():
    torch.manual_seed(0)
    return nn.Sequential(nn.Linear(4, 8, bias=False), nn.BatchNorm1d(8), nn.ReLU(),
                         nn.Sequential(nn.Linear(8, 3), nn.BatchNorm1d(3)))


def _aliases(params, bucket):
    spans, n = b2dist.bucket_layout(params)
    assert bucket.numel() == n
    for p, (off, k) in zip(params, spans):
        assert p.grad.data_ptr() == bucket.data_ptr() + 4 * off and p.grad.numel() == k and p.grad.shape == p.shape
    assert b2dist.grads_in_bucket(params, bucket)


def test_bucket_follows_parameter_groups_order():
    net = _net()
    groups = optim.parameter_groups(net)
    params = [p for g in groups for p in g]
    # the optimizer's order: the two Linear layers' parameters, then the two BatchNorms'
    assert [tuple(p.shape) for p in params] == [(8, 4), (3, 8), (3,), (8,), (8,), (3,), (3,)]
    spans, n = b2dist.bucket_layout(params)
    assert spans == [(0, 32), (32, 24), (56, 3), (59, 8), (67, 8), (75, 3), (78, 3)] and n == 81
    bucket = b2dist.attach_grad_bucket(params)
    assert bucket.dtype == torch.float32 and bucket.shape == (81,) and not bucket.any()
    _aliases(params, bucket)


def test_grads_stay_views_through_backward_and_zero():
    net = _net().train()
    params = [p for g in optim.parameter_groups(net) for p in g]
    x = torch.randn(5, 4)
    net(x).square().sum().backward()                   # gradients held before the bucket is attached are kept
    before = [p.grad.clone() for p in params]
    bucket = b2dist.attach_grad_bucket(params)
    _aliases(params, bucket)
    for p, g in zip(params, before):
        assert torch.equal(p.grad, g)
    net(x).square().sum().backward()                   # autograd accumulates in place
    _aliases(params, bucket)
    for p, g in zip(params, before):
        assert torch.allclose(p.grad, 2 * g, rtol=1e-5, atol=1e-6)
    off = 0
    for p in params:
        assert torch.equal(bucket[off:off + p.numel()], p.grad.reshape(-1))
        off += p.numel()
    for p in params:
        p.grad.zero_()                                 # what the optimizer's step does
    _aliases(params, bucket)
    assert not bucket.any()
    params[0].grad = None
    assert not b2dist.grads_in_bucket(params, bucket)


def test_refused_without_a_process_group():
    assert not dist.is_initialized()
    with pytest.raises(RuntimeError, match="initialised process group"):
        b2dist.enable_data_parallel(_net())


def test_set_to_none_refused_before_any_device_work():
    net = _net()
    params = [p for g in optim.parameter_groups(net) for p in g]
    handle = b2dist.DataParallel(net, params, b2dist.attach_grad_bucket(params), world=2, rank=0)
    opt = optim.plan(net, orf.ONE_CYCLE, 10, data_parallel=handle)
    with pytest.raises(ValueError, match="set_to_none"):
        opt.step(set_to_none=True)
    _aliases(params, handle.bucket)
    other = _net()
    with pytest.raises(ValueError, match="other parameters"):
        optim.plan(other, orf.ONE_CYCLE, 10, data_parallel=handle)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        b2dist.enable_data_parallel(_net())
        q.put((rank, "not refused"))
    except RuntimeError as e:
        q.put((rank, "refused" if "NCCL" in str(e) else "other error: %s" % e))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(120)
def test_gloo_group_refused_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=90) for _ in range(world)]
    finally:
        for p in procs:
            p.join(30)
            if p.is_alive():
                p.kill()
                p.join(10)
    assert sorted(res) == [(0, "refused"), (1, "refused")]


def test_select_keeps_each_frames_draws():
    """a rank's share of the whole batch's host draws: concatenated over the shares they are the whole batch's"""
    import numpy as np
    from b2second import config
    cfg = config.get_config("car.fhd")
    nb, npts = [3, 0, 5, 2], [40, 7, 11, 30]
    d = augment.draw(np.random.RandomState(0), cfg.augment, nb, npts)
    parts = [augment.select(d, a, b) for a, b in ((0, 1), (1, 3), (3, 4))]
    for f in ("loc_noise", "rot_noise", "frame", "perm"):
        np.testing.assert_array_equal(np.concatenate([getattr(p, f) for p in parts]), getattr(d, f))
    assert sum((p.num_gt for p in parts), []) == nb and sum((p.num_points for p in parts), []) == npts
    c = dbsample.Candidates(objects=np.arange(9, dtype=np.int32), group=np.arange(9, dtype=np.int32) % 2,
                            offsets=np.array([0, 2, 2, 6, 9], np.int32))
    s = dbsample.select(c, 1, 3)
    np.testing.assert_array_equal(s.offsets, [0, 0, 4])
    np.testing.assert_array_equal(s.objects, [2, 3, 4, 5])
    np.testing.assert_array_equal(s.group, [0, 1, 0, 1])
