"""Several GPUs, one process each: frame sharding for inference and data-parallel training.

Inference: no data-path collective inside a frame, ONE all-gather of the fixed-stride detection records per batch
(SURVEY.md §8e).  The reference evaluates on one GPU (train.py:271-277); sharding inference frames is new
functionality, so there is no reference call site to mirror beyond the per-frame contract of ``VoxelNet.forward``.

Training: the reference's ``--multi_gpu`` (second/pytorch/train.py:203-204, 237-270, 299-327) wraps the net in
``torch.nn.DataParallel`` and loads ``batch_size * num_gpu`` frames per step.  ``enable_data_parallel`` gives the same
step with one process per GPU::

    dist.init_process_group("nccl")                      # torch.distributed.run --nproc-per-node W
    torch.cuda.set_device(local_rank)
    dp = training.enable_data_parallel(net)              # broadcast rank 0's weights; grads become bucket views
    opt = optim.plan(net, train_config.optimizer, train_config.steps, data_parallel=dp)
    # per step, rank r holds frames frames_for_rank(W * B, r, W) of the global batch
    ret = net(example); ret["loss"].backward()
    opt.step()                                           # all-reduce (1/W) * sum of the grads, then clip/decay/Adam
    net.b2s_metrics.update_metrics_async(...)           # counts summed over ranks: whole-batch metrics on every rank

What matches DataParallel: each rank's BatchNorm uses its own share's batch statistics and rank 0's running buffers are
the ones that count (``sync_buffers()`` copies them to the other ranks before an evaluation or a save there); the
gradient is ``sum_r (1/W) * g_r`` (``loss = ret_dict["loss"].mean()`` over the replicas), clipped, decayed and stepped
identically on every rank; the metric buffers are those of the whole batch, with the replica-mean losses and the frame-0
figures of the global frame 0 (rank 0's first frame).

Layout: global frame ``g`` of a batch of ``W*B`` frames runs on rank ``g // B`` as local frame
``g % B`` (contiguous blocks, so rank-major gather order == global frame order).
Record per frame: ``det [post_max, code+2]`` (box, score, label) + ``count`` -> packed as one float32
tensor ``[B, post_max*(code+2) + 1]`` so a single collective moves everything.
"""
import torch
import torch.distributed as dist

from . import optim


def frames_for_rank(num_frames, rank, world):
    """contiguous block partition; returns (start, stop) global frame ids for ``rank``."""
    per = (num_frames + world - 1) // world
    start = min(rank * per, num_frames)
    return start, min(start + per, num_frames)


def pack_records(det, count):
    """det [B, post_max, S] f32, count [B] i32 -> [B, post_max*S + 1] f32 (count stored exactly: < 2^24)."""
    B = det.shape[0]
    return torch.cat([det.reshape(B, -1), count.to(det.dtype).view(B, 1)], dim=1).contiguous()


def unpack_records(rec, post_max, stride):
    det = rec[:, :post_max * stride].reshape(rec.shape[0], post_max, stride)
    count = rec[:, post_max * stride].round().to(torch.int32)
    return det, count


class DetectionGatherer:
    """pre-allocated send/recv buffers + one ``all_gather_into_tensor`` per batch (NCCL on GPUs, gloo in tests)."""

    def __init__(self, batch_per_rank, post_max, stride, device, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.B, self.post_max, self.stride = batch_per_rank, post_max, stride
        width = post_max * stride + 1
        self.send = torch.zeros(batch_per_rank, width, dtype=torch.float32, device=device)
        self.recv = torch.zeros(self.world * batch_per_rank, width, dtype=torch.float32, device=device)

    def gather_records(self, records):
        """records [B, post_max*S + 1]: the engine's ``det_record`` buffer (the NMS epilogue writes the detections AND
        the count straight into it, so there is no packing step) -> same return value as ``gather``.  The buffer is
        the collective's send buffer itself."""
        assert records.shape == self.send.shape and records.is_contiguous()
        if self.world == 1:
            self.recv.copy_(records)
        elif hasattr(dist, "all_gather_into_tensor") and records.is_cuda:
            dist.all_gather_into_tensor(self.recv, records, group=self.group)
        else:
            parts = list(self.recv.view(self.world, self.B, -1).unbind(0))
            dist.all_gather(parts, records, group=self.group)
        return unpack_records(self.recv, self.post_max, self.stride)

    def gather(self, det, count):
        """-> (det_all [W*B, post_max, S], count_all [W*B]) in global frame order, on every rank."""
        self.send.copy_(pack_records(det, count))
        if self.world == 1:
            self.recv.copy_(self.send)
        elif hasattr(dist, "all_gather_into_tensor") and self.send.is_cuda:
            dist.all_gather_into_tensor(self.recv, self.send, group=self.group)
        else:
            parts = list(self.recv.view(self.world, self.B, -1).unbind(0))
            dist.all_gather(parts, self.send, group=self.group)
        return unpack_records(self.recv, self.post_max, self.stride)


# ---- data-parallel training --------------------------------------------------------------------------------------------

def bucket_layout(params):
    """-> [(offset, numel)] of each parameter's gradient in one flat float32 bucket, in the order given (the optimizer's
    ``parameter_groups`` order), packed back to back; and the bucket's length.  Host only."""
    spans, off = [], 0
    for p in params:
        spans.append((off, p.numel()))
        off += p.numel()
    return spans, off


def attach_grad_bucket(params):
    """allocate one flat float32 gradient bucket on the parameters' device and make every ``p.grad`` a view into it
    (torch DDP's ``gradient_as_bucket_view``), keeping any gradient already held; -> the bucket.  Autograd accumulates
    into an existing ``.grad`` in place and the optimizer zeroes it in place, so the views persist across steps."""
    if not params:
        raise ValueError("no trainable parameter")
    spans, n = bucket_layout(params)
    dev = params[0].device
    for p in params:
        if p.dtype != torch.float32 or p.device != dev or not p.is_contiguous():
            raise TypeError("data-parallel parameters must be contiguous float32 tensors on one device")
    bucket = torch.zeros(n, dtype=torch.float32, device=dev)
    for p, (off, k) in zip(params, spans):
        view = bucket[off:off + k].view(p.shape)
        if p.grad is not None:
            view.copy_(p.grad)
        p.grad = view
    return bucket


def grads_in_bucket(params, bucket):
    """True when every ``p.grad`` is still its view of ``bucket`` (``bucket_layout``'s place)"""
    spans, n = bucket_layout(params)
    if bucket.numel() != n:
        return False
    base, size = bucket.data_ptr(), bucket.element_size()
    return all(p.grad is not None and p.grad.data_ptr() == base + off * size for p, (off, _) in zip(params, spans))


def _bn_buffers(net):
    return [b for m in net.modules() if isinstance(m, optim._BN_TYPES) for b in m.buffers(recurse=False)]


class DataParallel:
    """the data-parallel side of one network on one rank (see ``enable_data_parallel``): ``world``, ``rank``,
    ``group``, the parameters in ``optim.parameter_groups`` order and their gradient ``bucket``."""

    def __init__(self, net, params, bucket, world, rank, group=None):
        self.net = net
        self.params = params
        self.bucket = bucket
        self.world = int(world)
        self.rank = int(rank)
        self.group = group
        self.timing = None        # a list to collect (start, end) CUDA event pairs around each all-reduce

    def all_reduce_grads(self):
        """one collective on the bucket, ordered on the current stream: ``sum_r (1/W) * g_r`` on every rank (NCCL's
        AVG, a pre-multiplied sum by 1/W for floats, exact scaling for W a power of two).  No host sync."""
        if not grads_in_bucket(self.params, self.bucket):
            raise RuntimeError("a gradient is no longer a view of the data-parallel bucket (was .grad replaced or set "
                               "to None?)")
        ev = None
        if self.timing is not None:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        if self.world > 1:
            dist.all_reduce(self.bucket, op=dist.ReduceOp.AVG, group=self.group)
        if ev is not None:
            ev[1].record()
            self.timing.append(ev)

    def all_reduce_sum(self, t):
        """sum ``t`` over the ranks in place (the metrics' count record)"""
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    def sync_buffers(self):
        """broadcast rank 0's BatchNorm running buffers (DataParallel's replica 0 is the module itself; the other
        replicas' buffer updates are dropped).  Call it before evaluating or saving on a rank other than 0."""
        if self.world > 1:
            src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
            bufs = _bn_buffers(self.net)
            for b in bufs:
                dist.broadcast(b, src, group=self.group)
            torch.autograd.graph.increment_version(bufs)      # the drop-in's folded batch norms are keyed on it


def enable_data_parallel(net, group=None):
    """train ``net`` data-parallel over the ranks of ``group`` (default: the whole world), one process per GPU, with the
    reference's ``torch.nn.DataParallel`` semantics (see the module docstring); -> DataParallel, to pass to
    ``optim.plan(..., data_parallel=)``.  It is kept as ``net.b2s_data_parallel``, where the GPU metrics
    (``metrics.enable_gpu_metrics``) find it and sum their counts over the ranks.

    Refuses: no initialised process group, a backend other than NCCL, parameters not on this rank's CUDA device, two
    ranks on one device.  Broadcasts rank 0's parameters and buffers once and makes every ``p.grad`` a view of one flat
    float32 bucket in ``optim.parameter_groups`` order."""
    if not dist.is_available() or not dist.is_initialized():
        raise RuntimeError("enable_data_parallel needs an initialised process group (torch.distributed."
                           "init_process_group('nccl'))")
    backend = dist.get_backend(group)
    if backend != "nccl":
        raise RuntimeError("enable_data_parallel needs the NCCL backend, the process group uses %r" % backend)
    params = [p for g in optim.parameter_groups(net) for p in g]
    if not params:
        raise ValueError("no trainable parameter")
    dev = torch.device("cuda", torch.cuda.current_device())
    for p in list(net.parameters()) + list(net.buffers()):
        if p.device != dev:
            raise RuntimeError("parameters and buffers must be on this rank's device %s (torch.cuda.set_device), "
                               "found one on %s" % (dev, p.device))
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    uuids = [None] * world
    dist.all_gather_object(uuids, str(torch.cuda.get_device_properties(dev).uuid), group=group)
    if len(set(uuids)) != world:
        raise RuntimeError("two ranks share one GPU (devices %s); data-parallel training needs one device per rank"
                           % uuids)
    src = dist.get_global_rank(group, 0) if group is not None else 0
    state = list(net.parameters()) + list(net.buffers())
    with torch.no_grad():
        for t in state:
            dist.broadcast(t.data, src, group=group)
    # the drop-in's weight caches (packed planes, folded batch norms) are keyed on the autograd version
    torch.autograd.graph.increment_version(state)
    bucket = attach_grad_bucket(params)
    handle = DataParallel(net, params, bucket, world, rank, group)
    net.b2s_data_parallel = handle
    return handle
