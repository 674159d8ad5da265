"""Training metrics on the GPU: ``VoxelNet.update_metrics`` (second/pytorch/models/voxelnet.py:654-679 through
torchplus/metrics.py) and the log figures of train.py:335-373, in csrc/metrics.cu.

    net = metrics.enable_gpu_metrics(loss.enable_gpu_loss(training.enable_sparse_backward(net)))
    ret = net(example)
    ...
    m = net.update_metrics(ret["cls_loss_reduced"], ret["loc_loss_reduced"], ret["cls_preds"], labels, ret["cared"])

The reference's torchplus sequence synchronises with the host about two dozen times per call (``Scalar``'s
``if not scalar.eq(0.0)``, ``PrecisionRecall``'s ``if rec_count > 0`` / ``if prec_count > 0`` per threshold, the
``.cpu()`` of every value).  Here one launch pair updates the running buffers on the device and writes one float32
record; ``update_metrics`` reads it with one pinned device-to-host copy, and ``update_metrics_async`` returns a handle
whose ``result()`` does that copy later (the launch is capturable in a CUDA graph).

The running buffers are the reference's own (``rpn_acc.total/count``, ``rpn_metrics.prec_total/prec_count/rec_total/
rec_count``, ``rpn_cls_loss.*``, ``rpn_loc_loss.*``), updated in place in the reference's order and with its
conditionals, so ``state_dict()`` and checkpoints are unchanged.  ``plan`` reads the settings through the reference's
attribute names; sigmoid scores with background encoded as zeros (what every config uses) are covered, anything else
raises ``spec.UnsupportedNetwork``.
"""
import ctypes
import types

import numpy as np
import torch
from torch import nn

from .spec import UnsupportedNetwork

# the reference's PrecisionRecall thresholds (voxelnet.py:176-180); the mirror's rpn_metrics is built with them
THRESHOLDS = (0.1, 0.3, 0.5, 0.7, 0.8, 0.9, 0.95)
_CLEARED = ("rpn_acc", "rpn_metrics", "rpn_cls_loss", "rpn_loc_loss", "rpn_total_loss")   # what clear_metrics zeroes
METRIC_MODULES = ("rpn_acc", "rpn_precision", "rpn_recall") + _CLEARED[1:]          # voxelnet.py:172-184
MAX_THRESHOLDS = 16                                                                  # B2S_METRICS_MAX_THRESHOLDS


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


# ---- the reference's metric modules as buffer holders (torchplus/metrics.py), for the mirror -------------------------

class _Pair(nn.Module):
    """Scalar / Accuracy / Precision / Recall: the ``total`` and ``count`` buffers"""

    def __init__(self):
        super().__init__()
        self.register_buffer("total", torch.zeros(1))
        self.register_buffer("count", torch.zeros(1))

    def clear(self):
        self.total.zero_()
        self.count.zero_()


class _Accuracy(_Pair):
    def __init__(self, encode_background_as_zeros):
        super().__init__()
        self._ignore_idx, self._dim, self._threshold = -1, -1, 0.5
        self._encode_background_as_zeros = encode_background_as_zeros


class _PrecisionRecall(nn.Module):
    def __init__(self, thresholds, use_sigmoid_score, encode_background_as_zeros):
        super().__init__()
        for name in ("prec_total", "prec_count", "rec_total", "rec_count"):
            self.register_buffer(name, torch.zeros(len(thresholds)))
        self._ignore_idx, self._dim = -1, -1
        self._thresholds = list(thresholds)
        self._use_sigmoid_score = use_sigmoid_score
        self._encode_background_as_zeros = encode_background_as_zeros

    @property
    def thresholds(self):
        return self._thresholds

    def clear(self):
        self.rec_count.zero_()
        self.prec_count.zero_()
        self.prec_total.zero_()
        self.rec_total.zero_()


# ---- plan ------------------------------------------------------------------------------------------------------------

def plan(net):
    """-> MetricsPlan for a VoxelNet with the reference's metric modules (the reference's own network, or the mirror
    after ``enable_gpu_metrics``), read through the reference's attribute names."""
    acc, pr = net.rpn_acc, net.rpn_metrics
    if not (acc._encode_background_as_zeros and pr._encode_background_as_zeros):
        raise UnsupportedNetwork("encode_background_as_zeros = false is not supported")
    if not pr._use_sigmoid_score:
        raise UnsupportedNetwork("softmax scores (use_sigmoid_score = false) are not supported")
    th = pr._thresholds
    th = list(th) if isinstance(th, (list, tuple)) else [th]
    if any(isinstance(t, (list, tuple, np.ndarray, torch.Tensor)) for t in th):
        raise UnsupportedNetwork("rpn_metrics holds more than one threshold list")
    if not 1 <= len(th) <= MAX_THRESHOLDS:
        raise UnsupportedNetwork("rpn_metrics needs 1..%d thresholds, got %d" % (MAX_THRESHOLDS, len(th)))
    return MetricsPlan(net, [float(t) for t in th], float(acc._threshold), int(net._num_class))


class MetricsPlan:
    """the metrics of one network (see ``plan``)."""

    def __init__(self, net, thresholds, acc_threshold, num_class):
        self.net = net
        self.thresholds = thresholds
        self.acc_threshold = acc_threshold
        self.num_class = num_class
        self.last_status = None
        self._params = None
        self._count_log = (0, [False] * 3)

    def params(self):
        """b2s_metrics_params as a ctypes structure (host memory, read by the call)."""
        if self._params is None:
            L, _ = _lib()
            p = L.MetricsParams()
            p.num_thresholds = len(self.thresholds)
            for i, t in enumerate(self.thresholds):
                p.thresholds[i] = t           # float32, as torch compares a float32 score with a Python float
            p.acc_threshold = self.acc_threshold
            self._params = p
        return self._params

    def _buffers(self, dev):
        L, _ = _lib()
        n = self.net
        bufs = {"acc_total": n.rpn_acc.total, "acc_count": n.rpn_acc.count,
                "prec_total": n.rpn_metrics.prec_total, "prec_count": n.rpn_metrics.prec_count,
                "rec_total": n.rpn_metrics.rec_total, "rec_count": n.rpn_metrics.rec_count,
                "cls_total": n.rpn_cls_loss.total, "cls_count": n.rpn_cls_loss.count,
                "loc_total": n.rpn_loc_loss.total, "loc_count": n.rpn_loc_loss.count}
        b = L.MetricsBuffers()
        for name, t in bufs.items():
            if not (t.is_cuda and t.device == dev and t.dtype == torch.float32 and t.is_contiguous()):
                raise RuntimeError("metric buffer %s must be a contiguous float32 tensor on %s (net.metrics_to_float(), "
                                   "net.to(device)), got %s on %s" % (name, dev, t.dtype, t.device))
            setattr(b, name, t.data_ptr())
        return b

    def _inputs(self, cls_loss, loc_loss, cls_preds, labels, sampled, ret_dict, anchors_mask):
        """the launch arguments of one share's metrics, checked: the b2s_train_metrics(_count) inputs after num_anchors"""
        L, _ = _lib()
        B = int(cls_preds.shape[0])
        C = self.num_class
        cls = cls_preds.detach()
        L.require_cuda(cls, "cls_preds")
        if cls.dtype != torch.float32:
            raise TypeError("cls_preds must be float32, got %s" % cls.dtype)
        cls = cls.contiguous().view(B, -1, C)
        A = int(cls.shape[1])
        if labels.dtype not in (torch.int32, torch.int64):
            labels = labels.to(torch.int64)
        labels = labels.contiguous().view(B, A)
        if sampled.dtype not in (torch.bool, torch.uint8):
            raise TypeError("sampled must be the 0/1 bool weights (the loss's `cared`), got %s" % sampled.dtype)
        cared = sampled.contiguous().view(B, A).view(torch.uint8)
        scal = [None if t is None else t.detach().to(torch.float32).contiguous().view(-1)[:1]
                for t in (cls_loss, loc_loss)]
        extra = {"loc_loss": None, "cls_pos_loss": None, "cls_neg_loss": None, "dir_loss_reduced": None}
        if ret_dict is not None:
            for k in extra:
                if ret_dict.get(k) is not None:
                    extra[k] = ret_dict[k].detach().to(torch.float32).contiguous()
        loc_elem = extra["loc_loss"]
        code = 0
        if loc_elem is not None:
            code = int(loc_elem.shape[-1])
            loc_elem = loc_elem.view(B, A, code)
        mask = None
        if anchors_mask is not None:
            mask = anchors_mask.contiguous().view(B, A)
            mask = (mask if mask.dtype == torch.bool else mask != 0).view(torch.uint8)
        tensors = [("labels", labels), ("sampled", cared), ("cls_loss", scal[0]), ("loc_loss", scal[1])]
        tensors += [(k, v) for k, v in extra.items() if v is not None]
        if mask is not None:
            tensors.append(("anchors_mask", mask))
        for name, t in tensors:
            L.require_cuda(t, name)
        sc = [extra[k].view(-1)[:1] if extra[k] is not None else None
              for k in ("cls_pos_loss", "cls_neg_loss", "dir_loss_reduced")]
        args = [L.ptr(cls), C, L.ptr(labels), int(labels.dtype == torch.int64), L.ptr(cared), B, A,
                ctypes.byref(self.params()), L.ptr(scal[0]), L.ptr(scal[1]), L.ptr(loc_elem), code, L.ptr(mask),
                L.ptr(sc[0]), L.ptr(sc[1]), L.ptr(sc[2])]
        keep = (cls, labels, cared, scal, extra, mask)
        return args, keep, cls.device, B, A, code, [s is not None for s in sc]

    def update_metrics_async(self, cls_loss, loc_loss, cls_preds, labels, sampled, ret_dict=None, anchors_mask=None):
        """launch one step's metrics (VoxelNet.update_metrics' arguments: the reduced cls / loc losses, cls_preds,
        labels, and the 0/1 weights ``sampled`` -- the loss's ``cared``); -> MetricsHandle.  ``ret_dict`` (the loss
        dict) and ``anchors_mask`` (the example's, if any) add train.py's log figures.  No host synchronisation.

        Under data parallelism (``b2second.dist.enable_data_parallel(net)``) the arguments are this rank's share: its
        count record is summed over the ranks (one all-reduce) before the buffers are updated, so every rank's buffers
        and record are those of the whole batch, with the replica-mean losses and the global frame 0's figures."""
        dp = getattr(self.net, "b2s_data_parallel", None)
        if dp is not None:
            counts = self.count(cls_loss, loc_loss, cls_preds, labels, sampled, ret_dict, anchors_mask,
                                has_frame0=dp.rank == 0)
            dp.all_reduce_sum(counts)
            return self.finish(counts, 1.0 / dp.world)
        L, lib = _lib()
        args, keep, dev, B, A, code, have = self._inputs(cls_loss, loc_loss, cls_preds, labels, sampled, ret_dict,
                                                          anchors_mask)
        T = len(self.thresholds)
        record = torch.empty(L.METRICS_RECORD_HEAD + 2 * T, dtype=torch.float32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        ws_bytes = lib.b2s_train_metrics_workspace_bytes(B, A)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        bufs = self._buffers(dev)
        with torch.cuda.device(dev):
            L.check(lib.b2s_train_metrics(*args, ctypes.byref(bufs), L.ptr(record), L.ptr(ws), ws_bytes,
                                          L.ptr(status), L.stream()), "b2s_train_metrics")
        self.last_status = status        # device word; nonzero: a label outside [-1, num_class]
        return MetricsHandle(self, record, status, code, have)

    def count(self, cls_loss, loc_loss, cls_preds, labels, sampled, ret_dict=None, anchors_mask=None, has_frame0=True):
        """the first half of ``update_metrics_async`` on one share of a batch: -> its count record (device float32
        [METRICS_COUNT_HEAD + 2 * T], include/b2second.h B2S_METRICS_CNT_*).  Records of several shares add exactly;
        ``has_frame0`` False leaves the frame-0 figures zero, for shares that do not hold the batch's first frame."""
        L, lib = _lib()
        args, keep, dev, B, A, code, have = self._inputs(cls_loss, loc_loss, cls_preds, labels, sampled, ret_dict,
                                                          anchors_mask)
        T = len(self.thresholds)
        counts = torch.empty(L.METRICS_COUNT_HEAD + 2 * T, dtype=torch.float32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        ws_bytes = lib.b2s_train_metrics_workspace_bytes(B, A)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2s_train_metrics_count(*args, int(bool(has_frame0)), L.ptr(counts), L.ptr(ws), ws_bytes,
                                                L.ptr(status), L.stream()), "b2s_train_metrics_count")
        self.last_status = status
        self._count_log = (code, have)       # which log fields the last count's inputs held
        return counts

    def finish(self, counts, loss_scale=1.0):
        """the second half: update the running buffers from a (summed) count record, the five loss slots scaled by
        ``loss_scale`` (1/W for a sum over W ranks); -> MetricsHandle.  No host synchronisation."""
        L, lib = _lib()
        L.require_cuda(counts, "counts")
        T = len(self.thresholds)
        if counts.dtype != torch.float32 or counts.numel() != L.METRICS_COUNT_HEAD + 2 * T:
            raise ValueError("counts must be a float32 count record of %d entries" % (L.METRICS_COUNT_HEAD + 2 * T))
        dev = counts.device
        counts = counts.contiguous()
        record = torch.empty(L.METRICS_RECORD_HEAD + 2 * T, dtype=torch.float32, device=dev)
        bufs = self._buffers(dev)
        with torch.cuda.device(dev):
            L.check(lib.b2s_train_metrics_finish(L.ptr(counts), ctypes.byref(self.params()), float(loss_scale),
                                                 ctypes.byref(bufs), L.ptr(record), L.stream()),
                    "b2s_train_metrics_finish")
        code, have = self._count_log
        return MetricsHandle(self, record, self.last_status, code, have)

    def update_metrics(self, cls_loss, loc_loss, cls_preds, labels, sampled):
        """VoxelNet.update_metrics: the reference's dict of Python floats, read with one device-to-host copy."""
        return self.update_metrics_async(cls_loss, loc_loss, cls_preds, labels, sampled).result()


class MetricsHandle:
    """one launched step of metrics.  ``result()`` / ``step_log()`` copy the record to the host once (pinned memory,
    one copy and one wait) and build the reference's values from it; until then nothing waits for the device."""

    def __init__(self, plan_, record, status, code, have_scalars):
        self.plan = plan_
        self.record = record
        self.status = status
        self._code = code
        self._have = have_scalars
        self._host = None

    def _fetch(self):
        if self._host is None:
            h = torch.empty(self.record.shape, dtype=torch.float32, pin_memory=True)
            h.copy_(self.record, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
            self._host = h.numpy().copy()
        return self._host

    def result(self):
        """VoxelNet.update_metrics' dict (voxelnet.py:666-679)"""
        L, _ = _lib()
        r = self._fetch()
        rec = dict(zip(L.METRICS_REC, r))
        T = len(self.plan.thresholds)
        head = L.METRICS_RECORD_HEAD
        ret = {"loss": {"cls_loss": float(rec["cls_loss"]), "cls_loss_rt": float(rec["cls_loss_rt"]),
                        "loc_loss": float(rec["loc_loss"]), "loc_loss_rt": float(rec["loc_loss_rt"])},
               "rpn_acc": float(rec["rpn_acc"]), "pr": {}}
        for i, thresh in enumerate(self.plan.thresholds):
            ret["pr"][f"prec@{int(thresh*100)}"] = float(r[head + i])
            ret["pr"][f"rec@{int(thresh*100)}"] = float(r[head + T + i])
        return ret

    def step_log(self):
        """train.py's further log fields (train.py:335-373) from the same record: ``loss``: loc_elem, cls_pos_rt,
        cls_neg_rt, dir_rt (those whose inputs ``ret_dict`` held); ``misc``: num_pos, num_neg, num_anchors."""
        L, _ = _lib()
        r = self._fetch()
        rec = dict(zip(L.METRICS_REC, r))
        loss = {}
        if self._code:
            loss["loc_elem"] = [float(v) for v in r[L.METRICS_REC_LOC_ELEM:L.METRICS_REC_LOC_ELEM + self._code]]
        for have, key in zip(self._have, ("cls_pos_rt", "cls_neg_rt", "dir_rt")):
            if have:
                loss[key] = float(rec[key])
        misc = {k: int(rec[k]) for k in ("num_pos", "num_neg", "num_anchors")}
        return {"loss": loss, "misc": misc}


# ---- binding ---------------------------------------------------------------------------------------------------------

def _clear_metrics(self):
    """VoxelNet.clear_metrics (voxelnet.py:681-686): zero the five modules' buffers"""
    for name in _CLEARED:
        getattr(self, name).clear()


def _metrics_to_float(self):
    """VoxelNet.metrics_to_float (voxelnet.py:647-652)"""
    for name in _CLEARED:
        getattr(self, name).float()


def enable_gpu_metrics(net):
    """give ``net`` the reference's ``update_metrics`` on the GPU; returns ``net``.

    On the reference's VoxelNet this rebinds ``net.update_metrics`` and ``net.clear_metrics`` on the instance.  On the
    mirror (b2second.models.VoxelNet) it first adds the reference's metric modules with their buffers under the
    reference's names (rpn_acc, rpn_precision, rpn_recall, rpn_metrics, rpn_cls_loss, rpn_loc_loss, rpn_total_loss),
    so reference checkpoints load with them, and ``metrics_to_float``."""
    if not hasattr(net, "rpn_metrics"):
        ebz = bool(net._encode_background_as_zeros)
        mods = {"rpn_acc": _Accuracy(ebz), "rpn_precision": _Pair(), "rpn_recall": _Pair(),
                "rpn_metrics": _PrecisionRecall(THRESHOLDS, bool(net._use_sigmoid_score), ebz),
                "rpn_cls_loss": _Pair(), "rpn_loc_loss": _Pair(), "rpn_total_loss": _Pair()}
        dev = net.global_step.device
        for name, m in mods.items():
            setattr(net, name, m.to(dev))
        net.metrics_to_float = types.MethodType(_metrics_to_float, net)
    mp = plan(net)
    net.b2s_metrics = mp
    net.update_metrics = types.MethodType(
        lambda self, cls_loss, loc_loss, cls_preds, labels, sampled:
            mp.update_metrics(cls_loss, loc_loss, cls_preds, labels, sampled), net)
    net.clear_metrics = types.MethodType(_clear_metrics, net)
    return net
