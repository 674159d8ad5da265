"""The optimizer step on the GPU: everything second/pytorch/train.py does after ``loss.backward()`` (train.py:299,
323-325), in csrc/optim.cu.

    opt = optim.plan(net, train_config.optimizer, train_config.steps)
    ...
    loss.backward()
    gnorm = opt.step()      # clip_grad_norm_(10.0) + weight decay + Adam + schedule advance + zero_grad

``step`` is two kernel launches whatever the number of parameter tensors, with no host synchronisation; it returns
the gradient norm before clipping as a device scalar.  What it restates: ``torch.nn.utils.clip_grad_norm_``, the
reference's ``OptimWrapper.step`` over ``torch.optim.Adam`` (torchplus/train/fastai_optim.py:154-167,
second/pytorch/builder/optimizer_builder.py:68-87) with both decay forms (``fixed_weight_decay`` true: ``p *= 1 - wd *
lr`` before Adam, betas (., 0.99); false: Adam's L2 ``g += wd * p``, betas (0.9, 0.999)), and the ``OneCycle``,
``ExponentialDecay`` and ``ManualStepping`` schedules of torchplus/train/learning_schedules_fastai.py.  Anything else a
config could ask for (RMSprop, momentum SGD, amsgrad, a moving average, ``multi_phase`` schedules, parameters that are
not float32, hence mixed precision) raises ``spec.UnsupportedNetwork``.

The schedule is tabulated once: ``schedule_table`` evaluates the reference's own scalar expressions for every step
into a float64 table ``[total_step, 5]`` (lr, beta1, 1 - beta1^t, sqrt(1 - beta2^t), 1 - wd * lr) that lives in device
memory, and the kernels index it by a device step counter they advance themselves.  So the values are the reference's
Python doubles, the device needs no transcendental, and the step can be captured in a CUDA graph whose replays move
along the schedule (a per-step host staging row would need a copy per replay).  The table is 40 bytes per step.

Parameters are the reference's two groups, ``split_bn_bias(get_layer_groups(net))``: the ``requires_grad`` parameters
of the network's leaf modules that are not batch norms, then those of its batch norms, each in module order.  Frozen
parameters, and parameters held directly by a module that has children, are left alone as the reference leaves them.

``plan`` allocates every ``p.grad`` once and the kernel zeroes it, so the pointer tables stay fixed; they are rebuilt
when a gradient's address changed since the last step.  A parameter whose ``grad`` is ``None`` at a step is decayed
(decoupled form) but not stepped, as in torch; note that a parameter that never receives a gradient holds a zero
gradient here, which under the L2 form still decays it.  ``step(set_to_none=True)`` leaves ``grad = None`` as
``zero_grad()`` does in current torch, at the price of a table rebuild every step.

The kernels write parameters through raw pointers, so after every call ``step`` bumps the autograd version of each
parameter: the drop-in's weight caches (packed fp16 planes, folded batch norms) are keyed on it.  Replaying a captured
step does not run that host code; bump the versions (``opt.touch()``) before the next forward.

Data-parallel training (``b2second.dist.enable_data_parallel``): ``plan(..., data_parallel=handle)`` makes ``step``
enqueue one all-reduce of the flat gradient bucket (``sum_r (1/W) * g_r``) on the current stream before the clip, so
every rank clips, decays and steps on the same averaged gradient.  The gradients are views of that bucket and stay
so (zeroed in place), hence ``step(set_to_none=True)`` is refused there.

``state_dict`` / ``load_state_dict`` use ``torch.optim.Adam``'s format, so a checkpoint written by the reference's
``OptimWrapper`` resumes here and the other way round.
"""
import ctypes
from dataclasses import dataclass
from typing import Tuple

import numpy as np
import torch
from torch import nn

from .spec import UnsupportedNetwork

CLIP_NORM = 10.0                                     # train.py:323
ADAM_EPS = 1e-8                                      # torch.optim.Adam's default; the builder never sets it
HYPER_COLS = ("lr", "beta1", "bias_correction1", "bias_correction2_sqrt", "decay")
_BN_TYPES = (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d)


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


def _f32(v):
    return float(np.float32(float(v)))


@dataclass(frozen=True)
class OptimSettings:
    """``train_config.optimizer`` (second/protos/optimizer.proto) as optimizer_builder.build and
    lr_scheduler_builder.build read it.  Floats are protobuf's float32 values widened to Python floats."""
    decoupled: bool                                  # fixed_weight_decay
    weight_decay: float
    beta1: float                                     # what Adam is built with; a schedule without momentum keeps it
    beta2: float
    eps: float = ADAM_EPS
    clip_norm: float = CLIP_NORM
    schedule: str = "one_cycle"                      # one_cycle | exponential_decay | manual_stepping
    lr_max: float = 0.0                              # one_cycle
    moms: Tuple[float, ...] = ()
    div_factor: float = 0.0
    pct_start: float = 0.0
    initial_learning_rate: float = 0.0               # exponential_decay
    decay_length: float = 0.0
    decay_factor: float = 0.0
    staircase: bool = False
    boundaries: Tuple[float, ...] = ()               # manual_stepping
    rates: Tuple[float, ...] = ()


class _Node:
    """one view of a proto message or of the dict tree ``config.parse_prototxt`` gives for it"""

    def __init__(self, obj):
        self.obj = obj
        self.is_tree = isinstance(obj, dict)

    def which(self, oneof, names):
        if self.is_tree:
            have = [n for n in names if n in self.obj]
            return have[-1] if have else None
        return self.obj.WhichOneof(oneof)

    def sub(self, name):
        return _Node(self.obj[name][-1] if self.is_tree else getattr(self.obj, name))

    def value(self, name, default):
        if self.is_tree:
            return self.obj[name][-1] if name in self.obj else default
        return getattr(self.obj, name)

    def values(self, name):
        return list(self.obj.get(name, [])) if self.is_tree else list(getattr(self.obj, name))


def settings(optimizer_cfg):
    """-> OptimSettings from ``train_config.optimizer``: the proto message, or the dict ``config.parse_prototxt`` gives
    for that block (``tree["train_config"][-1]["optimizer"][-1]``).  An OptimSettings passes through."""
    if isinstance(optimizer_cfg, OptimSettings):
        return optimizer_cfg
    c = _Node(optimizer_cfg)
    kind = c.which("optimizer", ("rms_prop_optimizer", "momentum_optimizer", "adam_optimizer"))
    if kind != "adam_optimizer":
        raise UnsupportedNetwork("optimizer %s is not supported (adam_optimizer is)" % kind)
    if bool(c.value("use_moving_average", False)):
        raise UnsupportedNetwork("use_moving_average is not supported")
    adam = c.sub("adam_optimizer")
    if bool(adam.value("amsgrad", False)):
        raise UnsupportedNetwork("amsgrad: true is not supported")
    decoupled = bool(c.value("fixed_weight_decay", False))
    rate = adam.sub("learning_rate") if (not adam.is_tree or "learning_rate" in adam.obj) else _Node({})
    sched = rate.which("learning_rate", ("multi_phase", "one_cycle", "exponential_decay", "manual_stepping"))
    kw = dict(decoupled=decoupled, weight_decay=_f32(adam.value("weight_decay", 0.0)), beta1=0.9,
              beta2=0.99 if decoupled else 0.999, schedule=sched)
    if sched == "one_cycle":
        s = rate.sub(sched)
        kw.update(lr_max=_f32(s.value("lr_max", 0.0)), moms=tuple(_f32(v) for v in s.values("moms")),
                  div_factor=_f32(s.value("div_factor", 0.0)), pct_start=_f32(s.value("pct_start", 0.0)))
    elif sched == "exponential_decay":
        s = rate.sub(sched)
        kw.update(initial_learning_rate=_f32(s.value("initial_learning_rate", 0.0)),
                  decay_length=_f32(s.value("decay_length", 0.0)), decay_factor=_f32(s.value("decay_factor", 0.0)),
                  staircase=bool(s.value("staircase", False)))
    elif sched == "manual_stepping":
        s = rate.sub(sched)
        kw.update(boundaries=tuple(_f32(v) for v in s.values("boundaries")),
                  rates=tuple(_f32(v) for v in s.values("rates")))
    else:
        raise UnsupportedNetwork("learning rate schedule %s is not supported (one_cycle, exponential_decay and "
                                 "manual_stepping are)" % sched)
    return OptimSettings(**kw)


def _annealing_cos(start, end, pct):
    return end + (start - end) / 2 * (np.cos(np.pi * pct) + 1)


def _phase_values(total_step, phases):
    """LRSchedulerStep's rule: phases are (start fraction, function of the progress through the phase); a step belongs
    to the last phase that has begun and a phase ends where the next begins (the last at total_step)."""
    starts = [int(start * total_step) for start, _ in phases]
    if starts[0] != 0 or any(b <= a for a, b in zip(starts, starts[1:])):
        raise ValueError("schedule phases must start at step 0 and at increasing steps, got %s for %d steps"
                         % (starts, total_step))
    ends = starts[1:] + [total_step]
    out = []
    for (_, func), start, end in zip(phases, starts, ends):
        out.extend(float(func((step - start) / (end - start))) for step in range(start, min(end, total_step)))
    return out


def schedule(s: OptimSettings, total_step):
    """-> (lr, beta1) per step 0 .. total_step - 1 as two lists of Python floats, from the scalar expressions of
    OneCycle / ExponentialDecay / ManualStepping (learning_schedules_fastai.py:62-130)."""
    total_step = int(total_step)
    if total_step < 1:
        raise ValueError("total_step must be >= 1")
    moms = [s.beta1] * total_step
    if s.schedule == "one_cycle":
        if len(s.moms) != 2:
            raise ValueError("one_cycle needs two moms, got %r" % (s.moms,))
        low = s.lr_max / s.div_factor
        lrs = _phase_values(total_step, [(0, lambda p: _annealing_cos(low, s.lr_max, p)),
                                         (s.pct_start, lambda p: _annealing_cos(s.lr_max, low / 1e4, p))])
        moms = _phase_values(total_step, [(0, lambda p: _annealing_cos(s.moms[0], s.moms[1], p)),
                                          (s.pct_start, lambda p: _annealing_cos(s.moms[1], s.moms[0], p))])
    elif s.schedule == "exponential_decay":
        if not 0 < s.decay_length < 1:
            raise ValueError("decay_length must be in (0, 1)")
        if s.staircase:
            stride = int(s.decay_length * total_step)
            if stride < 1:
                raise ValueError("decay_length * total_step must be at least one step")
            phases, step, stage = [], 0, 1
            while step <= total_step:
                phases.append((step / total_step, lambda p, _d=s.initial_learning_rate * stage: _d))
                stage *= s.decay_factor
                step += stride
        else:
            # as the reference computes it: the continuous form does not multiply by initial_learning_rate
            phases = [(0, lambda p: pow(s.decay_factor, p / s.decay_length))]
        lrs = _phase_values(total_step, phases)
    elif s.schedule == "manual_stepping":
        if not all(0 < b < 1 for b in s.boundaries) or len(s.boundaries) + 1 != len(s.rates):
            raise ValueError("manual_stepping needs boundaries in (0, 1) and one more rate than boundaries")
        lrs = _phase_values(total_step, [(b, lambda p, _d=r: _d) for b, r in zip((0.0,) + s.boundaries, s.rates)])
    else:
        raise UnsupportedNetwork("learning rate schedule %s is not supported" % s.schedule)
    return lrs, moms


def schedule_table(s: OptimSettings, total_step):
    """-> float64 [total_step, 5], row ``i`` for the step taken after ``i`` earlier ones (Adam's t = i + 1): HYPER_COLS.
    Every entry is the Python double the reference's scheduler and torch.optim.Adam compute on the host."""
    lrs, moms = schedule(s, total_step)
    rows = [(lr, b1, 1 - b1 ** (i + 1), (1 - s.beta2 ** (i + 1)) ** 0.5, 1 - s.weight_decay * lr)
            for i, (lr, b1) in enumerate(zip(lrs, moms))]
    return np.array(rows, dtype=np.float64).reshape(len(rows), len(HYPER_COLS))


def parameter_groups(net):
    """-> the reference's two parameter groups, ``split_bn_bias(get_layer_groups(net))`` (fastai_optim.py:14-23,
    optimizer_builder.py:33-35): the ``requires_grad`` parameters of the leaf modules that are not batch norms, then
    those of the batch norms, in depth-first module order, each parameter once."""
    def leaves(m):
        kids = list(m.children())
        return [m] if not kids else [leaf for k in kids for leaf in leaves(k)]

    groups, seen = ([], []), set()
    for leaf in leaves(net):
        for p in leaf.parameters():
            if p.requires_grad and id(p) not in seen:
                seen.add(id(p))
                groups[isinstance(leaf, _BN_TYPES)].append(p)
    return list(groups)


def plan(net, optimizer_cfg, total_step, data_parallel=None):
    """-> OptimPlan for ``net``, the optimizer block (see ``settings``) and ``train_config.steps``; ``data_parallel``:
    the handle of ``b2second.dist.enable_data_parallel(net)``, to all-reduce the gradients in every ``step``."""
    return OptimPlan(settings(optimizer_cfg), parameter_groups(net), total_step, data_parallel=data_parallel)


class OptimPlan:
    """the optimizer of one network (see ``plan``)."""

    def __init__(self, s: OptimSettings, groups, total_step, data_parallel=None):
        self.settings = s
        self.groups = groups
        self.params = [p for g in groups for p in g]
        if not self.params:
            raise ValueError("no trainable parameter")
        if data_parallel is not None and [id(p) for p in data_parallel.params] != [id(p) for p in self.params]:
            raise ValueError("the data-parallel handle was made for other parameters (enable_data_parallel(net) on "
                             "the same network)")
        self.data_parallel = data_parallel
        dev = self.params[0].device
        for p in self.params:
            if p.dtype != torch.float32:
                raise UnsupportedNetwork("parameters must be float32, got %s (mixed precision and loss scaling are "
                                         "not supported)" % p.dtype)
            if p.device != dev or not p.is_contiguous():
                raise UnsupportedNetwork("parameters must be contiguous and on one device")
            if p.numel() >= 1 << 31:
                raise UnsupportedNetwork("a parameter tensor of 2^31 or more elements is not supported")
        self.total_step = int(total_step)
        self.table = schedule_table(s, self.total_step)
        self.device = dev
        self.hyper = torch.from_numpy(self.table).to(dev)
        self.exp_avg = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        self.exp_avg_sq = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        for p in self.params:
            if p.grad is None:
                p.grad = torch.zeros_like(p, memory_format=torch.contiguous_format)
        self.step_count = torch.zeros(1, dtype=torch.int64, device=dev)
        self.total_norm = torch.zeros(1, dtype=torch.float32, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)   # device word; see spconv._lib.STATUS_BITS
        self.table_builds = 0
        self._grad_ptrs = None
        self._device_tables = None
        self._params_c = None

    # ---- the step ----------------------------------------------------------------------------------------------
    def _c_params(self, zero_grad):
        if self._params_c is None:
            L, _ = _lib()
            s = self.settings
            both = []
            for z in (0, 1):
                c = L.OptimParams()
                c.weight_decay, c.beta2, c.eps, c.max_norm = s.weight_decay, s.beta2, s.eps, s.clip_norm
                c.total_step, c.decoupled, c.zero_grad = self.total_step, int(s.decoupled), z
                both.append(c)
            self._params_c = both
        return ctypes.byref(self._params_c[int(zero_grad)])

    def _build_tables(self, grad_ptrs):
        L, lib = _lib()
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("a gradient moved since the last optimizer step; take one eager step before capturing")
        chunks = []
        for t, p in enumerate(self.params):
            n = p.numel()
            chunks.extend((t, o, min(L.OPTIM_CHUNK, n - o), 0) for o in range(0, n, L.OPTIM_CHUNK))
        ptrs = np.array([[p.data_ptr() for p in self.params], grad_ptrs, [m.data_ptr() for m in self.exp_avg],
                         [v.data_ptr() for v in self.exp_avg_sq]], dtype=np.int64)
        tabs = {"ptrs": torch.from_numpy(ptrs).to(self.device),
                "chunks": torch.tensor(chunks, dtype=torch.int32).view(-1, 4).to(self.device),
                "num_chunks": len(chunks)}
        ws_bytes = lib.b2s_optim_workspace_bytes(len(chunks))
        tabs["ws"] = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
        tabs["ws_bytes"] = ws_bytes
        self._device_tables = tabs
        self._grad_ptrs = grad_ptrs
        self.table_builds += 1

    def step(self, set_to_none=False):
        """one training step's clip, decay, Adam update, schedule advance and zero_grad; -> the gradient norm before
        clipping (device float32 scalar).  No host synchronisation.  Under data parallelism the gradients are first
        averaged over the ranks, and ``set_to_none`` is refused (it would detach them from the bucket)."""
        dp = self.data_parallel
        if dp is not None and set_to_none:
            raise ValueError("step(set_to_none=True) would detach the gradients from the data-parallel bucket; "
                             "zero them in place (set_to_none=False)")
        L, lib = _lib()
        L.require_cuda(self.params[0], "parameters")
        grads = [p.grad for p in self.params]
        for g, p in zip(grads, self.params):
            if g is not None and (g.dtype != torch.float32 or not g.is_contiguous() or g.shape != p.shape or
                                  g.device != p.device):
                raise TypeError("gradients must be dense contiguous float32 tensors of their parameter's shape")
        grad_ptrs = [0 if g is None else g.data_ptr() for g in grads]
        if grad_ptrs != self._grad_ptrs:
            self._build_tables(grad_ptrs)
        t = self._device_tables
        n = len(self.params)
        base = t["ptrs"].data_ptr()
        with torch.cuda.device(self.device):
            if dp is not None:
                dp.all_reduce_grads()
            L.check(lib.b2s_optim_step(
                ctypes.c_void_p(base), ctypes.c_void_p(base + 8 * n), ctypes.c_void_p(base + 16 * n),
                ctypes.c_void_p(base + 24 * n), n, L.ptr(t["chunks"]), t["num_chunks"], L.ptr(self.hyper),
                L.ptr(self.step_count), self._c_params(not set_to_none), L.ptr(self.total_norm), L.ptr(t["ws"]),
                t["ws_bytes"], L.ptr(self.status), L.stream()), "b2s_optim_step")
        self.touch()
        if set_to_none:
            for p in self.params:
                p.grad = None
        return self.total_norm[0]

    def touch(self):
        """bump the autograd version of every stepped parameter, which the caches keyed on it (the drop-in's packed
        weights and folded batch norms) watch.  ``step`` calls it; call it yourself after replaying a captured step."""
        torch.autograd.graph.increment_version(self.params)

    # ---- what the training loop logs ---------------------------------------------------------------------------
    @property
    def global_step(self):
        """steps taken so far, read from the device counter (this synchronises)"""
        return int(self.step_count.item())

    @global_step.setter
    def global_step(self, value):
        self.step_count.fill_(int(value))

    def _row(self):
        return self.table[min(max(self.global_step, 0), self.total_step - 1)]

    @property
    def lr(self):
        """the learning rate of the next step (the table row the device counter points at; this synchronises)"""
        return float(self._row()[0])

    @property
    def mom(self):
        """beta1 of the next step"""
        return float(self._row()[1])

    # ---- checkpoints: torch.optim.Adam's format ----------------------------------------------------------------
    def state_dict(self):
        s = self.settings
        t = self.global_step
        row = self._row()
        state = {}
        if t > 0:
            for i in range(len(self.params)):
                state[i] = {"step": torch.tensor(float(t), dtype=torch.float32), "exp_avg": self.exp_avg[i],
                            "exp_avg_sq": self.exp_avg_sq[i]}
        groups, first = [], 0
        for g in self.groups:
            groups.append({"lr": float(row[0]), "betas": (float(row[1]), s.beta2), "eps": s.eps,
                           "weight_decay": 0 if s.decoupled else s.weight_decay, "amsgrad": False,
                           "params": list(range(first, first + len(g)))})
            first += len(g)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        """resume from ``torch.optim.Adam.state_dict()`` (what the reference's OptimWrapper saves) or from
        ``state_dict()``.  The moments are copied into this plan's buffers and the device step counter set from
        ``step``, which must be the same for every parameter that has state."""
        sizes = [len(g["params"]) for g in sd["param_groups"]]
        if sizes != [len(g) for g in self.groups]:
            raise ValueError("checkpoint has parameter groups of sizes %s, this network %s"
                             % (sizes, [len(g) for g in self.groups]))
        if any(g.get("amsgrad", False) for g in sd["param_groups"]):
            raise UnsupportedNetwork("amsgrad: true is not supported")
        order = [i for g in sd["param_groups"] for i in g["params"]]
        steps = set()
        with torch.no_grad():
            for k, idx in enumerate(order):
                st = sd["state"].get(idx)
                if st is None:
                    self.exp_avg[k].zero_()
                    self.exp_avg_sq[k].zero_()
                    continue
                if tuple(st["exp_avg"].shape) != tuple(self.params[k].shape):
                    raise ValueError("checkpoint moment %d has shape %s, the parameter %s"
                                     % (idx, tuple(st["exp_avg"].shape), tuple(self.params[k].shape)))
                self.exp_avg[k].copy_(st["exp_avg"])
                self.exp_avg_sq[k].copy_(st["exp_avg_sq"])
                steps.add(int(float(st["step"])))
        if len(steps) > 1:
            raise ValueError("parameters with different step counts (%s) are not supported" % sorted(steps))
        self.global_step = steps.pop() if steps else 0
