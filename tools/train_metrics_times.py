"""training-metric and weight-packing times (CUDA events and a host clock): python tools/train_metrics_times.py [N]

1. VoxelNet.update_metrics for car.fhd at batch 8 and nuscenes.all.pp.mhead at batch 4 (full anchor maps, synthetic
   logits and labels): N back-to-back calls of b2second.metrics (update_metrics: launch + one pinned copy per call;
   update_metrics_async: the launches alone) against the reference's torchplus sequence restated in torch on the same
   GPU (tests/metrics_ref.py), and the CUDA launches and runtime copies / synchronisations of one call of each
   (torch.profiler).  The host clock spans the enqueueing of the N calls, not the final synchronise.
2. One drop-in training step of car.fhd's sparse middle encoder (tools/train_step_times.py's setup: batch 8 of 29 k-point
   clouds, forward + backward with enable_sparse_backward) after a weight update, so that every layer repacks its
   tensor-core weights: device packing (b2s_pack_sparse_weights) against the host path (tc.pack_sparse_weights +
   pow2_scale + split_f16, one host read per packing).
Prints the card first and the SM clock sampled during the run last."""
import json
import sys

import _measure
import metrics_ref as mr
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
from train_step_times import middle_encoder

from b2second import metrics, tc

DEV = "cuda:0"


def timed(fn, n):
    """(us per call between CUDA events, us per call on the host clock) after one warm-up"""
    ms, host_ms = _measure.timed(fn, n, warmup=1, host=True)
    return ms * 1e3, host_ms * 1e3


def counts(fn):
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
    ev = prof.events()
    kernels = sum(1 for e in ev if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                  and "Memset" not in e.name)
    copies = sum(1 for e in ev if e.name.startswith("cudaMemcpy"))
    # the profiler's own flush on stop is a cudaDeviceSynchronize: not counted
    syncs = sum(1 for e in ev if e.name in ("cudaStreamSynchronize", "cudaEventSynchronize"))
    return kernels, copies, syncs


def metric_rows(N):
    print("\n== update_metrics, %d back-to-back calls ==" % N)
    print("%-24s %5s %8s | %-26s %10s %10s %8s %6s %6s" % ("config", "batch", "anchors", "path", "events us",
                                                            "host us", "kernels", "copies", "syncs"))
    for name, B in (("car.fhd", 8), ("nuscenes.all.pp.mhead", 4)):
        net = metrics.enable_gpu_metrics(_measure.mirror(name))
        C = int(net._num_class)
        A = int(net.anchors().shape[0])
        st = mr.make_steps(0, B, A, C, steps=1)[0]
        args = mr.to_torch(st, DEV)
        ref = mr.MetricsRef(device=DEV)
        paths = [("b2second update_metrics", lambda: net.update_metrics(*args)),
                 ("b2second ..._async", lambda: net.b2s_metrics.update_metrics_async(*args)),
                 ("torchplus sequence (torch)", lambda: ref.update(*args, C))]
        for label, fn in paths:
            t_ev, t_host = timed(fn, N)
            k, c, s = counts(fn)
            print("%-24s %5d %8d | %-26s %10.1f %10.1f %8d %6d %6d" % (name, B, A, label, t_ev, t_host, k, c, s))


def host_pack(w, transpose=False, flip=False):
    wt = (w.flip(0) if flip else w).transpose(1, 2).contiguous() if transpose else w
    wp = tc.pack_sparse_weights(wt)
    ws = tc.pow2_scale(wp)
    hi, lo = tc.split_f16(wp, ws)
    return hi, lo, torch.tensor([ws], dtype=torch.float32, device=w.device), \
        torch.tensor([1.0 / ws], dtype=torch.float32, device=w.device)


def packing_rows():
    print("\n== drop-in training step of car.fhd's middle encoder, batch 8, weights updated before every step ==")
    B = 8
    sp, mid, vf, coors = middle_encoder(B)
    convs = [m for m in mid.modules() if isinstance(m, sp.SparseConvolution)]
    g = None

    def step():
        nonlocal g
        with torch.no_grad():
            for m in convs:
                m.weight.mul_(1.0)               # a new weight version, as after an optimizer step
        out = mid(vf, coors, B)
        if g is None:
            g = torch.randn(out.shape, device=DEV)
        (out * g).sum().backward()

    device_pack = sp._pack_tc_weights
    res = {"device": [], "host": []}
    for rep in range(3):                      # alternate the two, three times
        for label, fn in (("device", device_pack), ("host", host_pack)):
            sp._pack_tc_weights = fn
            res[label].append(timed(step, 10))
    sp._pack_tc_weights = device_pack
    for label, v in res.items():
        ev = [x[0] for x in v]
        print("%-6s packing: %8.2f ms per step (events; min %.2f, max %.2f over 3 alternating runs of 10 steps)" % (
            label, np.median(ev) / 1e3, min(ev) / 1e3, max(ev) / 1e3))


def main():
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    _measure.require_gpu("train_metrics_times")
    print(json.dumps(_measure.card()))
    with _measure.clocks() as clk:
        metric_rows(N)
        packing_rows()
    print(json.dumps({"sm_clock": clk}))


if __name__ == "__main__":
    main()
