"""training-metric and weight-packing times (CUDA events and a host clock): python tools/train_metrics_times.py [N]

1. VoxelNet.update_metrics for car.fhd at batch 8 and nuscenes.all.pp.mhead at batch 4 (full anchor maps, synthetic
   logits and labels): N back-to-back calls of b2second.metrics (update_metrics: launch + one pinned copy per call;
   update_metrics_async: the launches alone) against the reference's torchplus sequence restated in torch on the same
   GPU (tests/metrics_ref.py), and the CUDA launches and runtime copies / synchronisations of one call of each
   (torch.profiler).
2. One drop-in training step of car.fhd's sparse middle encoder (tools/train_step_times.py's setup: batch 8 of 29 k-point
   clouds, forward + backward with enable_sparse_backward) after a weight update, so that every layer repacks its
   tensor-core weights: device packing (b2s_pack_sparse_weights) against the host path (tc.pack_sparse_weights +
   pow2_scale + split_f16, one host read per packing)."""
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import bench
import metrics_ref as mr
from b2second import config, loader, metrics, models, tc, training

N = int(sys.argv[1]) if len(sys.argv) > 1 else 50
DEV = "cuda:0"
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
sp = loader.product_spconv()
print(torch.cuda.get_device_name(0))
os.system("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv")


def timed(fn, n=N):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3, (time.perf_counter() - t0) / n * 1e6     # us (events, host clock)


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


print("\n== update_metrics, %d back-to-back calls ==" % N)
print("%-24s %5s %8s | %-26s %10s %10s %8s %6s %6s" % ("config", "batch", "anchors", "path", "events us", "host us",
                                                        "kernels", "copies", "syncs"))
for name, B in (("car.fhd", 8), ("nuscenes.all.pp.mhead", 4)):
    net = metrics.enable_gpu_metrics(models.build_network(config.get_config(name), sp).to(DEV))
    C = int(net._num_class)
    A = int(net.anchors().shape[0])
    st = mr.make_steps(0, B, A, C, steps=1)[0]
    args = mr.to_torch(st, DEV)
    ref = mr.MetricsRef(device=DEV)
    paths = [("b2second update_metrics", lambda: net.update_metrics(*args)),
             ("b2second ..._async", lambda: net.b2s_metrics.update_metrics_async(*args)),
             ("torchplus sequence (torch)", lambda: ref.update(*args, C))]
    for label, fn in paths:
        t_ev, t_host = timed(fn)
        k, c, s = counts(fn)
        print("%-24s %5d %8d | %-26s %10.1f %10.1f %8d %6d %6d" % (name, B, A, label, t_ev, t_host, k, c, s))

print("\n== drop-in training step of car.fhd's middle encoder, batch 8, weights updated before every step ==")
cfg = config.get_config("car.fhd")
net = models.build_network(cfg, sp)
models.synthetic_weights_(net, "car.fhd", seed=0)
net = net.cuda().train()
mid = training.enable_sparse_backward(net.middle_feature_extractor)
B = 8
feats, coors = [], []
for b, c in enumerate(bench.make_clouds("car.fhd", B, 29000)):
    res = net.voxel_generator.generate(c, cfg.max_voxels)
    n = res["voxel_num"]
    vf = torch.from_numpy(res["voxels"][:n]).sum(1) / torch.from_numpy(res["num_points_per_voxel"][:n]).clamp_min(1)[:, None]
    feats.append(vf[:, :4].float())
    coors.append(torch.from_numpy(np.pad(res["coordinates"][:n], ((0, 0), (1, 0)), constant_values=b)))
vf = torch.cat(feats).cuda()
coors = torch.cat(coors).int().cuda()
convs = [m for m in mid.modules() if isinstance(m, sp.SparseConvolution)]
g = None


def step():
    global g
    with torch.no_grad():
        for m in convs:
            m.weight.mul_(1.0)               # a new weight version, as after an optimizer step
    out = mid(vf, coors, B)
    if g is None:
        g = torch.randn(out.shape, device=DEV)
    (out * g).sum().backward()


def host_pack(w, transpose=False, flip=False):
    wt = (w.flip(0) if flip else w).transpose(1, 2).contiguous() if transpose else w
    wp = tc.pack_sparse_weights(wt)
    ws = tc.pow2_scale(wp)
    hi, lo = tc.split_f16(wp, ws)
    return hi, lo, torch.tensor([ws], dtype=torch.float32, device=w.device), \
        torch.tensor([1.0 / ws], dtype=torch.float32, device=w.device)


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
