"""CUDA-event and host time of the optimizer step: python tools/optim_step_times.py [iters]

Prints one JSON line.  Per network (the mirrors of car.fhd, pointpillars/car/xyres_16 and nuscenes/all.pp.mhead, each
with its config's decay form and schedule, random gradients): per step
  fused         b2second.optim step() (csrc/optim.cu: two kernels); ``fused_replay_gpu_ms`` is the same step captured
                in a CUDA graph and replayed, which takes the host out of the GPU figure
  torch         the reference's sequence restated with torch: clip_grad_norm_, the per-parameter decay loop of
                OptimWrapper.step (fixed_weight_decay configs), torch.optim.Adam (default foreach) with lr and betas set
                as the scheduler sets them, zero_grad(set_to_none=False) -- gradients are zeroed in place, as the torch
                of the reference's time did, so that every timed step has gradients
  torch_fused   the same with torch.optim.Adam(fused=True), the strongest torch baseline
each as ``*_gpu_ms`` (CUDA events around ITERS back-to-back steps after warm-ups) and ``*_host_ms`` (host clock around
the same loop before the final synchronise: what the host spends enqueueing a step), the device activities one step
launches (``*_launches``, counted with torch.profiler in a run of its own), and the byte floor: 4 B per parameter for
the norm pass, 16 B read + 12 B written + 4 B of zeroed gradient for the update, at the H100 SXM data-sheet 3.35 TB/s
(arithmetic, not a measurement).  Also prints the card name, its power limit and the SM clock sampled during the run.
"""
import sys

import _measure
import optim_ref as orf
import torch

from b2second import optim

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_PARAM = 4 + 16 + 12 + 4
TOTAL_STEP = 30000
NETWORKS = (("car.fhd", orf.ONE_CYCLE), ("pointpillars.car.xyres_16", orf.STAIRCASE),
            ("nuscenes.all.pp.mhead", orf.ONE_CYCLE))


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def build(name):
    net = _measure.mirror(name, spconv="oracle")
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    for p in net.parameters():
        p.grad = torch.randn(p.shape, generator=gen, device="cuda:0") * 0.01
    return net


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    _measure.require_gpu("optim_step_times")
    rows = []
    with _measure.clocks() as clk:
        for name, s in NETWORKS:
            row = {"config": name, "decay": "decoupled" if s.decoupled else "l2", "schedule": s.schedule}
            net = build(name)
            opt = optim.plan(net, s, TOTAL_STEP)
            row["tensors"] = len(opt.params)
            row["parameters"] = sum(p.numel() for p in opt.params)
            variants = {"fused": opt.step}
            for key, kw in (("torch", {}), ("torch_fused", {"fused": True})):
                twin = build(name)
                adam = orf.torch_adam(s, optim.parameter_groups(twin), **kw)
                step = [0]

                def chain(adam=adam, step=step):
                    i = step[0] % TOTAL_STEP
                    orf.torch_step(s, adam, float(opt.table[i, 0]), float(opt.table[i, 1]))
                    step[0] += 1
                variants[key] = chain
            for key, fn in variants.items():
                gpu, host = _measure.timed(fn, ITERS, warmup=10, host=True)
                row[key + "_gpu_ms"], row[key + "_host_ms"] = round(gpu, 4), round(host, 4)
            for key, fn in variants.items():
                row[key + "_launches"] = launches(fn)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                opt.step()
            row["fused_replay_gpu_ms"] = round(_measure.timed(graph.replay, ITERS, warmup=10), 4)
            nbytes = BYTES_PER_PARAM * row["parameters"]
            row["byte_floor"] = nbytes
            row["byte_floor_ms"] = round(nbytes / HBM_BYTES_PER_S * 1e3, 4)
            rows.append(row)
    _measure.report("optim_step_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
