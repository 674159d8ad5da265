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
(arithmetic, not a measurement).  Also prints the card name, its power limit and the SM clock read after each loop.
"""
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
sys.path.insert(0, os.path.join(REPO, "tests"))
import torch  # noqa: E402

import optim_ref as orf  # noqa: E402
from b2second import config, loader, models, optim  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 200
HBM_BYTES_PER_S = 3.35e12
BYTES_PER_PARAM = 4 + 16 + 12 + 4
TOTAL_STEP = 30000
NETWORKS = (("car.fhd", orf.ONE_CYCLE), ("pointpillars.car.xyres_16", orf.STAIRCASE),
            ("nuscenes.all.pp.mhead", orf.ONE_CYCLE))


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_ms(fn):
    """-> (GPU ms per call between CUDA events, host ms per call to enqueue)"""
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    h0 = time.perf_counter()
    for _ in range(ITERS):
        fn()
    h1 = time.perf_counter()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / ITERS, (h1 - h0) * 1e3 / ITERS


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def build(name):
    net = models.build_network(config.get_config(name), loader.oracle_spconv()).to("cuda:0")
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    for p in net.parameters():
        p.grad = torch.randn(p.shape, generator=gen, device="cuda:0") * 0.01
    return net


def main():
    assert torch.cuda.is_available(), "this tool times CUDA kernels: it needs a GPU"
    rows, clocks = [], []
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
            gpu, host = time_ms(fn)
            clocks.append(smi("clocks.sm"))
            row[key + "_gpu_ms"], row[key + "_host_ms"] = round(gpu, 4), round(host, 4)
        for key, fn in variants.items():
            row[key + "_launches"] = launches(fn)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            opt.step()
        row["fused_replay_gpu_ms"] = round(time_ms(graph.replay)[0], 4)
        clocks.append(smi("clocks.sm"))
        nbytes = BYTES_PER_PARAM * row["parameters"]
        row["byte_floor"] = nbytes
        row["byte_floor_ms"] = round(nbytes / HBM_BYTES_PER_S * 1e3, 4)
        rows.append(row)
    print(json.dumps({"tool": "optim_step_times", "device": torch.cuda.get_device_name(0),
                      "power_limit": smi("power.limit"), "sm_clock_after_each_loop": clocks, "iters": ITERS,
                      "results": rows}))


if __name__ == "__main__":
    main()
