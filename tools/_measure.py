"""The measurement code of every tool under tools/: how a time is taken and what is recorded beside it.

A tool starts with ``import _measure``, which puts the repository root, second.pytorch_b200 and tests on sys.path.
Measurement needs a CUDA device and never falls back to the CPU.  An absolute time is only worth something next to
the card and the power limit it was measured on, so every tool prints ``card()`` and the SM clock sampled while it ran.
"""
import contextlib
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(REPO, "tests"), REPO, os.path.join(REPO, "second.pytorch_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

import bench  # noqa: E402

CARD_FIELDS = ("device", "power_limit", "sm_clock_max")       # nvidia-smi's name, power.limit, clocks.max.sm
UNAVAILABLE = "unavailable"


def require_gpu(what):
    """raise unless a CUDA device is present; set the fp32 policy (no TF32 in cuDNN or cuBLAS)"""
    if not torch.cuda.is_available():
        raise RuntimeError("%s measures on a CUDA device and this machine has none" % what)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def parse_card(text):
    """the card fields of `nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader` output;
    a field the card reports as [N/A], or output that is not one such line, reads "unavailable"."""
    lines = text.strip().splitlines()
    fields = lines[0].rsplit(",", 2) if len(lines) == 1 else []
    if len(fields) != len(CARD_FIELDS):
        fields = [""] * len(CARD_FIELDS)
    fields = [f.strip() for f in fields]
    return {k: UNAVAILABLE if v in ("", "[N/A]", "N/A") else v for k, v in zip(CARD_FIELDS, fields)}


def card():
    """name, power limit and maximum SM clock of the current device, from one read-only nvidia-smi query"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        text = q.stdout if q.returncode == 0 else ""
    except (OSError, subprocess.SubprocessError):
        text = ""
    return parse_card(text)


@contextlib.contextmanager
def clocks():
    """sample the SM clock with bench.ClockSampler while the block runs; yields a dict that holds the sampler's
    summary once the block ends.  A block that ends before nvidia-smi's first sample waits (up to 5 s) for one, so the
    summary holds at least a clock read right after the block.  The sampler is stopped however the block ends, so no
    nvidia-smi outlives a tool."""
    sampler = bench.ClockSampler(torch.cuda.current_device())
    summary = {}
    sampler.start()
    try:
        yield summary
    finally:
        deadline = time.perf_counter() + 5
        while sampler.proc is not None and sampler.proc.poll() is None and not sampler.rows \
                and time.perf_counter() < deadline:
            time.sleep(0.02)
        summary.update(sampler.stop())


def timed(fn, iters, warmup=3, flush=None, host=False):
    """ms per call of fn() on the device, after `warmup` untimed calls.

    Without `flush`: CUDA events around `iters` back-to-back calls, the mean.  With host=True, also the host-clock ms
    per call spent in that loop before its final synchronise (what the host takes to enqueue a call).
    With a `flush` buffer: CUDA events around each call, the buffer written between calls to evict L2 (outside the
    event pair), the median.  The fp32 policy is left as the caller set it."""
    if not torch.cuda.is_available():
        raise RuntimeError("timed() measures on a CUDA device and this machine has none")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    if flush is not None:
        ts = []
        for i in range(iters):
            flush.fill_(i)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    h0 = time.perf_counter()
    for _ in range(iters):
        fn()
    h1 = time.perf_counter()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return (ms, (h1 - h0) * 1e3 / iters) if host else ms


def peak_bytes(fn):
    """torch.cuda.max_memory_allocated over one call of fn(), above what was allocated before it"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def mirror(name, batch=None, spconv="product", points=29000):
    """the mirror network of config `name` with seeded synthetic weights, on the GPU; with a batch, also that many
    bench.make_clouds clouds of `points` points (numpy, on the host)"""
    from b2second import config, loader, models
    sp = loader.product_spconv() if spconv == "product" else loader.oracle_spconv()
    net = models.build_network(config.get_config(name), sp)
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    return net if batch is None else (net, bench.make_clouds(name, batch, points))


def report(tool, results, sm_clock, **fields):
    """print and return the tool's one JSON line: the card, the SM clock summary of clocks(), the fields and the
    results"""
    line = json.dumps({"tool": tool, **card(), "sm_clock": sm_clock, **fields, "results": results})
    print(line, flush=True)
    return line
