"""clouds/s of the three serving loops over the same two alternating pinned batches:
python tools/stream_times.py [rounds] [steps]

For car.fhd and pointpillars.car.xyres_16 at B = 32 (29 k-point bench clouds, the seeded mirror network, host
detections), each round times, back to back with no L2 flush:
  resident  eng.infer(device clouds): the graph with the clouds already in HBM (bench.py's resident loop)
  net       net(example) on pinned host clouds (bench.py's e2e loop): copy, graph, read-back, sync, result dicts
  stream    net.b2s_fastpath.stream over `steps` such examples: the next batch's copy overlaps the current graph
  h2d       eng.load_points(pinned clouds) alone: what the copy of one batch takes
The loops alternate within every round; each is reported as (min, median, max) over the rounds.
"""
import collections
import itertools
import sys

import _measure
import torch

import bench
from b2second import fastpath

B = 32
POINTS = 29000


def spread(xs):
    xs = sorted(xs)
    return [round(xs[0], 3), round(xs[len(xs) // 2], 3), round(xs[-1], 3)]


def measure(name, rounds, steps):
    net, clouds = _measure.mirror(name, 2 * B, points=POINTS)
    net = fastpath.accelerate(net.eval(), max_points=POINTS + 1000, output="host")
    fast = net.b2s_fastpath
    eng = fast.engine(B)
    dev = eng.dev
    host = [bench.pinned_slab(clouds[s * B:(s + 1) * B]) for s in range(2)]
    devc = [bench.device_slab(h, dev) for h in host]
    anchors = torch.from_numpy(net.anchors()[None]).to(dev)
    examples = [{"points": host[k % 2], "anchors": anchors} for k in range(steps)]
    turn = itertools.count()
    loops = {
        "resident": lambda: _measure.timed(lambda: eng.infer(devc[next(turn) % 2]), steps),
        "net": lambda: _measure.timed(lambda: net({"points": host[next(turn) % 2], "anchors": anchors}), steps),
        "stream": lambda: _measure.timed(lambda: collections.deque(fast.stream(examples), maxlen=0), 1,
                                         warmup=1) / steps,
        "h2d": lambda: _measure.timed(lambda: eng.load_points(host[next(turn) % 2]), steps),
    }
    ms = {k: [] for k in loops}
    for _ in range(rounds):
        for k, fn in loops.items():
            ms[k].append(fn())
    eng.check_status()
    out = {"config": name, "batch": B, "points_per_cloud": POINTS}
    for k, v in ms.items():
        out[k] = {"ms_per_step": spread(v)}
        if k != "h2d":
            out[k]["clouds_per_s"] = spread([B / (t * 1e-3) for t in v])
    res = sorted(ms["resident"])[rounds // 2]
    out["stream_over_resident_ms"] = round(sorted(ms["stream"])[rounds // 2] / res, 4)
    out["net_over_resident_ms"] = round(sorted(ms["net"])[rounds // 2] / res, 4)
    del eng, fast, net
    torch.cuda.empty_cache()
    return out


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 100
    _measure.require_gpu("stream_times")
    with _measure.clocks() as clk:
        results = [measure(name, rounds, steps) for name in ("car.fhd", "pointpillars.car.xyres_16")]
    _measure.report("stream_times", results, clk, rounds=rounds, steps=steps,
                    timing="CUDA events around back-to-back steps (no L2 flush); stream: one stream of `steps` "
                           "examples, ms per example")


if __name__ == "__main__":
    main()
