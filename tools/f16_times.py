"""the half-precision mode (precision="f16") against the default fp32-grade mode of the fused engine:
python tools/f16_times.py [rounds] [steps]

Per config (car.fhd and pointpillars.car.xyres_16 at B = 32 on 29 k-point bench clouds, nuscenes.all.pp.largea at
B = 4 on 300 k-point clouds; the seeded mirror network), two engines on the same network, one per precision:
  resident   clouds/s of eng.infer(device clouds) (bench.py's resident loop: the graph with the clouds in HBM); the two
             precisions alternate within every round, reported as (min, median, max) over the rounds
  stages     ms per stage of one eager step with a CUDA event before each stage (engine.run_timed, mean of 5): the
             sparse encoder (sum of the sparse_conv* stages, rulebooks apart), "rpn" (the 3x3 layers of every block,
             stride 1 and 2), "rpn_1x1" (deblocks, heads and the fused tail), and the rest
  planes     bytes of fp16 operand planes each engine holds (engine.fp16_plane_bytes): the f16 engine allocates no lo
             planes, so the fp32 engine's "lo" is what the mode saves
"""
import sys

import _measure
import torch

from b2second.engine import InferenceEngine

CASES = [("car.fhd", 32, 29000), ("pointpillars.car.xyres_16", 32, 29000), ("nuscenes.all.pp.largea", 4, 300000)]
PRECISIONS = ("fp32", "f16")


def spread(xs):
    xs = sorted(xs)
    return [round(xs[0], 3), round(xs[len(xs) // 2], 3), round(xs[-1], 3)]


def stages(eng):
    t = eng.run_timed(iters=5)
    out = {"sparse_conv": sum(v for k, v in t.items() if k.startswith("sparse_conv")),
           "rulebooks": sum(v for k, v in t.items() if k.startswith("rulebook"))}
    out.update({k: v for k, v in t.items() if not k.startswith(("sparse_conv", "rulebook"))})
    return {k: round(v, 4) for k, v in out.items()}


def measure(name, B, points, rounds, steps):
    net, clouds = _measure.mirror(name, B, points=points)
    net = net.eval()
    engines = {p: InferenceEngine(net, batch_size=B, max_points=points + 1000, precision=p) for p in PRECISIONS}
    dev = engines["fp32"].dev
    frames = [torch.from_numpy(c).to(dev) for c in clouds]
    anchors = torch.from_numpy(net.anchors()[None]).to(dev)
    for eng in engines.values():
        eng.set_anchors(anchors)
    ms = {p: [] for p in PRECISIONS}
    for _ in range(rounds):
        for p, eng in engines.items():
            ms[p].append(_measure.timed(lambda: eng.infer(frames), steps))
    out = {"config": name, "batch": B, "points_per_cloud": points}
    for p, eng in engines.items():
        eng.check_status()
        out[p] = {"ms_per_step": spread(ms[p]), "clouds_per_s": spread([B / (t * 1e-3) for t in ms[p]]),
                  "stages_ms": stages(eng), "fp16_plane_bytes": eng.fp16_plane_bytes()}
    med = {p: sorted(ms[p])[rounds // 2] for p in PRECISIONS}
    out["f16_speedup_median"] = round(med["fp32"] / med["f16"], 4)
    out["lo_plane_bytes_saved"] = out["fp32"]["fp16_plane_bytes"]["lo"] - out["f16"]["fp16_plane_bytes"]["lo"]
    del engines, net
    torch.cuda.empty_cache()
    return out


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 50
    _measure.require_gpu("f16_times")
    with _measure.clocks() as clk:
        results = [measure(name, B, points, rounds, steps) for name, B, points in CASES]
    _measure.report("f16_times", results, clk, rounds=rounds, steps=steps,
                    timing="CUDA events around back-to-back resident steps (no L2 flush), precisions alternated "
                           "within each round; stages: one eager step with an event before each stage")


if __name__ == "__main__":
    main()
