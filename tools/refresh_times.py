"""What evaluating during training costs on the fused engine: python tools/refresh_times.py [rounds]

Per config (the seeded mirror network, B = 8, 29 k-point bench clouds, a candidate list that holds every anchor so the
seed-1 weights cannot overflow it), each round times, from the host clock around
work that ends in a device synchronise:
  refresh   net.load_state_dict(other weights) + the next net(example), minus that net(example) alone: what a refresh
            adds to the first call after eval() or a checkpoint load
  rebuild   a new FastPath on the same network, its engine and its first net(example) (graph capture included): what
            a newly accelerated copy of the network costs instead
and, for car.fhd and pointpillars.car.xyres_16, one eval pass over 3769 clouds (KITTI val) at B = 8 (the last batch
smaller):
  engine    net(example) on the fused engine after eval() (one refresh, then the graphs)
  dropin    the same examples' voxels through the module-by-module forward on the spconv drop-in, synchronised per batch
Each figure is (min, median, max) over the rounds.
"""
import sys
import time

import _measure
import numpy as np
import torch

from b2second import fastpath, models

B = 8
POINTS = 29000
KITTI_VAL = 3769
NAMES = ["car.fhd", "car.lite", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea",
         "nuscenes.all.pp.mhead"]


def spread(xs):
    xs = sorted(xs)
    return [round(xs[0], 3), round(xs[len(xs) // 2], 3), round(xs[-1], 3)]


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def refresh_vs_rebuild(name, rounds):
    net, clouds = _measure.mirror(name, B, points=POINTS)
    cand_cap = int(np.prod(net.anchors().shape[:-1]))      # every anchor: the seed-1 weights cannot overflow it
    net = fastpath.accelerate(net.eval(), max_points=POINTS + 1000, cand_cap=cand_cap)
    dev = next(net.parameters()).device
    example = {"points": [torch.from_numpy(c).to(dev) for c in clouds],
               "anchors": torch.from_numpy(net.anchors()[None]).to(dev)}
    states = [{k: v.clone() for k, v in net.state_dict().items()},
              models.synthetic_weights_(_measure.mirror(name), name, seed=1).state_dict()]
    for _ in range(3):
        net(example)
    ms = {"call": [], "load_and_call": [], "rebuild": []}
    for r in range(rounds):
        ms["call"].append(host_ms(lambda: net(example)))
        ms["load_and_call"].append(host_ms(lambda: (net.load_state_dict(states[(r + 1) % 2]), net(example))))

        def rebuild():
            fast = fastpath.FastPath(net, max_points=POINTS + 1000, cand_cap=cand_cap)
            fast(example)
        ms["rebuild"].append(host_ms(rebuild))
        torch.cuda.empty_cache()
    out = {"config": name, "batch": B, "points_per_cloud": POINTS,
           "refresh_ms": spread([a - c for a, c in zip(ms["load_and_call"], ms["call"])])}
    out.update({k + "_ms": spread(v) for k, v in ms.items()})
    del net
    torch.cuda.empty_cache()
    return out


def eval_pass(name, rounds):
    net, clouds = _measure.mirror(name, B, points=POINTS)
    dev = next(net.parameters()).device
    vg = net.voxel_generator
    anchors = torch.from_numpy(net.anchors()[None]).to(dev)
    sizes = [B] * (KITTI_VAL // B) + ([KITTI_VAL % B] if KITTI_VAL % B else [])
    batches = [[torch.from_numpy(clouds[i % B]).to(dev) for i in range(b)] for b in sizes]
    # the drop-in's input: the reference's voxel dict of each distinct batch size (voxelised once, on the GPU)
    voxels = {}
    for b in set(sizes):
        pts = torch.cat(batches[sizes.index(b)])
        offs = torch.tensor([0] + [int(c.shape[0]) for c in batches[sizes.index(b)]], device=dev).cumsum(0).int()
        res = vg.generate_device(pts, getattr(vg, "_max_voxels", 20000), frame_offsets=offs, batch=b)
        n = int(res["num_voxels"][0].item())
        voxels[b] = {"voxels": res["voxels"][:n], "num_points": res["num_points_per_voxel"][:n],
                     "coordinates": res["coordinates"][:n], "anchors": anchors.repeat(b, 1, 1)}
    plain = net.forward
    fast_net = fastpath.accelerate(net, max_points=POINTS + 1000)

    def engine():
        fast_net.eval()
        for pts in batches:
            fast_net({"points": pts, "anchors": anchors})

    def dropin():
        with torch.no_grad():
            for b in sizes:
                plain(voxels[b])
                torch.cuda.synchronize()
    engine()                  # builds both engines and captures their graphs
    dropin()
    ms = {"engine": [], "dropin": []}
    for _ in range(rounds):
        ms["engine"].append(host_ms(engine))
        ms["dropin"].append(host_ms(dropin))
    del net, fast_net
    torch.cuda.empty_cache()
    return {"config": name, "clouds": KITTI_VAL, "batch": B, "points_per_cloud": POINTS,
            **{k + "_s": spread([t / 1e3 for t in v]) for k, v in ms.items()}}


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    _measure.require_gpu("refresh_times")
    with _measure.clocks() as clk:
        results = {"refresh": [], "eval_pass": []}
        for kind, fn, names in (("refresh", refresh_vs_rebuild, NAMES),
                                ("eval_pass", eval_pass, ("car.fhd", "pointpillars.car.xyres_16"))):
            for n in names:
                results[kind].append(fn(n, rounds))
                print("%s %s done" % (kind, n), file=sys.stderr, flush=True)     # progress; the report is stdout
    _measure.report("refresh_times", results, clk, rounds=rounds,
                    timing="host clock around work ending in a device synchronise; (min, median, max) over rounds")


if __name__ == "__main__":
    main()
