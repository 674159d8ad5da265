"""ms per step the anchor-area mask adds to the fused engine (eager, a CUDA event before every stage, like
InferenceEngine.run_timed): python tools/anchor_mask_times.py [batch] [iters]

For each config: the "anchor_mask" stage of an engine built with anchor_area_threshold=1 (one memset + scatter, the two
scans of the summed-area table, the per-anchor lookup), the count map's size, and the whole step with and without the
mask.  pointpillars.car.xyres_16 has the threshold in its own eval config; car.fhd has it forced on (its config holds -1).
"""
import json
import sys

import _measure
import torch

from b2second.engine import InferenceEngine


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    ITERS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    _measure.require_gpu("anchor_mask_times")
    print(json.dumps(_measure.card()))
    with _measure.clocks() as clk:
        for name in ("pointpillars.car.xyres_16", "car.fhd"):
            pts = 20000
            net, uniq = _measure.mirror(name, min(B, 4), points=pts)
            net.eval()
            frames = [torch.from_numpy(uniq[i % len(uniq)]).cuda() for i in range(B)]
            row = {}
            for label, thr in (("off", None), ("on", 1.0)):
                eng = InferenceEngine(net, batch_size=B, max_points=pts + 1000, use_cuda_graph=False,
                                      anchor_area_threshold=thr)
                eng.load_points(frames)
                t = eng.run_timed(iters=ITERS)
                row[label] = (sum(t.values()), t.get("anchor_mask"), eng)
                if thr is not None:
                    kept = float(eng.anchors_mask.float().mean())
            eng = row["on"][2]
            map_mb = eng.am_ws_bytes / 1e6
            print("%-26s B=%d grid %dx%d  map %.1f MB  anchors %d  kept %.1f %%  anchor_mask stage %.3f ms  "
                  "step %.3f -> %.3f ms" % (name, B, eng.am_nx, eng.am_ny, map_mb, eng.A, 100 * kept, row["on"][1],
                                            row["off"][0], row["on"][0]))
    print(json.dumps({"sm_clock": clk}))


if __name__ == "__main__":
    main()
