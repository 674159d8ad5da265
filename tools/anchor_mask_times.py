"""ms per step the anchor-area mask adds to the fused engine (eager, a CUDA event before every stage, like
InferenceEngine.run_timed): python tools/anchor_mask_times.py [batch] [iters]

For each config: the "anchor_mask" stage of an engine built with anchor_area_threshold=1 (one memset + scatter, the two
scans of the summed-area table, the per-anchor lookup), the count map's size, and the whole step with and without the
mask.  pointpillars.car.xyres_16 has the threshold in its own eval config; car.fhd has it forced on (its config holds -1).
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
import torch  # noqa: E402

import bench  # noqa: E402
from b2second import config, loader, models  # noqa: E402
from b2second.engine import InferenceEngine  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
ITERS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
assert torch.cuda.is_available(), "this tool times CUDA kernels: it needs a GPU"
sp = loader.product_spconv()
print("device: %s" % torch.cuda.get_device_name(0))
for name in ("pointpillars.car.xyres_16", "car.fhd"):
    cfg = config.get_config(name)
    net = models.build_network(cfg, sp).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    pts = 20000
    uniq = bench.make_clouds(name, min(B, 4), pts)
    frames = [torch.from_numpy(uniq[i % len(uniq)]).cuda() for i in range(B)]
    row = {}
    for label, thr in (("off", None), ("on", 1.0)):
        eng = InferenceEngine(net, batch_size=B, max_points=pts + 1000, use_cuda_graph=False, anchor_area_threshold=thr)
        eng.load_points(frames)
        t = eng.run_timed(iters=ITERS)
        row[label] = (sum(t.values()), t.get("anchor_mask"), eng)
        if thr is not None:
            kept = float(eng.anchors_mask.float().mean())
    eng = row["on"][2]
    map_mb = eng.am_ws_bytes / 1e6
    print("%-26s B=%d grid %dx%d  map %.1f MB  anchors %d  kept %.1f %%  anchor_mask stage %.3f ms  step %.3f -> %.3f ms"
          % (name, B, eng.am_nx, eng.am_ny, map_mb, eng.A, 100 * kept, row["on"][1], row["off"][0], row["on"][0]))
