"""forward + backward time and peak memory of PointPillars' pillar feature net in training (CUDA events):
python tools/pfn_train_times.py [iters]

Two cases: pointpillars.car.xyres_16 at B = 2 (T = 100, at most 12 000 pillars per frame, 29 k-point bench clouds) and
nuscenes.all.pp.mhead at B = 3 (T = 60, at most 25 000 per frame, NuScenes-sized clouds), voxelized by the drop-in
VoxelGeneratorV2 on the GPU.  Each case times the VFE's forward + backward (loss = sum(out * G)) with
enable_pfn_training (b2s_pfn_train_forward / _backward) against the torch modules (TF32 off), after a warm-up, and
reports torch.cuda.max_memory_allocated of each path over the pass.  Prints the card name and power limit of the run."""
import json
import os
import subprocess
import sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
import numpy as np
import torch
import bench
from b2second import config, loader, models, training

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
CASES = [("pointpillars.car.xyres_16", 2, 29000), ("nuscenes.all.pp.mhead", 3, 300000)]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def batch(net, cfg, name, B, points):
    def t(a):
        return a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    vox, num, coors = [], [], []
    for b, c in enumerate(bench.make_clouds(name, B, points)):
        res = net.voxel_generator.generate(c, cfg.max_voxels)
        n = int(res["voxel_num"])
        vox.append(t(res["voxels"])[:n].cuda())
        num.append(t(res["num_points_per_voxel"])[:n].cuda())
        coors.append(torch.nn.functional.pad(t(res["coordinates"])[:n].cuda().int(), (1, 0), value=b))
    return torch.cat(vox).float().contiguous(), torch.cat(num).int(), torch.cat(coors).int().contiguous()


def measure(vfe, vox, num, coors, G):
    def step():
        out = vfe(vox, num, coors)
        (out * G).sum().backward()
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / ITERS, peak


def main():
    assert torch.cuda.is_available(), "pfn_train_times.py measures on a CUDA device"
    sp = loader.product_spconv()
    rows = []
    for name, B, points in CASES:
        cfg = config.get_config(name)
        res = {}
        for ours in (False, True):
            net = models.build_network(cfg, sp)
            models.synthetic_weights_(net, name, seed=0)
            net = net.cuda().train()
            if ours:
                training.enable_pfn_training(net)
            vox, num, coors = batch(net, cfg, name, B, points)
            G = torch.randn(vox.shape[0], 64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
            res["ours" if ours else "torch"] = measure(net.voxel_feature_extractor, vox, num, coors, G)
        N, T, F = vox.shape
        row = {"config": name, "batch": B, "pillars": N, "T": T, "real_points": int(num.sum()),
               "ms_ours": round(res["ours"][0], 3), "ms_torch": round(res["torch"][0], 3),
               "peak_MB_ours": round(res["ours"][1] / 2 ** 20, 1), "peak_MB_torch": round(res["torch"][1] / 2 ** 20, 1)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": card(), "iters": ITERS}))


if __name__ == "__main__":
    main()
