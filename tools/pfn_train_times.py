"""forward + backward time and peak memory of PointPillars' pillar feature net in training (CUDA events):
python tools/pfn_train_times.py [iters]

Two cases: pointpillars.car.xyres_16 at B = 2 (T = 100, at most 12 000 pillars per frame, 29 k-point bench clouds) and
nuscenes.all.pp.mhead at B = 3 (T = 60, at most 25 000 per frame, NuScenes-sized clouds), voxelized by the drop-in
VoxelGeneratorV2 on the GPU.  Each case times the VFE's forward + backward (loss = sum(out * G)) with
enable_pfn_training (b2s_pfn_train_forward / _backward) against the torch modules (TF32 off), after a warm-up, and
reports torch.cuda.max_memory_allocated of each path over the pass.  Prints the card name and power limit of the run."""
import sys

import _measure
import numpy as np
import torch

from b2second import training

CASES = [("pointpillars.car.xyres_16", 2, 29000), ("nuscenes.all.pp.mhead", 3, 300000)]


def batch(net, clouds):
    def t(a):
        return a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    vox, num, coors = [], [], []
    for b, c in enumerate(clouds):
        res = net.voxel_generator.generate(c, net.cfg.max_voxels)
        n = int(res["voxel_num"])
        vox.append(t(res["voxels"])[:n].cuda())
        num.append(t(res["num_points_per_voxel"])[:n].cuda())
        coors.append(torch.nn.functional.pad(t(res["coordinates"])[:n].cuda().int(), (1, 0), value=b))
    return torch.cat(vox).float().contiguous(), torch.cat(num).int(), torch.cat(coors).int().contiguous()


def measure(vfe, vox, num, coors, G, iters):
    def step():
        out = vfe(vox, num, coors)
        (out * G).sum().backward()
    return _measure.timed(step, iters), _measure.peak_bytes(step)


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    _measure.require_gpu("pfn_train_times")
    rows = []
    with _measure.clocks() as clk:
        for name, B, points in CASES:
            res = {}
            for ours in (False, True):
                net, clouds = _measure.mirror(name, B, points=points)
                net.train()
                if ours:
                    training.enable_pfn_training(net)
                vox, num, coors = batch(net, clouds)
                G = torch.randn(vox.shape[0], 64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
                res["ours" if ours else "torch"] = measure(net.voxel_feature_extractor, vox, num, coors, G, ITERS)
            N, T, F = vox.shape
            rows.append({"config": name, "batch": B, "pillars": N, "T": T, "real_points": int(num.sum()),
                         "ms_ours": round(res["ours"][0], 3), "ms_torch": round(res["torch"][0], 3),
                         "peak_MB_ours": round(res["ours"][1] / 2 ** 20, 1),
                         "peak_MB_torch": round(res["torch"][1] / 2 ** 20, 1)})
    _measure.report("pfn_train_times", rows, clk, iters=ITERS)

if __name__ == "__main__":
    main()
