"""forward + backward time and peak memory of the train-mode BatchNorm + ReLU pairs (CUDA events):
python tools/bn_train_times.py [iters]

Three cases: car.fhd's RPN at B = 8, pointpillars.car.xyres_16's RPN at B = 2 and car.fhd's middle encoder at B = 8, all
from bench clouds voxelized by the drop-in VoxelGeneratorV2 with synthetic weights, in train() with
enable_sparse_backward and enable_rpn_training, so every pair sees the layout it has in training.  One forward records
each pair's input; then, per pair, relu(bn(x)) forward + backward (loss = sum(y * G)) with enable_bn_relu_training
(b2s_bn_relu_train_forward / _backward) is timed against the torch modules after a warm-up, with the peak of
torch.cuda.max_memory_allocated over one pass, and the least time the pair's map traffic can take at 3.35 TB/s (3 map
passes forward, 5 backward).  For the two RPNs the whole rpn forward + backward is timed the same way with and without
the opt-in.  Prints the card name and power limit of the run."""
import copy
import sys

import _measure
import numpy as np
import torch

from b2second import bn_train, training

CASES = [("car.fhd", 8, "rpn"), ("pointpillars.car.xyres_16", 2, "rpn"), ("car.fhd", 8, "middle")]
HBM = 3.35e12                       # H100 SXM data-sheet HBM3 bandwidth, bytes/s


def network(name, B):
    """the drop-in network in train() with sparse backward and RPN training, and the inputs of its three stages"""
    net, clouds = _measure.mirror(name, B)
    net = training.enable_rpn_training(training.enable_sparse_backward(net)).train()

    def t(a):
        return a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    vox, num, coors = [], [], []
    for b, c in enumerate(clouds):
        res = net.voxel_generator.generate(c, net.cfg.max_voxels)
        n = int(res["voxel_num"])
        vox.append(t(res["voxels"])[:n].cuda())
        num.append(t(res["num_points_per_voxel"])[:n].cuda())
        coors.append(torch.nn.functional.pad(t(res["coordinates"])[:n].cuda().int(), (1, 0), value=b))
    return net, torch.cat(vox).float().contiguous(), torch.cat(num).int(), torch.cat(coors).int().contiguous()


def pair_times(bn, relu, x, iters):
    """(ms, peak bytes) of relu(bn(x)) forward + backward, fused and torch, on copies of the modules"""
    G = torch.randn(x.shape, device=x.device, generator=torch.Generator(x.device).manual_seed(0))
    G = G.contiguous(memory_format=torch.channels_last) if x.dim() == 4 and not x.is_contiguous() else G
    out = {}
    for fused in (True, False):
        seq = torch.nn.Sequential(copy.deepcopy(bn), copy.deepcopy(relu))
        for m in seq:
            m.__dict__.pop("forward", None)
        seq[0].__dict__.pop("_b2s_bn_train", None)
        if fused:
            training.enable_bn_relu_training(seq)
        xi = x.detach().clone().requires_grad_(True)

        def step():
            y = seq(xi)
            (y * G).sum().backward()
        out[fused] = _measure.timed(step, iters), _measure.peak_bytes(step)
    return out


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    _measure.require_gpu("bn_train_times")
    rows = []
    with _measure.clocks() as clk:
        for name, B, part in CASES:
            net, vox, num, coors = network(name, B)
            stage = net.rpn if part == "rpn" else net.middle_feature_extractor
            pairs = bn_train.select(stage)
            seen = {}
            hooks = [bn.register_forward_pre_hook(lambda m, i: seen.setdefault(id(m), i[0].detach().clone()))
                     for bn, _ in pairs]
            rpn_in = {}
            hooks.append(net.rpn.register_forward_pre_hook(lambda m, i: rpn_in.setdefault("x", i[0].detach().clone())))
            feats = net.voxel_feature_extractor(vox, num, coors)       # grad on: the layers take their training path
            net.rpn(net.middle_feature_extractor(feats, coors, B))
            for h in hooks:
                h.remove()
            tot = {"ours": 0.0, "torch": 0.0, "floor": 0.0}
            for i, (bn, relu) in enumerate(pairs):
                x = seen[id(bn)]
                t = pair_times(bn, relu, x, ITERS)
                floor = 8 * x.numel() * 4 / HBM * 1e3
                layout = "rows" if x.dim() == 2 or not x.is_contiguous() else "nchw"
                row = {"config": name, "batch": B, "stage": part, "pair": i, "shape": list(x.shape), "layout": layout,
                       "ms_ours": round(t[True][0], 4), "ms_torch": round(t[False][0], 4), "ms_floor": round(floor, 4),
                       "peak_MB_ours": round(t[True][1] / 2 ** 20, 1), "peak_MB_torch": round(t[False][1] / 2 ** 20, 1)}
                tot["ours"] += t[True][0]
                tot["torch"] += t[False][0]
                tot["floor"] += floor
                rows.append(row)
            summary = {"config": name, "batch": B, "stage": part, "pairs": len(pairs),
                       "ms_ours_sum": round(tot["ours"], 3), "ms_torch_sum": round(tot["torch"], 3),
                       "ms_floor_sum": round(tot["floor"], 3)}
            if part == "rpn":
                x = rpn_in["x"]
                for fused in (False, True):
                    if fused:
                        training.enable_bn_relu_training(net)
                    xi = x.clone().requires_grad_(True)

                    def step():
                        r = net.rpn(xi)
                        sum(v.float().sum() for v in r.values() if torch.is_tensor(v) and v.requires_grad).backward()
                    ms, peak = _measure.timed(step, ITERS), _measure.peak_bytes(step)
                    key = "ours" if fused else "torch"
                    summary["rpn_ms_" + key] = round(ms, 3)
                    summary["rpn_peak_MB_" + key] = round(peak / 2 ** 20, 1)
            rows.append(summary)
            del net
            torch.cuda.empty_cache()
    _measure.report("bn_train_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
