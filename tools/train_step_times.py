"""per-layer training times of car.fhd's sparse middle encoder (CUDA events): python tools/train_step_times.py [batch]

For every sparse conv of SpMiddleFHD on a batch of synthetic 29 k-point clouds (default batch 8): the forward, the input
gradient (dgrad) and the weight gradient (wgrad) of the b2second kernels, and the algorithmic wgrad rate
2 * pairs * Cin * Cout / t.  Then the whole middle encoder forward + backward (loss = sum(dense_out * G)) with
enable_sparse_backward, against the same layers restated in plain torch on the GPU (gather - mm - index_add_ over the
same rulebooks: what a training step costs without these kernels).  Prints the card first and the SM clock sampled
during the run last."""
import json
import sys

import _measure
import numpy as np
import torch

from b2second import loader, training

ITERS = 10


def middle_encoder(B):
    """car.fhd's drop-in middle encoder in train() with enable_sparse_backward, and its input from B bench clouds:
    (spconv, middle encoder, mean voxel features [N, 4], coordinates [N, 4] with the frame index first)"""
    net, clouds = _measure.mirror("car.fhd", B)
    net = net.train()
    mid = training.enable_sparse_backward(net.middle_feature_extractor)
    feats, coors = [], []
    for b, c in enumerate(clouds):
        res = net.voxel_generator.generate(c, net.cfg.max_voxels)
        n = res["voxel_num"]
        vf = torch.from_numpy(res["voxels"][:n]).sum(1) / torch.from_numpy(
            res["num_points_per_voxel"][:n]).clamp_min(1)[:, None]
        feats.append(vf[:, :4].float())
        coors.append(torch.from_numpy(np.pad(res["coordinates"][:n], ((0, 0), (1, 0)), constant_values=b)))
    return loader.product_spconv(), mid, torch.cat(feats).cuda(), torch.cat(coors).int().cuda()


def timed(fn, iters=ITERS):
    return _measure.timed(fn, iters, warmup=1) * 1e3     # us


def torch_conv(m, f, rb):
    w = m.weight.view(rb.K, m.in_channels, m.out_channels)
    out = torch.zeros(rb.num_out, m.out_channels, device=f.device, dtype=f.dtype)
    nbr = rb.nbr.long()
    for k in range(rb.K):
        o = torch.nonzero(nbr[:, k] >= 0).squeeze(1)
        out = out.index_add(0, o, f.index_select(0, nbr[o, k]) @ w[k])
    return out


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    _measure.require_gpu("train_step_times")
    print(json.dumps(_measure.card()))
    sp, mid, vf, coors = middle_encoder(B)
    seq = mid.middle_conv
    with _measure.clocks() as clk:
        # ---- per layer: record each sparse conv's input tensor and rulebook on one forward ----
        records = []
        x = sp.SparseConvTensor(vf, coors, mid.sparse_shape, B)
        for i in range(len(seq)):
            m = seq[i]
            if isinstance(m, sp.SparseConvolution):
                inp = x
                x = m(x)
                rb = inp.indice_dict[m.indice_key]
                records.append((i, m, inp, rb))
            elif x.indices.shape[0]:
                x.features = m(x.features)
        print("car.fhd middle encoder, batch %d, %d voxels, tensor pipe %s" % (B, vf.shape[0], sp.USE_TENSOR_CORES))
        print("%-6s %4s %4s %3s %8s %9s %10s %10s %10s %12s" % ("layer", "cin", "cout", "K", "rows", "pairs", "fwd us",
                                                                  "dgrad us", "wgrad us", "wgrad TFLOP/s"))
        tot = [0.0, 0.0, 0.0]
        for i, m, inp, rb in records:
            f = inp.features.detach().contiguous().float()
            dy = torch.randn(rb.num_out, m.out_channels, device="cuda")
            pairs = int((rb.nbr >= 0).sum())
            with torch.no_grad():
                t_f = timed(lambda: m._forward_rows(f, rb))
            # layer 0: the VFE output needs no input gradient
            t_d = timed(lambda: m._dgrad(dy, m.weight, rb, f.shape[0])) if i > 0 else float("nan")
            t_w = timed(lambda: m._wgrad(f, dy, rb))
            tot[0] += t_f
            tot[1] += 0.0 if i == 0 else t_d
            tot[2] += t_w
            print("%-6d %4d %4d %3d %8d %9d %10.1f %10.1f %10.1f %12.2f" % (
                i, m.in_channels, m.out_channels, rb.K, rb.num_out, pairs, t_f, t_d, t_w,
                2.0 * pairs * m.in_channels * m.out_channels / t_w / 1e6))
        print("sum    %62.1f %10.1f %10.1f" % tuple(tot))

        # ---- whole middle encoder: b2second kernels vs a plain torch restatement on the same rulebooks ----
        g = torch.randn(x.dense().shape, device="cuda")

        def step(use_torch):
            x = sp.SparseConvTensor(vf, coors, mid.sparse_shape, B)
            j = 0
            for i in range(len(seq)):
                m = seq[i]
                if isinstance(m, sp.SparseConvolution):
                    if use_torch:
                        _, _, inp, rb = records[j]
                        y = sp.SparseConvTensor(None, rb.out_indices, rb.out_shape, B)
                        y._features = torch_conv(m, x.features, rb)
                        y.indice_dict = x.indice_dict
                        x = y
                    else:
                        x = m(x)
                    j += 1
                elif x.indices.shape[0]:
                    x.features = m(x.features)
            out = x.dense()
            (out * g).sum().backward()
        t_ours = timed(lambda: step(False), 5)
        t_torch = timed(lambda: step(True), 5)
    print("middle encoder forward + backward: b2second %.2f ms (rulebooks and tile plans rebuilt every step, one host "
          "sync per strided layer), torch gather-mm-index_add %.2f ms (rulebooks reused, not timed) (x%.1f)" % (
              t_ours / 1e3, t_torch / 1e3, t_torch / t_ours))
    print(json.dumps({"sm_clock": clk}))


if __name__ == "__main__":
    main()
