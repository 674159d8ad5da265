"""the f16 training mode (precision="f16") against the default fp32-grade mode, per layer and per stage:
python tools/f16_train_times.py [rounds]

On the seeded mirror networks and bench clouds of 29 k points (CUDA events, _measure.timed):
  sparse   car.fhd at batch 8: every sparse conv of the middle encoder, forward, input gradient (dgrad) and weight
           gradient (wgrad) in each mode (SparseConvolution._forward_rows / _dgrad / _wgrad on the rulebooks of one
           forward; the splits of X and dY are included, as in a training step)
  rpn      car.fhd at batch 8 and pointpillars.car.xyres_16 at batch 2: every distinct covered 3x3 layer shape, forward,
           dgrad and wgrad in each mode (rpn_train's launchers; the splits included in forward and dgrad)
  totals   the whole middle encoder (car.fhd, batch 8) and the whole RPN (both configs) forward + backward in train()
The two modes alternate within every round; run `rounds` rounds (default 2) to show the spread.  One JSON line per
config and round, with the card, its power limit and the SM clock sampled during the round.
"""
import copy
import sys

import numpy as np
import torch
import torch.nn as nn

import _measure
from b2second import rpn_train, training

PRECISIONS = (("fp32", 3), ("f16", 1))
ITERS = 10


def us(fn, iters=ITERS):
    return round(_measure.timed(fn, iters, warmup=2) * 1e3, 1)


def middle_encoder(B):
    """car.fhd's drop-in middle encoder (train()) and its input: (spconv, module, voxel features, coordinates)"""
    from b2second import loader
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


def sparse_rows(B):
    sp, mid, vf, coors = middle_encoder(B)
    records = []
    x = sp.SparseConvTensor(vf, coors, mid.sparse_shape, B)
    with torch.no_grad():
        for i, m in enumerate(mid.middle_conv):
            if isinstance(m, sp.SparseConvolution):
                inp = x
                x = m(x)
                records.append((i, m, inp.features.detach().contiguous().float(), inp.indice_dict[m.indice_key]))
            elif x.indices.shape[0]:
                x.features = m(x.features)
    rows = []
    for i, m, f, rb in records:
        dy = torch.randn(rb.num_out, m.out_channels, device="cuda") * 2.0 ** -20
        row = {"layer": i, "cin": m.in_channels, "cout": m.out_channels, "K": rb.K, "rows": rb.num_out,
               "pairs": int((rb.nbr >= 0).sum())}
        for prec, p in PRECISIONS:
            with torch.no_grad():
                row[prec] = [us(lambda: m._forward_rows(f, rb, p)),
                             us(lambda: m._dgrad(dy, m.weight, rb, f.shape[0], None, p)) if i > 0 else None,
                             us(lambda: m._wgrad(f, dy, rb, None, None, p))]
        rows.append(row)
    g = torch.randn(mid(vf, coors, B).shape, device="cuda")

    def step():
        (mid(vf, coors, B) * g).sum().backward()
    total = {}
    for prec, _ in PRECISIONS:
        training.enable_sparse_backward(mid, precision=prec)
        total[prec] = round(_measure.timed(step, 5, warmup=2), 3)
    training.enable_sparse_backward(mid)
    return {"layers": rows, "middle_encoder_ms": total}


def rpn_layer(B, cin, cout, H, W):
    conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False).cuda()
    x = torch.relu(torch.randn(B, cin, H, W, device="cuda"))
    dy = torch.randn(B, cout, H, W, device="cuda") * 2.0 ** -20
    row = {"cin": cin, "cout": cout, "H": H, "W": W}
    for prec, p in PRECISIONS:
        w = rpn_train.pack_weights(conv, False, p)
        wt = rpn_train.pack_weights(conv, True, p)
        xs = rpn_train.split_halo(x, products=p)
        gs = rpn_train.split_halo(dy, products=p)
        row[prec] = [us(lambda: rpn_train.conv3x3(*rpn_train.split_halo(x, products=p), *w, B, H, W, cin, cout, p)),
                     us(lambda: rpn_train.conv3x3(*rpn_train.split_halo(dy, products=p), *wt, B, H, W, cout, cin, p)),
                     us(lambda: rpn_train.wgrad(*xs, *gs, B, H, W, cin, cout, p))]
    return row


def rpn_rows(name, B):
    net = _measure.mirror(name)
    rpn = net.rpn
    first = rpn.blocks[0][1]
    H, W = (int(v) * first.stride[0] for v in net.cfg.feature_map_size[1:])
    covered = {id(c) for c, _ in rpn_train.select(rpn)}
    shapes, h, w = [], H, W
    for blk in rpn.blocks:
        st = blk[1].stride[0]
        h, w = (h + 2 - 3) // st + 1, (w + 2 - 3) // st + 1
        shapes += [(m.in_channels, m.out_channels, h, w) for m in blk if id(m) in covered]
    layers = [dict(rpn_layer(B, *s), count=shapes.count(s)) for s in dict.fromkeys(shapes)]
    x = (torch.relu(torch.randn(B, first.in_channels, H, W, device="cuda")) *
         (torch.rand(B, 1, H, W, device="cuda") < 0.15)).requires_grad_(True)
    model = rpn_train.enable(copy.deepcopy(rpn)).cuda().train()
    with torch.no_grad():
        G = {k: torch.randn_like(v) for k, v in model(x).items()}

    def step():
        o = model(x)
        sum((o[k] * G[k]).sum() for k in G).backward()
    total = {}
    for prec, p in PRECISIONS:
        rpn_train.enable(model, p)
        total[prec] = round(_measure.timed(step, 5, warmup=2), 3)
    return {"layers": layers, "covered_layers": len(shapes), "rpn_ms": total}


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    _measure.require_gpu("f16_train_times")
    for r in range(rounds):
        for name, B, what in (("car.fhd", 8, "sparse"), ("car.fhd", 8, "rpn"), ("pointpillars.car.xyres_16", 2, "rpn")):
            with _measure.clocks() as clk:
                res = sparse_rows(B) if what == "sparse" else rpn_rows(name, B)
            _measure.report("f16_train_times", res, clk, config=name, batch=B, stage=what, round=r,
                            columns="us per call: [forward, dgrad, wgrad]; totals in ms")
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
