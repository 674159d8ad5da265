"""training times of the RPN's 3x3 stride-1 convolutions (CUDA events): python tools/rpn_train_times.py

For car.fhd at batch 8 and pointpillars.car.xyres_16 at batch 2 (their training batch sizes), per distinct covered
layer shape: forward, input gradient (dgrad) and weight gradient (wgrad) of b2second.rpn_train (the splits of X and dY
included in forward and dgrad), of cuDNN fp32 (allow_tf32 False) and, for information, of cuDNN TF32, with the
algorithmic rate 2 * B * H * W * 9 * Cin * Cout / t and each kernel's bound: f16 MMA work (3 products) at the data-sheet
989 TFLOP/s, or its L2 -> SM operand bytes.  Then the whole RPN forward + backward in train() mode, and the error of
each path's forward against float64 (max |y - y64| / max |y64|).  Prints the card, its power limit and the SM clock
sampled during the run."""
import copy
import json

import _measure
import torch
import torch.nn as nn
import torch.nn.functional as F

from b2second import rpn_train

ITERS = 20
DEV = "cuda:0"
MMA_PEAK = 989e12          # dense f16 wgmma, H100 SXM data sheet


def timed(fn, iters=ITERS):
    return _measure.timed(fn, iters) * 1e3     # us


def tf32(on):
    torch.backends.cudnn.allow_tf32 = on
    torch.backends.cuda.matmul.allow_tf32 = on


def layer_row(B, cin, cout, H, W):
    conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False).to(DEV)
    rpn_train.enable(nn.Sequential(conv))
    conv.train()
    x = torch.randn(B, cin, H, W, device=DEV)
    dy = torch.randn(B, cout, H, W, device=DEV) * 1e-6
    w = conv.weight.detach()
    flop = 2.0 * B * H * W * 9 * cin * cout
    x_hi, x_lo, xs = rpn_train.split_halo(x)
    w_hi, w_lo, w_inv = rpn_train.pack_weights(conv, False)
    wt_hi, wt_lo, wt_inv = rpn_train.pack_weights(conv, True)
    g_hi, g_lo, gs = rpn_train.split_halo(dy)
    ours = (timed(lambda: rpn_train.conv3x3(*rpn_train.split_halo(x), w_hi, w_lo, w_inv, B, H, W, cin, cout)),
            timed(lambda: rpn_train.conv3x3(*rpn_train.split_halo(dy), wt_hi, wt_lo, wt_inv, B, H, W, cout, cin)),
            timed(lambda: rpn_train.wgrad(x_hi, x_lo, xs, g_hi, g_lo, gs, B, H, W, cin, cout)))
    rows = []
    for on in (False, True):
        tf32(on)
        rows.append((timed(lambda: F.conv2d(x, w, padding=1)),
                     timed(lambda: torch.nn.grad.conv2d_input(x.shape, w, dy, padding=1)),
                     timed(lambda: torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=1))))
    tf32(False)
    y64 = F.conv2d(x.double(), w.double(), padding=1)
    tf32(True)
    e_tf32 = float((F.conv2d(x, w, padding=1).double() - y64).abs().max() / y64.abs().max())
    tf32(False)
    e_fp32 = float((F.conv2d(x, w, padding=1).double() - y64).abs().max() / y64.abs().max())
    y = rpn_train.conv3x3(x_hi, x_lo, xs, w_hi, w_lo, w_inv, B, H, W, cin, cout).permute(0, 3, 1, 2)
    e_ours = float((y.double() - y64).abs().max() / y64.abs().max())
    # bounds: forward / dgrad k_conv_tc (3 f16 products per term); wgrad: MMA, or L2 -> SM bytes of its jobs
    # (X hi/lo window 2 x 128 B x 10/8 per pixel and 64 input channels, dY hi/lo 4 B per channel up to 128)
    px = B * H * W
    jobs = 3 * (cin // 64) * ((cout + 127) // 128)
    l2_bytes = px * jobs * (2 * 128 * 10 / 8 + 4 * min(cout, 128))
    return flop, ours, rows[0], rows[1], (e_ours, e_fp32, e_tf32), 3 * flop / MMA_PEAK * 1e6, l2_bytes


def rpn_step(name, B):
    net = _measure.mirror(name)
    rpn = net.rpn
    first = rpn.blocks[0][1]
    H, W = (int(v) * first.stride[0] for v in net.cfg.feature_map_size[1:])
    x = (torch.relu(torch.randn(B, first.in_channels, H, W, device=DEV)) *
         (torch.rand(B, 1, H, W, device=DEV) < 0.15)).requires_grad_(True)
    torch_rpn = copy.deepcopy(rpn).to(DEV).train()
    ours = rpn_train.enable(copy.deepcopy(rpn)).to(DEV).train()
    out = torch_rpn(x)
    G = {k: torch.randn_like(v) for k, v in out.items()}

    def step(m):
        o = m(x)
        sum((o[k] * G[k]).sum() for k in G).backward()
    tf32(False)
    t_ours, t_fp32 = timed(lambda: step(ours), 5), timed(lambda: step(torch_rpn), 5)
    tf32(True)
    t_tf32 = timed(lambda: step(torch_rpn), 5)
    tf32(False)
    layers = [(c.in_channels, c.out_channels) for c, _ in rpn_train.select(rpn)]
    return rpn, H, W, layers, t_ours, t_fp32, t_tf32


def config_rows(name, B):
    """the whole-RPN line and the per-layer table of one config"""
    rpn, H, W, layers, t_ours, t_fp32, t_tf32 = rpn_step(name, B)
    print("\n%s, batch %d, RPN input %d x %d, %d covered layers" % (name, B, H, W, len(layers)))
    print("whole RPN forward + backward (train mode): b2second %.2f ms, cuDNN fp32 %.2f ms (x%.2f), cuDNN TF32 "
          "%.2f ms" % (t_ours / 1e3, t_fp32 / 1e3, t_fp32 / t_ours, t_tf32 / 1e3))
    shapes = []
    h, w = H, W
    for blk in rpn.blocks:
        st = blk[1].stride[0]
        h, w = (h + 2 - 3) // st + 1, (w + 2 - 3) // st + 1
        for m in blk:
            if type(m) is nn.Conv2d and m.stride == (1, 1) and rpn_train.qualifies(m, m.padding[0]):
                key = (m.in_channels, m.out_channels, h, w)
                if key not in shapes:
                    shapes.append(key)
    print("%9s %9s | %8s %8s %8s | %8s %8s %8s | %8s %8s %8s | %6s %6s %6s | %7s %7s | %8s %8s %8s" % (
        "cin>cout", "H x W", "fwd us", "dgrad", "wgrad", "fp32 fwd", "dgrad", "wgrad", "tf32 fwd", "dgrad",
        "wgrad", "TF/s f", "d", "w", "MMA us", "L2 GB", "err ours", "fp32", "tf32"))
    for cin, cout, h, w in shapes:
        flop, o, f, t, e, mma_us, l2 = layer_row(B, cin, cout, h, w)
        print("%4d>%-4d %4dx%-4d | %8.1f %8.1f %8.1f | %8.1f %8.1f %8.1f | %8.1f %8.1f %8.1f | %6.1f %6.1f %6.1f |"
              " %7.1f %7.2f | %8.1e %8.1e %8.1e" % (cin, cout, h, w, *o, *f, *t, *(flop / x / 1e6 for x in o),
                                                   mma_us, l2 / 1e9, *e))


def main():
    _measure.require_gpu("rpn_train_times")
    print(json.dumps(_measure.card()))
    with _measure.clocks() as clk:
        for name, B in (("car.fhd", 8), ("pointpillars.car.xyres_16", 2)):
            config_rows(name, B)
    print(json.dumps({"sm_clock": clk}))


if __name__ == "__main__":
    main()
