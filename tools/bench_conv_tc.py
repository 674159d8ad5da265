"""micro-benchmark of b2s_conv2d_tc alone (RPN 3x3 128->128 at car.fhd size), CUDA-event timed.
B2S_CONV_B = frames, B2S_CONV_ACC=0 skips the accuracy check, B2S_CONV_CLOCKS=1 samples the SM clock and its slowdown
reasons (the software power cap among them) over 4000 launches back to back."""
import json
import os

import _measure
import torch

from b2second import loader, tc


def main():
    _measure.require_gpu("bench_conv_tc")
    print(json.dumps(_measure.card()))
    L = loader.product_spconv()._lib
    lib = L.load()
    B, H, W, C = 8, 200, 176, 128
    B = int(os.environ.get("B2S_CONV_B", B))
    x = torch.randn(B, H + 2, W + 2, C, device="cuda")
    hi, lo = tc.split_f16(x)
    w = torch.randn(9, C, C, device="cuda") * 0.03
    ws = tc.pow2_scale(w)
    w_hi, w_lo = tc.split_f16(w, ws)
    scale = torch.full((C,), 1.0 / ws, device="cuda")
    shift = torch.zeros(C, device="cuda")
    o_hi = torch.zeros_like(hi)
    o_lo = torch.zeros_like(hi)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")

    def run():
        L.check(lib.b2s_conv2d_tc(L.ptr(hi), L.ptr(lo), B, H, W, C, L.ptr(w_hi), L.ptr(w_lo), 9, C, 128, L.ptr(scale),
                                  L.ptr(shift), 1, L.ptr(o_hi), L.ptr(o_lo), 1, C, L.ptr(status), L.stream()), "conv")
    with _measure.clocks() as clk:
        ms = _measure.timed(run, 10, flush=flush)
    flops = 2.0 * B * H * W * C * C * 9
    print("median %.3f ms  algorithmic %.1f TFLOP/s (x3 f16 MMAs issued: %.1f)" % (
        ms, flops / ms / 1e9, 3 * flops / ms / 1e9))
    print(json.dumps({"sm_clock": clk}))
    # accuracy of the merged hi+lo output against an fp64 cuDNN-free reference (frames 0..1)
    if os.environ.get("B2S_CONV_ACC", "1") == "1":
        nb = 2
        xin = (hi[:nb].double() + lo[:nb].double()).permute(0, 3, 1, 2)            # [nb, C, H+2, W+2] (halo = padding)
        wt = ((w_hi.double() + w_lo.double()) / ws).reshape(3, 3, C, C).permute(2, 3, 0, 1)  # [Cout, Cin, 3, 3]
        ref = torch.nn.functional.conv2d(xin, wt).clamp_(min=0).permute(0, 2, 3, 1)  # [nb, H, W, C]
        got = (o_hi[:nb, 1:-1, 1:-1].double() + o_lo[:nb, 1:-1, 1:-1].double())
        err = (got - ref).abs()
        print("max|err| %.3e  max|ref| %.3e  max-rel %.3e  rms-rel %.3e  mean signed %.3e" % (
            err.max().item(), ref.abs().max().item(),
            (err.max() / ref.abs().max()).item(), (err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item(),
            ((got - ref).mean() / ref.abs().mean()).item()))
    # is the tensor pipe power-capped?
    if os.environ.get("B2S_CONV_CLOCKS", "0") == "1":
        with _measure.clocks() as clk:
            ms = _measure.timed(run, 4000, warmup=0)
        print("back-to-back: %.3f ms/launch; SM clock %s" % (ms, json.dumps(clk)))


if __name__ == "__main__":
    main()
