"""micro-benchmark of b2s_conv2d_tc alone (RPN 3x3 128->128 at car.fhd size), CUDA-event timed.
B2S_CONV_DBG (diagnostic, wrong results; `make DIAG=1` builds only): 1 = no lo loads, 4 = no accumulator
drain.  B2S_CONV_B = frames."""
import os
import sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
import torch
from b2second import loader, tc
sp = loader.product_spconv()
L = sp._lib
lib = L.load()
B, H, W, C = 8, 200, 176, 128
B = int(os.environ.get("B2S_CONV_B", B))
x = torch.randn(B, H + 2, W + 2, C, device="cuda")
hi, lo = tc.split_f16(x)
w = torch.randn(9, C, C, device="cuda") * 0.03
ws = tc.pow2_scale(w)
w_hi, w_lo = tc.split_f16(w, ws)
scale = torch.full((C,), 1.0 / ws, device="cuda"); shift = torch.zeros(C, device="cuda")
o_hi = torch.zeros_like(hi); o_lo = torch.zeros_like(hi)
status = torch.zeros(1, dtype=torch.int32, device="cuda")
flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
def run():
    L.check(lib.b2s_conv2d_tc(L.ptr(hi), L.ptr(lo), B, H, W, C, L.ptr(w_hi), L.ptr(w_lo), 9, C, 128, L.ptr(scale),
                              L.ptr(shift), 1, L.ptr(o_hi), L.ptr(o_lo), 1, C, L.ptr(status), L.stream()), "conv")
for _ in range(3): run()
torch.cuda.synchronize()
ts = []
for i in range(10):
    flush.fill_(i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); run(); b.record(); torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
ms = sorted(ts)[len(ts) // 2]
flops = 2.0 * B * H * W * C * C * 9
print("B2S_CONV_DBG=%s B2S_CONV_HALO=%s  median %.3f ms  algorithmic %.1f TFLOP/s (x3 f16 MMAs issued: %.1f)" % (
    os.environ.get("B2S_CONV_DBG", "0"), os.environ.get("B2S_CONV_HALO", "0"), ms, flops / ms / 1e9, 3 * flops / ms / 1e9))
# accuracy of the merged hi+lo output against an fp64 cuDNN-free reference (frames 0..1)
if os.environ.get("B2S_CONV_ACC", "1") == "1":
    nb = 2
    xin = (hi[:nb].double() + lo[:nb].double()).permute(0, 3, 1, 2)            # [nb, C, H+2, W+2] (halo = padding)
    wt = ((w_hi.double() + w_lo.double()) / ws).reshape(3, 3, C, C).permute(2, 3, 0, 1)  # [Cout, Cin, 3, 3]
    ref = torch.nn.functional.conv2d(xin, wt).clamp_(min=0).permute(0, 2, 3, 1)  # [nb, H, W, C]
    got = (o_hi[:nb, 1:-1, 1:-1].double() + o_lo[:nb, 1:-1, 1:-1].double())
    err = (got - ref).abs()
    print("B2S_CONV_CHAIN=%s  max|err| %.3e  max|ref| %.3e  max-rel %.3e  rms-rel %.3e  mean signed %.3e" % (
        os.environ.get("B2S_CONV_CHAIN", "1"), err.max().item(), ref.abs().max().item(),
        (err.max() / ref.abs().max()).item(), (err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item(),
        ((got - ref).mean() / ref.abs().mean()).item()))
# SM clock / power while the kernel runs back to back (is the tensor pipe power-capped?)
if os.environ.get("B2S_CONV_CLOCKS", "0") == "1":
    import subprocess, threading
    rows = []
    pr = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,power.draw,clocks_event_reasons.sw_power_cap",
                           "--format=csv,noheader,nounits", "-lms", "50"], stdout=subprocess.PIPE, text=True)
    th = threading.Thread(target=lambda: [rows.append(l.strip()) for l in pr.stdout], daemon=True); th.start()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(4000): run()
    b.record(); torch.cuda.synchronize()
    pr.terminate()
    print("back-to-back: %.3f ms/launch; nvidia-smi samples (MHz, W, power-cap): %s" % (a.elapsed_time(b) / 4000, rows[3:-1][::4]))
