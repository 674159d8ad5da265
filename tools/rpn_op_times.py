"""per-launch times of the tensor-core RPN program (CUDA events, eager): python tools/rpn_op_times.py <config> [batch]"""
import json
import sys

import _measure
import torch

from b2second.engine import InferenceEngine, ctypes_ptr


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "pointpillars.car.xyres_16"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 32
    _measure.require_gpu("rpn_op_times")
    print(json.dumps(_measure.card()))
    pts = 300000 if "nuscenes" in name else 29000
    net, uniq = _measure.mirror(name, min(B, 4), points=pts)
    eng = InferenceEngine(net.eval(), batch_size=B, max_points=pts + 1000, use_cuda_graph=False)
    eng.infer([torch.from_numpy(uniq[i % len(uniq)]).cuda() for i in range(B)])
    torch.cuda.synchronize()
    L, lib = eng._L, eng.lib
    st = L.stream()
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
    tot = 0.0
    with _measure.clocks() as clk:
        for i, op in enumerate(eng.tc_plan):
            src, dst = eng.tc_bufs[op["src"]], eng.tc_bufs[op["dst"]]
            esz = dst[0].element_size()
            o_hi = ctypes_ptr(dst[0].data_ptr() + esz * op["dst_coff"])
            o_lo = ctypes_ptr(dst[1].data_ptr() + esz * op["dst_coff"]) if op["planes"] == 2 else None

            def run():
                L.check(lib.b2s_conv2d_tc_ex(
                    L.ptr(src[0]), L.ptr(src[1]), B, op["Hin"], op["Win"], op["cin"], L.ptr(op["w_hi"]),
                    L.ptr(op["w_lo"]), op["kh"], op["kw"], op["stride"], op["pad"], op["cout"], op["n_pad"],
                    L.ptr(op["scale"]), L.ptr(op["shift"]) if op["shift"] is not None else None,
                    1 if op["relu"] else 0, op["Hg"], op["Wg"], o_hi, o_lo, op["Hout"], op["Wout"],
                    1 if op["padded"] else 0, dst[0].shape[-1], op["out_mul"], op["off_h"], op["off_w"], None, None,
                    None, None, None, None, L.ptr(eng.status), st), "conv")
            ms = _measure.timed(run, 5, warmup=1, flush=flush)
            tot += ms
            px = B * op["Hg"] * op["Wg"]
            fl = 2.0 * px * op["taps"] * op["cin"] * op["cout"]
            byt = 4.0 * (B * op["Hin"] * op["Win"] * op["cin"] / (op["stride"] ** 2 if op["kh"] == 1 else 1)
                         + px * op["cout"] * (1 if op["planes"] == 2 else 1))
            print("%2d %-8s v2=%d k%dx%d s%d cin %3d cout %3d (n_pad %3d) grid %dx%d px %8d  %7.3f ms  %6.1f TFLOP/s  "
                  "~%5.0f GB/s" % (i, op["kind"], op["v2"], op["kh"], op["kw"], op["stride"], op["cin"], op["cout"],
                                   op["n_pad"], op["Hg"], op["Wg"], px, ms, fl / ms / 1e9, byt / ms / 1e6))
    print("total %.3f ms over %d launches" % (tot, len(eng.tc_plan)))
    print(json.dumps({"sm_clock": clk}))


if __name__ == "__main__":
    main()
