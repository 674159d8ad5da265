"""CUDA-event time of the training loss, forward + backward: python tools/loss_times.py [iters]

Prints one JSON line.  Per config (car.fhd at batch 8, nuscenes.all.pp.mhead at batch 4, each with its config's real
anchor count): milliseconds per forward + backward of
  fused  b2second.loss (csrc/loss.cu: three forward kernels, one backward kernel, plus the few torch allocations)
  torch  tests/loss_ref.py in float32 -- the reference's op chain (one-hot, cat, sigmoid, pow, log1p/exp, clamp, floor,
         cross-entropy, sums) -- and its autograd backward
on the same inputs (tests/loss_ref.make_case "a": mostly background, some ignored, a few positives), the kernels' HBM
byte bound (DESIGN.md section 5) and the time that bound takes at the H100 SXM data-sheet 3.35 TB/s (arithmetic, not a
measurement).  Also prints the card name, its power limit and the SM clock sampled during the run.
"""
import sys

import _measure
import loss_ref
import torch

from b2second import loss

HBM_BYTES_PER_S = 3.35e12


def byte_bound(B, A, C, nb, label_bytes):
    """HBM bytes of one forward + backward: every input element read once per pass, every output written once"""
    n = B * A
    count = n * (label_bytes + 4)                                  # labels, importance
    fwd_in = n * (4 * 7 + 4 * C + 4 * nb + label_bytes + 4 + 4 * 7 + 4 * 7)   # preds, labels, importance, targets,
    fwd_out = n * (4 * C + 4 * 7 + 1)                              # anchors (the yaw's sectors); per-anchor outputs
    bwd = fwd_in + n * (4 * 7 + 4 * C + 4 * nb)                    # the same reads, the three gradients
    return count + fwd_in + fwd_out + bwd


def main():
    ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    _measure.require_gpu("loss_times")
    dev = "cuda:0"
    rows = []
    with _measure.clocks() as clk:
        for name, B in (("car.fhd", 8), ("nuscenes.all.pp.mhead", 4)):
            net = _measure.mirror(name, spconv="oracle")
            lp = loss.plan(net)
            s = lp.settings
            A = int(net.anchors().shape[0])
            example, preds = loss_ref.make_case("a", B, A, s.num_class, s.num_dir_bins, s.dir_offset, seed=0)
            ex = {k: v.to(dev) for k, v in example.items()}
            ex["labels"] = ex["labels"].to(torch.int32)                # what b2second.targets.assign_batch gives
            pr = {k: v.to(dev).requires_grad_() for k, v in preds.items()}

            def fused():
                lp.loss(ex, pr)["loss"].backward()

            def chain():
                loss_ref.loss(s, ex, pr)["loss"].backward()

            row = {"config": name, "batch": B, "anchors": A, "num_class": s.num_class}
            row["fused_ms"] = round(_measure.timed(fused, ITERS), 4)
            row["torch_ms"] = round(_measure.timed(chain, ITERS), 4)
            nbytes = byte_bound(B, A, s.num_class, s.num_dir_bins, 4)
            row["byte_bound"] = nbytes
            row["byte_bound_ms"] = round(nbytes / HBM_BYTES_PER_S * 1e3, 4)
            rows.append(row)
    _measure.report("loss_times", rows, clk, iters=ITERS)


if __name__ == "__main__":
    main()
