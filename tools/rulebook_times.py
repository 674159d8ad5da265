"""where the rulebook stage of car.fhd's fused engine spends its time: python tools/rulebook_times.py [OUT_DIR]

For the bench workload (synthetic 29 k-point KITTI clouds, batch 32 and batch 1):
  * the `rulebook*` stage time of InferenceEngine.run_timed (CUDA events around each stage, eager replay);
  * every kernel and memset the rulebook stage issues, from torch.profiler with CUDA activities in a run of its own
    (launches are attributed to the stage whose window the host launched them in); the chrome traces go to OUT_DIR
    (default: rulebook_times under the system's temporary directory);
  * live rows per level and the bytes of the tables built for them (nbr, row_mask; capacity-sized for comparison).
Prints the card first, one table per batch, and the SM clock sampled during the run; writes the same with the results
to OUT_DIR/rulebook_times.json."""
import json
import os
import re
import sys
import tempfile

import _measure
import torch

from b2second.engine import InferenceEngine

ITERS = 10


def short(name):
    name = name.replace("(anonymous namespace)::", "")
    name = re.sub(r"[(<].*$", "", name)              # drop the argument list and template arguments
    return re.sub(r"^.*::", "", name) or name        # and the namespace


def profile_stage(eng, out, prefix="rulebook"):
    """{kernel or memset name: (launches per step, us per step)} of the stages named prefix*"""
    from torch.profiler import record_function
    cur = [None]

    def mark(name):
        if cur[0] is not None:
            cur[0].__exit__(None, None, None)
        cur[0] = record_function("stage:" + name)
        cur[0].__enter__()

    eng._mark = mark
    act = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.no_grad(), torch.profiler.profile(activities=act) as prof:
        for _ in range(ITERS):
            eng._launch()
            mark("end")
            cur[0].__exit__(None, None, None)
            cur[0] = None
        torch.cuda.synchronize()
    del eng._mark
    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, "trace_b%d.json" % eng.B)
    prof.export_chrome_trace(path)
    return stage_split(path, prefix)


def stage_split(path, prefix):
    """per-step {name: (launches, us)} of the device work launched inside the stage windows of a chrome trace"""
    windows = []
    with open(path) as f:
        trace = json.load(f)["traceEvents"]
    # host launch (cuda_runtime, by correlation id) -> stage window it falls in; device work -> its launch
    for e in trace:
        if e.get("cat") == "user_annotation" and e.get("name", "").startswith("stage:" + prefix):
            windows.append((e["ts"], e["ts"] + e["dur"]))
    in_stage = set()
    for e in trace:
        if e.get("cat") in ("cuda_runtime", "cuda_driver") and any(a <= e["ts"] <= b for a, b in windows):
            in_stage.add(e["args"].get("correlation"))
    acc = {}
    for e in trace:
        if e.get("cat") not in ("kernel", "gpu_memset") or e["args"].get("correlation") not in in_stage:
            continue
        nm = "memset" if e["cat"] == "gpu_memset" else short(e["name"])
        c, us = acc.get(nm, (0, 0.0))
        acc[nm] = (c + 1, us + e["dur"])
    return {k: (c / ITERS, us / ITERS) for k, (c, us) in sorted(acc.items(), key=lambda kv: -kv[1][1])}


def level_stats(eng):
    out = []
    for lyr in eng.layers:
        if not lyr["build_rb"]:
            continue
        lout, rb = lyr["out_level"], lyr["rb"]
        n = int(lout.n_dev[0].item())
        K = lyr["K"]
        masks = rb.get("row_mask") is not None
        out.append({"layer": lyr["index"], "kind": "subm" if lyr["subm"] else "strided", "K": K, "rows": n,
                    "cap": lout.cap, "table_bytes_live": 4 * n * K + (4 * n if masks else 0),
                    "table_bytes_cap": 4 * lout.cap * K + (4 * lout.cap if masks else 0)})
    return out


def run(B, out):
    net, clouds = _measure.mirror("car.fhd", B)
    eng = InferenceEngine(net.eval(), batch_size=B, max_points=30000, use_cuda_graph=False)
    eng.load_points([torch.from_numpy(c).cuda() for c in clouds])
    stages = eng.run_timed(iters=20)
    rb_ms = sum(v for k, v in stages.items() if k.startswith("rulebook"))
    step_ms = sum(stages.values())
    kernels = profile_stage(eng, out)
    levels = level_stats(eng)
    eng.check_status()
    print("car.fhd B=%d: rulebook stage %.3f ms of %.3f ms (run_timed, eager)  launches/step %d" % (
        B, rb_ms, step_ms, eng.kernel_launches_per_step()))
    print("  %-28s %8s %10s" % ("kernel / memset", "per step", "us/step"))
    for k, (c, us) in kernels.items():
        print("  %-28s %8.1f %10.1f" % (k, c, us))
    print("  %-28s %8.1f %10.1f" % ("sum", sum(c for c, _ in kernels.values()), sum(us for _, us in kernels.values())))
    print("  %-6s %-8s %3s %9s %9s %14s %14s" % ("layer", "kind", "K", "rows", "cap", "live bytes", "cap bytes"))
    for s in levels:
        print("  %-6d %-8s %3d %9d %9d %14d %14d" % (s["layer"], s["kind"], s["K"], s["rows"], s["cap"],
                                                    s["table_bytes_live"], s["table_bytes_cap"]))
    res = {"batch": B, "rulebook_ms": rb_ms, "step_ms_eager": step_ms,
           "rulebook_stages_ms": {k: v for k, v in stages.items() if k.startswith("rulebook")},
           "kernels": {k: {"per_step": c, "us_per_step": us} for k, (c, us) in kernels.items()}, "levels": levels,
           "launches_per_step": eng.kernel_launches_per_step()}
    del eng, net
    torch.cuda.empty_cache()
    return res


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "rulebook_times")
    _measure.require_gpu("rulebook_times")
    card = _measure.card()
    print(json.dumps(card))
    with _measure.clocks() as clk:
        results = [run(B, out) for B in (32, 1)]
    print(json.dumps({"sm_clock": clk}))
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "rulebook_times.json"), "w") as f:
        json.dump({**card, "sm_clock": clk, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
