"""per-layer eager stage times of the engine (CUDA events): python tools/layer_times.py [batch]

For every sparse layer on the tensor pipe it also prints what k_sparse_conv_tc moves and multiplies, counted on the
device from the engine's own tables (nbr, perm, tile_mask) after the timed runs:
  pairs     neighbour-table entries that name an input row
  kb_exec   (128-position tile, K block) pairs the kernel executes (K blocks the tile mask rules out are skipped)
  gath_MB   bytes gathered: every pair fetches its input row, hi and lo planes (pairs * 4 * C_in)
  halo_MB   bytes if each tile fetched each distinct input row once (distinct rows per tile * 4 * C_in)
  mma_us    executed fp16 MMA work (kb_exec * 128 rows * 64 * 3*C_out MACs: A_hi*[W_hi;W_lo] + A_lo*W_hi) at the
            H100 SXM data-sheet dense FP16 rate, 989 TFLOP/s
  l2_us     gath_MB at the L2-resident copy bandwidth this script measures on the same card
"""
import json
import sys

import _measure
import torch

from b2second.engine import InferenceEngine

TILE, BLOCK_K = 128, 64
PEAK_F16 = 989e12


def l2_copy_bandwidth(nbytes=16 << 20, iters=200):
    """bytes/s of a device copy whose source and destination (2 x 16 MB) stay resident in the 50 MB L2"""
    a = torch.empty(nbytes // 4, dtype=torch.float32, device="cuda").uniform_()
    b = torch.empty_like(a)
    return 2.0 * nbytes / (_measure.timed(lambda: b.copy_(a), iters, warmup=10) * 1e-3)


def gather_counts(lyr, n_out):
    """(pairs, executed (tile, K block) pairs, distinct input rows summed over tiles) of one tensor-pipe layer"""
    rb, K, cin = lyr["rb"], lyr["K"], lyr["cin_tc"]
    dev = rb["nbr"].device
    perm = rb.get("perm")
    rows = perm[:n_out].long() if perm is not None else torch.arange(n_out, device=dev)
    nb = rb["nbr"][rows].long()                                   # [pos, K] in the kernel's tile order
    tiles = (n_out + TILE - 1) // TILE
    pack = BLOCK_K // cin
    num_kb = (K + pack - 1) // pack
    if rb.get("tile_mask") is not None:
        m = rb["tile_mask"][:tiles].long() & ((1 << K) - 1)
        kb = torch.stack([((m >> (j * pack)) & ((1 << pack) - 1)) != 0 for j in range(num_kb)], 1)
        kb_exec = int(kb.sum(1).clamp(min=1).sum().item())
    else:
        kb_exec = tiles * num_kb
    tile_of = (torch.arange(n_out, device=dev) // TILE).unsqueeze(1).expand(-1, K)
    ok = nb >= 0
    key = tile_of[ok] * (int(nb.max().item()) + 1) + nb[ok]
    return int(ok.sum().item()), kb_exec, int(torch.unique(key).numel())


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    _measure.require_gpu("layer_times")
    print(json.dumps(_measure.card()))
    net, clouds = _measure.mirror("car.fhd", B)
    eng = InferenceEngine(net.eval(), batch_size=B, max_points=30000, use_cuda_graph=False)
    eng.load_points([torch.from_numpy(c).cuda() for c in clouds])
    with _measure.clocks() as clk:
        st = eng.run_timed(iters=5)
        l2_bw = l2_copy_bandwidth()
    stats = {s["index"]: s for s in eng.sparse_layer_stats()}
    print("batch %d, L2-resident copy bandwidth %.0f GB/s (read + write)" % (B, l2_bw / 1e9))
    tot = {"us": 0.0, "gath": 0, "halo": 0}
    for k, v in st.items():
        extra = ""
        if k.startswith("sparse_conv"):
            s = stats[int(k[len("sparse_conv"):])]
            lyr = eng.layers[s["index"]]
            extra = "  cin %d cout %d K %d rows %d pairs %d tc %s" % (s["cin"], s["cout"], s["K"], s["n_out"], s["pairs"],
                                                                      lyr["tc"])
            if lyr["tc"]:
                pairs, kb_exec, uniq = gather_counts(lyr, s["n_out"])
                gath, halo = pairs * 4 * lyr["cin_tc"], uniq * 4 * lyr["cin_tc"]
                mma_us = kb_exec * TILE * BLOCK_K * 3 * s["cout"] * 2 / PEAK_F16 * 1e6
                l2_us = gath / l2_bw * 1e6
                extra += ("\n%16s kb_exec %d gath_MB %.1f halo_MB %.1f (%.2f) mma_us %.1f l2_us %.1f gap_us %.1f"
                          % ("", kb_exec, gath / 1e6, halo / 1e6, halo / max(gath, 1), mma_us, l2_us,
                             v * 1e3 - max(mma_us, l2_us)))
                tot["us"] += v * 1e3
                tot["gath"] += gath
                tot["halo"] += halo
        print("%-16s %8.1f us%s" % (k, v * 1e3, extra))
    print("tensor-pipe sparse layers: %.1f us, gathered %.1f MB, per-tile halo %.1f MB"
          % (tot["us"], tot["gath"] / 1e6, tot["halo"] / 1e6))
    print(json.dumps({"sm_clock": clk}))


if __name__ == "__main__":
    main()
