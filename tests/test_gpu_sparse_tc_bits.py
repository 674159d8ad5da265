"""Bit-level regression of the tensor-pipe sparse convolution (b2s_sparse_conv_tc_plan): on every built (Cin, Cout)
pair, SubM and strided, the output planes must be the exact bits the kernel produced before its pipeline was
restructured.  Scheduling changes (which warp issues a load, how stages are recycled) may not change a single bit.

tests/golden/sparse_tc_bits.json holds SHA-256 digests of the fp16 hi/lo output planes (no plan, and rows grouped with
tile masks: both must give the same bits) and of the fp32 output rows.  Inputs are generated from fixed seeds, large
enough that every CTA walks several tiles.  Re-record with the kernel whose bits are the reference:
    python tests/test_gpu_sparse_tc_bits.py OUT.json
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse_tc_bits.json")
CASES = [(cin, cout, subm) for cin in (8, 16, 32, 64) for cout in (16, 32, 64) for subm in (True, False)]


def case_id(cin, cout, subm):
    return "cin%d_cout%d_%s" % (cin, cout, "subm" if subm else "strided")


def _inputs(cin, cout, subm):
    """features [n, cin] and coordinates of a noisy surface per frame (structured, differing neighbourhoods)"""
    rng = np.random.default_rng(1000 + 10 * cin + cout + (1 if subm else 0))
    shape, batch = (9, 96, 80), 4
    n = 24000
    b = rng.integers(batch, size=4 * n)
    y = rng.integers(shape[1], size=4 * n)
    x = rng.integers(shape[2], size=4 * n)
    z = np.clip(np.round(shape[0] / 2 + 2 * np.sin(x / 5.0) + rng.normal(0, 0.7, size=4 * n)), 0, shape[0] - 1)
    idx = np.unique(np.stack([b, z, y, x], 1).astype(np.int32), axis=0)[:n]
    feats = rng.standard_normal((idx.shape[0], cin)).astype(np.float32)
    w = (rng.standard_normal((27, cin, cout)) * 0.1).astype(np.float32)
    scale = (rng.random(cout) + 0.5).astype(np.float32)
    shift = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    return shape, batch, torch.from_numpy(feats), torch.from_numpy(idx), torch.from_numpy(w), scale, shift


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def run_case(product, cin, cout, subm):
    """{"planes": digest, "planes_planned": digest, "fp32": digest, "rows": n_out} of one case"""
    from b2second import tc
    L = product._lib
    lib = L.load()
    shape, batch, feats, idx, w, scale, shift = _inputs(cin, cout, subm)
    x = product.SparseConvTensor(feats.cuda(), idx.cuda(), shape, batch)
    s, p = ([1, 1, 1], [1, 1, 1]) if subm else ([2, 2, 2], [1, 1, 1])
    rb = product.ops.build_rulebook(x, [3, 3, 3], s, p, [1, 1, 1], subm)
    n_out = rb.num_out
    nbr = rb.nbr.contiguous()
    wp = tc.pack_sparse_weights(w.cuda())
    ws = tc.pow2_scale(wp)
    w_hi, w_lo = tc.split_f16(wp, ws)
    n_in = feats.shape[0]
    fbuf = torch.zeros(n_in, 2, cin, dtype=torch.float16, device="cuda")
    f_hi, f_lo = fbuf[:, 0], fbuf[:, 1]
    feats_d = feats.cuda()
    n_in_dev = torch.tensor([n_in], dtype=torch.int32, device="cuda")
    L.check(lib.b2s_split_f16(L.ptr(feats_d), L.ptr(f_hi), L.ptr(f_lo), L.ptr(n_in_dev), n_in, cin, cin, 2 * cin,
                              L.stream()), "b2s_split_f16")
    scale_d = torch.from_numpy(scale).cuda() / ws
    shift_d = torch.from_numpy(shift).cuda()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    perm = torch.zeros(n_out, dtype=torch.int32, device="cuda")
    tmask = torch.zeros((n_out + 127) // 128, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_sparse_tile_plan(L.ptr(nbr), None, 27, L.i3([3, 3, 3]), L.ptr(rb.num_out_dev), n_out, 1, L.ptr(perm),
                                     L.ptr(tmask), L.stream()), "b2s_sparse_tile_plan")
    out = {"rows": n_out}
    for key, pm, tm in (("planes", None, None), ("planes_planned", perm, tmask)):
        obuf = torch.full((n_out, 2, cout), 7.0, dtype=torch.float16, device="cuda")
        L.check(lib.b2s_sparse_conv_tc_plan(L.ptr(f_hi), L.ptr(f_lo), 2 * cin, n_in, cin, L.ptr(w_hi), L.ptr(w_lo),
                                            L.ptr(nbr), 27, L.ptr(rb.num_out_dev), n_out, L.ptr(pm), L.ptr(tm),
                                            L.ptr(scale_d), L.ptr(shift_d), 1, L.ptr(obuf[:, 0]), L.ptr(obuf[:, 1]),
                                            2 * cout, cout, L.ptr(status), L.stream()), "b2s_sparse_conv_tc_plan")
        torch.cuda.synchronize()
        out[key] = _digest(obuf)
    o32 = torch.full((n_out, cout), 7.0, device="cuda")
    L.check(lib.b2s_sparse_conv_tc(L.ptr(f_hi), L.ptr(f_lo), 2 * cin, n_in, cin, L.ptr(w_hi), L.ptr(w_lo), L.ptr(nbr),
                                   27, L.ptr(rb.num_out_dev), n_out, L.ptr(scale_d), L.ptr(shift_d), 0,
                                   L.ptr(o32), None, 0, cout, L.ptr(status), L.stream()), "b2s_sparse_conv_tc")
    torch.cuda.synchronize()
    out["fp32"] = _digest(o32)
    assert int(status.item()) == 0
    return out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("cin,cout,subm", CASES, ids=[case_id(*c) for c in CASES])
def test_sparse_conv_tc_bits_unchanged(product, cin, cout, subm):
    with open(FIXTURE) as f:
        want = json.load(f)[case_id(cin, cout, subm)]
    got = run_case(product, cin, cout, subm)
    assert got["rows"] == want["rows"]
    assert got["rows"] > 132 * 128 or not subm        # SubM cases: more tiles than SMs, so CTAs recycle stages
    assert got["planes"] == want["planes"], "fp16 hi/lo planes, no plan"
    assert got["planes_planned"] == want["planes"], "fp16 hi/lo planes, grouped rows + tile masks"
    assert got["fp32"] == want["fp32"], "fp32 rows"


if __name__ == "__main__":
    REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
    from b2second import loader
    sp = loader.product_spconv()
    rec = {}
    for c in CASES:
        r = run_case(sp, *c)
        assert r["planes"] == r["planes_planned"], c
        rec[case_id(*c)] = {"rows": r["rows"], "planes": r["planes"], "fp32": r["fp32"]}
        print(case_id(*c), r["rows"])
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
