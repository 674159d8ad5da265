"""Bit-level regression of the rulebook builders (csrc/rulebook.cu) and the tile plans built from them
(csrc/sparse_plan.cu).  Rulebooks are integers, so a rework of how they are built may not change a single value.

tests/golden/rulebook_bits.json holds SHA-256 digests of the live part of every table:
  * engine_b32 / engine_b1: every rulebook a car.fhd InferenceEngine builds on synth.kitti_cloud frames -- the output
    coordinates and row count of each level, nbr, row_mask, perm and tile_mask;
  * dropin_*: spconv.ops.build_rulebook (SubM and strided, several shapes and batches) and its tile plan;
  * overflow: b2s_rulebook_conv with cap_out below the live row count -- the overflow flag is raised, the row count is
    clamped and the rows that fit are the same as without the clamp.
Re-record with the build whose tables are the reference:
    python tests/test_gpu_rulebook_bits.py OUT.json
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rulebook_bits.json")
ROWS_OVERFLOW = 2          # B2S_STATUS_ROWS_OVERFLOW

# (name, spatial shape, batch, rows, ksize, stride, padding, subm)
DROPIN = [
    ("subm_9x96x80_b4", (9, 96, 80), 4, 24000, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
    ("subm_41x160x140_b2", (41, 160, 140), 2, 30000, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
    ("subm_5x33x47_b3", (5, 33, 47), 3, 3000, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
    ("strided_9x96x80_b4", (9, 96, 80), 4, 24000, (3, 3, 3), (2, 2, 2), (1, 1, 1), False),
    ("strided_41x160x140_b2", (41, 160, 140), 2, 30000, (3, 3, 3), (2, 2, 2), (1, 1, 1), False),
    ("strided_5x33x47_b3", (5, 33, 47), 3, 3000, (3, 3, 3), (2, 2, 2), (0, 1, 1), False),
    ("strided_k311_9x96x80_b4", (9, 96, 80), 4, 24000, (3, 1, 1), (2, 1, 1), (0, 0, 0), False),
]


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def _cloud(shape, batch, n, seed):
    """unique (b, z, y, x) rows of a noisy surface per frame, in random order"""
    rng = np.random.default_rng(seed)
    b = rng.integers(batch, size=4 * n)
    y = rng.integers(shape[1], size=4 * n)
    x = rng.integers(shape[2], size=4 * n)
    z = np.clip(np.round(shape[0] / 2 + 2 * np.sin(x / 5.0) + rng.normal(0, 0.7, size=4 * n)), 0, shape[0] - 1)
    idx = np.unique(np.stack([b, z, y, x], 1).astype(np.int32), axis=0)[:n]
    return torch.from_numpy(idx[rng.permutation(idx.shape[0])].copy())


def engine_case(product, B):
    import bench
    from b2second import config, models
    from b2second.engine import InferenceEngine
    cfg = config.get_config("car.fhd")
    net = models.build_network(cfg, product).eval()
    models.synthetic_weights_(net, "car.fhd", seed=0)
    eng = InferenceEngine(net.cuda(), batch_size=B, max_points=30000, use_cuda_graph=False)
    clouds = [torch.from_numpy(c).cuda() for c in bench.make_clouds("car.fhd", B, 29000)]
    eng.infer(clouds)
    torch.cuda.synchronize()
    eng.check_status()
    out = {}
    for lyr in eng.layers:
        if not lyr["build_rb"]:
            continue
        lout, rb = lyr["out_level"], lyr["rb"]
        n = int(lout.n_dev[0].item())
        d = {"num_out": n, "coors_out": _digest(lout.coors[:n]), "nbr": _digest(rb["nbr"][:n])}
        if rb.get("row_mask") is not None:
            d["row_mask"] = _digest(rb["row_mask"][:n])
        if rb.get("perm") is not None and lyr["tc"]:
            d["perm"] = _digest(rb["perm"][:n])
            d["tile_mask"] = _digest(rb["tile_mask"][:(n + 127) // 128])
        out["layer%d" % lyr["index"]] = d
    del eng
    torch.cuda.empty_cache()
    return out


def dropin_case(product, name, shape, batch, n, ksize, stride, padding, subm):
    idx = _cloud(shape, batch, n, seed=sum(map(ord, name))).cuda()
    x = product.SparseConvTensor(torch.zeros(idx.shape[0], 4, device="cuda"), idx, shape, batch)
    rb = product.ops.build_rulebook(x, list(ksize), list(stride), list(padding), [1, 1, 1], subm)
    m = rb.num_out
    d = {"num_out": m, "coors_out": _digest(rb.out_indices[:m]), "nbr": _digest(rb.nbr[:m]),
         "row_mask": _digest(rb.row_mask[:m])}
    perm, tmask = product.ops.tile_plan(rb)
    if perm is not None:
        d["perm"] = _digest(perm[:m])
        d["tile_mask"] = _digest(tmask[:(m + 127) // 128])
    torch.cuda.synchronize()
    return d


def overflow_case(product):
    """a strided conv whose output rows do not fit cap_out: the rows that fit are the unclamped call's first rows"""
    L = product._lib
    lib = L.load()
    shape, batch, ks, st, pd = (9, 96, 80), 4, (3, 3, 3), (2, 2, 2), (1, 1, 1)
    idx = _cloud(shape, batch, 24000, seed=4242).cuda()
    n_in = idx.shape[0]
    oshape = product.ops.get_conv_output_size(shape, ks, st, pd, (1, 1, 1))
    n_in_dev = torch.tensor([n_in], dtype=torch.int32, device="cuda")
    ws_bytes = lib.b2s_rulebook_conv_workspace_bytes(batch, L.i3(oshape))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    out = {}
    for tag, cap in (("full", n_in * 8), ("clamped", 10007)):
        coors = torch.full((cap, 4), -7, dtype=torch.int32, device="cuda")
        nbr = torch.full((cap, 27), -7, dtype=torch.int32, device="cuda")
        rmask = torch.full((cap,), 7, dtype=torch.int32, device="cuda")
        n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        L.check(lib.b2s_rulebook_conv(
            L.ptr(idx), L.ptr(n_in_dev), n_in, batch, L.i3(shape), L.i3(oshape), L.i3(ks), L.i3(st), L.i3(pd),
            L.i3((1, 1, 1)), L.ptr(coors), L.ptr(n_out), cap, L.ptr(nbr), None, None, 0, L.ptr(ws), ws_bytes,
            L.ptr(rmask), L.ptr(status), L.stream()), "b2s_rulebook_conv")
        torch.cuda.synchronize()
        out[tag] = (int(n_out.item()), int(status.item()), coors, nbr, rmask)
    n_full, st_full, c_full, nb_full, rm_full = out["full"]
    n_cl, st_cl, c_cl, nb_cl, rm_cl = out["clamped"]
    assert st_full == 0 and n_full > 10007
    assert st_cl == ROWS_OVERFLOW and n_cl == 10007
    assert torch.equal(c_cl, c_full[:n_cl]) and torch.equal(nb_cl, nb_full[:n_cl]) and torch.equal(rm_cl, rm_full[:n_cl])
    return {"num_out": n_cl, "status": st_cl, "coors_out": _digest(c_cl), "nbr": _digest(nb_cl),
            "row_mask": _digest(rm_cl)}


def _want(key):
    with open(FIXTURE) as f:
        return json.load(f)[key]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("B", [32, 1])
def test_engine_rulebooks_unchanged(product, B):
    want = _want("engine_b%d" % B)
    got = engine_case(product, B)
    assert sorted(got) == sorted(want)
    for layer in want:
        assert got[layer] == want[layer], layer


@pytest.mark.timeout(300)
@pytest.mark.parametrize("case", DROPIN, ids=[c[0] for c in DROPIN])
def test_dropin_rulebooks_unchanged(product, case):
    assert dropin_case(product, *case) == _want("dropin_" + case[0])


@pytest.mark.timeout(300)
def test_clamped_rows_unchanged(product):
    assert overflow_case(product) == _want("overflow")


if __name__ == "__main__":
    REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, "second.pytorch_b200"))
    from b2second import loader
    sp = loader.product_spconv()
    rec = {}
    for B in (32, 1):
        rec["engine_b%d" % B] = engine_case(sp, B)
        print("engine_b%d" % B, {k: v["num_out"] for k, v in rec["engine_b%d" % B].items()})
    for c in DROPIN:
        rec["dropin_" + c[0]] = dropin_case(sp, *c)
        print(c[0], rec["dropin_" + c[0]]["num_out"])
    rec["overflow"] = overflow_case(sp)
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
