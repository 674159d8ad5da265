"""The RPN background skip at 8x8-block granularity on the GPU:
  b2s_rpn_block_plan             against its numpy restatement (flags, work / background lists, counts)
  k_conv3x3_tc2 with a list      a hand-made block list (odd count, pairs straddling a block row and a frame, partial
                                 edge blocks) against the dense launch; background blocks from the fill warps; nothing
                                 else written
  fused engine (car.lite)        skip on vs off: bit-identical heads, candidates and detections
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from b2second import config, models
from test_host_rpn_plan import bg_plan_numpy

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H,W", [(200, 176), (160, 132)])
def test_block_plan_matches_numpy(product, H, W):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(H + W)
    B, nl = 3, 6
    occ = (rng.random((B, H, W)) < 0.002).astype(np.uint8)
    occ[1] = 0                                         # an empty frame: all of it is background
    occ[2, 90:130, 60:120] = 1
    occ[0, H - 1, W - 1] = 1                           # data in the partial corner block (W = 132)
    nb = B * (-(-H // 8)) * (-(-W // 8))
    d_occ = torch.from_numpy(occ).cuda()
    scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device="cuda")
    flags = torch.full((nl, nb), -1, dtype=torch.int32, device="cuda")
    work = torch.full((nl, nb), -1, dtype=torch.int32, device="cuda")
    bg = torch.full((nl, nb), -1, dtype=torch.int32, device="cuda")
    counts = torch.zeros(nl, 2, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_block_plan(L.ptr(d_occ), B, H, W, nl, L.ptr(scratch), L.ptr(flags), L.ptr(work), L.ptr(bg),
                                   L.ptr(counts), L.stream()), "b2s_rpn_block_plan")
    torch.cuda.synchronize()
    ref = bg_plan_numpy(occ, nl, tile=8)
    for l in range(nl):
        f = ref[l].reshape(-1)
        assert np.array_equal(flags[l].cpu().numpy(), f)
        nw = int(counts[l, 0])
        assert nw == int(f.sum()) and int(counts[l, 1]) == nb - nw
        assert np.array_equal(work[l, :nw].cpu().numpy(), np.nonzero(f)[0])
        assert np.array_equal(bg[l, :nb - nw].cpu().numpy(), np.nonzero(f == 0)[0])
        assert not ref[l][1].any()
    assert int(counts[0, 1]) > nb // 2


def test_block_list_launch_matches_dense_launch(product):
    """Listed blocks bit-identical to the dense launch, background blocks = the given field, the rest untouched."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, H, W, C = 2, 20, 36, 128                        # 3 x 5 blocks per frame: the last row and column are partial
    bh_n, bw_n = 3, 5
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(B, C, H, W, device="cuda", generator=g)
    w = torch.randn(C, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.1
    hi, lo = tc.split_f16(F.pad(x.permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).contiguous())
    wt = w.permute(2, 3, 0, 1).reshape(9, C, C).contiguous()
    ws = tc.pow2_scale(wt)
    w_hi, w_lo = tc.split_f16(wt, ws)
    scale_k = (scale / ws).contiguous()
    # the background "field": any halo-padded frame; the kernel copies it, it does not compute it
    field = torch.randn(2, H + 2, W + 2, C, device="cuda", generator=g).half()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")

    def launch(work, bg):
        out = [torch.full((B, H + 2, W + 2, C), v, dtype=torch.float16, device="cuda") for v in (-3.0, -5.0)]
        d = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
        wl, wn = (d(work), d([len(work)])) if work is not None else (None, None)
        bl, bn = (d(bg), d([len(bg)])) if bg is not None else (None, None)
        L.check(lib.b2s_conv2d_tc_ex(
            L.ptr(hi), L.ptr(lo), B, H, W, C, L.ptr(w_hi), L.ptr(w_lo), 3, 3, 1, 1, C, 128, L.ptr(scale_k), L.ptr(shift),
            1, H, W, L.ptr(out[0]), L.ptr(out[1]), H, W, 1, C, 1, 0, 0, L.ptr(wl), L.ptr(wn), L.ptr(bl), L.ptr(bn),
            L.ptr(field[0]) if bg is not None else None, L.ptr(field[1]) if bg is not None else None,
            L.ptr(status), L.stream()), "b2s_conv2d_tc_ex")
        torch.cuda.synchronize()
        return out

    dense = launch(None, None)
    # pairs (4, 5): a block-row boundary, (14, 15): a frame boundary; 29 is alone (odd count), partial in both axes
    work = [4, 5, 10, 12, 14, 15, 29]
    untouched = {0, 20}                                 # in neither list
    bg = [i for i in range(B * bh_n * bw_n) if i not in work and i not in untouched]
    got = launch(work, bg)
    assert int(status.item()) == 0
    for p in range(2):
        for blk in range(B * bh_n * bw_n):
            b, bh, bw = blk // (bh_n * bw_n), (blk // bw_n) % bh_n, blk % bw_n
            sl = (slice(1 + bh * 8, 1 + min(H, bh * 8 + 8)), slice(1 + bw * 8, 1 + min(W, bw * 8 + 8)))
            if blk in work:
                assert torch.equal(got[p][b][sl], dense[p][b][sl]), (p, blk)
            elif blk in untouched:
                assert bool((got[p][b][sl] == (-3.0, -5.0)[p]).all()), (p, blk)
            else:
                assert torch.equal(got[p][b][sl], field[p][sl]), (p, blk)
        # the halo is never written
        for t in (got[p][:, 0], got[p][:, -1], got[p][:, :, 0], got[p][:, :, -1]):
            assert bool((t == (-3.0, -5.0)[p]).all()), p


def test_engine_block_skip_is_bit_identical_car_lite(product, monkeypatch):
    from b2second import tc
    from b2second.engine import InferenceEngine
    name = "car.lite"
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    clouds = [torch.from_numpy(gu.make_cloud(name, s, n)).cuda() for s, n in ((0, 20000), (1, 29000), (2, 12000))]
    res = {}
    for bg_on in (True, False):
        if not bg_on:                                        # the reference: no layer tracks background blocks
            monkeypatch.setattr(tc, "background_layers", lambda plan: [])
        eng = InferenceEngine(net, batch_size=3, max_points=30000, use_cuda_graph=True)
        assert bool(eng.bg_idx) == bg_on
        eng.infer(clouds)
        res[bg_on] = (eng.detections(), eng.tc_heads.clone(), eng.cand_count.clone(),
                      eng.bg_counts.clone() if eng.bg_idx else None, getattr(eng, "bg_tiles", 0))
    on, off = res[True], res[False]
    assert float((on[3][:, 1].float() / on[4]).min()) > 0.1      # the skip really takes blocks away
    assert torch.equal(on[2], off[2])
    assert torch.equal(on[1], off[1])
    for a, b in zip(on[0], off[0]):
        assert a["box3d_lidar"].shape == b["box3d_lidar"].shape and a["box3d_lidar"].shape[0] > 0
        assert torch.equal(a["box3d_lidar"], b["box3d_lidar"]) and torch.equal(a["scores"], b["scores"])
