"""The RPN background skip at the granularity of 8-pixel-wide strips (8 x 4 in the engine, 8 x 2 too) on the GPU:
  b2s_rpn_strip_plan             against its numpy restatement (flags, work / background lists, counts)
  k_conv3x3_tc2 with a list      hand-made 8x2 / 8x4 strip lists (short tails, tiles straddling an 8x8 block row and a frame,
                                 partial bottom / right strips) against the dense launch; background strips from the
                                 fill warps, copied or (inside the field's constant margin) stored from its interior
                                 value; nothing else written
  fused engine (car.fhd, lite)   skip on vs off: bit-identical heads, candidates and detections
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from b2second import config, models
from test_host_rpn_strips import strip_plan_numpy

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows", [2, 4])
@pytest.mark.parametrize("H,W", [(200, 176), (160, 132), (163, 132)])
def test_strip_plan_matches_numpy(product, H, W, rows):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(H + W)
    B, nl = 3, 6
    occ = (rng.random((B, H, W)) < 0.002).astype(np.uint8)
    occ[1] = 0                                         # an empty frame: all of it is background
    occ[2, 90:130, 60:120] = 1
    occ[0, H - 1, W - 1] = 1                           # data in the partial corner strip
    ns = B * (-(-H // rows)) * (-(-W // 8))
    d_occ = torch.from_numpy(occ).cuda()
    scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device="cuda")
    flags = torch.full((nl, ns), -1, dtype=torch.int32, device="cuda")
    work = torch.full((nl, ns), -1, dtype=torch.int32, device="cuda")
    bg = torch.full((nl, ns), -1, dtype=torch.int32, device="cuda")
    counts = torch.zeros(nl, 2, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_strip_plan(L.ptr(d_occ), B, H, W, nl, rows, L.ptr(scratch), L.ptr(flags), L.ptr(work),
                                   L.ptr(bg), L.ptr(counts), L.stream()), "b2s_rpn_strip_plan")
    torch.cuda.synchronize()
    ref = strip_plan_numpy(occ, nl, rows)
    for l in range(nl):
        f = ref[l].reshape(-1)
        assert np.array_equal(flags[l].cpu().numpy(), f)
        nw = int(counts[l, 0])
        assert nw == int(f.sum()) and int(counts[l, 1]) == ns - nw
        assert np.array_equal(work[l, :nw].cpu().numpy(), np.nonzero(f)[0])
        assert np.array_equal(bg[l, :ns - nw].cpu().numpy(), np.nonzero(f == 0)[0])
        assert not ref[l][1].any()
    assert int(counts[0, 1]) > ns // 2


# B = 2, H = 21, W = 36, strips R rows high: ceil(21 / R) x 5 strips per frame, id = (b * strips_h + sh) * 5 + sw; the
# last strip row is one pixel high, strip column 4 four pixels wide.  8 / R consecutive entries make one warpgroup
# tile, two tiles one work item.  Each case: (R, work list, strips in neither list, bg_margin: -1 = a random field;
# m >= 0 = a field that is constant at least m pixels from every border and random nearer to it).
STRIP_CASES = [
    # R = 2, 13 entries: tile (18, 22, 50, 53) straddles the 8x8 block rows (strip rows 3 | 4) and reaches the bottom
    # edge, tile (54, 55, 61, 104) straddles the frames, the last tile holds the corner strip 109 and three repeats
    (2, [0, 4, 9, 17, 18, 22, 50, 53, 54, 55, 61, 104, 109], {5, 60, 107}, -1),
    (2, [0, 4, 9, 17, 18, 22, 50, 53, 54, 55, 61, 104, 109], {5, 60, 107}, 3),
    # R = 2, 11 entries: tile (55, 56, 108) ends in a repeat, and the last tile of the second work item is all repeats
    (2, [1, 2, 3, 4, 22, 23, 27, 54, 55, 56, 108], {5, 60, 107}, -1),
    # R = 4, 11 entries: tile (7, 12) straddles the 8x8 block rows, (14, 25) reaches the bottom edge, (29, 30) straddles
    # the frames, the last tile is the corner strip 59 and a repeat
    (4, [0, 4, 7, 12, 14, 25, 29, 30, 44, 57, 59], {5, 35, 50}, -1),
    (4, [0, 4, 7, 12, 14, 25, 29, 30, 44, 57, 59], {5, 35, 50}, 5),
]


@pytest.mark.parametrize("R,work,untouched,margin", STRIP_CASES)
def test_strip_list_launch_matches_dense_launch(product, R, work, untouched, margin):
    """Listed strips bit-identical to the dense launch, background strips = the given field, the rest untouched."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    B, H, W, C = 2, 21, 36, 128
    sh_n, sw_n = -(-H // R), 5
    assert len(work) % 8 != 0
    g = torch.Generator(device="cuda").manual_seed(12)
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
    if margin >= 0:                                     # constant interior: one random pixel's value
        field[:, 1 + margin:H + 1 - margin, 1 + margin:W + 1 - margin] = field[:, 1 + H // 2, 1 + W // 2][:, None, None]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")

    def launch(work, bg):
        out = [torch.full((B, H + 2, W + 2, C), v, dtype=torch.float16, device="cuda") for v in (-3.0, -5.0)]
        d = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
        wl, wn = (d(work), d([len(work)])) if work is not None else (None, None)
        bl, bn = (d(bg), d([len(bg)])) if bg is not None else (None, None)
        L.check(lib.b2s_conv2d_tc_ex2(
            L.ptr(hi), L.ptr(lo), B, H, W, C, L.ptr(w_hi), L.ptr(w_lo), 3, 3, 1, 1, C, 128, L.ptr(scale_k), L.ptr(shift),
            1, H, W, L.ptr(out[0]), L.ptr(out[1]), H, W, 1, C, 1, 0, 0, L.ptr(wl), L.ptr(wn), L.ptr(bl), L.ptr(bn),
            L.ptr(field[0]) if bg is not None else None, L.ptr(field[1]) if bg is not None else None, margin, R,
            L.ptr(status), L.stream()), "b2s_conv2d_tc_ex2")
        torch.cuda.synchronize()
        return out

    dense = launch(None, None)
    bg = [i for i in range(B * sh_n * sw_n) if i not in work and i not in untouched]
    got = launch(work, bg)
    assert int(status.item()) == 0
    for p in range(2):
        for s in range(B * sh_n * sw_n):
            b, sh, sw = s // (sh_n * sw_n), (s // sw_n) % sh_n, s % sw_n
            sl = (slice(1 + sh * R, 1 + min(H, sh * R + R)), slice(1 + sw * 8, 1 + min(W, sw * 8 + 8)))
            if s in work:
                assert torch.equal(got[p][b][sl], dense[p][b][sl]), (p, s)
            elif s in untouched:
                assert bool((got[p][b][sl] == (-3.0, -5.0)[p]).all()), (p, s)
            else:
                assert torch.equal(got[p][b][sl], field[p][sl]), (p, s)
        # the halo is never written
        for t in (got[p][:, 0], got[p][:, -1], got[p][:, :, 0], got[p][:, :, -1]):
            assert bool((t == (-3.0, -5.0)[p]).all()), p


@pytest.mark.parametrize("name", ["car.fhd", "car.lite"])
def test_engine_strip_skip_is_bit_identical(product, monkeypatch, name):
    from b2second import tc
    from b2second.engine import BG_ROWS, InferenceEngine
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    clouds = [torch.from_numpy(gu.make_cloud(name, s, n)).cuda() for s, n in ((0, 20000), (1, 29000), (2, 12000))]
    res = {}
    for bg_on in (True, False):
        if not bg_on:                                        # the reference: no layer tracks background strips
            monkeypatch.setattr(tc, "background_layers", lambda plan: [])
        eng = InferenceEngine(net, batch_size=3, max_points=30000, use_cuda_graph=True)
        assert bool(eng.bg_idx) == bg_on
        if bg_on:
            H, W = eng.tc_hw
            assert eng.bg_tiles == 3 * (-(-H // BG_ROWS)) * (-(-W // 8))
        eng.infer(clouds)
        res[bg_on] = (eng.detections(), eng.tc_heads.clone(), eng.cand_count.clone(),
                      eng.bg_counts.clone() if eng.bg_idx else None, getattr(eng, "bg_tiles", 0))
    on, off = res[True], res[False]
    assert float((on[3][:, 1].float() / on[4]).min()) > 0.1      # the skip really takes strips away
    assert torch.equal(on[2], off[2])
    assert torch.equal(on[1], off[1])
    for a, b in zip(on[0], off[0]):
        assert a["box3d_lidar"].shape == b["box3d_lidar"].shape and a["box3d_lidar"].shape[0] > 0
        assert torch.equal(a["box3d_lidar"], b["box3d_lidar"]) and torch.equal(a["scores"], b["scores"])
