"""Background strips filled only where a later launch reads them, background tail tiles written from the empty frame's
records, and a BEV map cleared only where it was written:
  b2s_rpn_strip_bands            against its numpy restatement (bands of every layer, the fused tail's work and
                                 background tiles, counts, nothing past the counts), and the coverage property: every
                                 pixel a computed strip of layer l + 1 reads, and every pixel of a computed tail tile,
                                 lies in a strip of the layer before that is computed or in the band
  b2s_rpn_tail_tc_ex             listed tiles bit-identical to the dense tail, background tiles equal to the given
                                 record field (stored from registers inside the margin, copied near the border),
                                 nothing else written
  b2s_to_bev_tc_ex               captured once, replayed over batches with fewer rows in other places: the planes and
                                 the occupancy map equal a zero-fill scatter's after every replay
  fused engine (car.fhd, lite)   one engine over three different batches: BEV planes, heads, candidates and detections
                                 bit-identical to a fresh engine per batch without background strips
"""
import numpy as np
import pytest
import torch

import golden_util as gu
from b2second import config, models
from rpn_bands_ref import strip_bands, tail_tiles
from test_host_rpn_strips import strip_plan_numpy

pytestmark = pytest.mark.gpu


def strips_to_pixels(mask, H, W, rows, width=8):
    return mask.repeat(rows, axis=1).repeat(width, axis=2)[:, :H, :W]


def dilate(mask):
    H, W = mask.shape[1:]
    pad = np.pad(mask, ((0, 0), (1, 1), (1, 1)))
    out = np.zeros_like(mask)
    for dy in range(3):
        for dx in range(3):
            out |= pad[:, dy:dy + H, dx:dx + W]
    return out


def run_bands(lib, L, occ, nl, rows):
    B, H, W = occ.shape
    ns = B * (-(-H // rows)) * (-(-W // 8))
    nt = B * (-(-H // 8)) * (-(-W // 16))
    d_occ = torch.from_numpy(occ).cuda()
    scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(nl, ns, dtype=torch.int32, device="cuda")
    work = torch.zeros(nl, ns, dtype=torch.int32, device="cuda")
    bg = torch.zeros(nl, ns, dtype=torch.int32, device="cuda")
    counts = torch.zeros(nl, 2, dtype=torch.int32, device="cuda")
    bands = torch.full((nl, ns), -1, dtype=torch.int32, device="cuda")
    band_counts = torch.full((nl + 1,), -1, dtype=torch.int32, device="cuda")
    tail = torch.full((2, nt), -1, dtype=torch.int32, device="cuda")
    tail_counts = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_strip_plan(L.ptr(d_occ), B, H, W, nl, rows, L.ptr(scratch), L.ptr(flags), L.ptr(work),
                                   L.ptr(bg), L.ptr(counts), L.stream()), "b2s_rpn_strip_plan")
    L.check(lib.b2s_rpn_strip_bands(L.ptr(flags), B, H, W, nl, rows, L.ptr(bands), L.ptr(band_counts),
                                    L.ptr(tail[0]), L.ptr(tail[1]), L.ptr(tail_counts), L.stream()),
            "b2s_rpn_strip_bands")
    torch.cuda.synchronize()
    return (flags.cpu().numpy(), bands.cpu().numpy(), band_counts.cpu().numpy(), tail.cpu().numpy(),
            tail_counts.cpu().numpy())


@pytest.mark.parametrize("H,W", [(200, 176), (163, 132)])
def test_strip_bands_match_numpy(product, H, W):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(H * W)
    B, nl, rows = 3, 6, 4
    occ = (rng.random((B, H, W)) < 0.002).astype(np.uint8)
    occ[1] = 0                                         # an empty frame: no band, no computed tail tile
    occ[2] = 1                                         # a full frame: every strip and tile computed, no band
    occ[0, H - 1, W - 1] = 1                           # data in the partial corner strip and tile
    flags, bands, band_counts, tail, tail_counts = run_bands(lib, L, occ, nl, rows)
    ref_flags = strip_plan_numpy(occ, nl, rows)
    ref = strip_bands(ref_flags, rows)
    assert int(band_counts[nl]) == -1                  # one count per layer
    for l in range(nl):
        assert np.array_equal(flags[l], ref_flags[l].reshape(-1))
        f = ref[l].reshape(-1)
        nb = int(band_counts[l])
        assert nb == int(f.sum()) and nb > 0
        assert np.array_equal(bands[l, :nb], np.nonzero(f)[0])
        assert (bands[l, nb:] == -1).all()
        assert not ref[l][1].any() and not ref[l][2].any()
    tiles = tail_tiles(ref_flags[-1], rows)
    assert tiles[0, -1, -1] and not tiles[1].any() and tiles[2].all()
    t = tiles.reshape(-1)
    nw = int(tail_counts[0])
    assert nw == int(t.sum()) and int(tail_counts[1]) == t.size - nw and int(tail_counts[2]) == -1
    assert np.array_equal(tail[0, :nw], np.nonzero(t)[0]) and (tail[0, nw:] == -1).all()
    assert np.array_equal(tail[1, :t.size - nw], np.nonzero(~t)[0]) and (tail[1, t.size - nw:] == -1).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_strip_bands_cover_what_is_read(product, seed):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(seed)
    B, nl, rows = 2, 6, 4
    H, W = int(rng.integers(40, 90)), int(rng.integers(40, 90))
    occ = (rng.random((B, H, W)) < rng.choice([0.001, 0.004, 0.02])).astype(np.uint8)
    flags, bands, band_counts, tail, tail_counts = run_bands(lib, L, occ, nl, rows)
    sh, sw = -(-H // rows), -(-W // 8)
    th, tw = -(-H // 8), -(-W // 16)
    computed_tiles = np.zeros(B * th * tw, bool)
    computed_tiles[tail[0, :int(tail_counts[0])]] = True
    for l in range(nl):
        computed = flags[l].reshape(B, sh, sw).astype(bool)
        band = np.zeros(B * sh * sw, bool)
        band[bands[l, :int(band_counts[l])]] = True
        filled = strips_to_pixels(computed | band.reshape(B, sh, sw), H, W, rows)
        if l + 1 < nl:   # the pixels the windows of layer l + 1's computed strips read (inside the image)
            read = dilate(strips_to_pixels(flags[l + 1].reshape(B, sh, sw).astype(bool), H, W, rows))
        else:            # the pixels of the computed tail tiles
            read = strips_to_pixels(computed_tiles.reshape(B, th, tw), H, W, 8, 16)
            assert (strips_to_pixels(computed, H, W, rows) <= read).all()      # every computed strip is in one
        assert not (read & ~filled).any(), l
        assert not (band.reshape(B, sh, sw) & computed).any()


@pytest.mark.parametrize("margin", [-1, 3])
def test_tail_lists_match_dense_tail(product, margin):
    """listed tiles bit-identical to the dense tail, background tiles = the given record field, the rest untouched."""
    from b2second import tc
    L = product._lib
    lib = L.load()
    net = models.build_network(config.get_config("car.fhd"), product).eval()
    models.synthetic_weights_(net, "car.fhd", seed=0)
    net = net.cuda()
    B, H, W = 2, 21, 36           # 3 x 3 tiles of 8 x 16 per frame, the last tile row and column partial
    plan = tc.plan_rpn(net.rpn, H, W)
    assert tc.fusable_tail(plan)
    d, h, S = plan["ops"][-2], plan["ops"][-1], plan["heads"]["stride"]
    n = h["cout"]
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.zeros(B, H + 2, W + 2, 128, device="cuda")
    x[:, 1:H + 1, 1:W + 1] = torch.rand(B, H, W, 128, device="cuda", generator=g)
    hi, lo = tc.split_f16(x)
    field = torch.randn(H, W, S, device="cuda", generator=g)
    if margin >= 0:                                     # constant interior: one pixel's record
        field[margin:H - margin, margin:W - margin] = field[H // 2, W // 2]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    # tile 13 = frame 1, tile (1, 1) lies >= 3 pixels from every border: stored from registers when margin = 3
    work, bg = [0, 4, 8, 10, 17], [1, 2, 5, 12, 13, 16]

    def launch(work, bg):
        out = torch.full((B, H, W, S), -3.0, device="cuda")
        dv = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
        wl, wn = (dv(work), dv([len(work)])) if work is not None else (None, None)
        bl, bn = (dv(bg), dv([len(bg)])) if bg is not None else (None, None)
        L.check(lib.b2s_rpn_tail_tc_ex(
            L.ptr(hi), L.ptr(lo), B, H, W, 128, L.ptr(d["w_hi"]), L.ptr(d["w_lo"]), d["cout"], L.ptr(d["scale"]),
            L.ptr(d["shift"]), L.ptr(h["w_hi"]), L.ptr(h["w_lo"]), n, h["n_pad"], L.ptr(h["scale"]), L.ptr(h["shift"]),
            L.ptr(out), S, L.ptr(wl), L.ptr(wn), L.ptr(bl), L.ptr(bn), L.ptr(field) if bg is not None else None,
            margin, L.ptr(status), L.stream()), "b2s_rpn_tail_tc_ex")
        torch.cuda.synchronize()
        return out

    dense = launch(None, None)
    got = launch(work, bg)
    assert int(status.item()) == 0
    for t in range(B * 9):
        b, th, tw = t // 9, (t // 3) % 3, t % 3
        sl = (b, slice(th * 8, min(H, th * 8 + 8)), slice(tw * 16, min(W, tw * 16 + 16)))
        if t in work:
            assert torch.equal(got[sl][..., :n], dense[sl][..., :n]), t
        elif t in bg:
            assert torch.equal(got[sl][..., :n], field[sl[1:]][..., :n]), t
        else:
            assert bool((got[sl] == -3.0).all()), t
    assert bool((got[..., n:] == -3.0).all())


def test_to_bev_tc_ex_replays_match_zero_fill_scatter(product):
    L = product._lib
    lib = L.load()
    B, D, H, W, C, cap = 3, 2, 20, 28, 32, 600
    coors = torch.zeros(cap, 4, dtype=torch.int32, device="cuda")
    feats = torch.zeros(cap, C, dtype=torch.float32, device="cuda")
    n_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    planes = [torch.zeros(B, H + 2, W + 2, C * D, dtype=torch.float16, device="cuda") for _ in range(2)]
    occ = torch.zeros(B, H, W, dtype=torch.uint8, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        L.check(lib.b2s_to_bev_tc_ex(L.ptr(feats), None, None, 0, L.ptr(coors), L.ptr(n_dev), cap, C, B, D, H, W,
                                     L.ptr(planes[0]), L.ptr(planes[1]), L.ptr(occ), L.stream()), "b2s_to_bev_tc_ex")
    # (seed, rows, y range): the second batch has fewer rows, all in the lower half, so most earlier pixels must clear
    for seed, n, (y0, y1) in ((0, 500, (0, H)), (1, 90, (H // 2, H)), (2, 300, (0, H))):
        rng = np.random.default_rng(seed)
        flat = rng.choice(B * D * (y1 - y0) * W, n, replace=False)
        b, r = np.divmod(flat, D * (y1 - y0) * W)
        z, r = np.divmod(r, (y1 - y0) * W)
        y, x = np.divmod(r, W)
        coors.zero_()
        coors[:n] = torch.from_numpy(np.stack([b, z, y + y0, x], 1).astype(np.int32)).cuda()
        feats.zero_()
        feats[:n] = torch.from_numpy(rng.standard_normal((n, C)).astype(np.float32)).cuda()
        n_dev.fill_(n - 5)                                                      # the last rows are beyond the count
        ref = [torch.full_like(planes[0], 7.0) for _ in range(2)]
        ref_occ = torch.full_like(occ, 9)
        L.check(lib.b2s_to_bev_tc(L.ptr(feats), None, None, 0, L.ptr(coors), L.ptr(n_dev), cap, C, B, D, H, W,
                                  L.ptr(ref[0]), L.ptr(ref[1]), L.ptr(ref_occ), L.stream()), "b2s_to_bev_tc")
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(planes[0], ref[0]) and torch.equal(planes[1], ref[1]), seed
        assert torch.equal(occ, ref_occ), seed
        assert int(ref_occ.sum()) > 0


@pytest.mark.parametrize("name", ["car.fhd", "car.lite"])
def test_engine_bands_over_a_batch_sequence(product, monkeypatch, name):
    from b2second import tc
    from b2second.engine import InferenceEngine
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    batches = [((0, 20000), (1, 29000), (2, 12000)),
               ((3, 6000), (4, 3000), (5, 9000)),              # fewer points: most earlier BEV pixels must clear
               ((6, 24000), (7, 29000), (8, 15000))]
    batches = [[torch.from_numpy(gu.make_cloud(name, s, n)).cuda() for s, n in bt] for bt in batches]
    eng = InferenceEngine(net, batch_size=3, max_points=30000, use_cuda_graph=True)
    assert len(eng.bg_idx) == 6
    got = []
    for clouds in batches:
        eng.infer(clouds)
        band = eng.bg_band_counts.clone()
        bg = eng.bg_counts[:, 1].clone()
        assert bool((band < bg).all())                 # the band is a strict part of the background
        assert 0 < int(eng.tail_counts[1]) < eng.tail_tiles     # some tail tiles are background
        got.append((eng.detections(), eng.tc_heads.clone(), eng.cand_count.clone(), eng.tc_bev[0].clone(),
                    eng.tc_bev[1].clone()))
    monkeypatch.setattr(tc, "background_layers", lambda plan: [])
    for clouds, on in zip(batches, got):
        ref = InferenceEngine(net, batch_size=3, max_points=30000, use_cuda_graph=True)
        assert not ref.bg_idx
        ref.infer(clouds)
        assert torch.equal(on[3], ref.tc_bev[0]) and torch.equal(on[4], ref.tc_bev[1])
        assert torch.equal(on[2], ref.cand_count)
        assert torch.equal(on[1], ref.tc_heads)
        for a, b in zip(on[0], ref.detections()):
            assert a["box3d_lidar"].shape == b["box3d_lidar"].shape
            assert torch.equal(a["box3d_lidar"], b["box3d_lidar"]) and torch.equal(a["scores"], b["scores"])
        del ref
