"""The NuScenes multi-head network (nuscenes/all.pp.mhead) on the H100: the new kernels against torch, and the fused
engine, ``accelerate(net)`` and the module-by-module path against the fixtures generated from the unmodified reference
(tests/golden/make_mhead_golden.py).  Bars as for the single-head networks (test_gpu_e2e.py)."""
import ctypes

import numpy as np
import pytest
import torch

import golden_util as gu
from b2second import spec
from test_mhead import CASES, IDS, NAME, build

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_convs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _example(net, pts, max_voxels, device):
    res = net.voxel_generator.generate(pts, max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    return {"anchors": torch.from_numpy(net.anchors()[None]).to(device),
            "voxels": torch.from_numpy(res["voxels"]).to(device),
            "num_points": torch.from_numpy(res["num_points_per_voxel"]).to(device),
            "coordinates": torch.from_numpy(coords).to(device)}


def test_pfn_radius_matches_the_module(product):
    L = product._lib
    lib = L.load()
    net = build(product).cuda()
    s = spec.spec_from_module(net)
    pts = gu.make_cloud(NAME, 0, 60000)
    ex = _example(net, pts, 30000, "cuda")
    N, T, Fn = ex["voxels"].shape
    with torch.no_grad():
        ref = net.voxel_feature_extractor(ex["voxels"], ex["num_points"], ex["coordinates"])
    p = s.pfn
    w, sc, sh = p["w"].cuda(), p["scale"].cuda(), p["shift"].cuda()
    assert w.shape[1] == Fn + 4
    slots = torch.arange(N * T, dtype=torch.int32, device="cuda").view(N, T)
    n_dev = torch.tensor([N], dtype=torch.int32, device="cuda")
    out = torch.zeros(N, 64, device="cuda")
    L.check(lib.b2s_pfn_ex(L.ptr(ex["voxels"]), Fn, L.ptr(slots), L.ptr(ex["num_points"].int()),
                           L.ptr(ex["coordinates"].int().contiguous()), L.ptr(n_dev), N, T, L.ptr(w), L.ptr(sc),
                           L.ptr(sh), 64, p["vx"], p["vy"], p["x_offset"], p["y_offset"], 1, L.ptr(out), L.stream()),
            "b2s_pfn_ex")
    torch.cuda.synchronize()
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5)
    # decoration 0 through the new entry point is b2s_pfn bit for bit
    w0 = torch.randn(64, Fn + 5, device="cuda")
    a, b = torch.zeros_like(out), torch.zeros_like(out)
    for fn, o, extra in ((lib.b2s_pfn, a, ()), (lib.b2s_pfn_ex, b, (0,))):
        L.check(fn(L.ptr(ex["voxels"]), Fn, L.ptr(slots), L.ptr(ex["num_points"].int()),
                   L.ptr(ex["coordinates"].int().contiguous()), L.ptr(n_dev), N, T, L.ptr(w0), L.ptr(sc), L.ptr(sh), 64,
                   p["vx"], p["vy"], p["x_offset"], p["y_offset"], *extra, L.ptr(o), L.stream()), "pfn")
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_crop_is_slicing_plus_zero_halo(product):
    L = product._lib
    lib = L.load()
    B, H, W, C, c = 2, 50, 44, 64, 5
    g = torch.Generator(device="cuda").manual_seed(0)
    src = [torch.randn(B, H + 2, W + 2, C, device="cuda", generator=g).half() for _ in range(2)]
    dst = [torch.full((B, H - 2 * c + 2, W - 2 * c + 2, C), 7.0, device="cuda").half() for _ in range(2)]
    L.check(lib.b2s_crop_nhwc(L.ptr(src[0]), L.ptr(src[1]), B, H, W, C, c, L.ptr(dst[0]), L.ptr(dst[1]), L.stream()),
            "b2s_crop_nhwc")
    torch.cuda.synchronize()
    for s_, d in zip(src, dst):
        want = torch.nn.functional.pad(s_[:, 1 + c:H + 1 - c, 1 + c:W + 1 - c], (0, 0, 1, 1, 1, 1))
        assert torch.equal(d.view(torch.int16), want.view(torch.int16))


def test_decode_segments_equals_per_segment_decode(product):
    """two head maps, one list per frame: the same candidates, bit for bit, as one b2s_decode_filter_strided per map,
    with the anchor ids shifted by the segment's base"""
    L = product._lib
    lib = L.load()
    B, code, ncls, nbins, cc = 2, 7, 10, 2, 8192
    g = torch.Generator(device="cuda").manual_seed(1)
    segs = [(12, 30, 40, 232), (8, 48, 48, 152)]        # (a_loc, H, W, record stride)
    recs = [torch.randn(B, h, w, S, device="cuda", generator=g) * 0.5 - 0.4 for a, h, w, S in segs]
    A = sum(a * h * w for a, h, w, _ in segs)
    anchors = torch.rand(A, code, device="cuda", generator=g) + 0.5
    mask = (torch.rand(B, A, device="cuda", generator=g) < 0.8).to(torch.uint8)
    thresh = 0.7                                         # ~6 % of the anchors pass: no list overflows

    def bufs(n):
        return [torch.zeros(n, cc, code, device="cuda"), torch.zeros(n, cc, device="cuda"),
                torch.zeros(n, cc, dtype=torch.int32, device="cuda"), torch.zeros(n, cc, dtype=torch.int32, device="cuda"),
                torch.zeros(n, cc, dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    desc, base, per_seg = [], 0, []
    for (a, h, w, S), r in zip(segs, recs):
        box, cls, dr = r.data_ptr(), r.data_ptr() + 4 * a * code, r.data_ptr() + 4 * a * (code + ncls)
        bs = h * w * S
        desc.append({"box": box, "cls": cls, "dir": dr, "box_batch_stride": bs, "cls_batch_stride": bs,
                     "dir_batch_stride": bs, "ch_stride": 1, "pix_stride": S, "a_loc": a, "H": h, "W": w,
                     "anchor_base": base})
        o = bufs(B)
        m = mask[:, base:base + a * h * w].contiguous()
        L.check(lib.b2s_decode_filter_strided(
            ctypes.c_void_p(box), ctypes.c_void_p(cls), ctypes.c_void_p(dr), bs, bs, bs, 1, S,
            L.ptr(anchors[base:]), L.ptr(m), B, a, h, w, code, ncls, nbins, thresh, *[L.ptr(t) for t in o], cc,
            L.ptr(status), L.stream()), "b2s_decode_filter_strided")
        per_seg.append((o, base, m))
        base += a * h * w
    got = bufs(B)
    L.check(lib.b2s_decode_filter_segments(L.head_segments(desc), len(desc), L.ptr(anchors), L.ptr(mask), A, B, code,
                                           ncls, nbins, thresh, *[L.ptr(t) for t in got], cc, L.ptr(status),
                                           L.stream()), "b2s_decode_filter_segments")
    torch.cuda.synchronize()
    assert int(status.item()) == 0

    def rows(o, b, shift=0):
        n = int(o[5][b].item())
        key = o[4][b, :n].long() + shift
        order = torch.argsort(key)
        return key[order], o[0][b, :n][order], o[1][b, :n][order], o[2][b, :n][order], o[3][b, :n][order]
    for b in range(B):
        parts = [rows(o, b, base) for o, base, _ in per_seg]
        want = [torch.cat([p[i] for p in parts]) for i in range(5)]
        have = rows(got, b)
        assert want[0].numel() > 100 and all(p[0].numel() > 0 for p in parts)
        assert torch.equal(have[0], want[0])                            # same candidates, global anchor ids
        for x, y in zip(have[1:], want[1:]):
            assert torch.equal(x, y)                                    # boxes, scores, labels, dirs bit-identical


def _anchor_scores(eng, b=0):
    """max over classes of the sigmoid score of every anchor of frame b, in global anchor order, from the engine's heads"""
    out = []
    for si, g in enumerate(eng.segments):
        if eng.rpn_impl == "tc":
            off = eng.tc_prog["segments"][si]["offsets"][1]
            t = eng.tc_seg_heads[g["name"]][b, :, :, off:off + g["a_loc"] * 10]          # [H, W, a_loc*ncls]
            t = t.reshape(g["H"] * g["W"], g["a_loc"], 10).permute(1, 0, 2)
        else:
            t = eng._keep[si][1][b].reshape(g["a_loc"], 10, g["H"] * g["W"]).permute(0, 2, 1)
        out.append(torch.sigmoid(t).max(-1)[0].reshape(-1))
    return torch.cat(out)


def _head_values(eng, flat_idx, which, per_anchor):
    """values of the concatenated ``box_preds`` / ``cls_preds`` [B, A, per_anchor] of network_forward at ``flat_idx``,
    read from the engine's head records (tc) or its torch head outputs (cudnn)"""
    idx = np.asarray(flat_idx, dtype=np.int64)
    c, a, b = idx % per_anchor, (idx // per_anchor) % eng.A, idx // (per_anchor * eng.A)
    out = np.zeros(idx.shape, np.float32)
    for si, g in enumerate(eng.segments):
        n = g["a_loc"] * g["H"] * g["W"]
        sel = (a >= g["base"]) & (a < g["base"] + n)
        loc = a[sel] - g["base"]
        al, hw = loc // (g["H"] * g["W"]), loc % (g["H"] * g["W"])
        y, x = hw // g["W"], hw % g["W"]
        if eng.rpn_impl == "tc":
            pg = eng.tc_prog["segments"][si]
            off = pg["offsets"][0 if which == "box" else 1]
            t = eng.tc_seg_heads[g["name"]].cpu().numpy()
            out[sel] = t[b[sel], y, x, off + al * per_anchor + c[sel]]
        else:
            t = eng._keep[si][0 if which == "box" else 1].cpu().numpy()
            out[sel] = t[b[sel], al * per_anchor + c[sel], y, x]
    return out


@pytest.mark.parametrize("rpn_impl,graph", [("tc", True), ("cudnn", False)])
@pytest.mark.parametrize("seed,n,path", CASES, ids=IDS)
def test_engine_matches_golden(product, seed, n, path, rpn_impl, graph):
    from b2second.engine import InferenceEngine
    fix = np.load(path)
    pts = gu.make_cloud(NAME, seed, n)
    net = build(product).cuda()
    eng = InferenceEngine(net, batch_size=1, max_points=n, max_voxels=int(fix["max_voxels"]), use_cuda_graph=graph,
                          rpn_impl=rpn_impl)
    assert eng.A == 324800 and [(g["H"], g["W"], g["a_loc"]) for g in eng.segments] == [(100, 100, 12), (160, 160, 8)]
    eng.infer([torch.from_numpy(pts).cuda()])
    if graph:
        eng.infer([torch.from_numpy(pts).cuda()])
    out = eng.detections()[0]
    assert int(eng.num_voxels[0].item()) == int(fix["voxel_num"])
    # candidate count: exact, except for anchors whose score lies within the head-tensor bar (1e-4 on the logit,
    # 5e-6 on a score near 0.05) of the threshold -- their side of it is not decided at fp32 parity
    near = int(((_anchor_scores(eng) - eng.score_thresh).abs() <= 5e-6).sum().item())
    assert abs(int(eng.cand_count[0].item()) - int(fix["num_pass_threshold"])) <= near
    np.testing.assert_allclose(_head_values(eng, fix["box_sel_idx"], "box", 7), fix["box_sel_val"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(_head_values(eng, fix["cls_sel_idx"], "cls", 10), fix["cls_sel_val"], rtol=0, atol=1e-4)
    gu.assert_detections_close({k: (v.numpy() if hasattr(v, "numpy") else v) for k, v in out.items()}, fix)


@pytest.mark.parametrize("entry", ["voxels", "points"])
def test_accelerate_runs_the_multihead_network(product, entry):
    from b2second import fastpath
    seed, n, path = CASES[0]
    fix = np.load(path)
    pts = gu.make_cloud(NAME, seed, n)
    net = build(product).cuda()
    ex = _example(net, pts, int(fix["max_voxels"]), "cuda")
    fastpath.accelerate(net, max_points=n, max_voxels=int(fix["max_voxels"]))
    eng = net.b2s_fastpath.engine(1)
    assert eng.rpn_impl == "tc" and eng.pfn_deco == 1
    if entry == "points":
        ex = {"anchors": ex["anchors"], "points": [torch.from_numpy(pts)], "metadata": [{"token": "m0"}]}
    out = net(ex)[0]
    gu.assert_detections_close({k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()}, fix)
    out2 = net(ex)[0]                                   # graph replay
    assert torch.equal(out2["box3d_lidar"], out["box3d_lidar"]) and torch.equal(out2["scores"], out["scores"])


def test_batch_of_three_equals_single_frames(product):
    from b2second.engine import InferenceEngine
    net = build(product).cuda()
    clouds = [gu.make_cloud(NAME, s, n) for s, n in ((0, 60000), (4, 30000), (1, 120000))]
    single = InferenceEngine(net, batch_size=1, max_points=120000, use_cuda_graph=False)
    ref = []
    for c in clouds:
        single.infer([torch.from_numpy(c).cuda()])
        ref.append((single.detections()[0], int(single.cand_count[0].item())))
    eng = InferenceEngine(net, batch_size=3, max_points=120000, use_cuda_graph=True)
    eng.infer([torch.from_numpy(c).cuda() for c in clouds])
    got = eng.detections()
    assert eng.cand_count.cpu().tolist() == [r[1] for r in ref]
    for g, (r, _) in zip(got, ref):
        assert r["box3d_lidar"].shape[0] > 0
        assert torch.equal(g["box3d_lidar"], r["box3d_lidar"]) and torch.equal(g["scores"], r["scores"])
        assert torch.equal(g["label_preds"], r["label_preds"])


@pytest.mark.parametrize("seed,n,path", CASES, ids=IDS)
def test_module_path_matches_golden(product, seed, n, path):
    fix = np.load(path)
    pts = gu.make_cloud(NAME, seed, n)
    net = build(product).cuda()
    ex = _example(net, pts, int(fix["max_voxels"]), "cuda")
    with torch.no_grad():
        pd = net.network_forward(ex["voxels"], ex["num_points"], ex["coordinates"], 1)
        out = net(ex)[0]
    np.testing.assert_allclose(pd["box_preds"].flatten()[torch.from_numpy(fix["box_sel_idx"]).cuda()].cpu().numpy(),
                               fix["box_sel_val"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(pd["cls_preds"].flatten()[torch.from_numpy(fix["cls_sel_idx"]).cuda()].cpu().numpy(),
                               fix["cls_sel_val"], rtol=0, atol=1e-4)
    gu.assert_detections_close({k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()}, fix)
