"""Kernel-level GPU parity (one C-ABI entry point at a time, against torch fp32 / the CPU oracle):
  b2s_pfn                      PillarFeatureNet (pointpillars.py:203-237) incl. pillars with more points than T
  b2s_to_bev_tc                scatter to the NHWC + halo fp16 hi/lo planes, from fp32 rows and from hi/lo rows
  b2s_decode_filter_strided    sigmoid / threshold / second_box_decode over a packed head record, anchors_mask,
                               candidate-cap overflow
  b2s_nms                      device-resident top-k + NMS + direction / range epilogue, rotated and aligned
  b2s_rbbox_overlap_host, b2s_rotate_iou_eval     rotated overlap matrices (SURVEY.md §8(f)2)
  multi-class NMS branch       fused engine vs the mirror's predict() (voxelnet.py:458-547)
"""
import dataclasses

import numpy as np
import pytest
import torch

import detect_ref as R
import golden_util as gu
from b2second import box_ops, config, models

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


# ------------------------------------------------------------------------------------------------ PFN
@pytest.mark.parametrize("F,T,n_pillars", [(4, 100, 700), (4, 60, 300), (5, 20, 50)])
def test_pfn_matches_torch_module(product, F, T, n_pillars):
    L = product._lib
    lib = L.load()
    g = torch.Generator().manual_seed(F * 100 + T)
    vs, rng = (0.16, 0.16, 4.0), (0.0, -39.68, -3.0, 69.12, 39.68, 1.0)
    pfn = models.PillarFeatureNet(num_input_features=F, num_filters=(64,), voxel_size=vs, pc_range=rng).eval()
    with torch.no_grad():
        lyr = pfn.pfn_layers[0]
        lyr.linear.weight.copy_(torch.randn(lyr.linear.weight.shape, generator=g) * 0.3)
        lyr.norm.weight.copy_(torch.rand(64, generator=g) + 0.5)
        lyr.norm.bias.copy_(torch.randn(64, generator=g) * 0.1)
        lyr.norm.running_mean.copy_(torch.randn(64, generator=g) * 0.1)
        lyr.norm.running_var.copy_(torch.rand(64, generator=g) + 0.5)
    num = torch.randint(1, T + 1, (n_pillars,), generator=g, dtype=torch.int32)
    num[:5] = T                                       # full pillars (no padded slot: max over real points only)
    num[5:10] = 1
    coors = torch.zeros(n_pillars, 4, dtype=torch.int32)
    coors[:, 2] = torch.randint(0, 496, (n_pillars,), generator=g)
    coors[:, 3] = torch.randint(0, 432, (n_pillars,), generator=g)
    voxels = torch.zeros(n_pillars, T, F)
    for i in range(n_pillars):
        n = int(num[i])
        cx = coors[i, 3].item() * vs[0] + rng[0]
        cy = coors[i, 2].item() * vs[1] + rng[1]
        voxels[i, :n, 0] = cx + torch.rand(n, generator=g) * vs[0]
        voxels[i, :n, 1] = cy + torch.rand(n, generator=g) * vs[1]
        voxels[i, :n, 2] = torch.rand(n, generator=g) * 4 - 3
        voxels[i, :n, 3:] = torch.rand(n, F - 3, generator=g)
    with torch.no_grad():
        ref = pfn(voxels, num, coors)
    sc, sh = (lyr.norm.weight / torch.sqrt(lyr.norm.running_var + lyr.norm.eps)), None
    sh = lyr.norm.bias - lyr.norm.running_mean * sc
    # device: points = the voxel slots flattened, slot table = identity (the pre-voxelised entry of the engine)
    pts = voxels.reshape(-1, F).cuda().contiguous()
    slots = torch.arange(n_pillars * T, dtype=torch.int32).view(n_pillars, T).cuda()
    out = torch.zeros(n_pillars, 64, device="cuda")
    n_dev = torch.tensor([n_pillars], dtype=torch.int32, device="cuda")
    w, scd, shd = lyr.linear.weight.detach().cuda().contiguous(), sc.detach().cuda().contiguous(), sh.detach().cuda().contiguous()
    numd, coorsd = num.cuda(), coors.cuda()
    L.check(lib.b2s_pfn(L.ptr(pts), F, L.ptr(slots), L.ptr(numd), L.ptr(coorsd), L.ptr(n_dev), n_pillars, T, L.ptr(w),
                        L.ptr(scd), L.ptr(shd), 64, vs[0], vs[1], pfn.x_offset, pfn.y_offset, L.ptr(out), L.stream()),
            "b2s_pfn")
    torch.cuda.synchronize()
    err = float((out.cpu() - ref).abs().max())
    assert err <= 2e-5 * max(1.0, float(ref.abs().max())), "PFN differs by %g" % err


# ------------------------------------------------------------------------------------------------ to_bev_tc
@pytest.mark.parametrize("D,C", [(2, 64), (1, 64)])
def test_to_bev_tc_scatter(product, D, C):
    from b2second import tc
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(D)
    B, H, W, n = 3, 20, 28, 500
    flat = rng.choice(B * D * H * W, n, replace=False)
    b, r = np.divmod(flat, D * H * W)
    z, r = np.divmod(r, H * W)
    y, x = np.divmod(r, W)
    coors = torch.from_numpy(np.stack([b, z, y, x], 1).astype(np.int32)).cuda()
    feats = torch.from_numpy(rng.standard_normal((n, C)).astype(np.float32)).cuda()
    n_dev = torch.tensor([n - 7], dtype=torch.int32, device="cuda")          # the last 7 rows are beyond the count
    ref = torch.zeros(B, H + 2, W + 2, C * D)
    fc, cc = feats.cpu(), coors.cpu()
    for i in range(n - 7):
        bb, zz, yy, xx = cc[i].tolist()
        ref[bb, yy + 1, xx + 1, torch.arange(C) * D + zz] = fc[i]
    r_hi, r_lo = tc.split_f16(ref)
    o_hi = torch.full((B, H + 2, W + 2, C * D), 7.0, dtype=torch.float16, device="cuda")   # stale contents must vanish
    o_lo = torch.full_like(o_hi, 7.0)
    occ = torch.full((B, H, W), 9, dtype=torch.uint8, device="cuda")
    L.check(lib.b2s_to_bev_tc(L.ptr(feats), None, None, 0, L.ptr(coors), L.ptr(n_dev), n, C, B, D, H, W, L.ptr(o_hi),
                              L.ptr(o_lo), L.ptr(occ), L.stream()), "b2s_to_bev_tc")
    torch.cuda.synchronize()
    assert torch.equal(o_hi.cpu(), r_hi) and torch.equal(o_lo.cpu(), r_lo)
    ref_occ = torch.zeros(B, H, W, dtype=torch.uint8)
    ref_occ[cc[:n - 7, 0].long(), cc[:n - 7, 2].long(), cc[:n - 7, 3].long()] = 1
    assert torch.equal(occ.cpu(), ref_occ)                         # occupancy map for b2s_rpn_bg_plan
    # rows that arrive already split (interleaved [row][hi | lo], as the last sparse layer writes them)
    buf = torch.zeros(n, 2, C, dtype=torch.float16, device="cuda")
    f_hi, f_lo = tc.split_f16(feats)
    buf[:, 0], buf[:, 1] = f_hi, f_lo
    o_hi.fill_(3.0)
    o_lo.fill_(3.0)
    L.check(lib.b2s_to_bev_tc(None, L.ptr(buf[:, 0]), L.ptr(buf[:, 1]), 2 * C, L.ptr(coors), L.ptr(n_dev), n, C, B, D, H, W,
                              L.ptr(o_hi), L.ptr(o_lo), None, L.stream()), "b2s_to_bev_tc")
    torch.cuda.synchronize()
    assert torch.equal(o_hi.cpu(), r_hi) and torch.equal(o_lo.cpu(), r_lo)


# ------------------------------------------------------------------------------------------------ decode + filter
def _decode_reference(box, cls, dirp, anchors, thresh, mask=None):
    """voxelnet.py:413-444,551-576 for one frame with torch ops: returns dict anchor -> (box7, score, label, dir)."""
    dec = box_ops.second_box_decode(box[None], anchors[None])[0]
    scores = torch.sigmoid(cls)
    top, lab = scores.max(-1)
    dl = dirp.max(-1)[1]
    keep = top >= thresh
    if mask is not None:
        keep &= mask.bool()
    return {int(a): (dec[a], float(top[a]), int(lab[a]), int(dl[a])) for a in torch.nonzero(keep).flatten().tolist()}


@pytest.mark.parametrize("ncls,a_loc,use_mask", [(1, 2, False), (4, 8, False), (10, 20, True), (1, 2, True)])
def test_decode_filter_strided_matches_torch(product, ncls, a_loc, use_mask):
    L = product._lib
    lib = L.load()
    g = torch.Generator().manual_seed(ncls * 10 + a_loc)
    B, H, W, code, nb = 2, 12, 10, 7, 2
    A = a_loc * H * W
    n_ch = a_loc * (code + ncls + nb)
    S = max(32, (n_ch + 3) // 4 * 4)
    heads = torch.randn(B, H, W, S, generator=g)
    offs = [0, a_loc * code, a_loc * (code + ncls)]
    heads[..., offs[1]:offs[2]] -= 1.0                                 # ~25 % of the anchors pass
    anchors = torch.cat([torch.rand(A, 3, generator=g) * 40, torch.rand(A, 3, generator=g) * 3 + 0.5,
                         torch.rand(A, 1, generator=g) * 3.14], 1)
    mask = (torch.rand(B, A, generator=g) < 0.5).to(torch.uint8) if use_mask else None
    thresh = 0.3
    cc = A
    hd, an = heads.cuda(), anchors.cuda().contiguous()
    md = mask.cuda() if use_mask else None
    cand_box = torch.zeros(B, cc, code, device="cuda")
    cand_score = torch.zeros(B, cc, device="cuda")
    cand_label = torch.zeros(B, cc, dtype=torch.int32, device="cuda")
    cand_dir = torch.zeros(B, cc, dtype=torch.int32, device="cuda")
    cand_anchor = torch.zeros(B, cc, dtype=torch.int32, device="cuda")
    cand_count = torch.zeros(B, dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    import ctypes

    def run(cap):
        status.zero_()
        L.check(lib.b2s_decode_filter_strided(
            ctypes.c_void_p(hd.data_ptr() + 4 * offs[0]), ctypes.c_void_p(hd.data_ptr() + 4 * offs[1]),
            ctypes.c_void_p(hd.data_ptr() + 4 * offs[2]), H * W * S, H * W * S, H * W * S, 1, S, L.ptr(an), L.ptr(md), B,
            a_loc, H, W, code, ncls, nb, thresh, L.ptr(cand_box), L.ptr(cand_score), L.ptr(cand_label),
            L.ptr(cand_dir), L.ptr(cand_anchor), L.ptr(cand_count), cap, L.ptr(status), L.stream()),
            "b2s_decode_filter_strided")
        torch.cuda.synchronize()
    run(cc)
    assert int(status.item()) == 0
    for b in range(B):
        # packed record -> the reference's [A, *] views: anchor a = (al, h, w), channel al*per + c at pixel (h, w)
        rec = heads[b]                                                   # [H, W, S]

        def view(off, per):
            return rec[..., off:off + a_loc * per].reshape(H, W, a_loc, per).permute(2, 0, 1, 3).reshape(A, per)
        ref = _decode_reference(view(offs[0], code), view(offs[1], ncls), view(offs[2], nb), anchors, thresh,
                                mask[b] if use_mask else None)
        n = int(cand_count[b].item())
        assert n == len(ref) and n > 0
        got_anchor = cand_anchor[b, :n].cpu().tolist()
        assert sorted(got_anchor) == sorted(ref)
        for i, a in enumerate(got_anchor):
            rbox, rscore, rlab, rdir = ref[a]
            assert abs(float(cand_score[b, i]) - rscore) <= 1e-6
            assert int(cand_label[b, i]) == rlab and int(cand_dir[b, i]) == rdir
            assert float((cand_box[b, i].cpu() - rbox).abs().max()) <= 1e-5 * max(1.0, float(rbox.abs().max()))
    # candidate-cap overflow: never writes past the cap, raises the status bit, counts keep counting
    full = cand_count.clone()
    cap = int(full.min().item()) // 2
    run(cap)
    assert int(status.item()) & 8
    assert bool((cand_count >= full).all())


# ------------------------------------------------------------------------------------------------ device NMS
def _nms_reference(oracle, boxes, scores, labels, dirs, anchors_idx, rotated, pre_max, post_max, thr, use_dir, dir_offset,
                   dir_limit, bins, rng6):
    order = np.lexsort((anchors_idx, -scores.astype(np.float64)))          # score desc, anchor asc
    order = order[:pre_max]
    b = boxes[order]
    corners = box_ops.corners_2d_np(b[:, :2], b[:, 3:5], b[:, 6]).astype(np.float32)
    standup = box_ops.standup_np(corners).astype(np.float32)
    ident = np.arange(len(order), dtype=np.int32)
    near = 0
    if rotated:
        siou = box_ops.standup_iou_np(standup, 0.0)
        keep, iou = oracle.utils.rotate_non_max_suppression_cpu(corners, ident, siou, thr, return_iou=True)
        near = int(((iou >= 0) & (np.abs(iou - thr) < 1e-4)).sum())       # pairs whose decision fp32 rounding may flip
    else:
        dets = np.concatenate([standup, scores[order][:, None]], 1).astype(np.float32)
        k = np.zeros(len(order), np.int32)
        nk = oracle.utils.non_max_suppression(dets, k, thr, 0)
        keep = k[:nk].tolist()
    keep = keep[:post_max]
    sel = order[keep]
    out_b = boxes[sel].copy()
    if use_dir:
        period = np.float32(2 * np.pi / bins)
        val = out_b[:, 6] - np.float32(dir_offset)
        dir_rot = val - np.floor(val / period + np.float32(dir_limit)) * period
        out_b[:, 6] = dir_rot + np.float32(dir_offset) + period * dirs[sel].astype(np.float32)
    m = np.ones(len(sel), bool)
    if rng6 is not None:
        m = np.all(out_b[:, :3] >= np.asarray(rng6[:3], np.float32), 1) & np.all(out_b[:, :3] <= np.asarray(rng6[3:], np.float32), 1)
    return out_b[m], scores[sel][m], labels[sel][m], near


@pytest.mark.parametrize("rotated,n,spread,thr,pre_max,post_max", [
    (True, 600, 40.0, 0.01, 1000, 100), (True, 3000, 70.0, 0.1, 1000, 100), (False, 2500, 60.0, 0.5, 1000, 300),
    (False, 5000, 30.0, 0.3, 500, 83), (True, 5, 10.0, 0.5, 1000, 100)])
def test_device_nms_matches_oracle(product, oracle, rotated, n, spread, thr, pre_max, post_max):
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(n + int(thr * 100))
    B, code, cc = 3, 7, 6000
    counts = [n, max(1, n // 3), 0]
    cand_box = np.zeros((B, cc, code), np.float32)
    cand_score = np.zeros((B, cc), np.float32)
    cand_label = np.zeros((B, cc), np.int32)
    cand_dir = np.zeros((B, cc), np.int32)
    cand_anchor = np.zeros((B, cc), np.int32)
    for b, m in enumerate(counts):
        cand_box[b, :m, :2] = rng.uniform(0, spread, (m, 2))
        cand_box[b, :m, 2] = rng.uniform(-3, 1, m)
        cand_box[b, :m, 3:6] = rng.uniform(1.0, 5.0, (m, 3))
        cand_box[b, :m, 6] = rng.uniform(-np.pi, np.pi, m)
        cand_score[b, :m] = rng.choice(np.linspace(0.3, 0.99, 400), m).astype(np.float32)    # plenty of tied scores
        cand_label[b, :m] = rng.integers(0, 4, m)
        cand_dir[b, :m] = rng.integers(0, 2, m)
        cand_anchor[b, :m] = rng.permutation(200000)[:m]
    rng6 = [5.0, 5.0, -2.5, spread - 5.0, spread - 5.0, 0.5]
    d = {k: torch.from_numpy(v).cuda() for k, v in dict(box=cand_box, score=cand_score, label=cand_label, dir=cand_dir,
                                                        anchor=cand_anchor).items()}
    cnt = torch.tensor(counts, dtype=torch.int32, device="cuda")
    ws_bytes = lib.b2s_nms_workspace_bytes(B, cc, pre_max)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    width = post_max * (code + 2) + 1
    recs = {}
    for key, r6 in (("range", L.f6(rng6)), ("none", None)):
        rec = torch.zeros(B, width, device="cuda")
        det_count = torch.zeros(B, dtype=torch.int32, device="cuda")
        L.check(lib.b2s_nms(L.ptr(d["box"]), L.ptr(d["score"]), L.ptr(d["label"]), L.ptr(d["dir"]), L.ptr(d["anchor"]),
                            L.ptr(cnt), B, cc, code, 1 if rotated else 0, pre_max, post_max, thr, 1, 0.78, 0.5, 2, r6,
                            L.ptr(rec), width, L.ptr(det_count), L.ptr(ws), ws_bytes, L.stream()), "b2s_nms")
        torch.cuda.synchronize()
        recs[key] = (rec.cpu(), det_count.cpu())
    rec, det_count = recs["range"]
    assert rec[:, -1].tolist() == [float(c) for c in det_count.tolist()]      # the count rides in the record
    lo, hi = np.asarray(rng6[:3], np.float32), np.asarray(rng6[3:], np.float32)
    for b, m in enumerate(counts):
        rb, rs, rl, near = _nms_reference(oracle, cand_box[b, :m], cand_score[b, :m], cand_label[b, :m], cand_dir[b, :m],
                                          cand_anchor[b, :m], rotated, pre_max, post_max, thr, True, 0.78, 0.5, 2, rng6)
        k = int(det_count[b].item())
        got = rec[b, :-1].view(post_max, code + 2)[:k].numpy()
        # without the range test: the keep list must pass the fp64 certificate, and the range test filters its rows
        k_all = int(recs["none"][1][b])
        rows = recs["none"][0][b, :-1].view(post_max, code + 2)[:k_all].numpy()
        inside = np.all(rows[:, :3] >= lo, 1) & np.all(rows[:, :3] <= hi, 1)
        assert k == int(inside.sum()) and np.array_equal(got, rows[inside])
        order = np.lexsort((cand_anchor[b, :m], -cand_score[b, :m].astype(np.float64)))[:pre_max]
        slot = {cand_box[b, s, :6].tobytes() + cand_score[b, s].tobytes(): s for s in order}
        kept = [slot[r[:6].tobytes() + r[7:8].tobytes()] for r in rows]
        b5 = np.ascontiguousarray(cand_box[b, order][:, [0, 1, 3, 4, 6]])
        c64 = R.bev_corners(b5)
        if rotated:
            ov = R.overlaps(c64, c64)
            iou, bound = np.triu(ov[-1], 1), R.corner_bound(b5, b5, ov)
        else:
            st = R.standup(c64)
            iou, bound = np.triu(R.aligned_iou(st, st, 1.0)[0], 1), R.aligned_bound(st, st, 1.0, R.corner_rounding(b5),
                                                                                     R.corner_rounding(b5))
        err = R.nms_certificate(order, kept, iou, bound, thr, post_max, inclusive=bool(rotated))
        assert err is None, "frame %d: %s" % (b, err)
        if near:                      # a pair within 1e-4 of the IoU threshold: the certificate above decides
            continue
        assert k == len(rs), "frame %d: %d kept, oracle %d" % (b, k, len(rs))
        np.testing.assert_array_equal(got[:, 7], rs)
        np.testing.assert_array_equal(got[:, 8].astype(np.int32), rl)
        np.testing.assert_array_equal(got[:, :6], rb[:, :6])
        np.testing.assert_allclose(got[:, 6], rb[:, 6], rtol=0, atol=1e-5)


# ------------------------------------------------------------------------------------------------ rotated overlaps
def _rboxes(rng, n, spread):
    return np.concatenate([rng.uniform(0, spread, (n, 2)), rng.uniform(1.0, 5.0, (n, 2)),
                           rng.uniform(-np.pi, np.pi, (n, 1))], 1).astype(np.float32)


@pytest.mark.parametrize("N,K,spread", [(200, 150, 25.0), (1, 300, 10.0), (64, 64, 8.0)])
def test_rbbox_iou_and_intersection_match_oracle(product, oracle, N, K, spread):
    rng = np.random.default_rng(N + K)
    a, q = _rboxes(rng, N, spread), _rboxes(rng, K, spread)
    ca = box_ops.corners_2d_np(a[:, :2], a[:, 2:4], a[:, 4]).astype(np.float32)
    cq = box_ops.corners_2d_np(q[:, :2], q[:, 2:4], q[:, 4]).astype(np.float32)
    sa, sq = box_ops.standup_np(ca), box_ops.standup_np(cq)
    # stand-up IoU matrix [N, K] (iou_jit(eps=0), box_np_ops.py:696-725)
    ix = np.clip(np.minimum(sa[:, None, 2], sq[None, :, 2]) - np.maximum(sa[:, None, 0], sq[None, :, 0]), 0, None)
    iy = np.clip(np.minimum(sa[:, None, 3], sq[None, :, 3]) - np.maximum(sa[:, None, 1], sq[None, :, 1]), 0, None)
    inter = ix * iy
    area = lambda s: (s[:, 2] - s[:, 0]) * (s[:, 3] - s[:, 1])
    siou = (inter / (area(sa)[:, None] + area(sq)[None, :] - inter)).astype(np.float32)
    for fn in ("rbbox_iou", "rbbox_intersection"):
        for st in (0.0, 0.2):
            ref = getattr(oracle.utils, fn)(ca, cq, siou, st)
            got = getattr(product.utils, fn)(ca, cq, siou, st)
            assert got.shape == (N, K) and float(np.abs(got - ref).max()) <= 2e-5 * max(1.0, float(ref.max()))
            differ = (got == 0) != (ref == 0)                       # slivers: one side clips to exactly nothing
            assert float(np.abs(got - ref)[differ].max(initial=0.0)) < 1e-4
    assert float(ref.max()) > 0.5                                    # the matrix is not trivially empty
    # device-resident rotate_iou_gpu_eval counterpart: all four criteria against the oracle's pieces
    iou = oracle.utils.rbbox_iou(ca, cq, siou, 0.0)
    inter_a = oracle.utils.rbbox_intersection(ca, cq, siou, 0.0)
    ad, qd = torch.from_numpy(a).cuda(), torch.from_numpy(q).cuda()
    for crit, ref in ((-1, iou), (2, inter_a), (0, inter_a / (a[:, 2] * a[:, 3])[:, None]),
                      (1, inter_a / (q[:, 2] * q[:, 3])[None, :])):
        got = product.utils.rotate_iou_eval(ad, qd, crit).cpu().numpy()
        assert float(np.abs(got - ref).max()) <= 3e-5 * max(1.0, float(ref.max())), crit


# ------------------------------------------------------------------------------------------------ multi-class NMS
@pytest.mark.parametrize("name,agnostic", [("all.fhd", False), ("nuscenes.all.pp.largea", True)])
def test_multiclass_nms_branch_on_the_fused_engine(product, name, agnostic):
    """use_multi_class_nms (voxelnet.py:458-547; off in the BASELINE configs, SURVEY §8(f)3): fused engine (per-class
    candidate lists -> per-class NMS -> class-order concat, all on the device) vs the mirror's predict() on the same
    CUDA backend."""
    from b2second import fastpath
    cfg = dataclasses.replace(config.get_config(name), use_multi_class_nms=True, nms_class_agnostic=agnostic)
    net = models.build_network(cfg, product).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    pts = gu.make_cloud(name, 3, 40000 if "nuscenes" in name else 20000)
    res = net.voxel_generator.generate(pts, cfg.max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    ex = {"anchors": torch.from_numpy(net.anchors()[None]).cuda(), "voxels": torch.from_numpy(res["voxels"]).cuda(),
          "num_points": torch.from_numpy(res["num_points_per_voxel"]).cuda(), "coordinates": torch.from_numpy(coords).cuda()}
    with torch.no_grad():
        ref = net(ex)[0]
    fastpath.accelerate(net, max_points=max(1000, pts.shape[0]))
    got = net(ex)[0]
    eng = next(iter(net.b2s_fastpath.engines.values()))
    assert eng.mc and ref["box3d_lidar"].shape[0] > 0 and len(set(ref["label_preds"].tolist())) > 1
    assert got["box3d_lidar"].shape == ref["box3d_lidar"].shape
    # class order is fixed; inside a class detections are in descending score order
    assert torch.equal(got["label_preds"], ref["label_preds"])
    for c in set(ref["label_preds"].tolist()):
        m = (ref["label_preds"] == c).cpu().numpy()
        fix = {k: ref[k].cpu().numpy()[m] for k in ("box3d_lidar", "scores", "label_preds")}
        gu.assert_detections_close({k: got[k].cpu().numpy()[m] for k in fix}, fix)


# ------------------------------------------------------------------------------------------------ RPN background tiles
def test_rpn_background_plan_matches_numpy_and_background_skip_is_bit_identical(product, monkeypatch):
    """b2s_rpn_bg_plan against its numpy restatement (tests/test_host_rpn_plan.py), and the fused engine with the
    background-tile skip on vs off (tiles copied from the layer's empty-frame response by the conv kernel's epilogue
    warps): bit-identical head tensors, candidates and detections."""
    import test_host_rpn_plan as hp
    from b2second import tc
    from b2second.engine import InferenceEngine
    L = product._lib
    lib = L.load()
    rng = np.random.default_rng(0)
    B, H, W, nl = 3, 200, 176, 6
    occ = (rng.random((B, H, W)) < 0.002).astype(np.uint8)
    occ[1] = 0                                         # an empty frame: everything is background in layer 1
    occ[2, 90:130, 60:120] = 1
    th, tw = -(-H // 16), -(-W // 16)
    nt = B * th * tw
    d_occ = torch.from_numpy(occ).cuda()
    scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(nl, nt, dtype=torch.int32, device="cuda")
    work = torch.full((nl, nt), -1, dtype=torch.int32, device="cuda")
    bg = torch.full((nl, nt), -1, dtype=torch.int32, device="cuda")
    counts = torch.zeros(nl, 2, dtype=torch.int32, device="cuda")
    L.check(lib.b2s_rpn_bg_plan(L.ptr(d_occ), B, H, W, nl, L.ptr(scratch), L.ptr(flags), L.ptr(work), L.ptr(bg),
                                L.ptr(counts), L.stream()), "b2s_rpn_bg_plan")
    torch.cuda.synchronize()
    ref = hp.bg_plan_numpy(occ, nl)
    for l in range(nl):
        f = ref[l].reshape(-1)
        assert np.array_equal(flags[l].cpu().numpy(), f)
        nw = int(counts[l, 0])
        assert nw == int(f.sum()) and int(counts[l, 1]) == nt - nw
        assert np.array_equal(work[l, :nw].cpu().numpy(), np.nonzero(f)[0])
        assert np.array_equal(bg[l, :nt - nw].cpu().numpy(), np.nonzero(f == 0)[0])
    assert int(counts[0, 1]) > nt // 3                 # layer 1 really skips a lot here
    # engine on / off
    name = "car.fhd"
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    clouds = [torch.from_numpy(gu.make_cloud(name, s, n)).cuda() for s, n in ((0, 20000), (1, 29000))]
    res = {}
    for bg_on in (True, False):
        if not bg_on:                                        # the reference: no layer tracks background tiles
            monkeypatch.setattr(tc, "background_layers", lambda plan: [])
        eng = InferenceEngine(net, batch_size=2, max_points=30000, use_cuda_graph=True)
        assert bool(eng.bg_idx) == bg_on
        eng.infer(clouds)
        res[bg_on] = (eng.detections(), eng.tc_heads.clone(), eng.cand_count.clone(),
                      eng.bg_counts.clone() if eng.bg_idx else None, getattr(eng, "bg_tiles", 0))
    on, off = res[True], res[False]
    assert torch.equal(on[2], off[2])
    skipped = on[3][:, 1].float() / on[4]
    assert float(skipped.min()) > 0.3, skipped              # border tiles without data are background too
    assert torch.equal(on[1], off[1])                        # the copied field is what the kernel computes: bit-identical
    for a, b in zip(on[0], off[0]):
        assert a["box3d_lidar"].shape == b["box3d_lidar"].shape and a["box3d_lidar"].shape[0] > 0
        assert torch.equal(a["box3d_lidar"], b["box3d_lidar"]) and torch.equal(a["scores"], b["scores"])
