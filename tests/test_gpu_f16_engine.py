"""The fused engine in the half-precision mode (precision="f16") on the H100:
  sparse      every sparse layer of the f16 engine (single-plane rows, the first layer's b2s_split_f16_ex, the planned
              launches with the rulebooks' perm and tile masks) against tests/tc_ref.sparse_ref on the engine's own
              input rows of the layer, with the per-element f16 bound and the BatchNorm fold term
  BEV         the f16 BEV plane bit-equal to the scatter of the last layer's rows (PointPillars: of fp16(PFN rows))
              into a zero map, bev_occ exactly the occupied pixels
  layers      every RPN op of the f16 engine against the float64 module layer it implements (tests/engine_ref.py),
              fed the engine's own output of the op before it, with the per-element f16 bound of
              tests/test_gpu_f16_fp64.py, the BatchNorm fold term and, for the ops k_conv_tc runs, its chain term; the
              crop op exact; the fused tail against the float64 deblock -> heads with the deblock's bound carried
              through the heads' weights; single-head and multi-head networks
  background  the shipped engine (background strips on) writes, bit for bit, the head records and BEV plane of the
              same engine without background strips
  serving     stream() equals net(example) bit for bit; refresh() after load_state_dict equals a newly built f16
              engine bit for bit; CUDA graphs on and off give identical results; output="host" works; the result dicts
              keep their float32 / int64 dtypes; the f16 engine holds no lo planes
  detections  on seeded car.fhd, xyres_16 and multi-head batches, the f16 engine's candidates against the float64
              decode of its own head maps (sigmoid and decode bounds of tests/detect_ref.py) and its NMS output against
              the keep-list certificate (detect_ref.nms_certificate), as tests/test_gpu_detect_fp64.py checks the
              detection kernels; the engine's detection records are those rows with the class labels
  capture     the CUDA graph is captured with Python's cyclic garbage collector off
  agreement   on seeded car.fhd and xyres_16 batches, the share of the fp32 mode's detections matched by an f16
              detection with the same label and BEV IoU >= 0.9 (printed, and asserted above a floor)
"""
import json
import os

import numpy as np
import pytest
import torch

import detect_ref as DR
import engine_ref as E
import golden_util as gu
import tc_ref
from b2second import config, fastpath, models

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11
FIELDS = ("box3d_lidar", "scores", "label_preds")
# the share of fp32-mode detections an f16 detection matches (label, BEV IoU >= 0.9) must stay above this floor; measured
# on an H100 80GB HBM3: car.fhd 0.984 (2994 of 3043), pointpillars.car.xyres_16 0.995 (9113 of 9160)
MATCH_FLOOR = 0.95


@pytest.fixture(autouse=True)
def _fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _net(product, name, seed=0):
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=seed)
    return net.cuda()


def _example(net, name, B, seed, points=20000):
    clouds = [torch.from_numpy(gu.make_cloud(name, seed + i, points)).cuda() for i in range(B)]
    return {"points": clouds, "anchors": torch.from_numpy(net.anchors()[None]).cuda(),
            "metadata": [{"token": "s%d" % (seed + i)} for i in range(B)]}


def _assert_same(got, want, what):
    """the result dicts equal bit for bit; -> the number of detections compared"""
    assert len(got) == len(want), what
    n = 0
    for g, w in zip(got, want):
        for k in FIELDS:
            assert g[k].dtype == w[k].dtype and torch.equal(g[k].cpu(), w[k].cpu()), "%s: %s" % (what, k)
        n += w["scores"].shape[0]
    return n


def _heads(eng):
    """the engine's fp32 head record maps (one per head segment)"""
    return [eng.tc_heads] if eng.segments is None else [eng.tc_seg_heads[g["name"]] for g in eng.segments]


def _assert_same_heads(a, b, what):
    """two engines' head records of their last batch equal bit for bit (they are written whether or not a frame has a
    detection above the score threshold)"""
    for x, y in zip(_heads(a), _heads(b)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), what


# ---- layers -----------------------------------------------------------------------------------------------------
class _Tap:
    """the engine's library with every f16 RPN launch followed by a copy of what it wrote"""
    HOOKED = ("b2s_conv2d_tc_ex3", "b2s_crop_nhwc_ex", "b2s_rpn_tail_tc_ex2")

    def __init__(self, eng):
        self.lib, self.eng, self.i, self.after = eng.lib, eng, 0, []

    def __getattr__(self, name):
        f = getattr(self.lib, name)
        if name not in self.HOOKED:
            return f

        def call(*args):
            ret = f(*args)
            eng = self.eng
            if name == "b2s_rpn_tail_tc_ex2":
                self.after.append(eng.tc_heads.clone())
            else:
                self.after.append(eng.tc_bufs[eng.tc_plan[self.i]["dst"]][0].clone())
            self.i += 1
            return ret
        return call


def _f16_extra(ref, ws, f16_out):
    """the f16 terms of the bound beyond tc_ref's ALPHA unit (tests/test_gpu_f16_fp64.py)"""
    rounding = ref.s * ((2 * U16 + U16 * U16) * ref.S1 + 2.0 ** -25 * (1 + U16) * (ref.Sw + ref.Sa / ws) + 2.0 ** -40)
    out = (U16 if f16_out else 2.0 ** -22) * ref.pre.abs() + 2.0 ** -25
    return rounding + out


def _check(got, ref, extra, what):
    err = (got.double() - ref.y).abs()
    bound = tc_ref.ALPHA * tc_ref._terms(ref, 1.0)[0] + extra
    ratio = float((err / bound).max()) if err.numel() else 0.0
    assert ratio <= 1.0, "%s: |y - y64| reaches %.3g x the f16 bound" % (what, ratio)
    return ratio


def _check_sparse(net, eng):
    """every sparse layer against float64 on the rows the engine fed it (layer 0: the mean VFE's fp32 rows, which the
    engine splits to one fp16 plane; then each layer's own fp16 output rows)"""
    from b2second import tc
    from test_gpu_engine_fp64 import sparse_modules
    mods = sparse_modules(net)
    assert len(mods) == len(eng.layers)
    feats = eng.vfe_out
    worst = 0.0
    for (conv, bn), lyr in zip(mods, eng.layers):
        assert lyr["tc"] and lyr["out_lo"] is None and lyr["out_stride"] == lyr["cout"]
        lin, lout = lyr["in_level"], lyr["out_level"]
        n_in, n_out = int(lin.n_dev[0]), int(lout.n_dev[0])
        assert n_out > 0
        x = feats[:n_in, :lyr["cin"]].double()
        K = lyr["K"]
        w = conv.weight.detach().float().reshape(K, lyr["cin"], lyr["cout"])
        ws = tc.pow2_scale(tc.pack_sparse_weights(w))
        s64, sh64 = E.fold64(bn)
        ds, dsh = E.fold_error(bn)
        ref = tc_ref.sparse_ref(x, w, lyr["rb"]["nbr"][:n_out], s64, sh64, lyr["relu"])
        got = lyr["out_hi"][:n_out].double()
        worst = max(worst, _check(got, ref, ds * ref.S1 + dsh + _f16_extra(ref, ws, True),
                                  "sparse layer %d" % lyr["index"]))
        feats = got
    return worst


def _check_bev(eng):
    """the f16 BEV plane == the scatter of the rows the RPN reads, into a zero map; bev_occ == the occupied pixels"""
    from b2second import tc
    fl = eng.final_level
    D, H, W = fl.shape
    n = int(fl.n_dev[0])
    co = fl.coors[:n].long()
    rows = tc.split_f16(eng.pfn_out[:n])[0] if eng.is_pillars else eng.layers[-1]["out_hi"][:n]
    assert eng.tc_bev[1] is None
    occ = torch.zeros(eng.B, H, W, dtype=torch.uint8, device="cuda")
    occ[co[:, 0], co[:, 2], co[:, 3]] = 1
    assert torch.equal(eng.bev_occ, occ), "BEV: bev_occ is not this batch's occupied pixels"
    ch = torch.arange(rows.shape[1], device="cuda") * D
    want = torch.zeros_like(eng.tc_bev[0])
    want[co[:, 0, None], co[:, 2, None] + 1, co[:, 3, None] + 1, ch[None, :] + co[:, 1, None]] = rows
    assert torch.equal(eng.tc_bev[0].view(torch.int16), want.view(torch.int16)), "BEV plane differs from the scatter"


@pytest.mark.parametrize("name", ["car.fhd", "car.lite", "pointpillars.car.xyres_16", "all.fhd",
                                  "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"])
def test_layers_against_fp64(product, name, monkeypatch):
    from b2second import tc
    from b2second.engine import InferenceEngine
    net = _net(product, name)
    B = 2
    monkeypatch.setattr(tc, "background_layers", lambda plan: [])
    points = 15000 if "nuscenes" not in name else 60000
    eng = InferenceEngine(net, batch_size=B, max_points=points + 1000, precision="f16")
    monkeypatch.undo()
    assert eng.products == 1 and not eng.bg_idx
    ex = _example(net, name, B, 11, points=points)
    eng.set_anchors(ex["anchors"])
    eng.infer(ex["points"])
    torch.cuda.synchronize()
    assert eng.check_status() & ~1 == 0
    if not eng.is_pillars:
        print("%s: worst error / f16 bound over the sparse layers %.3g" % (name, _check_sparse(net, eng)))
    _check_bev(eng)
    tap = _Tap(eng)
    eng.lib = tap
    try:
        with torch.no_grad():
            eng._launch("points")
        torch.cuda.synchronize()
    finally:
        eng.lib = tap.lib
    s = eng.spec
    refs = E.rpn_refs(s.rpn, None if getattr(s, "heads", None) is None else dict(s.heads))
    plan = eng.tc_prog
    E.assert_matches_plan(refs, plan)
    latest = {"in": eng.tc_bev[0].clone()}
    n_ops = len(eng.tc_plan) - (2 if eng.tc_tail_fused else 0)
    worst = 0.0
    for i, (r, op) in enumerate(zip(refs[:n_ops], eng.tc_plan[:n_ops])):
        src = latest[op["src"]]
        out = tap.after[i]
        if op["kind"] == "crop":
            c = op["crop"]
            want = torch.zeros_like(out)
            want[:, 1:-1, 1:-1] = src[:, 1 + c:src.shape[1] - 1 - c, 1 + c:src.shape[2] - 1 - c]
            assert torch.equal(out.view(torch.int16), want.view(torch.int16)), "%s: crop" % name
        else:
            x = src[:, 1:-1, 1:-1].double()
            ref, fold = E.op_ref(x, r, chains=not op["v2"])
            got = E.dst_view(out, op)
            worst = max(worst, _check(got, ref, fold + _f16_extra(ref, op["w_scale"], op["planes"] == 2),
                                      "%s op %d (%s)" % (name, i, op["kind"])))
        latest[op["dst"]] = out
    if eng.tc_tail_fused:
        d, h = eng.tc_plan[-2], eng.tc_plan[-1]
        rd, rh = refs[-2], refs[-1]
        x = latest[d["src"]][:, 1:-1, 1:-1].double()
        ref1, fold1 = E.op_ref(x, rd)
        delta = tc_ref.ALPHA * tc_ref._terms(ref1, 1.0)[0] + fold1 + _f16_extra(ref1, d["w_scale"], True)
        ref2, fold2 = E.op_ref(ref1.y, rh)
        carried, _ = E.op_ref(delta, dict(rh, w=rh["w"].abs(), bn=None, bias=None, relu=False))
        got = tap.after[-1][..., :h["cout"]]
        worst = max(worst, _check(got, ref2, fold2 + carried.y + _f16_extra(ref2, h["w_scale"], False),
                                  "%s fused tail" % name))
    print("%s: worst error / f16 bound over the RPN ops %.3g" % (name, worst))


@pytest.mark.parametrize("name", ["car.fhd", "car.lite"])
def test_background_strips_write_what_the_computed_run_writes(product, name, monkeypatch):
    """the shipped f16 engine (background strips, fused tail background tiles) == the same engine computing every
    strip, on a batch with an empty frame, a one-point frame and a frame at the map border"""
    from b2second import tc
    from b2second.engine import InferenceEngine
    net = _net(product, name)
    cfg = config.get_config(name)
    B = 4
    clouds = [gu.make_cloud(name, 3, 15000), np.zeros((0, 4), np.float32), gu.border_cloud(cfg, 4, 7),
              gu.make_cloud(name, 4, 3000)]
    pts = [torch.from_numpy(c).cuda() for c in clouds]
    shipped = InferenceEngine(net, batch_size=B, max_points=20000, precision="f16")
    assert shipped.bg_idx
    monkeypatch.setattr(tc, "background_layers", lambda plan: [])
    dense = InferenceEngine(net, batch_size=B, max_points=20000, precision="f16")
    monkeypatch.undo()
    anchors = torch.from_numpy(net.anchors()[None]).cuda()
    for eng in (shipped, dense):
        eng.set_anchors(anchors)
        for _ in range(2):                  # the second step clears what the first left
            eng.infer(pts)
        torch.cuda.synchronize()
    assert torch.equal(shipped.tc_heads.view(torch.int32), dense.tc_heads.view(torch.int32))
    assert torch.equal(shipped.tc_bev[0].view(torch.int16), dense.tc_bev[0].view(torch.int16))
    assert torch.equal(shipped.det_record, dense.det_record)


# ---- serving --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"])
def test_stream_graphs_and_output_host(product, name):
    B = 3
    nets = {}
    for graphs in (True, False):
        nets[graphs] = fastpath.accelerate(_net(product, name), max_points=40000, precision="f16",
                                           use_cuda_graph=graphs)
    net = nets[True]
    exs = [_example(net, name, B, 10 * k) for k in range(4)]
    calls = [net(ex) for ex in exs]
    eng = net.b2s_fastpath.engines[B]
    assert eng.precision == "f16" and eng.products == 1
    planes = eng.fp16_plane_bytes()
    assert planes["lo"] == 0 and planes["hi"] > 0
    for r in calls[0]:
        assert r["box3d_lidar"].dtype == torch.float32 and r["scores"].dtype == torch.float32
        assert r["label_preds"].dtype == torch.int64
    streamed = list(net.b2s_fastpath.stream(exs))
    n = 0
    for k, (g, w) in enumerate(zip(streamed, calls)):
        n += _assert_same(g, w, "%s stream batch %d" % (name, k))
    for k, ex in enumerate(exs):
        _assert_same(nets[False](ex), calls[k], "%s graphs off, batch %d" % (name, k))
        net(ex)
        _assert_same_heads(eng, nets[False].b2s_fastpath.engines[B], "%s graphs off, heads of batch %d" % (name, k))
    host = fastpath.accelerate(_net(product, name), max_points=40000, precision="f16", output="host")
    for k, ex in enumerate(exs[:2]):
        got = host(ex)
        assert got[0]["scores"].device.type == "cpu"
        _assert_same(got, calls[k], "%s output host, batch %d" % (name, k))
    assert n > 0 or "mhead" in name, "no detections: the comparison would prove little"


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.mhead"])
def test_refresh_after_load_state_dict(product, name):
    B = 2
    net = fastpath.accelerate(_net(product, name, seed=0), max_points=40000, precision="f16")
    ex = _example(net, name, B, 5)
    net(ex)
    eng = net.b2s_fastpath.engines[B]
    before = [h.clone() for h in _heads(eng)]
    state = _net(product, name, seed=1).state_dict()
    net.load_state_dict(state)
    got = net(ex)
    assert net.b2s_fastpath.refreshes == 1 and net.b2s_fastpath.engines[B] is eng
    fresh = fastpath.accelerate(_net(product, name, seed=1), max_points=40000, precision="f16")
    want = fresh(ex)
    _assert_same(got, want, "%s refresh" % name)
    _assert_same_heads(eng, fresh.b2s_fastpath.engines[B], "%s refresh, heads" % name)
    assert not all(torch.equal(a, b) for a, b in zip(before, _heads(eng))), \
        "the new weights changed nothing: the check would prove nothing"


# ---- detections -------------------------------------------------------------------------------------------------
def _head_maps(eng):
    """[(record map [B, H, W, S], channel offsets of box / cls / dir, a_loc, H, W, global anchor base)] of the engine's
    heads in anchor order"""
    if eng.segments is None:
        return [(eng.tc_heads, eng.tc_prog["heads"]["offsets"], eng.a_loc, eng.fH, eng.fW, 0)]
    return [(eng.tc_seg_heads[g["name"]], pg["offsets"], g["a_loc"], g["H"], g["W"], g["base"])
            for g, pg in zip(eng.segments, eng.tc_prog["segments"])]


def decode_ref(maps, anchors, b, code, ncls, nb, use_dir):
    """float64 reference of frame b's decode + score filter from packed head records, in the kernels' anchor order
    (anchor = base + a * H * W + pixel; record channel of anchor a: offset + a * channels + c): the per-class
    sigmoid and its bound, the decoded box and its bound, the direction bin (tests/test_gpu_detect_fp64.py's
    _decode_expect on the same values)"""
    t, x, d = [], [], []
    A = 0
    for rec, offs, a_loc, H, W, base in maps:
        assert base == A
        r = np.asarray(rec[b], np.float32).reshape(H * W, -1)

        def take(off, ch):
            return r[:, off:off + a_loc * ch].reshape(H * W, a_loc, ch).transpose(1, 0, 2).reshape(a_loc * H * W, ch)
        t.append(take(offs[0], code))
        x.append(take(offs[1], ncls))
        d.append(take(offs[2], nb) if use_dir else np.zeros((a_loc * H * W, 1), np.float32))
        A += a_loc * H * W
    t, x, d = np.concatenate(t), np.concatenate(x), np.concatenate(d)
    assert A == anchors.shape[0]
    s64, sb = DR.sigmoid64(x), DR.sigmoid_bound(x)
    o = DR.decode64(t, anchors)
    return dict(s64=s64, sb=sb, top=s64.max(1), o=o, ob=DR.decode_bound(t, anchors, o), dir=d.argmax(1), mask=None)


@pytest.mark.parametrize("name,points", [("car.fhd", 29000), ("pointpillars.car.xyres_16", 29000),
                                         ("nuscenes.all.pp.mhead", 300000)])
def test_detections_certificate(product, name, points, monkeypatch):
    import gc

    import bench
    from b2second.engine import InferenceEngine
    from test_gpu_detect_fp64 import _check_candidates, _check_frames, _Nms
    net = _net(product, name)
    B = 2
    eng = InferenceEngine(net, batch_size=B, max_points=points + 1000, precision="f16")
    s = eng.spec
    assert not eng.mc and s.num_direction_bins == 2
    # the graph is captured with the cyclic collector off
    seen, launch = [], eng._launch

    def spy(*a, **k):
        seen.append((torch.cuda.is_current_stream_capturing(), gc.isenabled()))
        return launch(*a, **k)
    monkeypatch.setattr(eng, "_launch", spy)
    eng.set_anchors(torch.from_numpy(net.anchors()[None]).cuda())
    eng.infer([torch.from_numpy(c).cuda() for c in bench.make_clouds(name, B, points, seed0=40)])
    torch.cuda.synchronize()
    eng.check_status()
    assert any(c for c, _ in seen) and all(not on for c, on in seen if c) and gc.isenabled()
    # decode + score filter of the engine's own head maps
    maps = [(m[0].cpu().numpy(),) + tuple(m[1:]) for m in _head_maps(eng)]
    anchors = eng.anchors.cpu().numpy()
    thr = float(np.float32(eng.score_thresh))
    cap, code = eng.cand_cap, eng.code
    cand = {k: getattr(eng, "cand_" + k).cpu().numpy() for k in ("box", "score", "label", "dir", "anchor", "count")}
    counts = [int(c) for c in cand["count"]]
    assert all(c <= cap for c in counts)
    for b in range(B):
        n = counts[b]
        ref = decode_ref(maps, anchors, b, code, s.num_class, s.num_direction_bins, s.use_direction_classifier)
        _check_candidates(ref, thr, cand["anchor"][b, :n], cand["score"][b, :n], cand["box"][b, :n],
                          cand["label"][b, :n], cand["dir"][b, :n], anchors.shape[0])
    # NMS of those candidates: rows naming their candidate slot, against the keep-list certificate
    slots = np.tile(np.arange(cap, dtype=np.int32), (B, 1))
    arrays = (cand["box"], cand["score"], slots, cand["dir"], cand["anchor"])
    nms = _Nms(product, *arrays, counts, cap)
    rng6 = list(s.post_center_range) if len(s.post_center_range) == 6 else None
    _check_frames(nms, arrays, counts, cap, 1 if s.use_rotate_nms else 0, eng.pre_max, eng.post_max, eng.iou_thresh,
                  1 if s.use_direction_classifier else 0, float(s.direction_offset), float(s.direction_limit_offset),
                  rng6=rng6)
    # the engine's records: the same rows, with the candidates' class labels
    rec, cnt = (t.cpu().numpy() for t in nms.last)
    mine = eng.det_record.cpu().numpy()
    S = code + 2
    kept = 0
    for b in range(B):
        k = int(cnt[b])
        assert mine[b, -1] == float(k)
        rows, got = (r[b, :eng.post_max * S].reshape(eng.post_max, S)[:k] for r in (rec, mine))
        np.testing.assert_array_equal(got[:, :code + 1], rows[:, :code + 1])
        np.testing.assert_array_equal(got[:, code + 1], cand["label"][b, rows[:, code + 1].astype(np.int64)])
        kept += k
    assert kept > 0, "no detections: the certificate would prove little"
    print("%s: %s candidates, %d detections certified" % (name, counts, kept))


# ---- agreement with the fp32 mode -----------------------------------------------------------------------------------
def _bev_iou(a, b):
    """BEV IoU matrix of float32 boxes a [N, >=7], b [K, >=7] (x, y, w, l, r at columns 0, 1, 3, 4, 6)"""
    ca = DR.bev_corners(a[:, [0, 1, 3, 4, 6]])
    cb = DR.bev_corners(b[:, [0, 1, 3, 4, 6]])
    return DR.overlaps(ca, cb)[-1]


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16"])
def test_detections_agree_with_the_fp32_mode(product, name, out_dir):
    import bench
    B = 8
    n32 = fastpath.accelerate(_net(product, name), max_points=30000)
    n16 = fastpath.accelerate(_net(product, name), max_points=30000, precision="f16")
    anchors = torch.from_numpy(n32.anchors()[None]).cuda()
    matched = total = n16_total = 0
    for k in range(4):
        clouds = [torch.from_numpy(c).cuda() for c in bench.make_clouds(name, B, 29000, seed0=100 + B * k)]
        ex = {"points": clouds, "anchors": anchors}
        for r32, r16 in zip(n32(ex), n16(ex)):
            b32, b16 = r32["box3d_lidar"].cpu().numpy(), r16["box3d_lidar"].cpu().numpy()
            l32, l16 = r32["label_preds"].cpu().numpy(), r16["label_preds"].cpu().numpy()
            total += b32.shape[0]
            n16_total += b16.shape[0]
            if b32.shape[0] == 0 or b16.shape[0] == 0:
                continue
            iou = _bev_iou(b32, b16)
            ok = (iou >= 0.9) & (l32[:, None] == l16[None, :])
            matched += int(ok.any(1).sum())
    assert total > 0
    share = matched / total
    line = {"config": name, "fp32_detections": total, "f16_detections": n16_total, "matched": matched,
            "share": share}
    print("f16 agreement:", json.dumps(line))
    with open(os.path.join(out_dir, "f16_agreement_%s.json" % name), "w") as f:
        json.dump(line, f)
    assert share >= MATCH_FLOOR, line
