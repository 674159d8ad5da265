"""The fused inference engine (``InferenceEngine``, as ``fastpath.accelerate`` and bench.py build it: rpn_impl "tc",
sparse_impl "tc", CUDA graph on, synthetic weights seed 0) checked stage by stage against float64 over a sequence of
three batches at the benchmark's batch sizes:
  batch 0  the benchmark's first batch (bench.make_clouds(name, 2B, points)[:B])
  batch 1  its second batch with an empty frame, a one-point frame and a frame whose points lie on the first and last
           row and column of the BEV map (computed strips beside background strips at the frame border)
  batch 2  a sparse batch (3000 points per frame: most BEV pixels of batch 1 must be cleared), the same three special
           frames at its first, middle and last position.
Every reference takes the engine's own input to the stage, so each bound is layer-local:
  voxels      per frame bit-equal to the CPU oracle's VoxelGeneratorV2; frame bases and num_voxels consistent
  rulebooks   each level's output coordinates (order included) and each table equal to the oracle's get_indice_pairs on
              the engine's input coordinates of the level (frames 0, 1, the special frames and B - 1)
  sparse      every live row of every layer against tc_ref.sparse_ref, weights and BatchNorm1d from the torch modules
              (folded in float64, plus the fold term of tests/engine_ref.py); the mean VFE / the PFN against fp32_ref
  BEV         the hi/lo planes bit-equal to the scatter of the last layer's rows into a zero map, bev_occ exactly the
              occupied pixels of this batch
  RPN ops     every op of tc_prog["ops"] of an engine without background strips against the float64 module layer it
              implements (engine_ref.rpn_refs) applied to the op's source buffer, with the tc_ref bound, the fold
              term and, for the ops k_conv_tc runs, its accumulation-chain term (engine_ref docstring; a zeroed lo
              plane of such an op is still rejected); the crop op exact
  fused tail  the head records against the float64 deblock -> heads, with the two-layer bound of check_fused_tail
  background  the shipped engine (background strips on): heads and BEV planes bit-equal to the run without them, and for
              every tracked layer every pixel the next layer's computed strips (or the fused tail's computed tiles)
              read bit-equal
and the engine's status is 0 after every step at B = 32.  At 300 k points the NuScenes frames hold more than max_voxels
pillars (the benchmark's clouds do), and there the status must be exactly the voxel-overflow bit: the engine drops the
extra pillars as the oracle's voxel generator does, and the voxel check compares the capped voxels bit for bit.
test_mutations_are_rejected shows the checks reject a BatchNorm fold
without eps, one head channel's shift dropped, one background strip of one frame copied from the previous batch, and
the lo plane of one op's output zeroed.

The per-op buffers of the RPN alternate (layer l + 2 overwrites layer l), so after each graph replay the same launch
sequence is run once more eagerly with every RPN launch followed by a copy of its destination; the final buffers of
that run must equal the replay's bit for bit, so the copies are what the graph computed.

Wall time on one H100 SXM (80 GB): pointpillars.car.xyres_16 18 s, all.fhd 15 s, car.fhd 15 s, the mutations 14 s,
car.lite 9 s, the NuScenes networks 7 s each; the whole file about 95 s.
"""
import numpy as np
import pytest
import torch

import engine_ref as E
import fp32_ref
import golden_util as gu
import tc_ref

pytestmark = pytest.mark.gpu

# (config, frames per batch, points per cloud): bench.py's batches
CONFIGS = [("car.fhd", 32, 29000), ("car.lite", 32, 29000), ("pointpillars.car.xyres_16", 32, 29000),
           ("all.fhd", 32, 29000), ("nuscenes.all.pp.largea", 4, 300000), ("nuscenes.all.pp.mhead", 4, 300000)]
SPARSE_POINTS = 3000
CHUNK = 4                    # frames per float64 reference chunk


@pytest.fixture(autouse=True)
def _fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---- inputs ------------------------------------------------------------------------------------------------------
border_cloud = gu.border_cloud


def batches(name, cfg, B, points, F):
    import bench
    bench_clouds = bench.make_clouds(name, 2 * B, points)
    sparse = [gu.make_cloud(name, 1000 + s, SPARSE_POINTS) for s in range(B)]
    r = np.asarray(cfg.point_cloud_range, np.float32)
    one = np.zeros((1, F), np.float32)
    one[0, :3] = 0.5 * (r[:3] + r[3:])
    specials = [np.zeros((0, F), np.float32), one, border_cloud(cfg, F, 7)]
    b1 = list(bench_clouds[B:])
    pos1 = [min(3, B - 3) + i for i in range(3)]                  # empty, one point, border: three neighbours
    pos2 = [0, B // 2, B - 1]
    for p, c in zip(pos1, specials):
        b1[p] = c
    for p, c in zip(pos2, specials):
        sparse[p] = c
    return [(list(bench_clouds[:B]), []), (b1, pos1), (sparse, pos2)]


def build_engine(product, name, B, points, skip=True, monkeypatch=None):
    from b2second import config, models, tc
    from b2second.engine import InferenceEngine
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    net = net.cuda()
    if not skip:
        monkeypatch.setattr(tc, "background_layers", lambda plan: [])
    eng = InferenceEngine(net, batch_size=B, max_points=points + 1000, use_cuda_graph=True, rpn_impl="tc",
                          sparse_impl="tc")
    if not skip:
        monkeypatch.undo()
        assert not eng.bg_idx
    return net, eng


# ---- the eager copy of a step --------------------------------------------------------------------------------------
class _Tap:
    """the engine's library with every RPN launch followed by a copy of what it wrote"""
    HOOKED = ("b2s_conv2d_tc_ex2", "b2s_crop_nhwc", "b2s_rpn_tail_tc_ex")

    def __init__(self, eng):
        self.lib, self.eng, self.i, self.after = eng.lib, eng, 0, []

    def __getattr__(self, name):
        f = getattr(self.lib, name)
        if name not in self.HOOKED:
            return f

        def call(*args):
            ret = f(*args)
            eng = self.eng
            if name == "b2s_rpn_tail_tc_ex":
                self.after.append((eng.tc_heads.clone(), None))
            else:
                dst = eng.tc_bufs[eng.tc_plan[self.i]["dst"]]
                self.after.append(tuple(None if t is None else t.clone() for t in dst))
            self.i += 1
            return ret
        return call


def step(eng, clouds, status):
    """one graph replay, then the same launches eagerly with copies -> per-op destination copies"""
    eng.infer([torch.from_numpy(c).cuda() for c in clouds])
    torch.cuda.synchronize()
    assert eng.check_status() == status
    final = {k: tuple(None if t is None else t.clone() for t in v) for k, v in eng.tc_bufs.items()}
    tap = _Tap(eng)
    eng.lib = tap
    try:
        with torch.no_grad():
            eng._launch("points")
    finally:
        eng.lib = tap.lib
    torch.cuda.synchronize()
    assert eng.check_status() == status
    for k, v in final.items():
        for a, b in zip(v, eng.tc_bufs[k]):
            if a is not None:
                assert torch.equal(bits(a), bits(b)), "the eager launch sequence differs from the graph in " + k
    return tap.after


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


# ---- 1. voxels -----------------------------------------------------------------------------------------------------
def expected_status(oracle, cfg, eng, clouds):
    """0, or B2S_STATUS_VOXEL_OVERFLOW (1) when some frame has more voxels than max_voxels: the engine then drops the
    extra voxels as the reference's voxel generator does"""
    gen = oracle.utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range, eng.T, eng.max_voxels + 1)
    return int(any(gen.generate(c, eng.max_voxels + 1)["voxel_num"] > eng.max_voxels for c in clouds))


def check_voxels(oracle, cfg, eng, clouds):
    B, T, mv = eng.B, eng.T, eng.max_voxels
    nv = eng.num_voxels.cpu().numpy()
    coors = eng.vox_coors.cpu().numpy()
    num = eng.vox_num.cpu().numpy()
    slots = eng.vox_slots.long()
    gen = oracle.utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range, T, mv)
    base, pbase = 0, 0
    for b, c in enumerate(clouds):
        ref = gen.generate(c, mv)
        n = int(ref["voxel_num"])
        assert nv[1 + b] == n, "voxels: frame %d has %d voxels, the oracle %d" % (b, nv[1 + b], n)
        sl = slice(base, base + n)
        assert (coors[sl, 0] == b).all(), "voxels: frame %d rows carry another frame index" % b
        assert np.array_equal(coors[sl, 1:], ref["coordinates"]), "voxels: frame %d coordinates" % b
        assert np.array_equal(num[sl], ref["num_points_per_voxel"]), "voxels: frame %d counts" % b
        s = slots[sl]
        live = s >= 0
        assert bool(((s[live] >= pbase) & (s[live] < pbase + c.shape[0])).all()), "voxels: frame %d slot outside its cloud" % b
        vox = torch.where(live[..., None], eng.points[s.clamp_min(0)], 0.0).cpu().numpy()
        assert np.array_equal(vox, ref["voxels"]), "voxels: frame %d voxels" % b
        base += n
        pbase += c.shape[0]
    assert nv[0] == base, "voxels: num_voxels[0] = %d, frames hold %d" % (nv[0], base)


# ---- 2. rulebooks --------------------------------------------------------------------------------------------------
def frame_rows(coors, n):
    """the frame index of each of the first n rows of a level; asserts the rows are grouped by frame (the index
    never decreases)"""
    b = coors[:n, 0]
    assert (np.diff(b) >= 0).all(), "rows are not grouped by frame"
    return b


def check_rulebooks(oracle, eng, frames):
    for lyr in eng.layers:
        if not lyr["build_rb"]:
            continue
        lin, lout = lyr["in_level"], lyr["out_level"]
        n_in, n_out = int(lin.n_dev[0]), int(lout.n_dev[0])
        cin, cout = lin.coors[:n_in].cpu().numpy(), lout.coors[:n_out].cpu().numpy()
        bi, bo = frame_rows(cin, n_in), frame_rows(cout, n_out)
        nbr = lyr["rb"]["nbr"][:n_out].cpu().numpy()
        for b in frames:
            ri, ro = np.nonzero(bi == b)[0], np.nonzero(bo == b)[0]
            idx = cin[ri].copy()
            idx[:, 0] = 0
            o_out, pairs, pnum = oracle.ops.get_indice_pairs(torch.from_numpy(idx), 1, lin.shape, lyr["kernel_size"],
                                                             lyr["stride"], lyr["padding"], lyr["dilation"], 0,
                                                             lyr["subm"])
            o_out = o_out.numpy()
            what = "rulebook of layer %d, frame %d" % (lyr["index"], b)
            assert len(ro) == o_out.shape[0], "%s: %d output rows, the oracle %d" % (what, len(ro), o_out.shape[0])
            assert np.array_equal(cout[ro, 1:], o_out[:, 1:]), what + ": output coordinates or their order"
            want = np.full((len(ro), lyr["K"]), -1, np.int64)
            pairs, pnum = pairs.numpy(), pnum.numpy()
            for k in range(lyr["K"]):
                want[pairs[k, 1, :pnum[k]], k] = ri[pairs[k, 0, :pnum[k]]]
            got = nbr[ro] if len(ro) else np.zeros((0, lyr["K"]))
            bad = np.argwhere(got != want)
            assert bad.size == 0, "%s: row %d offset %d is %d, the oracle %d" % (
                what, ro[bad[0][0]], bad[0][1], got[tuple(bad[0])], want[tuple(bad[0])])


# ---- 3. sparse layers, VFE, PFN ------------------------------------------------------------------------------------
def sparse_modules(net):
    """[(conv, bn or None)] of the sparse middle, in engine layer order"""
    mods = list(net.middle_feature_extractor.middle_conv._modules.values())
    out = []
    for i, m in enumerate(mods):
        if hasattr(m, "subm"):
            bn = mods[i + 1] if i + 1 < len(mods) and isinstance(mods[i + 1], torch.nn.BatchNorm1d) else None
            out.append((m, bn))
    return out


def check_sparse(net, eng, eps=None):
    from b2second import tc
    mods = sparse_modules(net)
    assert len(mods) == len(eng.layers)
    feats = eng.vfe_out
    for (conv, bn), lyr in zip(mods, eng.layers):
        assert lyr["tc"]
        lin, lout = lyr["in_level"], lyr["out_level"]
        n_in, n_out = int(lin.n_dev[0]), int(lout.n_dev[0])
        x = feats[:n_in, :lyr["cin"]].double()
        K = lyr["K"]
        w = conv.weight.detach().float().reshape(K, lyr["cin"], lyr["cout"])
        ws = tc.pow2_scale(tc.pack_sparse_weights(w))
        s64, sh64 = E.fold64(bn, eps)
        ds, dsh = E.fold_error(bn)
        assert bool(((lyr["scale_tc"].double() * ws - E.fold64(bn)[0]).abs() <= ds).all()), "fp32 fold of the scale"
        assert bool(((lyr["shift"].double() - E.fold64(bn)[1]).abs() <= dsh).all()), "fp32 fold of the shift"
        nbr = lyr["rb"]["nbr"][:n_out]
        ref = tc_ref.sparse_ref(x, w, nbr, s64, sh64, lyr["relu"])
        got = tc.merge_f16(lyr["out_hi"][:n_out], lyr["out_lo"][:n_out]).double()
        coors = lout.coors[:n_out]
        ck = E.Check("sparse layer %d" % lyr["index"], ws)
        ck.add(got, ref, ds * ref.S1 + dsh, lambda i: "frame %d, row %d (z %d, y %d, x %d), channel %d" % (
            int(coors[i[0], 0]), i[0], int(coors[i[0], 1]), int(coors[i[0], 2]), int(coors[i[0], 3]), i[1]))
        ck.done()
        feats = got


def check_vfe(eng):
    n = int(eng.num_voxels[0])
    s = eng.vox_slots[:n].long()
    vox = torch.where((s >= 0)[..., None], eng.points[s.clamp_min(0)], 0.0)
    ref = fp32_ref.vfe_ref(vox, eng.vox_num[:n], eng.vfe_nf, radius=eng.vfe_mode == 2)
    fp32_ref.assert_accurate(eng.vfe_out[:n], ref, "mean VFE")


def check_pfn(net, eng):
    n = int(eng.num_voxels[0])
    lyr = net.voxel_feature_extractor.pfn_layers[0]
    w = lyr.linear.weight.detach().float()
    s64, sh64 = E.fold64(lyr.norm)
    ds, dsh = E.fold_error(lyr.norm)
    vx, vy, xo, yo = eng.pfn_geom
    coors = eng.vox_coors[:n]
    for r0 in range(0, n, 8192):
        r1 = min(n, r0 + 8192)
        ref = fp32_ref.pfn_ref(eng.points, eng.vox_slots[r0:r1], eng.vox_num[r0:r1], coors[r0:r1], w, s64, sh64,
                               vx, vy, xo, yo, radius=eng.pfn_deco == 1)
        # fold term: |s32 - s64| * max_t S1_t + |sh32 - sh64|, with unit = max_t |s| S1_t
        extra = ds / s64.abs() * ref.unit + dsh
        ref = fp32_ref.Ref(ref.y, ref.bound + extra, ref.unit, ref.rest + extra)
        st = fp32_ref.error_stats(eng.pfn_out[r0:r1], ref)
        if st["ratio"] > 1.0:
            err = (eng.pfn_out[r0:r1].double() - ref.y).abs() / ref.bound
            i = int(err.argmax()) // err.shape[1]
            raise AssertionError("PFN: frame %d, row %d: %.3g x the bound" % (int(coors[r0 + i, 0]), r0 + i, st["ratio"]))
        assert st["rms"] <= fp32_ref.RHO, "PFN rows %d..%d: rms %.3g" % (r0, r1, st["rms"])


# ---- 4. BEV --------------------------------------------------------------------------------------------------------
def check_bev(eng):
    from b2second import tc
    fl = eng.final_level
    D, H, W = fl.shape
    n = int(fl.n_dev[0])
    co = fl.coors[:n].long()
    if eng.is_pillars:
        hi, lo = tc.split_f16(eng.pfn_out[:n])
    else:
        last = eng.layers[-1]
        hi, lo = last["out_hi"][:n], last["out_lo"][:n]
    C = hi.shape[1]
    occ = torch.zeros(eng.B, H, W, dtype=torch.uint8, device="cuda")
    occ[co[:, 0], co[:, 2], co[:, 3]] = 1
    assert torch.equal(eng.bev_occ, occ), "BEV: bev_occ is not this batch's occupied pixels (%d flagged, %d occupied)" % (
        int(eng.bev_occ.sum()), int(occ.sum()))
    ch = torch.arange(C, device="cuda") * D
    for p, (plane, rows) in enumerate(zip(eng.tc_bev, (hi, lo))):
        want = torch.zeros_like(plane)
        want[co[:, 0, None], co[:, 2, None] + 1, co[:, 3, None] + 1, ch[None, :] + co[:, 1, None]] = rows
        bad = (bits(plane) != bits(want)).any(-1).nonzero()
        assert bad.numel() == 0, "BEV %s plane: frame %d, pixel (%d, %d) (halo-padded) differs from the scatter%s" % (
            ("hi", "lo")[p], *bad[0].tolist(), " (stale: not occupied in this batch)"
            if not bool(occ[bad[0][0], (bad[0][1] - 1).clamp(0, H - 1), (bad[0][2] - 1).clamp(0, W - 1)]) else "")


# ---- 5. RPN ops ----------------------------------------------------------------------------------------------------
def interior(t, padded):
    return t[:, 1:-1, 1:-1] if padded else t


def merged(planes, padded=True):
    hi, lo = planes
    v = hi.double() if lo is None else hi.double() + lo.double()
    return interior(v, padded)


def op_inputs(eng, after, oi):
    """the source of op oi as the op read it: the copy after the last op before it that wrote that buffer"""
    src = eng.tc_plan[oi]["src"]
    if src == "in":
        return eng.tc_bev
    j = max(j for j in range(oi) if eng.tc_plan[j]["dst"] == src)
    return after[j]


def op_check(eng, after, refs, oi, eps=None, mutate=None):
    """op oi against float64 over chunks of frames; mutate(got, lo) -> a faulty copy of the output (or None)"""
    op, r = eng.tc_plan[oi], refs[oi]
    src = op_inputs(eng, after, oi)
    dst = after[oi]
    ck = E.Check("RPN op %d (%s, %s -> %s, channels %d..%d)" % (oi, op["kind"], op["src"], op["dst"], op["dst_coff"],
                                                               op["dst_coff"] + op["cout"]), op["w_scale"])
    for f0 in range(0, eng.B, CHUNK):
        f1 = min(eng.B, f0 + CHUNK)
        x = merged((src[0][f0:f1], None if src[1] is None else src[1][f0:f1]))
        ref, extra = E.op_ref(x, r, eps, chains=not op["v2"])
        got_hi = E.dst_view(dst[0][f0:f1], op)
        got_lo = None if dst[1] is None else E.dst_view(dst[1][f0:f1], op)
        got = got_hi.double() if got_lo is None else got_hi.double() + got_lo.double()
        if mutate is not None:
            got = mutate(got, got_lo)
        p = op["padded"]
        ck.add(got, ref, extra, lambda i: "frame %d, pixel (%d, %d), channel %d" % (
            f0 + i[0], op["off_h"] + op["out_mul"] * i[1], op["off_w"] + op["out_mul"] * i[2], op["dst_coff"] + i[3]))
    return ck.done()


def check_crop(eng, after, oi):
    op = eng.tc_plan[oi]
    src, dst = op_inputs(eng, after, oi), after[oi]
    c = op["crop"]
    for p in range(2):
        s = interior(src[p], True)[:, c:c + op["Hg"], c:c + op["Wg"]]
        assert torch.equal(bits(interior(dst[p], True)), bits(s.contiguous())), "crop op %d" % oi
        halo = dst[p].clone()
        halo[:, 1:-1, 1:-1] = 0
        assert not bool(halo.any()), "crop op %d: halo written" % oi


def check_rpn_ops(eng, after, refs):
    n_ops = len(eng.tc_plan) - (2 if eng.tc_tail_fused else 0)
    for oi in range(n_ops):
        if eng.tc_plan[oi]["kind"] == "crop":
            check_crop(eng, after, oi)
        else:
            op_check(eng, after, refs, oi)
    if eng.tc_tail_fused:
        check_fused_tail(eng, after, refs)


# ---- 6. fused tail -------------------------------------------------------------------------------------------------
def check_fused_tail(eng, after, refs, eps=None, mutate=None):
    """The tail computes y = ReLU(BN(deblock(x))) in registers and the records h = W_h y + b from it; y never reaches
    memory.  With y64 the float64 deblock + BN + ReLU of the engine's input x and bound_y its per-element bound (tc_ref
    + fold term: |y - y64| <= bound_y), and head64(v) = W_h v + b:
        |h - head64(y64)| <= |h - head64(y)| + |W_h (y - y64)|
                          <= bound_head(y) + |W_h| . bound_y,
    |W_h| the element-wise absolute head matrix.  bound_head(y) is the 3xF16 bound of the head layer on its actual
    input y; it grows with |y| (S1 = |W_h| |y|, Sa = sum |y|), and |y| <= |y64| + bound_y, so it is evaluated at
    |y64| + bound_y (the head's BN-free 1x1 conv has no fold term; its output is fp32, the 2^-22 |pre| term)."""
    d_op, h_op = eng.tc_plan[-2], eng.tc_plan[-1]
    rd, rh = refs[-2], refs[-1]
    src = op_inputs(eng, after, len(eng.tc_plan) - 2)
    rec = after[-1][0]
    ws_d, ws_h = d_op["w_scale"], h_op["w_scale"]
    n = h_op["cout"]
    ck = E.Check("fused tail (heads, channels 0..%d)" % n, ws_h)
    Wh = rh["w"][0].to("cuda")                                  # [n, Cin]
    bh = rh["bias"][rh["c0"]:rh["c1"]].to("cuda")
    for f0 in range(0, eng.B, CHUNK):
        f1 = min(eng.B, f0 + CHUNK)
        x = merged((src[0][f0:f1], src[1][f0:f1]))
        ry, ey = E.op_ref(x, rd, eps)
        unit, rest = tc_ref._terms(ry, ws_d)
        bound_y = tc_ref.ALPHA * unit + rest + ey
        y64 = ry.y
        del ry, unit, rest, ey
        ya = y64.abs() + bound_y
        pre = y64 @ Wh.t() + bh
        S1 = ya @ Wh.abs().t()
        Sa = ya.sum(-1, keepdim=True).expand_as(pre)
        Sw = Wh.abs().sum(1).expand_as(pre)
        ref = tc_ref.Ref(pre, pre, S1, Sa, Sw, torch.ones_like(pre))
        extra = bound_y @ Wh.abs().t()
        got = rec[f0:f1, :, :, :n].double()
        if mutate is not None:
            got = mutate(got, f0)
        ck.add(got, ref, extra, lambda i: "frame %d, pixel (%d, %d), channel %d" % (f0 + i[0], i[1], i[2], i[3]))
    return ck.done()


# ---- 7. background strips ------------------------------------------------------------------------------------------
def strips_to_pixels(mask, H, W, rows, width):
    return mask.repeat_interleave(rows, 1).repeat_interleave(width, 2)[:, :H, :W]


def dilate(m):
    return torch.nn.functional.max_pool2d(m[:, None].float(), 3, 1, 1)[:, 0] > 0


def read_masks(eng):
    """per background-tracked layer: [B, H, W] the pixels of its output that a later launch reads"""
    from b2second.engine import BG_ROWS
    H, W = eng.tc_hw
    B = eng.B
    sh, sw = -(-H // BG_ROWS), -(-W // 8)
    out = []
    for l in range(len(eng.bg_idx)):
        if l + 1 < len(eng.bg_idx):
            comp = eng.bg_flags[l + 1].view(B, sh, sw) != 0
            out.append(dilate(strips_to_pixels(comp, H, W, BG_ROWS, 8)))
        else:
            th, tw = -(-H // 8), -(-W // 16)
            t = torch.zeros(B * th * tw, dtype=torch.bool, device="cuda")
            t[eng.tail_work[:int(eng.tail_counts[0])].long()] = True
            out.append(strips_to_pixels(t.view(B, th, tw), H, W, 8, 16))
    return out


def check_background(eng, after, ref_eng, ref_after, masks, override=None):
    """override: {layer: planes} to use in place of the copies (a mutated copy)"""
    assert torch.equal(bits(eng.tc_heads), bits(ref_eng.tc_heads)), "background: head records differ"
    for p in range(2):
        assert torch.equal(bits(eng.tc_bev[p]), bits(ref_eng.tc_bev[p])), "background: BEV planes differ"
    for l, oi in enumerate(eng.bg_idx):
        got = (override or {}).get(l, after[oi])
        for p in range(2):
            diff = (bits(interior(got[p], True)) != bits(interior(ref_after[oi][p], True))).any(-1) & masks[l]
            bad = diff.nonzero()
            assert bad.numel() == 0, ("background: layer %d (op %d) %s plane, frame %d, pixel (%d, %d) is read by the "
                                      "next launch and differs from the run without background strips" % (
                                          l, oi, ("hi", "lo")[p], *bad[0].tolist()))


# ---- the test ------------------------------------------------------------------------------------------------------
def run_sequence(*args, **kw):
    """_run_sequence, with its engines and buffer copies freed before a failure is reported (a traceback would keep
    tens of GB of them alive into the next case)"""
    import gc
    msg = None
    try:
        _run_sequence(*args, **kw)
    except AssertionError as e:
        msg = str(e)
    gc.collect()
    torch.cuda.empty_cache()
    if msg is not None:
        raise AssertionError(msg)


def _run_sequence(product, oracle, monkeypatch, name, B, points, mutations=False):
    from b2second import config
    cfg = config.get_config(name)
    net, eng = build_engine(product, name, B, points, skip=False, monkeypatch=monkeypatch)
    heads = dict(eng.spec.heads) if eng.spec.heads is not None else None
    refs = E.rpn_refs(net.rpn, heads)
    E.assert_matches_plan(refs, eng.tc_prog)
    for r, op in zip(refs, eng.tc_plan):                        # the engine's fp32 folds within the derived bound
        if r["kind"] == "crop":
            continue
        s64, sh64, ds, dsh = E.scale_shift(r)
        if ds is not None:
            assert bool(((op["scale"].double().to(s64.device) * op["w_scale"] - s64).abs() <= ds).all())
            assert bool(((op["shift"].double().to(s64.device) - sh64).abs() <= dsh).all())
    skip_eng = None
    if name in ("car.fhd", "car.lite"):
        _, skip_eng = build_engine(product, name, B, points)
        assert len(skip_eng.bg_idx) == 6 and skip_eng.tc_tail_fused
    prev_skip = None
    for k, (clouds, special) in enumerate(batches(name, cfg, B, points, eng.F)):
        status = expected_status(oracle, cfg, eng, clouds)
        if B == 32:
            assert status == 0
        after = step(eng, clouds, status)
        check_voxels(oracle, cfg, eng, clouds)
        if eng.is_pillars:
            check_pfn(net, eng)
        else:
            check_vfe(eng)
            check_rulebooks(oracle, eng, sorted({0, 1, B - 1, *special}))
            check_sparse(net, eng)
        check_bev(eng)
        check_rpn_ops(eng, after, refs)
        if k == 0:
            chain_term_leaves_faults_visible(eng, after, refs)
        if skip_eng is not None:
            skip_after = step(skip_eng, clouds, status)
            masks = read_masks(skip_eng)
            check_background(skip_eng, skip_after, eng, after, masks)
            if mutations and k == 2:
                mutation_checks(eng, after, refs, skip_eng, skip_after, prev_skip, masks)
            prev_skip = skip_after
        del after


def chain_term_leaves_faults_visible(eng, after, refs):
    """the accumulation-chain term of k_conv_tc ops (engine_ref.op_ref) does not hide a fault of the size of a dropped
    product: the lo plane of one channel of a k_conv_tc op zeroed (tc_ref.f3) is rejected.  The op: the second one of
    the program when k_conv_tc runs it (the PointPillars 64 -> 64 conv whose terms share a sign over the background),
    else the first k_conv_tc op with hi/lo output."""
    n_ops = len(eng.tc_plan) - (2 if eng.tc_tail_fused else 0)
    cand = [i for i in range(n_ops) if not eng.tc_plan[i]["v2"] and eng.tc_plan[i]["kind"] != "crop"
            and eng.tc_plan[i]["planes"] == 2]
    if not cand:
        return
    oi = 1 if 1 in cand else cand[0]
    with pytest.raises(AssertionError, match=r"RPN op %d .*frame \d+, pixel" % oi):
        op_check(eng, after, refs, oi, mutate=lambda got, lo: tc_ref.f3(got, lo, cdim=3))


def mutation_checks(eng, after, refs, skip_eng, skip_after, prev_skip, masks):
    # a BatchNorm fold without eps, in the reference of the first RPN op
    with pytest.raises(AssertionError, match=r"RPN op 0 .*frame \d+, pixel \(\d+, \d+\)"):
        op_check(eng, after, refs, 0, eps=0.0)
    # one head channel's shift dropped: the channel with the largest bias, in a copy of the records
    ch = int(refs[-1]["bias"].abs().argmax())
    bias = float(refs[-1]["bias"][ch])

    def drop(got, f0):
        got = got.clone()
        got[..., ch] -= bias
        return got
    with pytest.raises(AssertionError, match=r"fused tail .*frame \d+, pixel \(\d+, \d+\), channel %d" % ch):
        check_fused_tail(eng, after, refs, mutate=drop)
    # the lo plane of one op's output zeroed (tc_ref.f3 on the channel whose lo plane carries most)
    with pytest.raises(AssertionError, match=r"RPN op 1 .*frame \d+"):
        op_check(eng, after, refs, 1, mutate=lambda got, lo: tc_ref.f3(got, lo, cdim=3))
    # one background strip of one frame copied from the previous batch: a strip the next launch reads that differs
    from b2second.engine import BG_ROWS
    H, W = eng.tc_hw
    for l, oi in enumerate(skip_eng.bg_idx):
        cur, old = skip_after[oi], prev_skip[oi]
        diff = (bits(interior(cur[0], True)) != bits(interior(old[0], True))).any(-1) & masks[l]
        comp = skip_eng.bg_flags[l].view(eng.B, -(-H // BG_ROWS), -(-W // 8)) != 0
        diff &= ~strips_to_pixels(comp, H, W, BG_ROWS, 8)        # a background strip of this batch
        hit = diff.nonzero()
        if hit.numel():
            b, y, x = hit[0].tolist()
            y0, x0 = y - y % BG_ROWS, x - x % 8
            bad = tuple(t.clone() for t in cur)
            for p in range(2):
                bad[p][b, 1 + y0:1 + y0 + BG_ROWS, 1 + x0:1 + x0 + 8] = old[p][b, 1 + y0:1 + y0 + BG_ROWS, 1 + x0:1 + x0 + 8]
            with pytest.raises(AssertionError, match=r"background: layer %d .*frame %d, pixel" % (l, b)):
                check_background(skip_eng, skip_after, eng, after, masks, override={l: bad})
            break
    else:
        raise AssertionError("no background strip read by the next launch differs from the previous batch")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name,B,points", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_engine_against_float64(product, oracle, monkeypatch, name, B, points):
    run_sequence(product, oracle, monkeypatch, name, B, points)


@pytest.mark.timeout(900)
def test_mutations_are_rejected(product, oracle, monkeypatch):
    """car.fhd at B = 32: each check fails on a faulty copy of a buffer or of the reference, naming the stage, the frame
    and the pixel"""
    run_sequence(product, oracle, monkeypatch, "car.fhd", 32, 29000, mutations=True)
