"""A GPU training step, layer by layer against float64, at the reference's training batch (train_input_reader.batch_size:
car.fhd 8, car.lite 12, all.fhd 3, pointpillars.car.xyres_16 2), over three steps on one network and one optimizer.

The network is the drop-in's (synthetic weights, seed 0) wrapped as train() runs it: enable_sparse_backward,
enable_gpu_loss, enable_gpu_metrics, enable_rpn_training, .train(), stepped by optim.plan(net, ONE_CYCLE, 100), TF32 off.
  step 0  bench.make_clouds(name, 2B, 29000)[:B], each frame with ground-truth boxes drawn near anchors
  step 1  the next B clouds with the special frames of tests/train_ref.py (an empty cloud, a frame without ground
          truth, boxes and points on the first and last BEV row and column, a crowded frame) spread over the batch
  step 2  a sparse batch (3000 points per frame) with special frames at the first, middle and last position: fewer
          voxels and smaller rulebooks than the step before, so a stale workspace or table would show.
For B < 4 the special frames take the place of ordinary ones over steps 1 and 2, each at least once.

Module forward hooks and autograd hooks (on the tensors and on the backward nodes) capture every layer the project
implements; every reference takes the kernel's own captured fp32 input, so each bound is local to one layer:
  voxels      per frame bit-equal to the oracle's VoxelGeneratorV2 (capped at the config's max_voxels)
  anchor mask (xyres_16) bit-equal to tests/anchor_mask_ref.py on the voxels' coordinates
  targets     per frame equal to tests/targets_ref.assign (the log components of the box targets within 4 ulp)
  rulebooks   each table the sparse layers use, for frames 0, B - 1 and the special frames, equal to the oracle's
              get_indice_pairs on the layer's input coordinates
  sparse      every SparseConvolution: forward rows against float64 with the module's current weights (those the
              previous step wrote), dX against the transposed-table contraction of the captured dY, dW against
              tc_ref.wgrad_ref, each with the tc_ref bound in the domain of the split's power-of-two scales (the
              exponents of tests/train_range_ref.py, which the splits follow bit for bit)
  dense()     the BEV map is the exact scatter of the last layer's rows; b2s_from_bev's row gradient the exact gather
  RPN 3x3     every layer rpn_train marked: y, dX and dW with train_ref.check_conv3x3_train, the weight scale the one
              pack_weights returned.  On top of the tc_ref bound each carries the accumulation-chain term of its
              kernel: y and dX run k_conv_tc (fp32 output), whose accumulator cuts every wgmma result toward zero
              (engine_ref.op_ref's term); dW runs b2s_conv2d_wgrad_tc, whose chains of 12 truncated wgmmas per 64-pixel
              strip are drained with round-to-nearest into 2048-pixel slab sums (train_ref.wgrad_chain_term).  Over
              ReLU outputs the cuts of one output share a sign and add up: without the terms, y of the xyres_16
              64 -> 64 layer reaches 1.26x the tc_ref bound, dX of car.lite 1.06x, dW of car.fhd 1.24x and 1.14x RHO
  loss        the six scalars within 1e-5 relative and every element of the three prediction gradients within
              C_REL eps32 |g64| + C_MAX eps32 max|g64| (test_gpu_loss.py's bound, the maximum taken per frame: the
              frames' normalisers differ by decades) against loss_ref.reference_run in float64
  optimizer   every parameter element and both Adam moments against optim_ref.ref_step from the captured fp32 state,
              within optim_ref.step_bounds; the gradient norm within 1e-7 relative
  metrics     the running buffers and the returned dict bit-equal to tests/metrics_ref.py on the same inputs
  status      voxelizer, targets, loss, metrics and optimizer status words 0 after every step.
BatchNorm, ReLU, the stride-2 convs, the deblocks, the heads, the VFE and the pillar scatter are torch's: their captured
outputs are the next checked layer's inputs.  The worst error / bound ratio per layer kind and step goes to
train_fp64_errors.json in the output directory.

test_mutations_are_rejected shows the checks bite: the RPN weight planes cached without the weight's version (stale
after the step), the lo plane of one sparse layer's dY split zeroed, one frame's loss normaliser replaced by the batch's
positive count, one parameter's Adam moment left from the previous step.

Worst error / bound ratios measured on one H100 SXM (80 GB): sparse forward 0.64, dX 0.55, dW 0.58; RPN forward 0.37,
dX 0.35, dW 0.38; loss 0.80; optimizer 0.72.

Wall time on one H100 SXM (80 GB): car.fhd 45 s, car.lite 33 s, the mutations 14 s, all.fhd 11 s,
pointpillars.car.xyres_16 9 s; the whole file about 2 minutes.
"""
import gc
import json
import os

import numpy as np
import pytest
import torch

import anchor_mask_ref as amr
import golden_util as gu
import loss_ref as lr
import metrics_ref as mr
import optim_ref as orf
import tc_ref
import targets_ref as tgr
import train_ref as tr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CONFIGS = [("car.fhd", 8), ("car.lite", 12), ("all.fhd", 3), ("pointpillars.car.xyres_16", 2)]
POINTS, SPARSE_POINTS = 29000, 3000
TOTAL_STEP = 100

_errors = {}


@pytest.fixture(scope="module", autouse=True)
def _report(out_dir):
    yield
    with open(os.path.join(out_dir, "train_fp64_errors.json"), "w") as f:
        json.dump(_errors, f, indent=1, sort_keys=True)


@pytest.fixture(autouse=True)
def _fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _note(ctx, kind, ratio):
    key = "%s/step%d/%s" % (ctx["name"], ctx["step"], kind)
    if ctx.get("record", True):
        _errors[key] = max(_errors.get(key, 0.0), float(ratio))


# ---- the network and the batches ----------------------------------------------------------------------------------
def build(product, name):
    from b2second import config, loss, metrics, models, optim, training
    cfg = config.get_config(name)
    net = models.build_network(cfg, product)
    models.synthetic_weights_(net, name, seed=0)
    net = metrics.enable_gpu_metrics(loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV))))
    net = training.enable_rpn_training(net).train()
    return cfg, net, optim.plan(net, orf.ONE_CYCLE, TOTAL_STEP)


def batches(name, cfg, B):
    """-> [(clouds, {position: special frame})] of the three steps"""
    import bench
    F = cfg.num_point_features
    clouds = bench.make_clouds(name, 2 * B, POINTS)
    sparse = [gu.make_cloud(name, 1000 + s, SPARSE_POINTS) for s in range(B)]
    out = [(list(clouds[:B]), {}), (list(clouds[B:]), {}), (sparse, {})]
    for k, where in tr.special_layout(B):
        out[k] = (out[k][0], where)
        for p, kind in where.items():
            if kind == "empty":
                out[k][0][p] = np.zeros((0, F), np.float32)
            elif kind == "border":
                out[k][0][p] = gu.border_cloud(cfg, F, 7)
    return out


# ---- 1. voxels, anchor mask, targets -------------------------------------------------------------------------------
def voxelize(product, oracle, cfg, clouds):
    """device voxels of the batch, checked frame by frame against the oracle -> (example part, expected status)"""
    B, mv, T = len(clouds), cfg.max_voxels, cfg.max_points_per_voxel
    gen = product.utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range, T, mv)
    offs = np.cumsum([0] + [c.shape[0] for c in clouds]).astype(np.int32)
    pts = torch.from_numpy(np.concatenate(clouds, 0)).to(DEV)
    res = gen.generate_device(pts, mv, frame_offsets=torch.from_numpy(offs).to(DEV), batch=B)
    counts = res["num_voxels"].cpu().numpy()
    og = oracle.utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range, T, mv + 1)
    overflow = 0
    row = 0
    for b, c in enumerate(clouds):
        overflow |= int(og.generate(c, mv + 1)["voxel_num"] > mv)
        ref = og.generate(c, mv)
        n = int(ref["voxel_num"])
        assert counts[1 + b] == n, "voxels: frame %d has %d voxels, the oracle %d" % (b, counts[1 + b], n)
        co = res["coordinates"][row:row + n].cpu().numpy()
        assert (co[:, 0] == b).all() and np.array_equal(co[:, 1:], ref["coordinates"]), "voxels: frame %d coordinates" % b
        assert np.array_equal(res["voxels"][row:row + n].cpu().numpy(), ref["voxels"]), "voxels: frame %d voxels" % b
        assert np.array_equal(res["num_points_per_voxel"][row:row + n].cpu().numpy(), ref["num_points_per_voxel"]), \
            "voxels: frame %d counts" % b
        row += n
    assert counts[0] == row
    ex = {"voxels": res["voxels"][:row], "num_points": res["num_points_per_voxel"][:row],
          "coordinates": res["coordinates"][:row]}
    return ex, res["status"], overflow


def anchor_mask(cfg, plan, coords, B):
    """the anchor-area mask where the config sets anchor_area_threshold (else None), checked against the restatement"""
    if cfg.anchor_area_threshold < 0:
        return None
    from b2second import anchor_mask as am, inputs
    mask = inputs.anchor_area_mask(coords, B, plan.anchors, cfg.voxel_size, cfg.point_cloud_range, cfg.grid_size,
                                   cfg.anchor_area_threshold)
    boxes = am.anchor_boxes(plan.anchors, cfg.voxel_size, cfg.point_cloud_range, cfg.grid_size)
    want = amr.anchor_area_mask_np(coords.cpu().numpy(), B, boxes, cfg.grid_size, cfg.anchor_area_threshold)
    assert np.array_equal(mask.cpu().numpy(), want), "anchor-area mask"
    return mask


def assign(plan, frames, mask):
    """assign_batch of the frames' ground truth, checked frame by frame against targets_ref.assign"""
    gt = np.concatenate([f[0] for f in frames])
    cls = np.concatenate([f[1] for f in frames])
    imp = np.concatenate([f[2] for f in frames])
    offs = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
    r = plan.assign_batch(torch.from_numpy(gt).to(DEV), torch.from_numpy(offs).to(DEV), torch.from_numpy(cls).to(DEV),
                          torch.from_numpy(imp).to(DEV), mask)
    mask_np = mask.cpu().numpy() if mask is not None else None
    for b, (g, c, i) in enumerate(frames):
        seg = (c - 1) if plan.assign_per_class else np.zeros(len(c), np.int32)
        labels, tg, im, _, _ = tgr.assign(plan, g, seg, c, i, None if mask_np is None else mask_np[b])
        pos = np.flatnonzero(labels > 0)
        try:
            tgr.check_frame(r["labels"][b], r["reg_targets"][b], r["importance"][b],
                                {"labels": labels, "importance_out": im, "pos": pos, "targets": tg[pos]})
        except AssertionError as e:
            raise AssertionError("targets: frame %d: %s" % (b, e))
    return r


# ---- capture -------------------------------------------------------------------------------------------------------
def _grads_by_shape(gi, *tensors):
    """the gradients of a backward node matched to its inputs by shape (None where autograd computed none)"""
    out = []
    for t in tensors:
        out.append(next((g.detach() for g in gi if g is not None and g.shape == t.shape), None))
    return out


class Capture:
    """forward hooks on the project's layers, and hooks on their backward nodes, recording one step"""

    def __init__(self, net, product):
        from b2second import rpn_train
        self.rpn_train = rpn_train
        self.sparse = [m for m in net.middle_feature_extractor.modules() if isinstance(m, product.SparseConvolution)]
        self.rpn = [m for m in net.rpn.modules() if getattr(m, "_b2s_rpn_train", False)]
        assert self.rpn, "no RPN layer on the tensor pipe"
        hs = [m.register_forward_hook(self._sparse(i)) for i, m in enumerate(self.sparse)]
        hs += [m.register_forward_hook(self._conv(i)) for i, m in enumerate(self.rpn)]
        if self.sparse:
            hs.append(net.middle_feature_extractor.middle_conv.register_forward_hook(self._rows))
            hs.append(net.middle_feature_extractor.register_forward_hook(self._dense))
        hs.append(net.rpn.register_forward_hook(self._heads))
        self.handles = hs
        self.reset()

    def reset(self):
        self.rec = {"sparse": [None] * len(self.sparse), "rpn": [None] * len(self.rpn), "bev": {}, "heads": {},
                    "head_grads": {}}

    def close(self):
        for h in self.handles:
            h.remove()

    def _sparse(self, i):
        def hook(mod, args, out):
            inp = args[0]
            r = {"x": inp.features.detach(), "in_idx": inp.indices, "in_shape": list(inp.spatial_shape),
                 "rb": inp.indice_dict[mod.indice_key], "w": mod.weight.detach().clone(), "y": out.features.detach(),
                 "mod": mod}
            x_req, w = inp.features, mod.weight

            def bw(gi, go):
                r["dy"] = go[0].detach()
                r["dx"], r["dw"] = _grads_by_shape(gi, x_req, w)
            node = out.features.grad_fn
            assert type(node).__name__.startswith("_SparseConvFunction"), \
                "sparse layer %d did not run the drop-in's _SparseConvFunction (%s)" % (i, type(node).__name__)
            node.register_hook(bw)
            self.rec["sparse"][i] = r
        return hook

    def _conv(self, i):
        def hook(mod, args, out):
            x = args[0]
            r = {"x": x.detach(), "y": out.detach(), "w": mod.weight.detach().clone(),
                 "w_inv": float(self.rpn_train.pack_weights(mod, False)[2])}

            def bw(gi, go):
                r["dy"] = go[0].detach()
                r["dx"], r["dw"] = _grads_by_shape(gi, x, mod.weight)
            assert type(out.grad_fn).__name__.startswith("Conv3x3TC"), "RPN layer %d did not run Conv3x3TC" % i
            out.grad_fn.register_hook(bw)
            self.rec["rpn"][i] = r
        return hook

    def _rows(self, mod, args, out):
        self.rec["bev"].update(rows=out.features.detach(), idx=out.indices, shape=list(out.spatial_shape),
                               B=out.batch_size)

    def _dense(self, mod, args, out):
        bev = self.rec["bev"]
        bev["map"] = out.detach()
        node = out.grad_fn
        while node is not None and "DenseFunction" not in type(node).__name__:
            node = node.next_functions[0][0]
        assert node is not None, "dense() did not run _DenseFunction"

        def bw(gi, go):
            bev["dmap"], bev["drows"] = go[0].detach(), gi[0].detach()
        node.register_hook(bw)

    def _heads(self, mod, args, out):
        for k in ("box_preds", "cls_preds", "dir_cls_preds"):
            t = out[k]
            self.rec["heads"][k] = t.detach()
            t.register_hook(lambda g, k=k: self.rec["head_grads"].__setitem__(k, g.detach()))


# ---- 2. layer checks -----------------------------------------------------------------------------------------------
def check_rulebooks(oracle, rec, frames):
    seen = set()
    for li, r in enumerate(rec["sparse"]):
        rb, mod = r["rb"], r["mod"]
        if id(rb) in seen:
            continue
        seen.add(id(rb))
        cin = r["in_idx"].cpu().numpy()
        n_out = rb.num_out
        cout = rb.out_indices[:n_out].cpu().numpy()
        nbr = rb.nbr[:n_out].cpu().numpy()
        for f in frames:
            idx = cin[cin[:, 0] == f].copy()
            idx[:, 0] = 0
            o_out, pairs, pnum = oracle.ops.get_indice_pairs(torch.from_numpy(idx), 1, r["in_shape"], mod.kernel_size,
                                                             mod.stride, mod.padding, mod.dilation, 0, rb.subm)
            msg = tr.compare_rulebook(cin, cout, nbr, f, o_out.numpy(), pairs.numpy(), pnum.numpy())
            assert msg is None, "rulebook of sparse layer %d: %s" % (li, msg)


def check_sparse(ctx, rec, mutate_dx=None):
    from b2second import tc
    for li, r in enumerate(rec["sparse"]):
        rb = r["rb"]
        K, cin, cout = rb.K, r["mod"].in_channels, r["mod"].out_channels
        w = r["w"].reshape(K, cin, cout)
        nbr = rb.nbr[:rb.num_out]
        ws = tc.pow2_scale(w)
        fwd, dxr, dwr, ex, eg = tr.sparse_refs(r["x"], r["dy"], w, nbr)
        what = "%s step %d: sparse layer %d (%d -> %d, K %d)" % (ctx["name"], ctx["step"], li, cin, cout, K)
        _note(ctx, "sparse forward", tr.scaled_check(r["y"], fwd, ws, ex, what + " forward")["ratio"])
        del fwd
        if r["dx"] is not None:
            got = r["dx"] if mutate_dx is None or mutate_dx[0] != li else mutate_dx[1](r, w, nbr, eg)
            _note(ctx, "sparse dX", tr.scaled_check(got, dxr, ws, eg, what + " dX")["ratio"])
        else:
            assert li == 0, "sparse layer %d returned no input gradient" % li
        del dxr
        _note(ctx, "sparse dW", tr.scaled_check(r["dw"].reshape(K, cin, cout), dwr, 1.0, ex + eg, what + " dW")["ratio"])


def dy_lo_plane_zeroed(r, w, nbr, eg):
    """dX as it would be had the lo plane of the dY split been zero: the lo plane's contribution taken off in float64"""
    _, lo = tc_ref.hi_lo(r["dy"], 2.0 ** eg)
    delta = tc_ref.sparse_ref(lo, w.transpose(1, 2).contiguous(), tr.transpose_table(nbr, r["x"].shape[0])).y
    return r["dx"].double() - delta * 2.0 ** -eg


def check_bev(rec):
    bev = rec["bev"]
    D, H, W = bev["shape"]
    B = bev["B"]
    rows, idx = bev["rows"], bev["idx"]
    want = tr.scatter_rows(rows, idx, B, D, H, W)
    assert torch.equal(bev["map"].view(want.shape), want), "dense(): the BEV map is not the scatter of the rows"
    dmap = bev["dmap"].reshape(want.shape)
    assert torch.equal(bev["drows"], tr.gather_rows(dmap, idx)), "from_bev: the row gradient is not the gather"


def check_rpn(ctx, rec, layers=None, parts=("forward", "dX", "dW")):
    """the RPN 3x3 layers (all, or those listed) against float64 with train_ref.check_conv3x3_train"""
    for li, r in enumerate(rec["rpn"]):
        if layers is not None and li not in layers:
            continue
        w = r["w"]
        what = "%s step %d: RPN layer %d (%d -> %d, %dx%d)" % (ctx["name"], ctx["step"], li, w.shape[1], w.shape[0],
                                                               r["x"].shape[2], r["x"].shape[3])
        st = tr.check_conv3x3_train(r["x"], r["dy"], r["y"], r["dx"], r.get("dw"), w, 1.0 / r["w_inv"], what, parts)
        for part, v in st.items():
            _note(ctx, "rpn " + part, v["ratio"])


def check_loss(ctx, net, ex, ret, rec, mutate=None):
    s = net.b2s_loss.settings
    B = ex["labels"].shape[0]
    cpu = {k: ex[k].cpu() for k in ("labels", "reg_targets", "importance", "anchors")}
    preds = {k: v.cpu() for k, v in rec["heads"].items()}
    out64, g64 = lr.reference_run(s, cpu, preds, torch.float64)
    lr.check_scalars([float(ret[k].detach()) for k in lr.SCALARS], [float(out64[k]) for k in lr.SCALARS],
                   "%s step %d: loss" % (ctx["name"], ctx["step"]))
    grads = {k: rec["head_grads"][k].cpu().double().numpy().reshape(g64[k].shape) for k in g64}
    if mutate is not None:
        grads = mutate(grads)
    worst = 0.0
    for k, want in g64.items():
        got = grads[k]
        assert np.isfinite(got).all(), k
        for b in range(B):
            bound = lr.C_REL * lr.EPS32 * np.abs(want[b]) + lr.C_MAX * lr.EPS32 * np.abs(want[b]).max()
            err = np.abs(got[b] - want[b])
            ratio = float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0
            worst = max(worst, ratio)
            if ratio > 1.0:
                i = np.unravel_index(np.argmax(err / np.maximum(bound, 1e-300)), err.shape)
                raise AssertionError("%s step %d: loss gradient %s, frame %d, element %s: %.3g x the bound (%.9g, "
                                     "float64 %.9g, frame max %.3g)" % (ctx["name"], ctx["step"], k, b, i, ratio,
                                                                        got[b][i], want[b][i], np.abs(want[b]).max()))
    _note(ctx, "loss", worst)


def normaliser_of_the_batch(ex):
    """one frame's gradients as if its loss normaliser were the batch's positive count"""
    pos = (ex["labels"] > 0).sum(1).cpu().numpy()
    b = int(np.flatnonzero((pos > 0) & (pos < pos.sum()))[0])

    def mutate(grads):
        grads = {k: v.copy() for k, v in grads.items()}
        for k in grads:
            grads[k][b] *= pos[b] / pos.sum()
        return grads
    return b, mutate


def check_optimizer(ctx, opt, before, after, k, stale_moment=None):
    s = opt.settings
    p, g, m, v = ([t.cpu().numpy().astype(np.float64) if t is not None else None for t in ts] for ts in before[:4])
    g = [t.astype(np.float32) for t in g]
    total, info = orf.ref_step(s, p, g, m, v, opt.table[k, 0], opt.table[k, 1], k + 1)
    got_total = before[4]
    assert abs(got_total - total) <= 1e-7 * total, "%s step %d: gradient norm %.9g, float64 %.9g" % (
        ctx["name"], ctx["step"], got_total, total)
    worst = 0.0
    gp, gm, gv = after
    for i in range(len(p)):
        d = orf.step_bounds(s, info[i], p[i], m[i], v[i])
        got_m = gm[i] if stale_moment != i else before[2][i]
        for name, got, want, bound in (("m", got_m, m[i], d[0]), ("v", gv[i], v[i], d[1]), ("p", gp[i], p[i], d[2])):
            ratio = float((np.abs(got.cpu().numpy().astype(np.float64) - want) / np.maximum(bound, 1e-300)).max())
            worst = max(worst, ratio)
            assert ratio <= 1.0, "%s step %d: optimizer %s of parameter %d: %.3g x its bound" % (
                ctx["name"], ctx["step"], name, i, ratio)
    _note(ctx, "optimizer", worst)


def metric_state(net):
    b = {"acc_total": net.rpn_acc.total, "acc_count": net.rpn_acc.count,
         "prec_total": net.rpn_metrics.prec_total, "prec_count": net.rpn_metrics.prec_count,
         "rec_total": net.rpn_metrics.rec_total, "rec_count": net.rpn_metrics.rec_count,
         "cls_total": net.rpn_cls_loss.total, "cls_count": net.rpn_cls_loss.count,
         "loc_total": net.rpn_loc_loss.total, "loc_count": net.rpn_loc_loss.count}
    return {k: v.detach().cpu().numpy().copy() for k, v in b.items()}


def check_metrics(ctx, net, ex, ret, state0):
    got = net.update_metrics(ret["cls_loss_reduced"], ret["loc_loss_reduced"], ret["cls_preds"], ex["labels"],
                             ret["cared"])
    ref = mr.MetricsRef(device=DEV)
    ref.load(state0)
    want = ref.update(ret["cls_loss_reduced"].detach(), ret["loc_loss_reduced"].detach(), ret["cls_preds"].detach(),
                      ex["labels"], ret["cared"], net.b2s_metrics.num_class)
    assert json.dumps(got, sort_keys=True) == json.dumps(want, sort_keys=True), \
        "%s step %d: metrics %r, the restatement %r" % (ctx["name"], ctx["step"], got, want)
    st, ws = metric_state(net), ref.state()
    for k in mr.BUFFERS:
        assert np.array_equal(st[k].view(np.int32), ws[k].view(np.int32)), "%s step %d: metric buffer %s" % (
            ctx["name"], ctx["step"], k)


# ---- the sequence --------------------------------------------------------------------------------------------------
def run_sequence(*args, **kw):
    """_run_sequence, with its captures freed before a failure is reported"""
    msg = None
    try:
        _run_sequence(*args, **kw)
    except AssertionError as e:
        msg = str(e)
    gc.collect()
    torch.cuda.empty_cache()
    if msg is not None:
        raise AssertionError(msg)


def _run_sequence(product, oracle, monkeypatch, name, B, mutations=False):
    from b2second import targets
    if mutations:
        stale_rpn_planes(monkeypatch)
    cfg, net, opt = build(product, name)
    plan = targets.plan(net.target_assigner, cfg.feature_map_size)
    anchors = net.anchors().reshape(-1, 7)
    assert np.array_equal(anchors, plan.anchors[:, :7])
    anchors_b = torch.from_numpy(anchors).to(DEV)[None].repeat(B, 1, 1)
    cap = Capture(net, product)
    try:
        for k, (clouds, where) in enumerate(batches(name, cfg, B)):
            if mutations and k == 2:
                break
            ctx = {"name": name, "step": k, "record": not mutations}
            cap.reset()
            ex, vox_status, overflow = voxelize(product, oracle, cfg, clouds)
            mask = anchor_mask(cfg, plan, ex["coordinates"], B)
            rng = np.random.default_rng(100 * k + 1)
            frames = [tr.gt_boxes(plan, rng, where.get(b, "ordinary")) for b in range(B)]
            ex.update(assign(plan, frames, mask))
            ex["anchors"] = anchors_b
            ret = net(ex)
            ret["loss"].backward()
            state0 = metric_state(net)
            check_metrics(ctx, net, ex, ret, state0)
            before = ([p.detach().clone() for p in opt.params], [p.grad.detach().clone() for p in opt.params],
                      [m.clone() for m in opt.exp_avg], [v.clone() for v in opt.exp_avg_sq])
            norm = float(opt.step())
            after = ([p.detach().clone() for p in opt.params], [m.clone() for m in opt.exp_avg],
                     [v.clone() for v in opt.exp_avg_sq])
            torch.cuda.synchronize()
            status = {"voxelizer": int(vox_status.item()), "targets": int(plan.last_status.item()),
                      "loss": int(net.b2s_loss.last_status.item()), "metrics": int(net.b2s_metrics.last_status.item()),
                      "optimizer": int(opt.status.item())}
            assert status == {"voxelizer": overflow, "targets": 0, "loss": 0, "metrics": 0, "optimizer": 0}, status
            assert overflow == 0, "a frame holds more than max_voxels voxels"
            rec = cap.rec
            if mutations and k == 1:
                # the planes cached at step 0 are served again: the forward no longer sees the stepped weights
                with pytest.raises(AssertionError, match=r"RPN layer 0 .* forward"):
                    check_rpn(ctx, rec, layers=[0], parts=("forward",))
                # the first parameter's first moment as it was before this step
                with pytest.raises(AssertionError, match=r"optimizer m of parameter 0"):
                    check_optimizer(ctx, opt, before + (norm,), after, k, stale_moment=0)
                break
            if cap.sparse:
                special = sorted({0, B - 1, *where})
                check_rulebooks(oracle, rec, special)
                check_sparse(ctx, rec)
                check_bev(rec)
            check_rpn(ctx, rec)
            check_loss(ctx, net, ex, ret, rec)
            check_optimizer(ctx, opt, before + (norm,), after, k)
            if mutations and k == 0:
                with pytest.raises(AssertionError, match=r"sparse layer 1 .* dX"):
                    check_sparse(ctx, rec, mutate_dx=(1, dy_lo_plane_zeroed))
                b, mutate = normaliser_of_the_batch(ex)
                with pytest.raises(AssertionError, match=r"loss gradient .*frame %d" % b):
                    check_loss(ctx, net, ex, ret, rec, mutate=mutate)
            del rec, ret, before, after
            cap.reset()
    finally:
        cap.close()


def stale_rpn_planes(monkeypatch):
    """rpn_train.pack_weights with its cache keyed on the weight's storage alone, not on its version"""
    from b2second import rpn_train
    orig = rpn_train.pack_weights

    def unversioned(conv, transpose):
        w = conv.weight
        key = (w.data_ptr(), str(w.device), transpose)
        cache = conv.__dict__.setdefault("_stale_planes", {})
        hit = cache.get(transpose)
        if hit is not None and hit[0] == key:
            return hit[1]
        val = orig(conv, transpose)
        cache[transpose] = (key, val)
        return val
    monkeypatch.setattr(rpn_train, "pack_weights", unversioned)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name,B", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_training_step_against_float64(product, oracle, monkeypatch, name, B):
    run_sequence(product, oracle, monkeypatch, name, B)


@pytest.mark.timeout(1200)
def test_mutations_are_rejected(product, oracle, monkeypatch):
    """car.lite at B = 12, steps 0 and 1: each check fails on a faulty copy of a captured value, or on the network run
    with the RPN weight planes cached without the weight's version"""
    run_sequence(product, oracle, monkeypatch, "car.lite", 12, mutations=True)
