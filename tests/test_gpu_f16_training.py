"""The f16 training mode on the GPU (training.enable_sparse_backward / enable_rpn_training with precision="f16").

Per layer shape, each single-product contraction against float64 with the f16 bound of tests/f16_train_ref.py, and on
every shape some element beyond tc_ref's 3xF16 bound (so the check is not vacuous and the kernel really runs one product):
  sparse   every tensor-pipe layer shape of car.fhd, car.lite and all.fhd on a random table: the forward (fp32 rows,
           b2s_sparse_conv_tc_plan_ex2), the input gradient where the layer takes it on the tensor pipe (the forward
           contraction over a transposed table with W^T) and the weight gradient (b2s_sparse_conv_wgrad_tc_ex), the last
           bit-identical with and without the tile mask, and every result bit-identical over two runs;
  RPN 3x3  every covered layer shape of car.fhd and pointpillars.car.xyres_16: forward and input gradient
           (b2s_conv2d_tc_ex3, products 1, fp32 output) and weight gradient (b2s_conv2d_wgrad_tc_ex).
The single-plane splits and packs are bit-equal to the hi planes (and scales) of the 3xF16 calls, non-finite values
included; Inf and NaN in dY reach exactly the outputs fp32 arithmetic makes non-finite; the sparse middle encoder's layers
and the RPN forward + backward of car.fhd and xyres_16 are captured in CUDA graphs and replayed bit for bit.

test_training_curves trains the car.fhd and xyres_16 mirror networks for 100 steps in each mode on one fixed synthetic
batch and gates only that both losses stay finite and decrease; the curves go to f16_training_curves.json in the output
directory.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import f16_train_ref as fr
import tc_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SPARSE_CONFIGS = ["car.fhd", "car.lite", "all.fhd"]
RPN_CONFIGS = ["car.fhd", "pointpillars.car.xyres_16"]


@pytest.fixture(autouse=True)
def _fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


_errors = {}


@pytest.fixture(scope="module", autouse=True)
def _report(out_dir):
    yield
    with open(os.path.join(out_dir, "f16_training_errors.json"), "w") as f:
        json.dump(_errors, f, indent=1, sort_keys=True)


def check(got, ref, sa, sb, n, what, mask=None):
    """f16_train_ref.check, its worst ratio and share beyond the 3xF16 bound kept for f16_training_errors.json"""
    ratio, beyond = fr.check(got, ref, sa, sb, n, what, mask)
    _errors[what] = {"ratio": round(ratio, 4), "beyond_3xf16": round(beyond, 4)}


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


# ---- sparse --------------------------------------------------------------------------------------------------------
def sparse_shapes(product, name):
    """[(cin, cin_tc, cout, K, dgrad on the tensor pipe)] of the config's tensor-pipe sparse layers"""
    from b2second import config, models, tc
    lib = product._lib.load()
    net = models.build_network(config.get_config(name), product)
    out = []
    for m in net.modules():
        if isinstance(m, product.SparseConvolution):
            K = int(np.prod(m.kernel_size))
            cin_tc = m._wgrad_tc_cin(lib, K)
            if cin_tc is None:
                continue
            key = (m.in_channels, cin_tc, m.out_channels, K,
                   tc.sparse_tc_channels(lib, m.out_channels, m.in_channels, K) == m.out_channels)
            if key not in out:
                out.append(key)
    assert out
    return out


def _table(g, n_rows, n_src, K, present=0.4):
    nbr = torch.randint(0, n_src, (n_rows, K), device=DEV, generator=g, dtype=torch.int32)
    nbr[torch.rand(n_rows, K, device=DEV, generator=g) >= present] = -1
    return nbr


def sp_conv(sp, x_split, w, table, n_out, cout, products, transpose=False):
    """one sparse contraction through the drop-in's launcher: fp32 rows [n_out, cout] and the weights' scale"""
    hi, lo, stride, inv_x = x_split.planes()
    w_hi, w_lo, ws, inv_w = sp._pack_tc_weights(w, transpose=transpose, products=products)
    out = torch.full((n_out, cout), float("nan"), device=DEV)
    n_dev = torch.tensor([n_out], dtype=torch.int32, device=DEV)
    scale = (inv_x * inv_w).expand(cout).contiguous()
    st = sp._conv_tc((hi, lo, stride), (w_hi, w_lo), table, table.shape[1], n_dev, n_out, (None, None), scale, None,
                     False, out, products=products)
    assert int(st.item()) == 0
    return out, float(ws)


def sp_wgrad(sp, x_split, g_split, nbr, cin_tc, cout, products, plan=(None, None)):
    L = sp._lib
    lib = L.load()
    x_hi, x_lo, xs, inv_x = x_split.planes()
    g_hi, g_lo, gs, inv_g = g_split.planes()
    n_out, K = nbr.shape
    dw = torch.full((K, cin_tc, cout), float("nan"), device=DEV)
    nbytes = lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(n_out, K, cin_tc, cout)
    work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=DEV)
    n_dev = torch.tensor([n_out], dtype=torch.int32, device=DEV)
    L.check(lib.b2s_sparse_conv_wgrad_tc_ex(
        L.ptr(x_hi), L.ptr(x_lo), xs, x_hi.shape[0], cin_tc, L.ptr(g_hi), L.ptr(g_lo), gs, cout, L.ptr(nbr), K,
        L.ptr(n_dev), n_out, L.ptr(plan[0]), L.ptr(plan[1]), L.ptr(inv_x * inv_g), L.ptr(dw), L.ptr(work), nbytes,
        products, L.stream()), "b2s_sparse_conv_wgrad_tc_ex")
    return dw


def tile_plan(sp, nbr):
    L = sp._lib
    n_out, K = nbr.shape
    perm = torch.empty(n_out, dtype=torch.int32, device=DEV)
    tmask = torch.empty((n_out + 127) // 128, dtype=torch.int32, device=DEV)
    n_dev = torch.tensor([n_out], dtype=torch.int32, device=DEV)
    L.check(L.load().b2s_sparse_tile_plan(L.ptr(nbr), None, K, None, L.ptr(n_dev), n_out, 1, L.ptr(perm), L.ptr(tmask),
                                          L.stream()), "b2s_sparse_tile_plan")
    return perm, tmask


@pytest.mark.parametrize("name", SPARSE_CONFIGS)
def test_sparse_layers_against_float64(product, name):
    sp = product
    for j, (cin, cin_tc, cout, K, dgrad) in enumerate(sparse_shapes(product, name)):
        what = "%s sparse %d -> %d, K %d" % (name, cin, cout, K)
        g = torch.Generator(device=DEV).manual_seed(300 + j)
        n_in, n_out = 6000, 5000
        x = torch.randn(n_in, cin, device=DEV, generator=g)
        if j:
            x = torch.relu(x)
        w = torch.randn(K, cin, cout, device=DEV, generator=g) * (2.0 / (K * cin)) ** 0.5
        dy = torch.randn(n_out, cout, device=DEV, generator=g) * 2.0 ** -20
        nbr = _table(g, n_out, n_in, K)
        x_split, g_split = sp._GradSplit(x, cin_tc, 1), sp._GradSplit(dy, products=1)
        sa, sg = 1.0 / float(x_split.planes()[3]), 1.0 / float(g_split.planes()[3])
        # forward
        y, ws = sp_conv(sp, x_split, w, nbr, n_out, cout, 1)
        check(y, tc_ref.sparse_ref(x, w, nbr), sa, ws, K * cin_tc, what + " forward")
        assert torch.equal(_bits(y), _bits(sp_conv(sp, x_split, w, nbr, n_out, cout, 1)[0])), what + " forward bits"
        # input gradient over a transposed table
        if dgrad:
            nbrT = _table(g, n_in, n_out, K)
            dx, wts = sp_conv(sp, g_split, w, nbrT, n_in, cin, 1, transpose=True)
            check(dx, tc_ref.sparse_ref(dy, w.transpose(1, 2).contiguous(), nbrT), sg, wts, K * cout, what + " dX")
        # weight gradient, in the tile plan's row order with and without the mask
        plan = tile_plan(sp, nbr)
        dw = sp_wgrad(sp, x_split, g_split, nbr, cin_tc, cout, 1, plan)
        assert torch.equal(_bits(dw), _bits(sp_wgrad(sp, x_split, g_split, nbr, cin_tc, cout, 1, (plan[0], None)))), \
            what + " dW with and without the tile mask"
        assert torch.equal(_bits(dw), _bits(sp_wgrad(sp, x_split, g_split, nbr, cin_tc, cout, 1, plan))), what + " dW bits"
        check(dw[:, :cin], tc_ref.wgrad_ref(x, dy, nbr), sa, sg, n_out, what + " dW")


# ---- RPN 3x3 ---------------------------------------------------------------------------------------------------------
def rpn_shapes(name):
    """[(cin, cout, H, W)] of the config's covered RPN layers at their map sizes"""
    from b2second import config, loader, models, rpn_train
    cfg = config.get_config(name)
    net = models.build_network(cfg, loader.product_spconv())
    rpn = net.rpn
    covered = {id(c) for c, _ in rpn_train.select(rpn)}
    H, W = (int(v) * rpn.blocks[0][1].stride[0] for v in cfg.feature_map_size[1:])
    out = []
    h, w = H, W
    for blk in rpn.blocks:
        st = blk[1].stride[0]
        h, w = (h + 2 - 3) // st + 1, (w + 2 - 3) // st + 1
        for m in blk:
            if id(m) in covered and (m.in_channels, m.out_channels, h, w) not in out:
                out.append((m.in_channels, m.out_channels, h, w))
    assert out
    return out


def _dense_layer(cin, cout, g):
    conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(cout, cin, 3, 3, device=DEV, generator=g) * (2.0 / (9 * cin)) ** 0.5)
    return conv


def dense_f16(conv, x, dy):
    """forward, dX and dW of rpn_train's launchers with products = 1 -> (y, dx, dw, scales)"""
    from b2second import rpn_train
    B, cin, H, W = x.shape
    cout = conv.out_channels
    x_hi, x_lo, xs = rpn_train.split_halo(x, products=1)
    g_hi, g_lo, gs = rpn_train.split_halo(dy, products=1)
    assert x_lo is None and g_lo is None
    w_hi, w_lo, w_inv = rpn_train.pack_weights(conv, False, 1)
    wt_hi, wt_lo, wt_inv = rpn_train.pack_weights(conv, True, 1)
    assert w_lo is None and wt_lo is None
    y = rpn_train.conv3x3(x_hi, None, xs, w_hi, None, w_inv, B, H, W, cin, cout, 1).permute(0, 3, 1, 2)
    dx = rpn_train.conv3x3(g_hi, None, gs, wt_hi, None, wt_inv, B, H, W, cout, cin, 1).permute(0, 3, 1, 2)
    dw = rpn_train.wgrad(x_hi, None, xs, g_hi, None, gs, B, H, W, cin, cout, 1)
    return y, dx, dw, (1.0 / float(xs), 1.0 / float(gs), 1.0 / float(w_inv), 1.0 / float(wt_inv))


@pytest.mark.parametrize("name", RPN_CONFIGS)
def test_rpn_layers_against_float64(name):
    for j, (cin, cout, H, W) in enumerate(rpn_shapes(name)):
        what = "%s RPN %d -> %d at %d x %d" % (name, cin, cout, H, W)
        g = torch.Generator(device=DEV).manual_seed(500 + j)
        B = 2
        conv = _dense_layer(cin, cout, g)
        x = torch.relu(torch.randn(B, cin, H, W, device=DEV, generator=g))
        dy = torch.randn(B, cout, H, W, device=DEV, generator=g) * 2.0 ** -20
        y, dx, dw, (sa, sg, ws, wts) = dense_f16(conv, x, dy)
        w = conv.weight.detach()
        check(y, tc_ref.dense_ref(x, w, padding=1), sa, ws, 9 * cin, what + " forward")
        check(dx, tc_ref.dense_ref(dy, w.transpose(0, 1).flip(2, 3).contiguous(), padding=1), sg, wts, 9 * cout,
                 what + " dX")
        check(dw, fr.dense_wgrad_ref(x, dy), sa, sg, B * H * W, what + " dW")
        y2, dx2, dw2, _ = dense_f16(conv, x, dy)
        for a, b, part in ((y, y2, "forward"), (dx, dx2, "dX"), (dw, dw2, "dW")):
            assert torch.equal(_bits(a), _bits(b)), "%s %s: two runs differ" % (what, part)


# ---- splits and packs ------------------------------------------------------------------------------------------------
def _with_nonfinite(t):
    t = t.clone()
    flat = t.view(-1)
    flat[3], flat[17], flat[40] = float("inf"), float("-inf"), float("nan")
    return t


def test_single_planes_equal_the_hi_planes(product):
    """b2s_split_f16_autoscale_ex, b2s_split_halo_f16_autoscale_ex, b2s_pack_sparse_weights_ex and
    b2s_pack_conv2d_weights_ex with products 1 write the hi plane (and the scale) of the products 3 calls, bit for bit"""
    from b2second import rpn_train
    sp = product
    g = torch.Generator(device=DEV).manual_seed(9)
    for n, c, cp, mag in ((1000, 4, 8, 1.0), (777, 16, 16, 2.0 ** -30), (513, 64, 64, 2.0 ** 20), (0, 32, 32, 1.0)):
        x = torch.randn(n, c, device=DEV, generator=g) * mag
        if n:
            x = _with_nonfinite(x)
        h3, _, s3_, sc3 = sp._GradSplit(x, cp, 3).planes()
        h1, l1, s1_, sc1 = sp._GradSplit(x, cp, 1).planes()
        assert l1 is None and torch.equal(_bits(h1[:n]), _bits(h3[:n])) and torch.equal(_bits(sc1), _bits(sc3)), (n, c)
    for K, cin, cout in ((27, 4, 16), (27, 16, 32), (3, 64, 64), (27, 32, 64)):
        w = torch.randn(K, cin, cout, device=DEV, generator=g) * 0.1
        w.view(-1)[5] = float("inf")
        for transpose, flip in ((False, False), (True, False), (True, True)):
            if transpose and cout not in (8, 16, 32, 64):
                continue
            p3 = sp._pack_tc_weights(w, transpose, flip, 3)
            p1 = sp._pack_tc_weights(w, transpose, flip, 1)
            assert p1[1] is None and torch.equal(_bits(p1[0]), _bits(p3[0]))
            assert torch.equal(_bits(p1[2]), _bits(p3[2])) and torch.equal(_bits(p1[3]), _bits(p3[3]))
    for layout in ("nchw", "nhwc"):
        x = torch.randn(2, 64, 13, 21, device=DEV, generator=g) * 2.0 ** -12
        x = _with_nonfinite(x)
        if layout == "nhwc":
            x = x.contiguous(memory_format=torch.channels_last)
        h3, _, s3 = rpn_train.split_halo(x)
        h1, l1, s1 = rpn_train.split_halo(x, products=1)
        assert l1 is None and torch.equal(_bits(h1), _bits(h3)) and torch.equal(_bits(s1), _bits(s3))
    for cin, cout in ((64, 64), (128, 256), (256, 128)):
        conv = _dense_layer(cin, cout, g)
        for transpose in (False, True):
            a = rpn_train.pack_weights(conv, transpose, 3)
            b = rpn_train.pack_weights(conv, transpose, 1)
            assert b[1] is None and torch.equal(_bits(b[0]), _bits(a[0])) and torch.equal(_bits(b[2]), _bits(a[2]))


# ---- Inf and NaN -----------------------------------------------------------------------------------------------------
def _check_nonfinite(got, finite, what):
    bad = torch.isfinite(got) != finite
    assert not bool(bad.any()), "%s: %d elements finite where fp32 is not or the reverse (expected %d non-finite)" % (
        what, int(bad.sum()), int((~finite).sum()))


@pytest.mark.parametrize("val", [float("inf"), float("-inf"), float("nan")], ids=["+inf", "-inf", "nan"])
def test_nonfinite_dy_passes_through(product, val):
    """1-3 poisoned elements of dY: dX and dW are non-finite exactly where fp32 arithmetic makes them so, and the rest
    meets the f16 bound of the same inputs with the poisoned elements set to 0"""
    sp = product
    rng = np.random.default_rng(3)
    g = torch.Generator(device=DEV).manual_seed(3)
    # dense 3x3, poisoned pixels at least 2 from the border
    B, cin, cout, H, W = 2, 64, 128, 29, 37
    conv = _dense_layer(cin, cout, g)
    x = torch.relu(torch.randn(B, cin, H, W, device=DEV, generator=g))
    dy = torch.randn(B, cout, H, W, device=DEV, generator=g) * 2.0 ** -20
    pts = [(int(rng.integers(B)), int(rng.integers(cout)), int(rng.integers(2, H - 2)), int(rng.integers(2, W - 2)))
           for _ in range(3)]
    clean = dy.clone()
    for p in pts:
        dy[p] = val
    _, dx, dw, (sa, sg, ws, wts) = dense_f16(conv, x, dy)
    bad_dx = torch.zeros_like(dx, dtype=torch.bool)
    bad_dw = torch.zeros_like(dw, dtype=torch.bool)
    for b, c, yy, xx in pts:
        bad_dx[b, :, yy - 1:yy + 2, xx - 1:xx + 2] = True
        bad_dw[c] = True
    _check_nonfinite(dx, ~bad_dx, "dense dX")
    _check_nonfinite(dw, ~bad_dw, "dense dW")
    w = conv.weight.detach()
    check(dx, tc_ref.dense_ref(clean, w.transpose(0, 1).flip(2, 3).contiguous(), padding=1), sg, wts, 9 * cout,
             "dense dX (finite part)", ~bad_dx)
    check(dw, fr.dense_wgrad_ref(x, clean), sa, sg, B * H * W, "dense dW (finite part)", ~bad_dw)
    # sparse: poisoned rows with every neighbour present
    n_in, n_out, K, cin, cout = 3000, 2500, 27, 32, 64
    x = torch.relu(torch.randn(n_in, cin, device=DEV, generator=g))
    w = torch.randn(K, cin, cout, device=DEV, generator=g) * (2.0 / (K * cin)) ** 0.5
    nbr = _table(g, n_out, n_in, K)
    full = torch.randint(0, n_in, (3, K), device=DEV, generator=g, dtype=torch.int32)
    rows = rng.choice(n_out, 3, replace=False)
    nbr[torch.from_numpy(rows).to(DEV)] = full
    nbrT = _table(g, n_in, n_out, K)
    dy = torch.randn(n_out, cout, device=DEV, generator=g) * 2.0 ** -20
    clean = dy.clone()
    chans = rng.integers(cout, size=3)
    dy[torch.from_numpy(rows).to(DEV), torch.from_numpy(chans).to(DEV)] = val
    g_split = sp._GradSplit(dy, products=1)
    dx, wts = sp_conv(sp, g_split, w, nbrT, n_in, cin, 1, transpose=True)
    dw = sp_wgrad(sp, sp._GradSplit(x, cin, 1), g_split, nbr, cin, cout, 1)
    bad_dx = torch.zeros_like(dx, dtype=torch.bool)
    bad_dw = torch.zeros_like(dw, dtype=torch.bool)
    for o, co in zip(rows, chans):
        bad_dx[(nbrT.long() == int(o)).any(1)] = True
        bad_dw[:, :, int(co)] = True                     # the row has every neighbour: every (k, ci) pairs with it
    _check_nonfinite(dx, ~bad_dx, "sparse dX")
    _check_nonfinite(dw, ~bad_dw, "sparse dW")
    sg = 1.0 / float(g_split.planes()[3])
    check(dx, tc_ref.sparse_ref(clean, w.transpose(1, 2).contiguous(), nbrT), sg, wts, K * cout,
             "sparse dX (finite part)", ~bad_dx)


# ---- CUDA graphs -----------------------------------------------------------------------------------------------------
def _capture(fn):
    """fn() eagerly, then captured once and replayed twice -> (eager outputs, replayed outputs)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = [t.clone() for t in fn()]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = fn()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    return eager, outs, graph


def test_sparse_middle_encoder_in_a_graph(product):
    """car.fhd's middle encoder in f16 mode: every layer's forward, dX and dW (the drop-in's own functions, on the
    rulebooks of one forward) captured in one CUDA graph, replayed bit for bit"""
    import bench
    from b2second import config, models, training
    sp = product
    name, B = "car.fhd", 2
    cfg = config.get_config(name)
    net = models.build_network(cfg, sp)
    models.synthetic_weights_(net, name, seed=0)
    net = net.to(DEV).train()
    mid = training.enable_sparse_backward(net.middle_feature_extractor, precision="f16")
    feats, coors = [], []
    for b, c in enumerate(bench.make_clouds(name, B, 20000)):
        res = net.voxel_generator.generate(c, cfg.max_voxels)
        n = res["voxel_num"]
        vf = torch.from_numpy(res["voxels"][:n]).sum(1) / torch.from_numpy(res["num_points_per_voxel"][:n]).clamp_min(1)[:, None]
        feats.append(vf[:, :4].float())
        coors.append(torch.from_numpy(np.pad(res["coordinates"][:n], ((0, 0), (1, 0)), constant_values=b)))
    x = sp.SparseConvTensor(torch.cat(feats).to(DEV), torch.cat(coors).int().to(DEV), mid.sparse_shape, B)
    records = []
    with torch.no_grad():
        for m in mid.middle_conv:
            if isinstance(m, sp.SparseConvolution):
                inp = x
                x = m(x)
                records.append((m, inp.features.detach().contiguous().float(), inp.indice_dict[m.indice_key]))
            elif x.indices.shape[0]:
                x.features = m(x.features)
    assert records and all(m._b2s_products == 1 for m, _, _ in records)
    g = torch.Generator(device=DEV).manual_seed(1)
    dys = [torch.randn(rb.num_out, m.out_channels, device=DEV, generator=g) * 2.0 ** -18 for m, _, rb in records]

    def layers():
        outs = []
        for (m, f, rb), dy in zip(records, dys):
            y, xs = m._forward_rows(f, rb)
            gs = sp._GradSplit(dy, products=1)
            outs += [y, m._dgrad(dy, m.weight, rb, f.shape[0], gs), m._wgrad(f, dy, rb, gs, xs)]
        return outs

    eager, outs, graph = _capture(layers)
    assert len(outs) == 3 * len(records)
    for i, (a, b) in enumerate(zip(eager, outs)):
        assert torch.equal(_bits(a), _bits(b)), "layer %d output %d differs after graph replay" % (i // 3, i % 3)
    del graph


@pytest.mark.parametrize("name", RPN_CONFIGS)
def test_rpn_forward_backward_in_a_graph(name):
    """the RPN in train() with its 3x3 layers in f16 mode: forward + backward captured in one CUDA graph, replayed with
    the eager run's bits (cuDNN deterministic for the torch layers)"""
    from b2second import config, loader, models, rpn_train, training
    cfg = config.get_config(name)
    net = models.build_network(cfg, loader.product_spconv())
    models.synthetic_weights_(net, name, seed=0)
    net = training.enable_rpn_training(net.to(DEV), precision="f16")
    rpn = net.rpn.train()
    assert all(c._b2s_products == 1 for c, _ in rpn_train.select(rpn))
    first = rpn.blocks[0][1]
    H, W = (int(v) * first.stride[0] for v in cfg.feature_map_size[1:])
    g = torch.Generator(device=DEV).manual_seed(2)
    x = (torch.relu(torch.randn(2, first.in_channels, H, W, device=DEV, generator=g)) *
         (torch.rand(2, 1, H, W, device=DEV, generator=g) < 0.15)).requires_grad_(True)
    with torch.no_grad():
        out = rpn(x)
    G = {k: torch.randn(v.shape, device=DEV, generator=g) for k, v in out.items()}
    params = [p for p in rpn.parameters() if p.requires_grad]
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        def step():
            o = rpn(x)
            loss = sum((o[k] * G[k]).sum() for k in G)
            return [loss.detach()] + list(torch.autograd.grad(loss, [x] + params))

        eager, outs, graph = _capture(step)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved
    for i, (a, b) in enumerate(zip(eager, outs)):
        assert torch.equal(_bits(a), _bits(b)), "%s: output %d differs after graph replay" % (name, i)
    del graph


# ---- a short training comparison --------------------------------------------------------------------------------------
def train_curve(product, name, B, precision, steps):
    """losses of `steps` optimizer steps of the mirror network (seed-0 weights) on one fixed synthetic batch"""
    import bench
    import optim_ref as orf
    import train_ref as tr
    from b2second import config, inputs, loss, models, optim, targets, training
    cfg = config.get_config(name)
    net = models.build_network(cfg, product)
    models.synthetic_weights_(net, name, seed=0)
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV), precision=precision))
    net = training.enable_rpn_training(net, precision=precision).train()
    opt = optim.plan(net, orf.ONE_CYCLE, steps)
    plan = targets.plan(net.target_assigner, cfg.feature_map_size)
    clouds = bench.make_clouds(name, B, 29000)
    gen = product.utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range, cfg.max_points_per_voxel,
                                         cfg.max_voxels)
    offs = np.cumsum([0] + [c.shape[0] for c in clouds]).astype(np.int32)
    pts = torch.from_numpy(np.concatenate(clouds, 0)).to(DEV)
    res = gen.generate_device(pts, cfg.max_voxels, frame_offsets=torch.from_numpy(offs).to(DEV), batch=B)
    n = int(res["num_voxels"][0].item())
    ex = {"voxels": res["voxels"][:n], "num_points": res["num_points_per_voxel"][:n],
          "coordinates": res["coordinates"][:n]}
    mask = None
    if cfg.anchor_area_threshold >= 0:
        mask = inputs.anchor_area_mask(ex["coordinates"], B, plan.anchors, cfg.voxel_size, cfg.point_cloud_range,
                                       cfg.grid_size, cfg.anchor_area_threshold)
    rng = np.random.default_rng(1)
    frames = [tr.gt_boxes(plan, rng, "ordinary") for _ in range(B)]
    gt = np.concatenate([f[0] for f in frames])
    cls = np.concatenate([f[1] for f in frames])
    imp = np.concatenate([f[2] for f in frames])
    goffs = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
    ex.update(plan.assign_batch(torch.from_numpy(gt).to(DEV), torch.from_numpy(goffs).to(DEV),
                                torch.from_numpy(cls).to(DEV), torch.from_numpy(imp).to(DEV), mask))
    ex["anchors"] = torch.from_numpy(net.anchors().reshape(-1, 7)).to(DEV)[None].repeat(B, 1, 1)
    losses = []
    for _ in range(steps):
        ret = net(dict(ex))
        ret["loss"].backward()
        opt.step()
        losses.append(ret["loss"].detach())
    return [float(v) for v in torch.stack(losses).cpu()]


@pytest.mark.timeout(900)
def test_training_curves(product, out_dir):
    steps = 100
    curves = {}
    for name, B in (("car.fhd", 4), ("pointpillars.car.xyres_16", 2)):
        for precision in ("fp32", "f16"):
            c = train_curve(product, name, B, precision, steps)
            curves["%s/%s" % (name, precision)] = c
            assert np.isfinite(c).all(), "%s %s: a loss is not finite" % (name, precision)
            assert np.mean(c[-10:]) < np.mean(c[:10]), "%s %s: the loss does not decrease (%r ... %r)" % (
                name, precision, c[:3], c[-3:])
        torch.cuda.empty_cache()
    with open(os.path.join(out_dir, "f16_training_curves.json"), "w") as f:
        json.dump(curves, f)
    for k, c in curves.items():
        print("%s: %s" % (k, " ".join("%.4f" % v for v in c[::10] + [c[-1]])))
