"""GPU tests of the training tensor-pipe convolutions at the edges of the fp32 range: the automatically scaled splits
bit for bit against the numpy model of tests/train_range_ref.py, the sparse training layer (enable_sparse_backward) and
the RPN's Conv3x3TC against float64 across the fp32 exponent range, Inf and NaN carried through every layer where
torch's fp32 arithmetic carries them, a whole car.fhd training step with a non-finite input, and the weight packs at
the exponent clamp."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import optim_ref as orf
import tc_ref
import train_range_ref as trr
from b2second import config, loader, loss, metrics, models, optim, rpn_train, tc, training

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16_SENT = 0x5A5A            # a finite fp16 pattern no split of these inputs writes


@pytest.fixture
def fp32_torch():
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _lib():
    sp = loader.product_spconv()
    return sp, sp._lib, sp._lib.load()


def _assert_planes(got_hi, got_lo, want_hi, want_lo, what):
    gh, gl = got_hi.cpu().numpy(), got_lo.cpu().numpy()
    assert trr.same_bits(gh, want_hi), what + ": hi plane"
    assert trr.same_bits(gl, want_lo), what + ": lo plane"


# ---- A. the split rule, bit for bit ------------------------------------------------------------------------------
CASES = trr.crafted_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_split_rows_autoscale_bits(name):
    """b2s_split_f16_autoscale: 6 live rows of 5 floats into 8 channels (3 padded) of an interleaved [row][hi | lo]
    buffer; two rows past num_rows_dev hold inf, NaN and FLT_MAX and change nothing, their planes stay untouched"""
    _, L, lib = _lib()
    x = CASES[name]
    rows, cols = x.shape
    dead = np.array([[np.inf, np.nan, trr.FLT_MAX, -np.inf, 1.0], [np.nan] * 5], np.float32)
    xd = torch.from_numpy(np.concatenate([x, dead])).to(DEV)
    buf = torch.full((rows + 2, 2, 8), 0, dtype=torch.int16, device=DEV).fill_(F16_SENT).view(torch.float16)
    sc = torch.full((2,), 7.0, device=DEV)
    n_dev = torch.tensor([rows], dtype=torch.int32, device=DEV)
    L.check(lib.b2s_split_f16_autoscale(L.ptr(xd), L.ptr(buf[:, 0]), L.ptr(buf[:, 1]), L.ptr(n_dev), rows + 2, cols,
                                        8, 16, L.ptr(sc), L.stream()), "b2s_split_f16_autoscale")
    torch.cuda.synchronize()
    e = trr.exponent(x)
    hi, lo = trr.split(x, e)
    pad = np.zeros((rows, 3), np.float16)
    _assert_planes(buf[:rows, 0], buf[:rows, 1], np.concatenate([hi, pad], 1), np.concatenate([lo, pad], 1), name)
    assert bool((buf[rows:].view(torch.int16) == F16_SENT).all()), "rows past num_rows_dev were written"
    assert float(sc[0]) == 2.0 ** -e


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_split_halo_autoscale_bits(name, layout):
    """b2s_split_halo_f16_autoscale of a [1, 16, 3, 5] map holding the crafted values twice over: interior bits of the
    model, a zero halo, 2^-e, and B2S_STATUS_F16_RANGE exactly when an element is not finite"""
    _, L, lib = _lib()
    v = CASES[name].ravel()
    B, C, H, W = 1, 16, 3, 5
    flat = np.resize(np.concatenate([v, v[::-1]]), B * C * H * W)
    flat[-1] = v[-1]                                                   # the last element of the map: the case's last
    x = torch.from_numpy(flat.reshape(B, C, H, W).astype(np.float32)).to(DEV)
    if layout == "nhwc":
        x = x.contiguous(memory_format=torch.channels_last)
    planes = torch.full((2, B, H + 2, W + 2, C), 0, dtype=torch.int16, device=DEV).fill_(F16_SENT).view(torch.float16)
    sc = torch.full((2,), 7.0, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    L.check(lib.b2s_split_halo_f16_autoscale(L.ptr(x), 0 if layout == "nchw" else 1, B, C, H, W, L.ptr(planes[0]),
                                             L.ptr(planes[1]), L.ptr(sc), L.ptr(status), L.stream()),
            "b2s_split_halo_f16_autoscale")
    torch.cuda.synchronize()
    xn = x.cpu().numpy()
    e = trr.exponent(xn)
    hi, lo = trr.split(xn.transpose(0, 2, 3, 1), e)                    # NHWC interior
    _assert_planes(planes[0, :, 1:-1, 1:-1], planes[1, :, 1:-1, 1:-1], hi, lo, name)
    ring = torch.ones(H + 2, W + 2, dtype=torch.bool)
    ring[1:-1, 1:-1] = False
    assert bool((planes[:, :, ring].view(torch.int16) == 0).all()), "halo not zero"
    assert float(sc[0]) == 2.0 ** -e
    assert (int(status.item()) & 16 != 0) == (not np.isfinite(xn).all()), int(status.item())


def test_inference_split_saturates():
    """b2s_split_f16 (inference) keeps its contract: +-inf saturate to +-65504 in both planes, NaN stays NaN"""
    _, L, lib = _lib()
    x = torch.tensor([[np.inf, -np.inf, np.nan, 70000.0, 1.0, 0, 0, 0]], dtype=torch.float32, device=DEV)
    buf = torch.zeros(1, 2, 8, dtype=torch.float16, device=DEV)
    L.check(lib.b2s_split_f16(L.ptr(x), L.ptr(buf[:, 0]), L.ptr(buf[:, 1]), None, 1, 8, 8, 16, L.stream()),
            "b2s_split_f16")
    hi, lo = buf[0, 0].cpu().double().numpy(), buf[0, 1].cpu().double().numpy()
    assert hi[0] == 65504 and lo[0] == 65504 and hi[1] == -65504 and lo[1] == -65504
    assert np.isnan(hi[2]) and hi[3] == 65504 and lo[3] == 4496 and hi[4] == 1 and lo[4] == 0


# ---- shared helpers of B, C, E -------------------------------------------------------------------------------------
def _check(got, ref, ws, k, what, mask=None):
    """tc_ref.assert_accurate of got * 2^k against ref (both in the scaled domain), on the elements of `mask`.  An fp32
    output rounded in the subnormal range is off by up to 2^-149 before the scaling: that much is taken off the error
    first (torch's fp32 result has the same rounding)."""
    g = got.detach().double() * 2.0 ** k
    y = ref.y
    if mask is not None:
        g, ref = g[mask], tc_ref.Ref(*[f[mask] for f in ref])
        y = ref.y
    d = g - y
    g = y + torch.sign(d) * (d.abs() - 2.0 ** (k - 149)).clamp_min(0.0)
    return tc_ref.assert_accurate(g, ref, ws, what)


def _scaled_exp(t):
    return trr.exponent(t.detach().cpu().numpy())


def _zero_nonfinite(t):
    return torch.where(torch.isfinite(t), t, torch.zeros_like(t))


# ---- sparse layer (enable_sparse_backward) -------------------------------------------------------------------------
SPARSE_SHAPE, SPARSE_BATCH = (20, 40, 40), 2


def _sparse_coords(seed):
    """random voxels and a dense 9^3 cube in batch 0 (rows whose every neighbour is present, in both tables)"""
    rng = np.random.default_rng(seed)
    D, H, W = SPARSE_SHAPE
    flat = rng.choice(SPARSE_BATCH * D * H * W, size=2500, replace=False)
    b, r = np.divmod(flat, D * H * W)
    z, r = np.divmod(r, H * W)
    y, x = np.divmod(r, W)
    cz, cy, cx = np.meshgrid(np.arange(5, 14), np.arange(10, 19), np.arange(10, 19), indexing="ij")
    cube = np.stack([np.zeros(cz.size, int), cz.ravel(), cy.ravel(), cx.ravel()], 1)
    idx = np.unique(np.concatenate([np.stack([b, z, y, x], 1), cube]).astype(np.int32), axis=0)
    return torch.from_numpy(idx[rng.permutation(idx.shape[0])]).to(DEV), rng


def _sparse_layer(cin, cout, table, seed, w=None):
    sp = loader.product_spconv()
    idx, rng = _sparse_coords(seed)
    if table == "subm":
        conv = sp.SubMConv3d(cin, cout, 3, bias=False, indice_key="k")
    else:
        conv = sp.SparseConv3d(cin, cout, 3, 2, padding=1, bias=False)
    if w is None:
        w = torch.from_numpy(rng.uniform(-1, 1, (27, cin, cout)).astype(np.float32)) * (6.0 / (27 * cin)) ** 0.5
    with torch.no_grad():
        conv.weight.copy_(w.view(conv.weight.shape))
    conv = training.enable_sparse_backward(conv.to(DEV)).train()
    return sp, conv, idx, rng


def _run_sparse(sp, conv, feats, idx, dy_of):
    """-> (forward rows, dX, dW [K, Cin, Cout], nbr, dY) through _SparseConvFunction"""
    x = feats.detach().clone().requires_grad_(True)
    t = sp.SparseConvTensor(x, idx, SPARSE_SHAPE, SPARSE_BATCH)
    conv.weight.grad = None
    out = conv(t)
    rb = t.indice_dict[conv.indice_key]
    dy = dy_of(rb)
    out.features.backward(dy)
    K = rb.K
    return (out.features.detach(), x.grad.detach(), conv.weight.grad.detach().view(K, conv.in_channels, -1), rb.nbr,
            dy)


def _transpose_table(nbr, n_in):
    """nbrT [n_in, K]: the output row that reads input row i through offset k, -1 if none"""
    n_out, K = nbr.shape
    t = torch.full((n_in, K), -1, dtype=torch.int64, device=nbr.device)
    for k in range(K):
        ok = nbr[:, k] >= 0
        t[nbr[ok, k].long(), k] = torch.nonzero(ok).flatten()
    return t.int()


def _sparse_refs(x, dy, w, nbr):
    """float64 (forward, dX, dW) Refs in the scaled domain of each operand's own exponent, and the exponents"""
    ex, eg = _scaled_exp(x), _scaled_exp(dy)
    xs, gs = _zero_nonfinite(x) * 2.0 ** ex, _zero_nonfinite(dy) * 2.0 ** eg
    fwd = tc_ref.sparse_ref(xs, w, nbr)
    dxr = tc_ref.sparse_ref(gs, w.transpose(1, 2).contiguous(), _transpose_table(nbr, x.shape[0]))
    dwr = tc_ref.wgrad_ref(xs, gs, nbr)
    return fwd, dxr, dwr, ex, eg


SPARSE_PAIRS = [(4, 16), (32, 32), (64, 64)]
EXPS = (-40, -24, -12, 0, 12, 16, 24, 40)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("e", EXPS)
@pytest.mark.parametrize("table", ["subm", "strided"])
@pytest.mark.parametrize("cin,cout", SPARSE_PAIRS)
def test_sparse_layer_magnitudes(cin, cout, table, e):
    """X = randn * 2^e, dY = randn * 2^-e: forward rows, dX and dW of the training layer against float64, checked as
    got * 2^k against the reference of the operands under the split's own exponents k (exact powers of two)"""
    sp, conv, idx, rng = _sparse_layer(cin, cout, table, seed=cin + cout + (table == "subm"))
    g = torch.Generator(device=DEV).manual_seed(e + 100)
    feats = torch.randn(idx.shape[0], cin, device=DEV, generator=g) * 2.0 ** e
    y, dx, dw, nbr, dy = _run_sparse(sp, conv, feats, idx,
                                     lambda rb: torch.randn(rb.num_out, cout, device=DEV, generator=g) * 2.0 ** -e)
    w = conv.weight.detach().view(27, cin, cout)
    ws = tc.pow2_scale(w)
    fwd, dxr, dwr, ex, eg = _sparse_refs(feats, dy, w, nbr)
    _check(y, fwd, ws, ex, "forward")
    _check(dx, dxr, ws, eg, "dX")
    _check(dw, dwr, 1.0, ex + eg, "dW")


# ---- dense RPN layer (Conv3x3TC) -------------------------------------------------------------------------------------
def _dense_layer(cin, cout, seed, w=None):
    g = torch.Generator().manual_seed(seed)
    conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False)
    with torch.no_grad():
        conv.weight.copy_((torch.rand(conv.weight.shape, generator=g) * 2 - 1) * (6.0 / (9 * cin)) ** 0.5
                          if w is None else w)
    conv = conv.to(DEV).train()
    rpn_train.enable(nn.Sequential(conv))
    return conv


def _run_dense(conv, x, dy):
    x = x.detach().clone().requires_grad_(True)
    conv.weight.grad = None
    y = conv(x)
    y.backward(dy)
    return y.detach(), x.grad.detach(), conv.weight.grad.detach().clone()


def _dense_nbr(B, H, W):
    b, h, w = torch.meshgrid(torch.arange(B, device=DEV), torch.arange(H, device=DEV), torch.arange(W, device=DEV),
                             indexing="ij")
    cols = []
    for ky in range(3):
        for kx in range(3):
            hh, ww = h + ky - 1, w + kx - 1
            ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
            cols.append(torch.where(ok, (b * H + hh.clamp(0, H - 1)) * W + ww.clamp(0, W - 1), -1).reshape(-1))
    return torch.stack(cols, 1).int()


def _rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _dense_refs(x, dy, w):
    B, _, H, W = x.shape
    ex, eg = _scaled_exp(x), _scaled_exp(dy)
    xs, gs = _zero_nonfinite(x) * 2.0 ** ex, _zero_nonfinite(dy) * 2.0 ** eg
    fwd = tc_ref.dense_ref(xs, w, padding=1)
    dxr = tc_ref.dense_ref(gs, w.flip(2, 3).transpose(0, 1), padding=1)
    dwr = tc_ref.wgrad_ref(_rows(xs), _rows(gs), _dense_nbr(B, H, W))
    return fwd, dxr, dwr, ex, eg


def _dw_rows(dw):
    """torch [Cout, Cin, 3, 3] -> [9, Cin, Cout], the layout of wgrad_ref"""
    return dw.permute(2, 3, 1, 0).reshape(9, dw.shape[1], dw.shape[0])


DENSE_SHAPES = [(64, 128), (128, 128)]
# (X exponent, dY exponent): dY from 2^-140 (fp32 subnormals) to 2^100, paired so that dW stays in the fp32 range
DENSE_EXPS = list(zip(EXPS, (100, 60, -60, -20, 20, 60, 80, -140)))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("ex,ey", DENSE_EXPS)
@pytest.mark.parametrize("cin,cout", DENSE_SHAPES)
def test_dense_layer_magnitudes(cin, cout, ex, ey):
    """Conv3x3TC on a 2 x 37 x 45 map, X = randn * 2^ex, dY = randn * 2^ey: forward, dX and dW against float64 in the
    scaled domain of the splits"""
    conv = _dense_layer(cin, cout, seed=cin + cout)
    g = torch.Generator().manual_seed(ex * 7 + ey)
    x = (torch.randn(2, cin, 37, 45, generator=g) * 2.0 ** ex).to(DEV)
    dy = (torch.randn(2, cout, 37, 45, generator=g) * 2.0 ** ey).to(DEV)
    y, dx, dw = _run_dense(conv, x, dy)
    w = conv.weight.detach()
    ws = tc.pow2_scale(w)
    fwd, dxr, dwr, kx, kg = _dense_refs(x, dy, w)
    _check(y, fwd, ws, kx, "forward")
    _check(dx, dxr, ws, kg, "dX")
    _check(_dw_rows(dw), dwr, 1.0, kx + kg, "dW")


# ---- C. Inf and NaN per layer --------------------------------------------------------------------------------------
POISONS = [("+inf", float("inf"), 1), ("-inf", float("-inf"), 2), ("nan", float("nan"), 3)]


def _poison_sparse_rows(rng, nbr, count, full):
    """`count` distinct rows; full: rows with every neighbour present (the analogue of keeping away from the border)"""
    cand = torch.nonzero((nbr >= 0).all(1)).flatten().cpu().numpy() if full else np.arange(nbr.shape[0])
    assert cand.size >= count
    return rng.choice(cand, size=count, replace=False)


def _check_nonfinite(got, finite, what):
    """isfinite(got) is exactly `finite` (Inf and NaN not told apart)"""
    bad = torch.isfinite(got) != finite
    assert not bool(bad.any()), "%s: %d elements finite where torch is not or the reverse (expected %d non-finite)" % (
        what, int(bad.sum()), int((~finite).sum()))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("target", ["x", "dy"])
@pytest.mark.parametrize("poison", POISONS, ids=lambda p: p[0])
@pytest.mark.parametrize("table", ["subm", "strided"])
@pytest.mark.parametrize("cin,cout", SPARSE_PAIRS)
def test_sparse_layer_nonfinite(cin, cout, table, poison, target):
    """1-3 elements of X (or dY) set to +inf, -inf or NaN: the non-finite outputs are exactly those torch's fp32
    arithmetic makes non-finite (every channel of a row that reads a poisoned element; every (k, ci, co) that pairs one
    with a partner), the rest meets the float64 bound of the same inputs with the poisoned elements set to 0"""
    name, val, count = poison
    sp, conv, idx, rng = _sparse_layer(cin, cout, table, seed=cin + cout + (table == "subm"))
    g = torch.Generator(device=DEV).manual_seed(count)
    feats = torch.randn(idx.shape[0], cin, device=DEV, generator=g)
    state = {}

    def dy_of(rb):
        dy = torch.randn(rb.num_out, cout, device=DEV, generator=g) * 2.0 ** -20
        if target == "dy":
            rows = _poison_sparse_rows(rng, rb.nbr, count, True)
            chans = rng.integers(cout, size=count)
            dy[torch.from_numpy(rows).to(DEV), torch.from_numpy(chans).to(DEV)] = val
            state["p"] = (rows, chans)
        return dy

    if target == "x":
        rows = rng.choice(idx.shape[0], size=count, replace=False)
        chans = rng.integers(cin, size=count)
        feats[torch.from_numpy(rows).to(DEV), torch.from_numpy(chans).to(DEV)] = val
        state["p"] = (rows, chans)
    y, dx, dw, nbr, dy = _run_sparse(sp, conv, feats, idx, dy_of)
    K = nbr.shape[1]
    rows, chans = state["p"]
    w = conv.weight.detach().view(K, cin, cout)
    nbr_l = nbr.long()
    bad_y = torch.zeros_like(y, dtype=torch.bool)
    bad_dx = torch.zeros_like(dx, dtype=torch.bool)
    bad_dw = torch.zeros_like(dw, dtype=torch.bool)
    if target == "x":
        for i, ci in zip(rows, chans):
            reads = nbr_l == int(i)                                         # [n_out, K]
            bad_y[reads.any(1)] = True
            bad_dw[reads.any(0), int(ci), :] = True
    else:
        nbrT = _transpose_table(nbr, idx.shape[0]).long()
        for o, co in zip(rows, chans):
            bad_dx[(nbrT == int(o)).any(1)] = True
            bad_dw[(nbr_l[int(o)] >= 0), :, int(co)] = True
    _check_nonfinite(y, ~bad_y, "forward")
    _check_nonfinite(dx, ~bad_dx, "dX")
    _check_nonfinite(dw, ~bad_dw, "dW")
    ws = tc.pow2_scale(w)
    fwd, dxr, dwr, ex, eg = _sparse_refs(feats, dy, w, nbr)
    _check(y, fwd, ws, ex, "forward (finite part)", ~bad_y)
    _check(dx, dxr, ws, eg, "dX (finite part)", ~bad_dx)
    _check(dw, dwr, 1.0, ex + eg, "dW (finite part)", ~bad_dw)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("target", ["x", "dy"])
@pytest.mark.parametrize("poison", POISONS, ids=lambda p: p[0])
@pytest.mark.parametrize("cin,cout", DENSE_SHAPES)
def test_dense_layer_nonfinite(cin, cout, poison, target):
    """Conv3x3TC with 1-3 elements of X (or dY) at +inf, -inf or NaN, at least 2 pixels from the border: non-finite
    exactly on the 3x3 neighbourhood of a poisoned pixel (forward, dX) and on its channel's slice of dW; the rest meets
    the float64 bound with the poisoned elements set to 0"""
    name, val, count = poison
    B, H, W = 2, 37, 45
    conv = _dense_layer(cin, cout, seed=cin + cout)
    g = torch.Generator().manual_seed(count)
    rng = np.random.default_rng(count)
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    dy = (torch.randn(B, cout, H, W, generator=g) * 2.0 ** -20).to(DEV)
    t, C = (x, cin) if target == "x" else (dy, cout)
    pts = [(int(rng.integers(B)), int(rng.integers(C)), int(rng.integers(2, H - 2)), int(rng.integers(2, W - 2)))
           for _ in range(count)]
    for p in pts:
        t[p] = val
    y, dx, dw = _run_dense(conv, x, dy)
    bad_y = torch.zeros_like(y, dtype=torch.bool)
    bad_dx = torch.zeros_like(dx, dtype=torch.bool)
    bad_dw = torch.zeros_like(dw, dtype=torch.bool)
    for b, c, yy, xx in pts:
        if target == "x":
            bad_y[b, :, yy - 1:yy + 2, xx - 1:xx + 2] = True
            bad_dw[:, c] = True
        else:
            bad_dx[b, :, yy - 1:yy + 2, xx - 1:xx + 2] = True
            bad_dw[c] = True
    _check_nonfinite(y, ~bad_y, "forward")
    _check_nonfinite(dx, ~bad_dx, "dX")
    _check_nonfinite(dw, ~bad_dw, "dW")
    w = conv.weight.detach()
    ws = tc.pow2_scale(w)
    fwd, dxr, dwr, kx, kg = _dense_refs(x, dy, w)
    _check(y, fwd, ws, kx, "forward (finite part)", ~bad_y)
    _check(dx, dxr, ws, kg, "dX (finite part)", ~bad_dx)
    _check(_dw_rows(dw), dwr, 1.0, kx + kg, "dW (finite part)", ~_dw_rows(bad_dw))


# ---- D. the step guard end to end ----------------------------------------------------------------------------------
@pytest.mark.timeout(900)
@pytest.mark.parametrize("bad", [float("inf"), float("nan")], ids=["inf", "nan"])
def test_nonfinite_voxel_reaches_the_step_guard(bad, fp32_torch, monkeypatch):
    """car.fhd with enable_sparse_backward, enable_gpu_loss, enable_gpu_metrics and enable_rpn_training, one voxel
    feature at +inf (or NaN), stepped by optim.plan, against the same network on the fp32 path (no tensor pipe in the
    sparse convs, the RPN on cuDNN): in both the loss is not finite, B2S_STATUS_OPT_NONFINITE is raised and the same
    parameters turn NaN"""
    from test_gpu_loss import _car_lite_example
    name = "car.fhd"
    cfg = config.get_config(name)
    sp = loader.product_spconv()
    ex = None
    res = []
    for tensor_pipe in (True, False):
        monkeypatch.setattr(sp, "USE_TENSOR_CORES", tensor_pipe)
        net = models.build_network(cfg, sp)
        models.synthetic_weights_(net, name, seed=0)
        net = metrics.enable_gpu_metrics(loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV))))
        if tensor_pipe:
            net = training.enable_rpn_training(net)
        net = net.train()
        if ex is None:
            ex = _car_lite_example(net, cfg)
            ex["voxels"] = ex["voxels"].clone()
            ex["voxels"][17, 0, 0] = bad
        opt = optim.plan(net, orf.ONE_CYCLE, 100)
        r = net(ex)
        r["loss"].backward()
        lossv = float(r["loss"].detach())
        opt.step()
        torch.cuda.synchronize()
        res.append((lossv, int(opt.status.item()), {k: torch.isnan(p.detach()) for k, p in net.named_parameters()}))
    for lossv, status, _ in res:
        assert not np.isfinite(lossv), lossv
        assert status & 256, status
    for k, m in res[1][2].items():
        assert torch.equal(res[0][2][k], m), k


# ---- E. weight packs at the exponent clamp -------------------------------------------------------------------------
WEIGHT_KINDS = {"tiny": (2.0 ** -120, 60), "subnormal": (2.0 ** -130, 70)}


def _weights(shape, kind, seed):
    """max|w| exactly 2^-120, or all weights fp32 subnormals (max 2^-130)"""
    m, _ = WEIGHT_KINDS[kind]
    g = torch.Generator().manual_seed(seed)
    w = (torch.rand(shape, generator=g) * 2 - 1) * m
    w.view(-1)[w.numel() // 2] = -m
    return w


@pytest.mark.parametrize("kind", sorted(WEIGHT_KINDS))
def test_layers_on_weights_at_the_clamp(kind):
    """a sparse and a dense training layer whose weights need the clamped scale 2^126: forward and dX against float64,
    in the domain of the weights times 2^a (so that the reference's weights are normal floats)"""
    m, ea = WEIGHT_KINDS[kind]
    a = 126                                                            # the pack's scale: the clamp
    # sparse SubM 32 -> 32
    w = _weights((27, 32, 32), kind, 1)
    sp, conv, idx, rng = _sparse_layer(32, 32, "subm", seed=5, w=w)
    g = torch.Generator(device=DEV).manual_seed(3)
    feats = torch.randn(idx.shape[0], 32, device=DEV, generator=g) * 2.0 ** ea
    y, dx, dw, nbr, dy = _run_sparse(sp, conv, feats, idx,
                                     lambda rb: torch.randn(rb.num_out, 32, device=DEV, generator=g) * 2.0 ** ea)
    wd = w.to(DEV)
    assert tc.pow2_scale(wd) == 2.0 ** a
    fwd, dxr, _, ex, eg = _sparse_refs(feats, dy, wd * 2.0 ** a, nbr)
    _check(y, fwd, 1.0, ex + a, "sparse forward")
    _check(dx, dxr, 1.0, eg + a, "sparse dX")
    # dense 64 -> 64
    w = _weights((64, 64, 3, 3), kind, 2)
    conv = _dense_layer(64, 64, seed=2, w=w)
    gg = torch.Generator().manual_seed(4)
    x = (torch.randn(1, 64, 21, 19, generator=gg) * 2.0 ** ea).to(DEV)
    dyd = (torch.randn(1, 64, 21, 19, generator=gg) * 2.0 ** ea).to(DEV)
    y, dx, _ = _run_dense(conv, x, dyd)
    fwd, dxr, _, kx, kg = _dense_refs(x, dyd, w.to(DEV) * 2.0 ** a)
    _check(y, fwd, 1.0, kx + a, "dense forward")
    _check(dx, dxr, 1.0, kg + a, "dense dX")
