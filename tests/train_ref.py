"""TEST INFRASTRUCTURE for tests/test_gpu_train_fp64.py, CPU-importable: the batches of the training sequence (which
special frame sits where), ground-truth boxes drawn near anchors, the rulebook comparison against the oracle's
get_indice_pairs and the exact scatter / gather of the dense() boundary, all in numpy or plain torch.

The special frames of a training batch:
  empty     a cloud without points (its ground truth is ordinary: every anchor of it sees zero features)
  no_gt     points but no ground truth: every anchor negative (or ignored), the loss normaliser clamped to 1
  border    points on the first and last row and column of the BEV map, and boxes on anchors of those rows / columns
  crowded   CROWDED ground-truth boxes
"""
import numpy as np

SPECIALS = ("empty", "no_gt", "border", "crowded")
CROWDED = 64
ORDINARY_GT = 12


def special_layout(B):
    """-> [(step, {position: special})] for the second and third batch of a sequence at batch size B.  Step 1 (the
    second batch) holds the four special frames, spread over the batch, as far as B allows; step 2 (the sparse batch)
    holds them at the first, middle and last position, those step 1 could not place first.  Every special frame
    appears at least once for B >= 2."""
    pos1 = [1, B // 3 + 1, 2 * B // 3, B - 2] if B >= 6 else list(range(min(len(SPECIALS), B)))
    first = dict(zip(pos1, SPECIALS))
    shown = set(first.values())
    order = [s for s in SPECIALS if s not in shown] + [s for s in SPECIALS if s in shown]
    pos2 = sorted({0, B // 2, B - 1})
    second = dict(zip(pos2, order[:len(pos2)]))
    return [(1, first), (2, second)]


def anchor_segments(plan):
    """segment index of every anchor of a b2second.targets.TargetPlan"""
    seg = np.zeros(plan.num_anchors, np.int64)
    for i, s in enumerate(plan.segments):
        seg[s.begin:s.end] = i
    return seg


def border_anchors(plan):
    """indices of the anchors centred on the first or last BEV row or column of the anchor grid, per side"""
    a = plan.anchors
    out = []
    for col, fn in ((0, np.min), (0, np.max), (1, np.min), (1, np.max)):
        v = a[:, col]
        out.append(np.flatnonzero(v == fn(v)))
    return out


def gt_boxes(plan, rng, kind):
    """-> (boxes float32 [G, 7], classes int32 [G] (1-based), importance float32 [G]) for one frame: boxes copied from
    anchors, moved by up to 0.5 m in x and y, with a random yaw (as the loss tests draw them); `kind` a special frame
    name or "ordinary".  In per-class plans a box's class is its anchor's."""
    if kind == "no_gt":
        return np.zeros((0, 7), np.float32), np.zeros(0, np.int32), np.zeros(0, np.float32)
    if kind == "border":
        idx = np.concatenate([rng.choice(side, 4, replace=False) for side in border_anchors(plan)])
    else:
        idx = rng.integers(0, plan.num_anchors, CROWDED if kind == "crowded" else ORDINARY_GT)
    gt = plan.anchors[idx, :7].astype(np.float32).copy()
    gt[:, :2] += rng.uniform(-0.5, 0.5, (len(idx), 2)).astype(np.float32)
    gt[:, 6] = rng.uniform(-np.pi, np.pi, len(idx)).astype(np.float32)
    cls = (anchor_segments(plan)[idx] + 1 if plan.assign_per_class else np.ones(len(idx))).astype(np.int32)
    imp = rng.uniform(0.5, 2.0, len(idx)).astype(np.float32)
    return gt, cls, imp


def compare_rulebook(cin, cout, nbr, frame, o_out, pairs, pnum):
    """one frame of a rulebook against the oracle's get_indice_pairs on the frame's input coordinates.
    cin [n_in, 4] / cout [n_out, 4] (b, z, y, x) and nbr [n_out, K] of the layer (numpy); o_out, pairs, pnum the
    oracle's result for the frame alone.  The output rows of the frame must be the oracle's set of coordinates (the
    drop-in's order within a frame is its own), and every row's neighbour through every offset the oracle's.
    -> None, or a message naming the first difference."""
    ri = np.flatnonzero(cin[:, 0] == frame)
    ro = np.flatnonzero(cout[:, 0] == frame)
    if len(ro) != o_out.shape[0]:
        return "frame %d: %d output rows, the oracle %d" % (frame, len(ro), o_out.shape[0])
    key = lambda c: (c[:, 0].astype(np.int64) * 65536 + c[:, 1]) * 65536 + c[:, 2]      # noqa: E731  (z, y, x)
    ours = key(cout[ro, 1:].astype(np.int64))
    theirs = key(o_out[:, 1:].astype(np.int64))
    order = np.argsort(ours)
    pos = np.searchsorted(ours[order], theirs)
    pos = np.minimum(pos, len(ours) - 1) if len(ours) else pos
    if len(theirs) and not np.array_equal(ours[order][pos], theirs):
        return "frame %d: output coordinates differ from the oracle's" % frame
    row_of = ro[order[pos]]                                   # our row of each oracle output row
    K = nbr.shape[1]
    want = np.full((len(cout), K), -1, np.int64)
    for k in range(K):
        want[row_of[pairs[k, 1, :pnum[k]]], k] = ri[pairs[k, 0, :pnum[k]]]
    got = nbr[ro].astype(np.int64)
    bad = np.argwhere(got != want[ro])
    if bad.size:
        r, k = bad[0]
        return "frame %d: row %d offset %d is %d, the oracle %d" % (frame, ro[r], k, got[r, k], want[ro][r, k])
    return None


def scatter_rows(rows, idx, B, D, H, W):
    """dense() of fp32 rows [n, C] at (b, z, y, x): [B, C, D, H, W], zero elsewhere (torch, exact)"""
    import torch
    out = torch.zeros(B, rows.shape[1], D, H, W, dtype=rows.dtype, device=rows.device)
    i = idx.long()
    out[i[:, 0], :, i[:, 1], i[:, 2], i[:, 3]] = rows
    return out


def gather_rows(dmap, idx):
    """the backward of scatter_rows: the gradient of every row gathered at its position"""
    i = idx.long()
    return dmap[i[:, 0], :, i[:, 1], i[:, 2], i[:, 3]]


# ---- float64 references of the training convolutions, in the domain of the splits' power-of-two scales ---------------
# The training splits (b2s_split_f16_autoscale, b2s_split_halo_f16_autoscale) scale each operand by 2^e with e the
# exponent of tests/train_range_ref.py; the kernels undo it exactly.  Checked in that domain, the tc_ref bound's
# absolute 2^-25 terms mean what they mean for operands of magnitude up to 2^13.

def exponent(t):
    import train_range_ref as trr
    return trr.exponent(t.detach().cpu().numpy())


def scaled(t, k):
    """float64 t * 2^k with non-finite elements set to 0"""
    import torch
    return torch.where(torch.isfinite(t), t, torch.zeros_like(t)).double() * 2.0 ** k


def rows(t):
    """[B, C, H, W] -> [B*H*W, C] pixel rows"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def dense_nbr(B, H, W, device):
    """[B*H*W, 9] input pixel of each output pixel and tap (ky * 3 + kx) of a pad-1 3x3 conv, -1 past the border"""
    import torch
    b, h, w = torch.meshgrid(torch.arange(B, device=device), torch.arange(H, device=device),
                             torch.arange(W, device=device), indexing="ij")
    cols = []
    for ky in range(3):
        for kx in range(3):
            hh, ww = h + ky - 1, w + kx - 1
            ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
            cols.append(torch.where(ok, (b * H + hh.clamp(0, H - 1)) * W + ww.clamp(0, W - 1), -1).reshape(-1))
    return torch.stack(cols, 1).int()


def dw_rows(dw):
    """torch [Cout, Cin, 3, 3] -> [9, Cin, Cout], the layout of tc_ref.wgrad_ref"""
    return dw.permute(2, 3, 1, 0).reshape(9, dw.shape[1], dw.shape[0])


def transpose_table(nbr, n_in):
    """nbrT [n_in, K]: the output row that reads input row i through offset k, -1 if none"""
    import torch
    n_out, K = nbr.shape
    t = torch.full((n_in, K), -1, dtype=torch.int64, device=nbr.device)
    for k in range(K):
        ok = nbr[:, k] >= 0
        t[nbr[ok, k].long(), k] = torch.nonzero(ok).flatten()
    return t.int()


def sparse_refs(x, dy, w, nbr):
    """float64 (forward, dX, dW) tc_ref.Refs of a sparse training layer in the scaled domain of each operand's own
    exponent, and the exponents"""
    import tc_ref
    ex, eg = exponent(x), exponent(dy)
    xs, gs = scaled(x, ex), scaled(dy, eg)
    fwd = tc_ref.sparse_ref(xs, w, nbr)
    dxr = tc_ref.sparse_ref(gs, w.transpose(1, 2).contiguous(), transpose_table(nbr, x.shape[0]))
    dwr = tc_ref.wgrad_ref(xs, gs, nbr)
    return fwd, dxr, dwr, ex, eg


def scaled_check(got, ref, ws, k, what, mask=None, extra=None):
    """tc_ref's per-element bound (plus `extra`, a derived term of the same shape) and its aggregate check of got * 2^k
    against ref, both in the scaled domain, on the elements of `mask`.  An fp32 output rounded in the subnormal range
    is off by up to 2^-149 before the scaling: that much is taken off the error first (torch's fp32 result has the
    same rounding).  -> {"ratio", "rms"}: the worst error / bound and the aggregate over RHO's unit"""
    import torch
    import tc_ref
    g = got.detach().double() * 2.0 ** k
    if mask is not None:
        g, ref = g[mask], tc_ref.Ref(*[f[mask] for f in ref])
        extra = None if extra is None else extra[mask]
    d = g - ref.y
    g = ref.y + torch.sign(d) * (d.abs() - 2.0 ** (k - 149)).clamp_min(0.0)
    err = (g - ref.y).abs()
    unit, rest = tc_ref._terms(ref, ws)
    if extra is not None:
        rest = rest + extra
    bound = tc_ref.ALPHA * unit + rest
    ratio, rms = 0.0, 0.0
    if err.numel():
        ratio = float((err / bound).max())
        excess = (err - rest).clamp_min(0.0)
        den = float((ref.s * ref.S1).pow(2).mean().sqrt())
        if den > 0:
            rms = float(excess.pow(2).mean().sqrt()) / den
        elif float(excess.max()) > 0.0:
            rms = float("inf")
    assert ratio <= 1.0, "%s: |y - y64| reaches %.3g x the bound" % (what, ratio)
    assert rms <= tc_ref.RHO, "%s: rms error %.3g x rms(|s| S1), above RHO = %.3g" % (what, rms, tc_ref.RHO)
    return {"ratio": ratio, "rms": rms}


def conv3x3_chain_ref(xs, w):
    """a 3x3 pad-1 conv of Conv3x3TC (forward, or dX with w the flipped transposed weight) as b2s_conv2d_tc_ex with fp32
    output computes it, i.e. on k_conv_tc: xs [B, C, H, W] float64 in the split's scaled domain, w [Cout, Cin, 3, 3]
    -> (tc_ref.Ref with NHWC fields, the accumulation-chain term of engine_ref.op_ref).  k_conv_tc's accumulator cuts
    every wgmma result toward zero; over ReLU outputs (all of one sign) the cuts of one output add up instead of
    cancelling, which tc_ref's ALPHA (calibrated on random-sign data) does not cover."""
    import engine_ref
    r = {"w": w.double().permute(2, 3, 0, 1).reshape(9, w.shape[0], w.shape[1]), "k": 3, "stride": 1, "pad": 1,
         "bn": None, "bias": None, "relu": False, "c0": 0, "c1": w.shape[0]}
    return engine_ref.op_ref(xs.permute(0, 2, 3, 1), r, chains=True)


WG_ROWS, WG_WIDTH, WG_SLAB = 8, 8, 32          # b2s_conv2d_wgrad_tc: 8 x 8-pixel strips, 32 strips per slab partial


def wgrad_chain_term(xs, gs, slabs_per_chunk=8):
    """the accumulation-chain term of the RPN weight gradient (csrc/conv_train.cu, b2s_conv2d_wgrad_tc) for
    dW[tap][ci][co] = sum_px X[px + tap][ci] dY[px][co], xs [B, Cin, H, W] / gs [B, Cout, H, W] float64 in the splits'
    scaled domain -> [9, Cin, Cout] (the layout of tc_ref.wgrad_ref), in the kernel's order:
      strips of 8 rows x 8 pixels, numbered (frame, strip row, strip column); per strip and tap a chain of 4 k16 steps
      (strip rows 2k, 2k + 1: 16 pixels), three wgmmas each (dY_hi X_hi, dY_hi X_lo, dY_lo X_hi) into one accumulator
      that is cut to fp32 toward zero after every wgmma; the chain's result added with round-to-nearest to the tap's
      running sum of its slab (32 strips); the slab partials added in slab order with round-to-nearest.
    With P_q the exact chain sum after step q and S1_q = sum |x g| over step q's pixels, the three results of step q
    are at most |P_(q-1)| + S1_q, |P_(q-1)| + S1_q and |P_q| in magnitude (to first order), a cut errs by less than
    2^-23 of its result and a round-to-nearest add by 2^-24 of its result:
        E = 2^-23 sum_strips sum_q (2 (|P_(q-1)| + S1_q) + |P_q|) + 2^-24 (sum_strips |R_s| + sum_slabs |T_j|)
    with R_s the slab's running sum after strip s and T_j the sum of the slab partials after slab j.  (engine_ref's
    E_chain for k_conv_tc, in this kernel's reduction order.)"""
    import torch
    import torch.nn.functional as F
    B, cin, H, W = xs.shape
    cout = gs.shape[1]
    sh, sw = -(-H // WG_ROWS), -(-W // WG_WIDTH)
    Hs, Ws = sh * WG_ROWS, sw * WG_WIDTH
    n = B * sh * sw

    def strips(t):
        """[B, Hs, Ws, C] -> [n, 4 steps, 16 pixels, C] in the kernel's strip and step order"""
        C = t.shape[-1]
        t = t.view(B, sh, WG_ROWS, sw, WG_WIDTH, C).permute(0, 1, 3, 2, 4, 5)
        return t.reshape(n, WG_ROWS // 2, 2 * WG_WIDTH, C)

    g = F.pad(gs.permute(0, 2, 3, 1), (0, 0, 0, Ws - W, 0, Hs - H))             # past the map: zero terms
    gst, gabs = strips(g), None
    gabs = gst.abs()
    xp = F.pad(xs.permute(0, 2, 3, 1), (0, 0, 1, 1 + Ws - W, 1, 1 + Hs - H))
    out = torch.zeros(9, cin, cout, dtype=torch.float64, device=xs.device)
    chunk = slabs_per_chunk * WG_SLAB
    for ky in range(3):
        for kx in range(3):
            xst = strips(xp[:, ky:ky + Hs, kx:kx + Ws].contiguous())
            walk = torch.zeros(cin, cout, dtype=torch.float64, device=xs.device)
            drain = walk.clone()
            partials = []
            for s0 in range(0, n, chunk):
                s1 = min(n, s0 + chunk)
                a, b = xst[s0:s1], gst[s0:s1]
                step = torch.einsum("spkc,spkd->spcd", a, b)
                s1q = torch.einsum("spkc,spkd->spcd", a.abs(), gabs[s0:s1])
                P = step.cumsum(1)
                walk += (2 * ((P - step).abs() + s1q) + P.abs()).sum((0, 1))
                Q = P[:, -1]
                del step, s1q, P
                for j0 in range(0, s1 - s0, WG_SLAB):
                    R = Q[j0:j0 + WG_SLAB].cumsum(0)
                    drain += R.abs().sum(0)
                    partials.append(R[-1])
            drain += torch.stack(partials).cumsum(0).abs().sum(0)
            out[ky * 3 + kx] = 2.0 ** -23 * walk + 2.0 ** -24 * drain
    return out


def check_conv3x3_train(x, dy, y, dx, dw, w, ws, what, parts=("forward", "dX", "dW")):
    """one Conv3x3TC training layer against float64: y = conv(x, w) and dX (k_conv_tc: the tc_ref bound plus
    conv3x3_chain_ref's term), dW (b2s_conv2d_wgrad_tc: the tc_ref bound plus wgrad_chain_term), each in the domain of
    the splits' scales.  x, dy [B, C, H, W] fp32 (NCHW or channels_last), w [Cout, Cin, 3, 3], ws the weight pack's
    power-of-two scale; dx None: not checked.  -> {part: {"ratio", "rms"}}"""
    kx, kg = exponent(x), exponent(dy)
    xs, gs = scaled(x, kx), scaled(dy, kg)
    out = {}
    if "forward" in parts:
        ref, extra = conv3x3_chain_ref(xs, w)
        out["forward"] = scaled_check(y.permute(0, 2, 3, 1), ref, ws, kx, what + " forward", extra=extra)
        del ref, extra
    if "dX" in parts and dx is not None:
        ref, extra = conv3x3_chain_ref(gs, w.flip(2, 3).transpose(0, 1))
        out["dX"] = scaled_check(dx.permute(0, 2, 3, 1), ref, ws, kg, what + " dX", extra=extra)
        del ref, extra
    if "dW" in parts:
        import tc_ref
        B, _, H, W = x.shape
        ref = tc_ref.wgrad_ref(rows(xs), rows(gs), dense_nbr(B, H, W, x.device))
        out["dW"] = scaled_check(dw_rows(dw), ref, 1.0, kx + kg, what + " dW", extra=wgrad_chain_term(xs, gs))
    return out
