"""TEST INFRASTRUCTURE: float64 references of the fused engine's stages, read off the torch modules.

The RPN program of the engine (b2second.tc.plan_rpn / plan_rpn_multihead) is a list of ops, each one launch over one
buffer.  ``rpn_refs`` walks the modules on its own -- blocks (ZeroPad2d + Conv2d + BN + ReLU, or a padded Conv2d),
deblocks (ConvTranspose2d k = s, or Conv2d k = s), the 1x1 heads packed into one record, the multi-head network's crop
and small-head convs -- and returns one float64 layer per op, in the order the ops run: the weights come from the
modules, never from the packed w_hi / w_lo, and BatchNorm is folded in float64.  ``op_ref`` applies one such layer to
an NHWC map and returns a tests/tc_ref.py ``Ref`` over the op's output grid.

BatchNorm fold.  The kernels get scale and shift folded in fp32 (b2second.spec.fold_bn, b2second.tc._fold_bn2d):
    s32 = fl(gamma / fl(sqrt(fl(var + fl(eps)))))          sh32 = fl(beta - fl(mean * s32))
With u = 2^-24 and eps <= var + eps: fl(var + fl(eps)) = (var + eps)(1 + t), |t| <= 2u(1 + u); the square root and the
division add one rounding each, so |s32 / s64 - 1| <= 3u + O(u^2) <= 4u.  For the shift,
    sh32 - sh64 = mean (s64 - s32) - mean s32 e4 + e5 (beta - fl(mean s32)),  |e4|, |e5| <= u,
so |sh32 - sh64| <= 5u |mean s64| + u |sh64| + O(u^2) <= 6u |mean s64| + 2u |sh64|.  (``fold_error``; the tests also
check the engine's actual fp32 values against it.)  A layer y = s * acc + sh with |acc| <= S1 = sum |a w| therefore
carries, on top of the 3xF16 bound of tc_ref, the fold term
    E_fold = ds * S1 + dsh,     ds = 4u |s64|,  dsh = 6u |mean s64| + 2u |sh64|,
and ReLU, 1-Lipschitz, keeps it.  (The bound of tc_ref is evaluated with s64 in place of s32: the two differ by 4u
relative, far inside ALPHA's 2x margin.)

Accumulation chains of k_conv_tc.  The tensor pipe's fp32 accumulate is not round-to-nearest: the result of every wgmma
is cut to fp32 toward zero.  tc_ref's ALPHA is calibrated on random-sign data, where those cuts partly cancel; when the
terms of one output share a sign (a constant input, as over the empty background of a PointPillars BEV map after its
first layer) they add up, and ALPHA alone does not cover them.  k_conv_tc reduces K in chains of CHAIN = 4 K blocks
(64 channels of one tap each), each chain in the tensor core's accumulator: per 16-channel step q three wgmmas
(A_lo B_hi, A_hi B_lo, A_hi B_hi), then the chain's accumulator is added to a running fp32 sum with round-to-nearest.
A cut to fp32 toward zero errs by less than one ulp, at most 2^-23 |A| for a result A.  With P_q the exact partial sum
of the chain after step q and S1_q = sum |a w| over the step's 16 channels, the three results of step q are at most
|P_(q-1)| + S1_q, |P_(q-1)| + S1_q and |P_q| in magnitude, and with Q_c the running sum after chain c
    E_chain = |s| (2^-23 sum_q (2 (|P_(q-1)| + S1_q) + |P_q|) + 2^-24 sum_c |Q_c|)
bounds the accumulator cuts and the drains (to first order: the operands are the hi/lo planes, within 2^-22 of a, w).
``op_ref(..., chains=True)`` adds it, computing the reduction in k_conv_tc's order; the ops k_conv3x3_tc2 runs (``v2``)
meet the tc_ref bound without it.

``Check`` accumulates the per-element check of tc_ref (|y - y64| <= ALPHA * unit + rest, plus the extra term) and its
aggregate rms over chunks of frames, and names the worst element: stage, frame, pixel or row, channel.
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

import tc_ref

U = 2.0 ** -24
# k_conv_tc (csrc/conv_tc.cu): K blocks of 64 channels (one tap each), 16-channel MMA steps, chains of 4 K blocks
BLOCK_K, MMA_K, CHAIN = 64, 16, 4


# ---- BatchNorm ---------------------------------------------------------------------------------------------------
def fold64(bn, eps=None):
    """eval-mode BatchNorm -> (scale, shift) in float64.  eps=None: the module's eps."""
    eps = bn.eps if eps is None else eps
    v = bn.running_var.detach().double()
    m = bn.running_mean.detach().double()
    w = bn.weight.detach().double() if bn.weight is not None else torch.ones_like(v)
    b = bn.bias.detach().double() if bn.bias is not None else torch.zeros_like(v)
    s = w / torch.sqrt(v + eps)
    return s, b - m * s


def fold_error(bn):
    """(ds, dsh): per-channel bounds on |s32 - s64| and |sh32 - sh64| of the fp32 fold (module docstring)."""
    s, sh = fold64(bn)
    m = bn.running_mean.detach().double()
    return 4 * U * s.abs(), 6 * U * (m * s).abs() + 2 * U * sh.abs()


# ---- the RPN walk ------------------------------------------------------------------------------------------------
def _conv_taps(w):
    """Conv2d weight [Cout, Cin, kh, kw] -> [taps = ky * kw + kx, Cout, Cin]"""
    return w.detach().double().permute(2, 3, 0, 1).reshape(-1, w.shape[0], w.shape[1])


def _layer(kind, w, k, stride, pad, bn, relu, shift=None, out_mul=1, off=(0, 0), coff=0):
    return {"kind": kind, "w": w, "k": k, "stride": stride, "pad": pad, "bn": bn, "relu": relu, "bias": shift,
            "out_mul": out_mul, "off": off, "coff": coff}


def _block_layers(block):
    """one RPN block -> [conv layer]: a ZeroPad2d pads the conv after it"""
    out, pad, cur = [], 0, None
    for m in block.children():
        if isinstance(m, nn.ZeroPad2d):
            p = m.padding
            assert len(set(p)) == 1
            pad = p[0]
        elif isinstance(m, nn.Conv2d):
            assert m.kernel_size[0] == m.kernel_size[1] and m.stride[0] == m.stride[1] and m.bias is None
            cur = _layer("block", _conv_taps(m.weight), m.kernel_size[0], m.stride[0], pad + m.padding[0], None, False)
            pad = 0
        elif isinstance(m, nn.BatchNorm2d):
            cur["bn"] = m
        elif isinstance(m, nn.ReLU):
            cur["relu"] = True
            out.append(cur)
            cur = None
        else:
            raise AssertionError("unexpected module %s in an RPN block" % type(m).__name__)
    assert cur is None
    return out


def _deblock_layers(deblock, coff):
    """ConvTranspose2d k = s: one 1x1 layer per output sub-grid position (a, c); Conv2d k = s: one strided layer"""
    up, bn, relu = list(deblock.children())
    assert isinstance(bn, nn.BatchNorm2d) and isinstance(relu, nn.ReLU) and up.bias is None
    k = up.kernel_size[0]
    if isinstance(up, nn.ConvTranspose2d):
        w = up.weight.detach().double()                                  # [Cin, Cout, k, k]
        return [_layer("deblock", w[:, :, a, c].t().unsqueeze(0), 1, 1, 0, bn, True, out_mul=k, off=(a, c),
                       coff=coff) for a in range(k) for c in range(k)]
    return [_layer("deblock", _conv_taps(up.weight), k, k, 0, bn, True, coff=coff)]


def _heads_layer(head):
    hd = [head.conv_box, head.conv_cls] + ([head.conv_dir_cls] if head._use_direction_classifier else [])
    w = torch.cat([h.weight.detach().double()[:, :, 0, 0] for h in hd], 0)
    b = torch.cat([h.bias.detach().double() for h in hd], 0)
    return _layer("heads", w.unsqueeze(0), 1, 1, 0, None, False, shift=b)


def _split(layers):
    """a layer -> one op per <= 128 output channels (the kernels' n_pad)"""
    out = []
    for L in layers:
        cout = L["w"].shape[1]
        for c0 in range(0, cout, 128):
            c1 = min(cout, c0 + 128)
            d = dict(L, c0=c0, c1=c1)
            d["w"] = L["w"][:, c0:c1]
            d["coff"] = L["coff"] + c0
            out.append(d)
    return out


def rpn_refs(rpn, heads=None):
    """-> [one float64 layer per op of tc.plan_rpn(rpn) (heads None) / tc.plan_rpn_multihead(rpn, heads)]"""
    layers, coff = [], 0
    for bi, block in enumerate(rpn.blocks):
        layers += _block_layers(block)
        j = bi - rpn._upsample_start_idx
        if j >= 0:
            dl = _deblock_layers(rpn.deblocks[j], coff)
            coff += dl[0]["w"].shape[1]
            layers += dl
    if heads is None:
        return _split(layers + [_heads_layer(rpn)])
    small = heads["small"]
    convs = [dict(c, kind="head_conv") for c in _block_layers(nn.Sequential(*small.net.children()))]
    return _split(layers + [_heads_layer(heads["large"])]) + [{"kind": "crop"}] + \
        _split(convs + [_heads_layer(small)])


def assert_matches_plan(refs, plan):
    """every op of the plan is the layer the walk puts there: kind, kernel, stride, padding, channels, sub-grid"""
    ops = plan["ops"]
    assert len(refs) == len(ops), (len(refs), len(ops))
    for i, (r, op) in enumerate(zip(refs, ops)):
        assert r["kind"] == op["kind"], (i, r["kind"], op["kind"])
        if r["kind"] == "crop":
            continue
        taps, cout, cin = r["w"].shape
        got = (op["kh"], op["kw"], op["stride"], op["pad"], op["cin"], op["cout"], op["out_mul"], op["off_h"],
               op["off_w"], op["dst_coff"], op["relu"])
        want = (r["k"], r["k"], r["stride"], r["pad"], cin, cout, r["out_mul"], r["off"][0], r["off"][1], r["coff"],
                r["relu"])
        assert got == want, (i, op["kind"], got, want)


def scale_shift(r, eps=None):
    """(scale64 or None, shift64 or None, ds, dsh) of one layer over its output channel slice"""
    if r["bn"] is None:
        sh = None if r["bias"] is None else r["bias"][r["c0"]:r["c1"]]
        return None, sh, None, None
    s, sh = fold64(r["bn"], eps)
    ds, dsh = fold_error(r["bn"])
    sl = slice(r["c0"], r["c1"])
    return s[sl], sh[sl], ds[sl], dsh[sl]


def op_ref(x, r, eps=None, chains=False):
    """x [n, H, W, Cin] float64 (the op's source map without its halo) -> (Ref with [n, Hg, Wg, Cout] fields, the extra
    term of the same shape: E_fold, plus E_chain when `chains`).  eps: BatchNorm eps of the fold (None: the module's).
    The reduction runs in the order of k_conv_tc: taps, then 64-channel blocks, then 16-channel MMA steps."""
    w = r["w"].to(x.device)
    k, st, pad = r["k"], r["stride"], r["pad"]
    n, H, W, cin = x.shape
    Hg, Wg = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
    xp = F.pad(x, (0, 0, pad, pad, pad, pad))
    inside = F.pad(torch.ones(n, H, W, 1, dtype=x.dtype, device=x.device), (0, 0, pad, pad, pad, pad))
    cout = w.shape[1]
    y = torch.zeros(n, Hg, Wg, cout, dtype=torch.float64, device=x.device)
    S1, Sa, Sw = y.clone(), y.clone(), y.clone()
    if chains:
        assert cin % BLOCK_K == 0
        part, walk, drain = y.clone(), y.clone(), y.clone()      # chain partial sum P, sum of |A_t|, sum of |Q_c|
    kb = 0
    for t in range(k * k):
        dy, dx = divmod(t, k)
        sl = (slice(None), slice(dy, dy + st * (Hg - 1) + 1, st), slice(dx, dx + st * (Wg - 1) + 1, st))
        a = xp[sl]
        wt = w[t].t()
        Sa += a.abs().sum(-1, keepdim=True)
        Sw += inside[sl] * wt.abs().sum(0)
        if not chains:
            y += a @ wt
            S1 += a.abs() @ wt.abs()
            continue
        for c0 in range(0, cin, MMA_K):
            if c0 % BLOCK_K == 0 and kb % CHAIN == 0 and kb:             # a chain ends: drained into the running sum
                drain += (y + part).abs()
                y += part
                part.zero_()
            if c0 % BLOCK_K == 0:
                kb += 1
            ac, wc = a[..., c0:c0 + MMA_K], wt[c0:c0 + MMA_K]
            step, s1 = ac @ wc, ac.abs() @ wc.abs()
            walk += 2 * (part.abs() + s1) + (part + step).abs()
            part += step
            S1 += s1
    if chains:
        drain += (y + part).abs()
        y += part
    scale, shift, ds, dsh = scale_shift(r, eps)
    ref = tc_ref._finish(y, S1, Sa, Sw, scale, shift, r["relu"], 3)
    extra = torch.zeros_like(y) if ds is None else ds.to(x.device) * S1 + dsh.to(x.device)
    if chains:
        extra = extra + ref.s * (2.0 ** -23 * walk + 2.0 ** -24 * drain)
    return ref, extra


def crop_size(h0):
    return int(np.round(h0 * 0.1))


# ---- the check ---------------------------------------------------------------------------------------------------
class Check:
    """per-element |got - y64| <= ALPHA * unit + rest + extra (tc_ref) over chunks, and the aggregate
    rms((|got - y64| - rest - extra)+) / rms(|s| S1) <= RHO; the failure message names the worst element."""

    def __init__(self, stage, ws):
        self.stage, self.ws = stage, ws
        self.worst, self.where = 0.0, None
        self.ex2, self.den2, self.n = 0.0, 0.0, 0

    def add(self, got, ref, extra, locate):
        """got, ref fields, extra: one shape; locate(index tuple) -> text naming the element"""
        err = (got.to(ref.y.device, torch.float64) - ref.y).abs()
        unit, rest = tc_ref._terms(ref, self.ws)
        rest = rest + extra
        bound = tc_ref.ALPHA * unit + rest
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        ratio = torch.nan_to_num(ratio, nan=float("inf"))
        m = float(ratio.max()) if ratio.numel() else 0.0
        if m > self.worst:
            idx = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
            self.worst = m
            self.where = "%s, |y - y64| = %.4g, bound %.4g, y64 = %.6g" % (
                locate(tuple(int(i) for i in idx)), float(err[idx]), float(bound[idx]), float(ref.y[idx]))
        self.ex2 += float((err - rest).clamp_min(0.0).pow(2).sum())
        self.den2 += float((ref.s * ref.S1).pow(2).sum())
        self.n += err.numel()

    def done(self):
        assert self.worst <= 1.0, "%s: %s reaches %.3g x the bound" % (self.stage, self.where, self.worst)
        rms = (self.ex2 / self.den2) ** 0.5 if self.den2 > 0 else (0.0 if self.ex2 == 0 else float("inf"))
        assert rms <= tc_ref.RHO, "%s: rms error %.3g x rms(|s| S1) over %d elements, above RHO = %.3g" % (
            self.stage, rms, self.n, tc_ref.RHO)
        return self.worst, rms


# ---- chaining the ops --------------------------------------------------------------------------------------------
def dst_channels(plan, name):
    """channels per pixel of an op's destination map: the buffer's, or for a head record the widest op into it"""
    if name in plan["buffers"]:
        return plan["buffers"][name][2]
    return max(op["dst_coff"] + op["cout"] for op in plan["ops"] if op["dst"] == name)


def dst_view(t, op, padded=None):
    """the elements of a destination map [n, Hout(+2), Wout(+2), C] one op writes: its sub-grid and channel slice"""
    p = (1 if op["padded"] else 0) if padded is None else padded
    h0, w0, m = p + op["off_h"], p + op["off_w"], op["out_mul"]
    return t[:, h0:h0 + m * (op["Hg"] - 1) + 1:m, w0:w0 + m * (op["Wg"] - 1) + 1:m,
             op["dst_coff"]:op["dst_coff"] + op["cout"]]


def run_chain(refs, plan, x):
    """x [n, H, W, C] float64 -> {buffer name: float64 map without halo} after every op of the program has run on the
    float64 results of the ops before it"""
    maps = {"in": x}
    n = x.shape[0]
    for r, op in zip(refs, plan["ops"]):
        src = maps[op["src"]]
        if r["kind"] == "crop":
            c = op["crop"]
            assert c == crop_size(src.shape[1])
            maps[op["dst"]] = src[:, c:src.shape[1] - c, c:src.shape[2] - c]
            continue
        if op["dst"] not in maps:
            maps[op["dst"]] = torch.zeros(n, op["Hout"], op["Wout"], dst_channels(plan, op["dst"]),
                                          dtype=torch.float64, device=x.device)
        dst_view(maps[op["dst"]], op, padded=0)[...] = op_ref(src, r)[0].y
    return maps
