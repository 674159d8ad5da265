"""Host side of the tensor-core kernels (csrc/conv_tc.cu, conv_tc2.cu, sparse_conv_tc.cu): 3xF16 weight
preparation and the RPN layer plan.

RPNV2 for the sparse-conv configs (second/pytorch/models/rpn.py:467-497 with layer_strides [1], upsample
strides [1]) is: 6 x [Conv3x3 pad1 + BN + ReLU] -> deblock ConvTranspose2d(k=1,s=1) + BN + ReLU -> three 1x1
heads.  Each becomes one b2s_conv2d_tc launch on NHWC halo-padded fp16 hi/lo planes; the three heads are one launch
writing a packed 32-float record per pixel (box | cls | dir | pad) that b2s_decode_filter_strided reads.
"""
import numpy as np
import torch
from torch import nn


def pow2_scale(w):
    """power of two s with max|w| * s in (2^12, 2^13]: fp16 keeps 11 significant bits down to 2^-14, so after this
    scaling the lo plane of every weight above 2^-17 of the largest one is a NORMAL fp16 (full 22-bit split);
    2^13 leaves three binades of head-room below the fp16 maximum.  The kernels multiply by 1/s in the epilogue.
    max|w| is taken over the finite elements (1 when none is non-zero), and the exponent is clamped to [-126, 126] so
    that s and 1/s are normal floats -- the rule of the device-side packs and splits (csrc/autoscale.cuh)."""
    a = w.detach().abs()
    a = a[torch.isfinite(a)]
    m = float(a.max()) if a.numel() else 0.0
    if m <= 0.0:
        return 1.0
    return float(2.0 ** min(max(13 - int(np.ceil(np.log2(m))), -126), 126))


def split_f16(t, scale=1.0):
    """fp32 tensor -> (hi, lo) torch.float16 planes of t*scale: hi = fp16(t*scale), lo = fp16(t*scale - hi)
    (3xF16 split, csrc/tc_common.cuh; the device-side counterpart is b2s_split_f16)."""
    t = t.detach().float().contiguous() * float(scale)
    hi = t.clamp(-65504.0, 65504.0).half()
    lo = (t - hi.float()).clamp(-65504.0, 65504.0).half()
    return hi.contiguous(), lo.contiguous()


def weight_planes(t, scale, products):
    """the weight operand planes of a tensor-core kernel: (hi, lo) of split_f16 for products = 3 (3xF16), (hi, None)
    for products = 1 (the f16 mode: one fp16 plane, bit for bit the hi plane of the 3xF16 split)"""
    hi, lo = split_f16(t, scale)
    return (hi, lo) if products == 3 else (hi, None)


def merge_f16(hi, lo):
    return hi.float() + lo.float()


SPARSE_TC_CIN = (8, 16, 32, 64)      # 3 or 4 input features are zero-padded to 8 (one 16-byte row chunk)
SPARSE_TC_COUT = (16, 32, 64)
SPARSE_BLOCK_K = 64                  # fp16 channels per 128-byte K block


def sparse_tc_cin(cin):
    """channel count the tensor-core sparse kernel sees for a layer with `cin` inputs (None: not covered)."""
    if cin in SPARSE_TC_CIN:
        return cin
    if cin < 8:
        return 8
    return None


def sparse_tc_channels(lib, cin, cout, K):
    """input width the tensor-core sparse kernel sees for a (cin -> cout, K offsets) layer -- sparse_tc_cin(cin) -- or
    None when the layer runs on the fp32 FMA kernel (b2s_sparse_conv): a width the library was not built for
    (b2s_sparse_conv_tc_supported) or more than 27 kernel offsets, which only the FMA kernel covers."""
    cin_tc = sparse_tc_cin(cin)
    if cin_tc is None or K > 27 or not lib.b2s_sparse_conv_tc_supported(cin_tc, cout):
        return None
    return cin_tc


def wants_tile_plan(subm, K):
    """whether a rulebook gets a tile plan (csrc/sparse_plan.cu: rows grouped by neighbourhood shape + per-tile offset
    masks) for b2s_sparse_conv_tc_plan.  SubM rulebooks with more than 3 offsets do: an ``indice_key`` shares them
    between layers.  A strided conv uses its table once, so the plan would cost more than it saves."""
    return bool(subm and K > 3)


def pack_sparse_weights(w):
    """spconv weight [K, Cin, Cout] -> the K-major B operand b2s_sparse_conv_tc expects (fp32, before the split).
    Cin is zero-padded to sparse_tc_cin(Cin).  Cin = 64: [K, Cout, 64].  Cin < 64: PACK = 64/Cin kernel offsets
    share one 128-byte K block, rows packed [ceil(K/PACK), Cout, 64] with column (offset-in-pack * Cin + cin) and
    zero columns past K."""
    K, cin0, cout = w.shape
    cin = sparse_tc_cin(cin0)
    assert cin is not None, "Cin %d is not covered by the tensor-core sparse kernel" % cin0
    wt = torch.zeros(K, cout, cin, dtype=torch.float32, device=w.device)
    wt[:, :, :cin0] = w.detach().float().transpose(1, 2)               # [K, Cout, Cin]
    if cin >= SPARSE_BLOCK_K:
        return wt.contiguous()
    pack = SPARSE_BLOCK_K // cin
    nkb = (K + pack - 1) // pack
    out = torch.zeros(nkb * pack, cout, cin, dtype=wt.dtype, device=wt.device)
    out[:K] = wt
    return out.view(nkb, pack, cout, cin).permute(0, 2, 1, 3).reshape(nkb, cout, SPARSE_BLOCK_K).contiguous()


def _fold_bn2d(bn):
    scale = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).detach().float().contiguous()
    shift = (bn.bias - bn.running_mean * scale).detach().float().contiguous()
    return scale, shift


def _pad_rows(w, n_pad):
    """[taps, Cout, Cin] -> [taps, n_pad, Cin] (zero rows)."""
    taps, cout, cin = w.shape
    if cout == n_pad:
        return w.contiguous()
    out = torch.zeros(taps, n_pad, cin, dtype=w.dtype, device=w.device)
    out[:, :cout] = w
    return out.contiguous()


def _n_pad(cout):
    for n in (32, 64, 128):
        if cout <= n:
            return n
    raise ValueError("Cout %d > 128 not supported by the tensor-core RPN" % cout)


def supported(rpn, heads=None):
    """True when every layer of this RPNV2 (or, with ``heads`` = the spec's [("large", m), ("small", m)], of this
    multi-head network) maps onto b2s_conv2d_tc_ex (channels % 64 == 0, kernels <= 4x4)."""
    try:
        if heads is None:
            plan_rpn(rpn, 64, 64, dry=True)
        else:
            plan_rpn_multihead(rpn, dict(heads), 64, 64, dry=True)
        return True
    except (ValueError, AssertionError, AttributeError):
        return False


def _conv_out(n, k, s, pad):
    return (n + 2 * pad - k) // s + 1


def plan_rpn(rpn, H, W, dry=False, products=3):
    """RPNV2 (second/pytorch/models/rpn.py:469-497 blocks, :264-299 deblocks, :386-420 heads) on an H x W BEV map ->
    {"buffers": {name: (h, w, c)}, "ops": [conv op dicts in execution order], "heads": {...}}.

    Every op is one b2s_conv2d_tc_ex launch: conv k x k / stride / pad, or one (a, c) sub-grid of a k = s
    ConvTranspose2d; output channels are cut into slices of <= 128 (the kernel's n_pad) and `torch.cat` of the
    deblock outputs is a channel offset into the shared "cat" buffer.  ``products`` = 3: 3xF16 weight planes (w_hi,
    w_lo); 1: the f16 mode, w_hi only (w_lo None)."""
    bufs, ops, emit, (cur, h, w), _ = _plan_backbone(rpn, H, W, dry, products)
    heads = [rpn.conv_box, rpn.conv_cls] + ([rpn.conv_dir_cls] if rpn._use_direction_classifier else [])
    offs, stride_s = _emit_heads(emit, heads, cur, "heads", h, w)
    return {"buffers": bufs, "ops": ops, "in_channels": ops[0]["cin"],
            "heads": {"offsets": offs, "stride": stride_s, "H": h, "W": w}}


def plan_rpn_multihead(rpn, heads, H, W, dry=False, products=3):
    """VoxelNetNuscenesMultiHead (second/pytorch/models/net_multi_head.py:121-176) on an H x W BEV map: the RPNNoHead
    backbone up to the concatenated map, then
      large head: its 1x1 box | cls | dir convs packed into one fp32 record per pixel of the concat map ("heads_large");
      small head: a "crop" op (b2s_crop_nhwc: stage 0 cropped by c = round(0.1 H0) on every side into a zero-halo map),
                  three Conv3x3 64 -> 64 + BN + ReLU, and its packed 1x1 heads ("heads_small").
    ``heads`` = {"large": module, "small": module}.  Records wider than 128 channels are two launches (dst_coff 0 / 128).
    -> {"buffers", "ops", "in_channels", "stage0", "crop", "segments": [{"name", "buffer", "offsets", "stride", "H", "W",
    "a_loc"}, large first]} -- the order of the reference's torch.cat, hence of the anchors."""
    bufs, ops, emit, (cur, h, w), (s0, h0, w0) = _plan_backbone(rpn, H, W, dry, products)
    segs = []

    def packed(m, src, name, hh, ww):
        hd = [m.conv_box, m.conv_cls] + ([m.conv_dir_cls] if m._use_direction_classifier else [])
        offs, stride_s = _emit_heads(emit, hd, src, "heads_" + name, hh, ww)
        segs.append({"name": name, "buffer": "heads_" + name, "offsets": offs, "stride": stride_s, "H": hh, "W": ww,
                     "a_loc": int(m._num_anchor_per_loc)})

    large, small = heads["large"], heads["small"]
    packed(large, cur, "large", h, w)
    c0 = bufs[s0][2]
    c = int(np.round(h0 * 0.1))
    hc, wc = h0 - 2 * c, w0 - 2 * c
    assert hc >= 1 and wc >= 1, "stage-0 map too small for the small head's crop"
    bufs["crop"] = (hc, wc, c0)
    ops.append({"kind": "crop", "src": s0, "dst": "crop", "crop": c, "cin": c0, "cout": c0, "Hin": h0, "Win": w0,
                "Hg": hc, "Wg": wc, "Hout": hc, "Wout": wc, "kh": 0, "kw": 0, "taps": 0, "stride": 1, "pad": 0,
                "n_pad": 0, "relu": False, "out_mul": 1, "off_h": 0, "off_w": 0, "dst_coff": 0, "planes": 2,
                "padded": True, "shift": None, "v2": False})
    mods = list(small.net.children())
    assert len(mods) % 3 == 0
    src = "crop"
    for li in range(0, len(mods), 3):
        conv, bn, relu = mods[li:li + 3]
        assert isinstance(conv, nn.Conv2d) and conv.kernel_size == (3, 3) and conv.stride == (1, 1) and \
            conv.padding == (1, 1) and conv.bias is None and conv.groups == 1
        assert isinstance(bn, nn.BatchNorm2d) and isinstance(relu, nn.ReLU)
        wt = conv.weight.detach()
        wt = wt.permute(2, 3, 0, 1).reshape(9, wt.shape[0], wt.shape[1])
        sc, sh = _fold_bn2d(bn)
        dst = "small%s" % "ab"[(li // 3) % 2]
        bufs[dst] = (hc, wc, wt.shape[1])
        emit("head_conv", src, dst, wt, 3, 3, 1, 1, sc, sh, True, hc, wc, hc, wc, hc, wc)
        src = dst
    packed(small, src, "small", hc, wc)
    return {"buffers": bufs, "ops": ops, "in_channels": ops[0]["cin"], "stage0": s0, "crop": c, "segments": segs}


def _emit_heads(emit, heads, src, dst, h, w):
    """box | cls | dir 1x1 convs packed into one fp32 record per pixel (bias as shift, padded to 4 channels);
    -> (channel offsets of the heads in the record, record stride)."""
    wt = torch.cat([hd.weight.detach()[:, :, 0, 0] for hd in heads], 0).unsqueeze(0)     # [1, sum Cout, Cin]
    bias = torch.cat([hd.bias.detach() for hd in heads], 0).float().contiguous()
    pad = (-wt.shape[1]) % 4
    if pad:
        wt = torch.cat([wt, torch.zeros(1, pad, wt.shape[2], device=wt.device, dtype=wt.dtype)], 1)
        bias = torch.cat([bias, torch.zeros(pad, device=bias.device)])
    stride_s = max(32, wt.shape[1])
    emit("heads", src, dst, wt.contiguous(), 1, 1, 1, 0, None, bias, False, h, w, h, w, h, w, planes=1, padded=False)
    offs = np.cumsum([0] + [hd.weight.shape[0] for hd in heads]).tolist()
    return offs, stride_s


def _plan_backbone(rpn, H, W, dry, products=3):
    """blocks + deblocks of an RPN (RPNV2 or RPNNoHead) -> (buffers, ops, emit, (output buffer, h, w),
    (stage-0 buffer, h, w))."""
    bufs, ops = {}, []

    def emit(kind, src, dst, w_t_co_ci, kh, kw, stride, pad, scale, shift, relu, hin, win, hg, wg, hout, wout,
             out_mul=1, off=(0, 0), dst_coff=0, planes=2, padded=True):
        taps, cout, cin = w_t_co_ci.shape
        assert taps == kh * kw and cin % 64 == 0, "input channels must be multiples of 64"
        for c0 in range(0, cout, 128):
            c1 = min(cout, c0 + 128)
            n_pad = _n_pad(c1 - c0)
            d = {"kind": kind, "src": src, "dst": dst, "kh": kh, "kw": kw, "taps": taps, "stride": stride, "pad": pad,
                 "cin": cin, "cout": c1 - c0, "n_pad": n_pad, "relu": relu, "Hin": hin, "Win": win, "Hg": hg, "Wg": wg,
                 "Hout": hout, "Wout": wout, "out_mul": out_mul, "off_h": off[0], "off_w": off[1],
                 "dst_coff": dst_coff + c0, "planes": planes, "padded": padded,
                 "shift": None if shift is None else shift[c0:c1].float().contiguous(),
                 # the weights-stationary N=256 kernel takes this op (conv_tc.cu dispatch)
                 "v2": (kh == 3 and kw == 3 and stride == 1 and pad == 1 and n_pad == 128 and planes == 2 and padded
                        and out_mul == 1)}
            if not dry:
                # weights pre-scaled by a power of two (exact), undone by the epilogue scale
                wp = _pad_rows(w_t_co_ci[:, c0:c1].float(), n_pad)
                ws = pow2_scale(wp)
                d["w_hi"], d["w_lo"] = weight_planes(wp, ws, products)
                d["w_scale"] = ws
                base = torch.ones(c1 - c0, dtype=torch.float32, device=wp.device) if scale is None \
                    else scale[c0:c1].float()
                d["scale"] = (base / ws).contiguous()
            ops.append(d)

    cur, h, w = "in", H, W
    stage0 = None
    ups = []                                   # (buffer, channels) of each deblock output, in order
    up_start = rpn._upsample_start_idx
    cat_hw = None
    up_filters = [list(db.children())[0].out_channels for db in rpn.deblocks]
    for bi, block in enumerate(rpn.blocks):
        mods = list(block.children())
        i, li = 0, 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, nn.ZeroPad2d):
                assert tuple(m.padding) == (1, 1, 1, 1)
                conv, bn, relu = mods[i + 1], mods[i + 2], mods[i + 3]
                assert conv.padding == (0, 0)
                i += 4
            else:
                conv, bn, relu = mods[i], mods[i + 1], mods[i + 2]
                assert conv.padding == (1, 1)
                i += 3
            assert isinstance(conv, nn.Conv2d) and conv.kernel_size == (3, 3) and conv.bias is None
            assert conv.stride[0] == conv.stride[1] and conv.stride[0] in (1, 2, 4)
            assert isinstance(bn, nn.BatchNorm2d) and isinstance(relu, nn.ReLU)
            st = conv.stride[0]
            wt = conv.weight.detach()                                   # [Cout, Cin, 3, 3]
            wt = wt.permute(2, 3, 0, 1).reshape(9, wt.shape[0], wt.shape[1])   # [tap=ky*3+kx, Cout, Cin]
            sc, sh = _fold_bn2d(bn)
            ho, wo = _conv_out(h, 3, st, 1), _conv_out(w, 3, st, 1)
            dst = "b%d%s" % (bi, "ab"[li % 2])
            bufs[dst] = (ho, wo, wt.shape[1])
            emit("block", cur, dst, wt, 3, 3, st, 1, sc, sh, True, h, w, ho, wo, ho, wo)
            cur, h, w = dst, ho, wo
            li += 1
        if bi == 0:
            stage0 = (cur, h, w)
        j = bi - up_start
        if j >= 0:
            up, bn, relu = list(rpn.deblocks[j].children())
            assert up.bias is None and isinstance(bn, nn.BatchNorm2d)
            sc, sh = _fold_bn2d(bn)
            coff = sum(up_filters[:j])
            k = up.kernel_size[0]
            assert up.kernel_size == (k, k) and up.stride == (k, k) and k in (1, 2, 4)
            if isinstance(up, nn.ConvTranspose2d):
                hu, wu = h * k, w * k
                if cat_hw is None:
                    cat_hw = (hu, wu)
                assert cat_hw == (hu, wu), "deblock outputs must share one resolution"
                wt = up.weight.detach()                                  # [Cin, Cout, k, k]
                for a in range(k):
                    for c in range(k):
                        emit("deblock", cur, "cat", wt[:, :, a, c].t().unsqueeze(0).contiguous(), 1, 1, 1, 0, sc, sh, True,
                             h, w, h, w, hu, wu, out_mul=k, off=(a, c), dst_coff=coff)
            else:                                                        # Conv2d(k, stride k): upsample_stride < 1
                hu, wu = _conv_out(h, k, k, 0), _conv_out(w, k, k, 0)
                if cat_hw is None:
                    cat_hw = (hu, wu)
                assert cat_hw == (hu, wu), "deblock outputs must share one resolution"
                wt = up.weight.detach()                                  # [Cout, Cin, k, k]
                wt = wt.permute(2, 3, 0, 1).reshape(k * k, wt.shape[0], wt.shape[1])
                emit("deblock", cur, "cat", wt, k, k, k, 0, sc, sh, True, h, w, hu, wu, hu, wu, dst_coff=coff)
            ups.append(up_filters[j])
    if ups:
        bufs["cat"] = (cat_hw[0], cat_hw[1], sum(ups))
        cur, h, w = "cat", cat_hw[0], cat_hw[1]
    return bufs, ops, emit, (cur, h, w), stage0


# the fields of an op that plan_rpn* derives from the weights: the device operands and the host power of two behind
# "scale"
OP_OPERANDS = ("w_hi", "w_lo", "scale", "shift")


def plan_layout(plan):
    """a plan of plan_rpn* without its weight-derived fields: what the engine's buffers and launches depend on"""
    out = {k: v for k, v in plan.items() if k != "ops"}
    out["ops"] = [{k: v for k, v in op.items() if k not in OP_OPERANDS + ("w_scale",)} for op in plan["ops"]]
    return out


def fusable_tail(plan):
    """True when the program ends with ONE k = s = 1 deblock 128 -> 128 (+BN+ReLU) whose output only feeds the packed heads
    (<= 32 channels): the shape b2s_rpn_tail_tc runs as a single kernel (car.fhd, car.lite; all.fhd packs 104 head
    channels, the multi-scale RPNs concatenate several deblocks)."""
    ops = plan["ops"]
    if len(ops) < 2:
        return False
    d, h = ops[-2], ops[-1]
    return bool(h["kind"] == "heads" and d["kind"] == "deblock" and h["src"] == d["dst"]
                and sum(1 for o in ops if o["dst"] == d["dst"]) == 1
                and (d["kh"], d["kw"], d["stride"], d["out_mul"], d["dst_coff"]) == (1, 1, 1, 1, 0)
                and d["cin"] == 128 and d["cout"] == 128 and d["relu"] and d["planes"] == 2
                and h["cin"] == 128 and h["n_pad"] == 32 and h["planes"] == 1 and not h["relu"])


def background_layers(plan):
    """indices of the leading ops of an RPN program that form a chain of 3x3 stride-1 pad-1 128-out layers starting at
    the BEV input (the ops the weights-stationary kernel takes): background blocks are only tracked through those."""
    idx, src = [], "in"
    for i, op in enumerate(plan["ops"]):
        if op["v2"] and op["src"] == src and op["dst_coff"] == 0 and op["cout"] == op["n_pad"]:
            idx.append(i)
            src = op["dst"]
        else:
            break
    return idx
