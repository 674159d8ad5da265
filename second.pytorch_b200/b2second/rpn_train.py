"""Training of the RPN's 3x3 stride-1 convolutions on the tensor pipe (csrc/conv_train.cu).

``training.enable_rpn_training(net)`` rebinds the ``forward`` of every covered ``nn.Conv2d`` in a sequential container
under ``net.rpn`` to ``Conv3x3TC`` and the ``forward`` of a ``nn.ZeroPad2d(1)`` directly in front of a covered
``padding=0`` conv to the identity (the pair is one pad-1 conv; the halo of the split input is the pad, so the padded
copy is never built).  A subclass that does not override ``forward`` counts (see ``sequences`` and ``plain``), so the
reference's own ``change_default_args`` convs inside torchplus' ``Sequential`` are covered as well as the mirror's.
Covered: 3x3 kernel, stride 1, no dilation, no groups, no bias, zero padding 1 (or 0 after the pad), ``C_in`` a
multiple of 64, ``C_out`` in {64, 128, 256} -- every 3x3 layer of car.fhd and car.lite and every stride-1 3x3 layer of
all.fhd, xyres_16 and all.pp.largea.  Stride-2 convs, deblocks and heads stay the torch modules; BatchNorm2d + ReLU
pairs are ``enable_bn_relu_training``'s (b2second.bn_train).

The rebound forward takes the kernels only in ``train()`` mode with grad enabled on float32 CUDA input; otherwise it is
``nn.Conv2d.forward`` (and the pad pads), so ``eval()`` and the state dict are unchanged.

Conv3x3TC, all on the caller's stream without a host sync (the layer can be captured):
  forward   x (NCHW or channels_last) -> halo planes of x * 2^ex (b2s_split_halo_f16_autoscale) -> b2s_conv2d_tc_ex with
            the packed weights (b2s_pack_conv2d_weights), fp32 NHWC out, returned as a channels_last NCHW tensor;
  backward  dY -> halo planes of dY * 2^ey -> dX through b2s_conv2d_tc_ex with W'[tap] = W[8 - tap]^T, and dW through
            b2s_conv2d_wgrad_tc from the saved X planes and the dY planes.

``enable(net, products=1)`` (``training.enable_rpn_training(net, precision="f16")``) runs the same layers in the f16 mode:
every plane is the hi plane alone (the ``*_ex`` splits and packs with products = 1), the forward and input gradient are
b2s_conv2d_tc_ex3 launches with products = 1 and fp32 output, and the weight gradient is b2s_conv2d_wgrad_tc_ex with
products = 1 -- one f16 wgmma product per MAC instead of three.  The product count is stored per conv
(``_b2s_products``).
"""
import types

import torch
import torch.nn as nn

from . import loader

LAYOUT_NCHW, LAYOUT_NHWC = 0, 1      # B2S_LAYOUT_*
COUT_BUILT = (64, 128, 256)


def _lib():
    sp = loader.product_spconv()
    return sp._lib, sp._lib.load()


def plain(m, cls):
    """True when ``m`` is a ``cls`` whose class does not override ``forward`` (``cls`` itself, or a subclass such as the
    reference's ``change_default_args`` layers, which only change constructor defaults)."""
    return isinstance(m, cls) and type(m).forward is cls.forward


def sequences(root):
    """-> [list of children] of every sequential container under ``root`` (``root`` included), in module order:
    ``nn.Sequential``, torchplus' ``Sequential`` (a plain ``nn.Module``) and the ``spconv`` drop-in's
    ``SparseSequential``, each of which runs its children in ``_modules`` order."""
    return [list(m._modules.values()) for m in root.modules()
            if isinstance(m, nn.Sequential) or type(m).__name__ in ("Sequential", "SparseSequential")]


def qualifies(conv, padding):
    """True when ``conv`` (an nn.Conv2d) is covered once its input is padded by ``padding`` - conv.padding."""
    return (plain(conv, nn.Conv2d) and tuple(conv.kernel_size) == (3, 3) and tuple(conv.stride) == (1, 1)
            and tuple(conv.dilation) == (1, 1) and conv.groups == 1 and conv.bias is None
            and conv.padding_mode == "zeros" and tuple(conv.padding) == (padding, padding)
            and conv.in_channels % 64 == 0 and conv.out_channels in COUT_BUILT)


def _is_pad1(m):
    return plain(m, nn.ZeroPad2d) and tuple(m.padding) == (1, 1, 1, 1)


def select(rpn):
    """-> [(conv, pad or None)] of the covered layers under ``rpn``, in module order."""
    out = []
    for mods in sequences(rpn):
        for i, m in enumerate(mods):
            if not plain(m, nn.Conv2d):
                continue
            if qualifies(m, 1):
                out.append((m, None))
            elif i > 0 and _is_pad1(mods[i - 1]) and qualifies(m, 0):
                out.append((m, mods[i - 1]))
    return out


def _active(conv, x):
    return conv.training and torch.is_grad_enabled() and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4


def _conv_forward(self, x):
    if _active(self, x):
        return Conv3x3TC.apply(x, self.weight, self)
    return nn.Conv2d.forward(self, x)


def _pad_forward(self, x):
    # the paired conv decides with the same test on the same tensor, so the pad is skipped exactly when the conv runs
    # Conv3x3TC (a pad-1 conv)
    return x if _active(self._b2s_rpn_conv, x) else nn.ZeroPad2d.forward(self, x)


def enable(net, products=3):
    """rebind the covered layers under ``net.rpn`` (or ``net`` itself when it has no ``rpn``) with ``products`` tensor-pipe
    products per MAC (3: 3xF16, 1: the f16 mode); idempotent apart from the product count, which a second call sets;
    never raises on a layer it does not cover.  Returns ``net``."""
    rpn = getattr(net, "rpn", net)
    for conv, pad in select(rpn):
        conv._b2s_products = products
        if getattr(conv, "_b2s_rpn_train", False):
            continue
        if pad is not None:
            pad.__dict__["_b2s_rpn_conv"] = conv      # a plain attribute: not a submodule, not in the state dict
            pad.forward = types.MethodType(_pad_forward, pad)
        conv.forward = types.MethodType(_conv_forward, conv)
        conv._b2s_rpn_train = True
    return net


# ---- planes and weights --------------------------------------------------------------------------------------------

def split_halo(t, status=None, products=3):
    """fp32 map [B, C, H, W] (contiguous or channels_last) -> (hi, lo) fp16 [B, H+2, W+2, C] planes of t * 2^e with a zero
    halo, and 2^-e as a [1] device tensor.  products = 1: the hi plane only, lo is None."""
    L, lib = _lib()
    B, C, H, W = (int(v) for v in t.shape)
    if t.is_contiguous():
        layout = LAYOUT_NCHW
    elif t.is_contiguous(memory_format=torch.channels_last):
        layout = LAYOUT_NHWC
    else:
        t, layout = t.contiguous(), LAYOUT_NCHW
    sc = torch.empty(2, dtype=torch.float32, device=t.device)
    if products == 1:
        hi = torch.empty(B, H + 2, W + 2, C, dtype=torch.float16, device=t.device)
        L.check(lib.b2s_split_halo_f16_autoscale_ex(L.ptr(t), layout, B, C, H, W, L.ptr(hi), None, L.ptr(sc),
                                                    L.ptr(status), 1, L.stream()), "b2s_split_halo_f16_autoscale_ex")
        return hi, None, sc[:1]
    planes = torch.empty(2, B, H + 2, W + 2, C, dtype=torch.float16, device=t.device)
    L.check(lib.b2s_split_halo_f16_autoscale(L.ptr(t), layout, B, C, H, W, L.ptr(planes[0]), L.ptr(planes[1]),
                                             L.ptr(sc), L.ptr(status), L.stream()), "b2s_split_halo_f16_autoscale")
    return planes[0], planes[1], sc[:1]


def pack_weights(conv, transpose, products=3):
    """the b2s_conv2d_tc_ex weight planes of ``conv`` ([G, 9, n_pad, n_in] hi / lo) and 1/s as a [1] device tensor,
    cached on the weight's (data_ptr, _version) and the product count like the sparse convs' planes (products = 1: the
    hi plane only, lo None)."""
    w = conv.weight
    key = (w.data_ptr(), w._version, str(w.device), transpose, products)
    cache = conv.__dict__.setdefault("_b2s_rpn_planes", {})
    hit = cache.get(transpose)
    if hit is not None and hit[0] == key:
        return hit[1]
    L, lib = _lib()
    cout, cin = int(w.shape[0]), int(w.shape[1])
    n_in, n_out = (cout, cin) if transpose else (cin, cout)
    planes = torch.empty(2 if products == 3 else 1, (n_out + 127) // 128, 9, min(n_out, 128), n_in, dtype=torch.float16,
                         device=w.device)
    sc = torch.empty(3, dtype=torch.float32, device=w.device)
    wd = w.detach()
    if not wd.is_contiguous():
        wd = wd.contiguous()
    if products == 1:
        L.check(lib.b2s_pack_conv2d_weights_ex(L.ptr(wd), cout, cin, int(transpose), L.ptr(planes[0]), None, L.ptr(sc),
                                               1, L.stream()), "b2s_pack_conv2d_weights_ex")
        val = (planes[0], None, sc[1:2])
        cache[transpose] = (key, val)
        return val
    L.check(lib.b2s_pack_conv2d_weights(L.ptr(wd), cout, cin, int(transpose), L.ptr(planes[0]), L.ptr(planes[1]),
                                        L.ptr(sc), L.stream()), "b2s_pack_conv2d_weights")
    val = (planes[0], planes[1], sc[1:2])
    cache[transpose] = (key, val)
    return val


def conv3x3(x_hi, x_lo, x_scale, w_hi, w_lo, w_inv, B, H, W, cin, cout, products=3):
    """3x3 stride-1 pad-1 conv of halo planes -> fp32 [B, H, W, cout]: one b2s_conv2d_tc_ex launch per 128 output
    channels, epilogue scale = (input's 2^-e) * (weights' 1/s), computed on the device.  products = 1: single planes
    (x_lo, w_lo None) through b2s_conv2d_tc_ex3 with products = 1 and fp32 output."""
    L, lib = _lib()
    out = torch.empty(B, H, W, cout, dtype=torch.float32, device=x_hi.device)
    n_pad = int(w_hi.shape[2])
    epi = (x_scale * w_inv).expand(n_pad).contiguous()
    for g in range(int(w_hi.shape[0])):
        cg = min(128, cout - 128 * g)
        if products == 1:
            L.check(lib.b2s_conv2d_tc_ex3(
                L.ptr(x_hi), None, B, H, W, cin, L.ptr(w_hi[g]), None, 3, 3, 1, 1, cg, n_pad, L.ptr(epi), None, 0, H, W,
                L.ptr(out[..., 128 * g:]), None, H, W, 0, cout, 1, 0, 0, None, None, None, None, None, None, -1, 8, 1, 1,
                None, L.stream()), "b2s_conv2d_tc_ex3")
            continue
        L.check(lib.b2s_conv2d_tc_ex(
            L.ptr(x_hi), L.ptr(x_lo), B, H, W, cin, L.ptr(w_hi[g]), L.ptr(w_lo[g]), 3, 3, 1, 1, cg, n_pad, L.ptr(epi),
            None, 0, H, W, L.ptr(out[..., 128 * g:]), None, H, W, 0, cout, 1, 0, 0, None, None, None, None, None, None,
            None, L.stream()), "b2s_conv2d_tc_ex")
    return out


def wgrad(x_hi, x_lo, x_scale, g_hi, g_lo, g_scale, B, H, W, cin, cout, products=3):
    L, lib = _lib()
    dw = torch.empty(cout, cin, 3, 3, dtype=torch.float32, device=x_hi.device)
    nbytes = int(lib.b2s_conv2d_wgrad_tc_workspace_bytes(B, H, W, cin, cout))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=x_hi.device)
    if products == 1:
        L.check(lib.b2s_conv2d_wgrad_tc_ex(L.ptr(x_hi), None, L.ptr(g_hi), None, B, H, W, cin, cout, L.ptr(x_scale),
                                           L.ptr(g_scale), L.ptr(dw), L.ptr(ws), nbytes, 1, L.stream()),
                "b2s_conv2d_wgrad_tc_ex")
        return dw
    L.check(lib.b2s_conv2d_wgrad_tc(L.ptr(x_hi), L.ptr(x_lo), L.ptr(g_hi), L.ptr(g_lo), B, H, W, cin, cout,
                                    L.ptr(x_scale), L.ptr(g_scale), L.ptr(dw), L.ptr(ws), nbytes, L.stream()),
            "b2s_conv2d_wgrad_tc")
    return dw


class Conv3x3TC(torch.autograd.Function):
    """y = conv2d(x, weight, padding=1) of a covered ``conv`` on the tensor pipe; see the module docstring."""

    @staticmethod
    def forward(ctx, x, weight, conv):
        B, cin, H, W = (int(v) for v in x.shape)
        cout = int(weight.shape[0])
        if cin != conv.in_channels:
            raise RuntimeError("Conv3x3TC: input has %d channels, the conv takes %d" % (cin, conv.in_channels))
        # the product count goes to the helpers only in the f16 mode: the default mode calls them as it always has
        kw = {} if getattr(conv, "_b2s_products", 3) == 3 else {"products": 1}
        x_hi, x_lo, x_scale = split_halo(x, **kw)
        w_hi, w_lo, w_inv = pack_weights(conv, False, **kw)
        y = conv3x3(x_hi, x_lo, x_scale, w_hi, w_lo, w_inv, B, H, W, cin, cout, **kw)
        ctx.save_for_backward(x_hi, x_lo, x_scale)
        ctx.conv, ctx.shape, ctx.kw = conv, (B, cin, H, W, cout), kw
        return y.permute(0, 3, 1, 2)                    # NCHW view of NHWC storage: channels_last

    @staticmethod
    def backward(ctx, dy):
        x_hi, x_lo, x_scale = ctx.saved_tensors
        B, cin, H, W, cout = ctx.shape
        kw = ctx.kw
        if not (dy.is_contiguous() or dy.is_contiguous(memory_format=torch.channels_last)):
            dy = dy.contiguous(memory_format=torch.channels_last)
        g_hi, g_lo, g_scale = split_halo(dy, **kw)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            wt_hi, wt_lo, wt_inv = pack_weights(ctx.conv, True, **kw)
            dx = conv3x3(g_hi, g_lo, g_scale, wt_hi, wt_lo, wt_inv, B, H, W, cout, cin, **kw).permute(0, 3, 1, 2)
        if ctx.needs_input_grad[1]:
            dw = wgrad(x_hi, x_lo, x_scale, g_hi, g_lo, g_scale, B, H, W, cin, cout, **kw)
        return dx, dw, None
