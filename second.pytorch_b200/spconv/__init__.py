"""``spconv`` drop-in (1.x API surface used by second.pytorch) on hand-written sm_100a CUDA.

Import this package as ``spconv`` (put ``second.pytorch_b200`` on ``sys.path``) and the reference's
``second/pytorch/models`` runs on it unchanged.  What second.pytorch touches (SURVEY.md §8b):

  SparseConvTensor    second/pytorch/models/middle.py:199-200,206 ; resnet.py:54-64
  SparseModule        resnet.py:32,69
  SparseSequential    middle.py:145
  SubMConv3d, SparseConv3d   middle.py:146-189 (wrapped by torchplus ``change_default_args(bias=False)``,
                      torchplus/tools.py:11-46 -> ``bias`` is a named __init__ parameter here)
  ops.nms, utils.*    see ops.py / utils/__init__.py

All arithmetic happens in libb2second.so (include/b2second.h).  No CPU fallback: tensors must be
CUDA tensors and the library must be built, otherwise calls raise.
"""
import math
import os

import numpy as np
import torch
from torch import nn

from . import _lib
from . import ops  # noqa: F401
from . import utils  # noqa: F401

__version__ = "1.2.1+b2second"

# sparse convolutions run on the tensor pipe (b2s_sparse_conv_tc, fp32-grade 3xF16 split) where the library covers the
# channel counts; False / env B2S_SPCONV_TC=0 forces the fp32 FMA kernel (b2s_sparse_conv) everywhere
USE_TENSOR_CORES = os.environ.get("B2S_SPCONV_TC", "1") != "0"


def _pow2_at_least(n):
    c = 1024
    while c < n:
        c <<= 1
    return c


class SparseConvTensor:
    """features [N,C] fp32 (CUDA), indices [N,4] int32 (b,z,y,x), spatial_shape (D,H,W), batch_size."""

    def __init__(self, features, indices, spatial_shape, batch_size, grid=None):
        self._features = features
        self._hilo = None   # (hi, lo, row stride in halves): fp16 hi/lo planes of the rows (tensor-core layers)
        self.indices = indices if indices.dtype == torch.int32 else indices.int()
        self.spatial_shape = [int(s) for s in spatial_shape]
        self.batch_size = int(batch_size)
        self.indice_dict = {}
        self.grid = grid
        self._hash = None   # (keys u64-as-int64 [cap], vals int32 [cap], cap)

    # ``features`` is read AND assigned by the reference (resnet.py:54-64).  Layers that run on the tensor pipe keep
    # their output as fp16 hi/lo planes (the next sparse layer consumes those directly); the fp32 rows are
    # materialised (hi + lo, exact) only when somebody actually reads ``.features``.
    @property
    def features(self):
        if self._features is None and self._hilo is not None:
            hi, lo, stride = self._hilo
            n, c = hi.shape
            out = torch.empty(n, c, dtype=torch.float32, device=hi.device)
            if n > 0:
                lib = _lib.load()
                _lib.check(lib.b2s_merge_f16(_lib.ptr(hi), _lib.ptr(lo), _lib.ptr(out), None, n, c, stride,
                                             _lib.stream()), "b2s_merge_f16")
            self._features = out
        return self._features

    @features.setter
    def features(self, value):
        self._features = value
        self._hilo = None

    @property
    def spatial_size(self):
        return int(np.prod(self.spatial_shape))

    def find_indice_pair(self, key):
        if key is None:
            return None
        return self.indice_dict.get(key, None)

    # -- coordinate -> row locator ---------------------------------------------------------------
    def _locator(self):
        if self._hash is None:
            _lib.require_cuda(self.indices, "SparseConvTensor.indices")
            lib = _lib.load()
            idx = self.indices.contiguous()
            n = idx.shape[0]
            dev = idx.device
            cap = _pow2_at_least(2 * max(n, 1))
            keys = torch.empty(cap, dtype=torch.int64, device=dev)
            vals = torch.empty(cap, dtype=torch.int32, device=dev)
            n_dev = torch.tensor([n], dtype=torch.int32, device=dev)
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            _lib.check(lib.b2s_hash_build(_lib.ptr(idx), _lib.ptr(n_dev), n, _lib.i3(self.spatial_shape),
                                          _lib.ptr(keys), _lib.ptr(vals), cap, _lib.ptr(status), _lib.stream()),
                       "b2s_hash_build")
            self._hash = (keys, vals, cap)
        return self._hash

    def dense(self, channels_first=True):
        feats = self.features
        _lib.require_cuda(feats, "SparseConvTensor.features")
        feats = feats.contiguous().float()
        if channels_first or self.spatial_shape[0] == 1:
            layout = 0 if channels_first else 1
            if feats.requires_grad and torch.is_grad_enabled():
                return _DenseFunction.apply(feats, self, layout)     # training: the gradient flows back to the rows
            return self._to_bev(feats, layout)
        # channels_last with D>1: [B,D,H,W,C] is not a BEV layout; go through NCDHW once
        return self.dense(True).permute(0, 2, 3, 4, 1).contiguous()

    def _to_bev(self, feats, layout):
        """fp32 rows -> [B,C,D,H,W] (layout 0) or [B,H,W,C] (layout 1, D == 1) through b2s_to_bev."""
        lib = _lib.load()
        idx = self.indices.contiguous()
        n, C = feats.shape
        D, H, W = self.spatial_shape
        B = self.batch_size
        dev = feats.device
        n_dev = torch.tensor([n], dtype=torch.int32, device=dev)
        if layout == 0:
            out = torch.empty(B, C, D, H, W, dtype=torch.float32, device=dev)
        else:
            out = torch.empty(B, D, H, W, C, dtype=torch.float32, device=dev)
        _lib.check(lib.b2s_to_bev(_lib.ptr(feats), _lib.ptr(idx), _lib.ptr(n_dev), n, C, B, D, H, W,
                                  _lib.ptr(out), layout, _lib.stream()), "b2s_to_bev")
        return out

    @property
    def sparity(self):
        return self.indices.shape[0] / np.prod(self.spatial_shape) / self.batch_size


class _DenseFunction(torch.autograd.Function):
    """SparseConvTensor.dense() with its backward: the gradient of each row is gathered from the dense gradient at the
    row's position (b2s_from_bev)."""

    @staticmethod
    def forward(ctx, feats, x, layout):
        ctx.x, ctx.layout, ctx.shape = x, layout, feats.shape
        return x._to_bev(feats, layout)

    @staticmethod
    def backward(ctx, grad):
        x = ctx.x
        n, C = ctx.shape
        D, H, W = x.spatial_shape
        grad = grad.contiguous().float()
        drows = torch.empty(n, C, dtype=torch.float32, device=grad.device)
        if n > 0:
            lib = _lib.load()
            n_dev = torch.tensor([n], dtype=torch.int32, device=grad.device)
            _lib.check(lib.b2s_from_bev(_lib.ptr(grad), _lib.ptr(x.indices.contiguous()), _lib.ptr(n_dev), n, C,
                                        x.batch_size, D, H, W, ctx.layout, _lib.ptr(drows), _lib.stream()),
                       "b2s_from_bev")
        return drows, None, None


class _SparseConvFunction(torch.autograd.Function):
    """one sparse convolution of the module path with its backward (torch.ops.spconv.indice_conv_backward upstream):
      dX  the forward contraction over the transposed table with W'[k] = W[k]^T (SparseConvolution._dgrad),
      dW  b2s_sparse_conv_wgrad_tc on the tensor pipe, else b2s_sparse_conv_wgrad,
      db  dY summed over the rows.
    Only the gradients autograd asks for are computed.  The weight is saved for backward, so autograd's version check
    refuses a backward after an in-place change of the weight."""

    @staticmethod
    def forward(ctx, feats, weight, bias, conv, rb):
        ctx.conv, ctx.rb, ctx.products = conv, rb, conv._b2s_products
        ctx.save_for_backward(feats, weight)
        out, ctx.x_split = conv._forward_rows(feats, rb, ctx.products)
        return out

    @staticmethod
    def backward(ctx, dy):
        feats, weight = ctx.saved_tensors
        conv, rb, products = ctx.conv, ctx.rb, ctx.products
        dy = dy.contiguous().float()
        split = _GradSplit(dy, products=products)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = conv._dgrad(dy, weight, rb, feats.shape[0], split, products)
        if ctx.needs_input_grad[1]:
            dw = conv._wgrad(feats, dy, rb, split, ctx.x_split, products).view_as(weight)
        if ctx.needs_input_grad[2]:
            db = dy.sum(0)
        return dx, dw, db, None, None


class _GradSplit:
    """fp32 rows [n, c] as fp16 hi/lo planes of `channels` (>= c, zero padded) halves, scaled by a power of two picked on
    the device (b2s_split_f16_autoscale), made on first use -- dY shared by the tensor-pipe dgrad and wgrad, and X for the
    wgrad: (hi, lo, row stride in halves, 2^-e as a [1] device tensor).  products = 1 (the f16 mode): the hi plane only,
    lo is None."""

    def __init__(self, t, channels=None, products=3):
        self.t, self.channels, self.products, self._planes = t, channels, products, None

    def planes(self):
        if self._planes is None and self.products == 1:
            t = self.t
            n, c = t.shape
            cp = self.channels or c
            hi = torch.empty(max(n, 1), cp, dtype=torch.float16, device=t.device)
            sc = torch.empty(2, dtype=torch.float32, device=t.device)
            _lib.check(_lib.load().b2s_split_f16_autoscale_ex(_lib.ptr(t), _lib.ptr(hi), None, None, n, c, cp, cp,
                                                              _lib.ptr(sc), 1, _lib.stream()),
                       "b2s_split_f16_autoscale_ex")
            self._planes = (hi, None, cp, sc[:1])
        if self._planes is None:
            t = self.t
            n, c = t.shape
            cp = self.channels or c
            buf = torch.empty(max(n, 1), 2, cp, dtype=torch.float16, device=t.device)
            sc = torch.empty(2, dtype=torch.float32, device=t.device)
            lib = _lib.load()
            _lib.check(lib.b2s_split_f16_autoscale(_lib.ptr(t), _lib.ptr(buf[:, 0]), _lib.ptr(buf[:, 1]), None, n, c, cp,
                                                   2 * cp, _lib.ptr(sc), _lib.stream()), "b2s_split_f16_autoscale")
            self._planes = (buf[:, 0], buf[:, 1], 2 * cp, sc[:1])
        return self._planes


class SparseModule(nn.Module):
    """marker base class: modules that take / return a SparseConvTensor."""
    pass


def is_spconv_module(module):
    return isinstance(module, SparseModule)


def _fold_bn(bn):
    """eval-mode BatchNorm1d -> per-channel (scale, shift); cached on the module until a parameter/buffer changes."""
    ts = [t for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var) if t is not None]
    key = tuple((t.data_ptr(), t._version) for t in ts)
    cached = getattr(bn, "_b2s_folded", None)
    if cached is not None and cached[0] == key:
        return cached[1], cached[2]
    with torch.no_grad():
        w = bn.weight if bn.weight is not None else torch.ones_like(bn.running_mean)
        b = bn.bias if bn.bias is not None else torch.zeros_like(bn.running_mean)
        scale = (w / torch.sqrt(bn.running_var + bn.eps)).float().contiguous()
        shift = (b - bn.running_mean * scale).float().contiguous()
    bn._b2s_folded = (key, scale, shift)
    return scale, shift


class SparseSequential(SparseModule):
    """runs sparse modules on the tensor and dense modules on ``.features`` (children '0','1',...).

    In eval mode a (sparse conv, BatchNorm1d, ReLU) triple -- the only pattern second.pytorch builds
    (middle.py:146-191) -- is executed as ONE kernel with the BN scale/shift and ReLU in the epilogue.
    """

    def __init__(self, *args, **kwargs):
        super().__init__()
        if len(args) == 1 and isinstance(args[0], dict):
            for key, module in args[0].items():
                self.add_module(key, module)
        else:
            for idx, module in enumerate(args):
                self.add_module(str(idx), module)
        for name, module in kwargs.items():
            if name in self._modules:
                raise ValueError("name exists.")
            self.add_module(name, module)
        self.fuse_bn_relu = True

    def __getitem__(self, idx):
        if not (-len(self) <= idx < len(self)):
            raise IndexError("index {} is out of range".format(idx))
        if idx < 0:
            idx += len(self)
        return list(self._modules.values())[idx]

    def __len__(self):
        return len(self._modules)

    def add(self, module, name=None):
        if name is None:
            name = str(len(self._modules))
            if name in self._modules:
                raise KeyError("name exists")
        self.add_module(name, module)

    def forward(self, input):
        mods = list(self._modules.values())
        i = 0
        while i < len(mods):
            module = mods[i]
            if is_spconv_module(module):
                assert isinstance(input, SparseConvTensor)
                if (self.fuse_bn_relu and not self.training and isinstance(module, SparseConvolution)
                        and i + 1 < len(mods) and isinstance(mods[i + 1], nn.BatchNorm1d)
                        and mods[i + 1].track_running_stats and module.bias is None):
                    relu = i + 2 < len(mods) and isinstance(mods[i + 2], nn.ReLU)
                    scale, shift = _fold_bn(mods[i + 1])
                    input = module(input, _epilogue=(scale, shift, relu))
                    i += 3 if relu else 2
                    continue
                input = module(input)
            elif isinstance(input, SparseConvTensor):
                if input.indices.shape[0] != 0:
                    input.features = module(input.features)
            else:
                input = module(input)
            i += 1
        return input


def _pack_tc_weights(w, transpose=False, flip=False, products=3):
    """fp32 weight [K, Cin, Cout] -> (hi, lo, s, 1/s): the fp16 planes of W[k] (transpose: W[k]^T, flip: W[K-1-k]^T) in
    the tensor-core kernel's packed layout, pre-scaled by the power of two s of b2second.tc.pow2_scale, with s and 1/s as
    [1] device tensors.  b2s_pack_sparse_weights reduces max|w| on the device, so nothing is read on the host; the
    planes and the scale are bit for bit tc.split_f16(tc.pack_sparse_weights(...), tc.pow2_scale(...)) for finite weights
    (a non-finite weight is packed as itself, not saturated).  products = 1 (the f16 mode): the hi plane only, lo is
    None."""
    lib = _lib.load()
    K, cin, cout = (int(v) for v in w.shape)
    n_in, n_out = (cout, cin) if transpose else (cin, cout)
    n_in_pad = 8 if n_in <= 8 else n_in
    pack = 64 // n_in_pad
    hi = torch.empty((K + pack - 1) // pack, n_out, 64, dtype=torch.float16, device=w.device)
    sc = torch.empty(3, dtype=torch.float32, device=w.device)
    if products == 1:
        _lib.check(lib.b2s_pack_sparse_weights_ex(_lib.ptr(w), K, cin, cout, int(transpose), int(flip), _lib.ptr(hi), None,
                                                  _lib.ptr(sc), 1, _lib.stream()), "b2s_pack_sparse_weights_ex")
        return hi, None, sc[0:1], sc[1:2]
    lo = torch.empty_like(hi)
    _lib.check(lib.b2s_pack_sparse_weights(_lib.ptr(w), K, cin, cout, int(transpose), int(flip), _lib.ptr(hi),
                                           _lib.ptr(lo), _lib.ptr(sc), _lib.stream()), "b2s_pack_sparse_weights")
    return hi, lo, sc[0:1], sc[1:2]


def _conv_tc(x, w, table, K, n_dev, n_out, plan, scale, shift, relu, out, out_lo=None, products=3):
    """one b2s_sparse_conv_tc_plan launch for the first n_out rows of `table`: fp16 input planes x = (hi, lo, row stride)
    as wide as Cin, packed weight planes w = (hi, lo), plan = ops.tile_plan's (perm, tile_mask); `out` as wide as Cout
    is fp32 rows, or with `out_lo` the hi plane of fp16 hi/lo rows.  -> the status word, None when there are no rows.
    products = 1 (the f16 training mode): single planes (the lo entries None) and fp32 rows out, through
    b2s_sparse_conv_tc_plan_ex2."""
    if n_out == 0:
        return None
    (hi, lo, stride), (w_hi, w_lo), (perm, tmask) = x, w, plan
    status = torch.zeros(1, dtype=torch.int32, device=out.device)
    if products == 1:
        _lib.check(_lib.load().b2s_sparse_conv_tc_plan_ex2(
            _lib.ptr(hi), None, stride, hi.shape[0], hi.shape[1], _lib.ptr(w_hi), None, _lib.ptr(table), K,
            _lib.ptr(n_dev), n_out, _lib.ptr(perm), _lib.ptr(tmask), _lib.ptr(scale), _lib.ptr(shift), int(relu),
            _lib.ptr(out), None, out.stride(0), out.shape[1], 1, 1, _lib.ptr(status), _lib.stream()),
            "b2s_sparse_conv_tc_plan_ex2")
        return status
    _lib.check(_lib.load().b2s_sparse_conv_tc_plan(
        _lib.ptr(hi), _lib.ptr(lo), stride, hi.shape[0], hi.shape[1], _lib.ptr(w_hi), _lib.ptr(w_lo), _lib.ptr(table), K,
        _lib.ptr(n_dev), n_out, _lib.ptr(perm), _lib.ptr(tmask), _lib.ptr(scale), _lib.ptr(shift), int(relu),
        _lib.ptr(out), _lib.ptr(out_lo), out.stride(0), out.shape[1], _lib.ptr(status), _lib.stream()),
        "b2s_sparse_conv_tc_plan")
    return status


def _conv_fma(x, w, table, n_dev, n_out, scale, shift, relu, out):
    """one b2s_sparse_conv launch (fp32 FMA) over `table` for its first n_out rows: fp32 rows x through w [K, Cin, Cout]
    into out [n_out, Cout]"""
    if n_out == 0:
        return
    K, cin, cout = w.shape
    _lib.check(_lib.load().b2s_sparse_conv(_lib.ptr(x), cin, _lib.ptr(w), _lib.ptr(table), K, _lib.ptr(n_dev), n_out,
                                           _lib.ptr(scale), _lib.ptr(shift), int(relu), _lib.ptr(out), cout,
                                           _lib.stream()), "b2s_sparse_conv")


def _triple(v):
    if isinstance(v, (list, tuple, np.ndarray)):
        assert len(v) == 3
        return [int(x) for x in v]
    return [int(v)] * 3


class SparseConvolution(SparseModule):
    def __init__(self, ndim, in_channels, out_channels, kernel_size=3, stride=1, padding=0, dilation=1,
                 groups=1, bias=True, subm=False, output_padding=0, transposed=False, inverse=False,
                 indice_key=None):
        super().__init__()
        assert groups == 1, "groups != 1 is not used by second.pytorch"
        assert ndim == 3 and not transposed and not inverse
        self.ndim = ndim
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _triple(kernel_size)
        self.conv1x1 = int(np.prod(self.kernel_size)) == 1
        self.stride = _triple(stride)
        self.padding = _triple(padding)
        self.dilation = _triple(dilation)
        self.transposed = transposed
        self.inverse = inverse
        self.output_padding = _triple(output_padding)
        self.groups = groups
        self.subm = subm
        self.indice_key = indice_key
        self.weight = nn.Parameter(torch.Tensor(*self.kernel_size, in_channels, out_channels))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            fan_in, _ = nn.init._calculate_fan_in_and_fan_out(self.weight)
            bound = 1 / math.sqrt(fan_in)
            nn.init.uniform_(self.bias, -bound, bound)

    def _tc_weights(self, cin_tc, products=3):
        """fp16 hi/lo planes of the (power-of-two scaled) weight in the tensor-core kernel's layout, the scale as a [1]
        device tensor and its inverse per output channel; cached until the parameter or the product count changes
        (products = 1: the hi plane only, lo None)."""
        w = self.weight
        key = (w.data_ptr(), w._version, str(w.device), products)
        cached = getattr(self, "_b2s_tc_w", None)
        if cached is None or cached[0] != key:
            K = int(np.prod(self.kernel_size))
            with torch.no_grad():
                wk = w.detach().float().contiguous().view(K, self.in_channels, self.out_channels)
                # the 3xF16 call keeps its form (products is passed only in the f16 mode)
                hi, lo, ws, inv = _pack_tc_weights(wk) if products == 3 else _pack_tc_weights(wk, products=products)
                inv = inv.expand(self.out_channels).contiguous()
            cached = (key, hi, lo, ws, inv)
            self._b2s_tc_w = cached
        return cached[1:]

    def forward(self, input, _epilogue=None):
        assert isinstance(input, SparseConvTensor)
        record = self.training and torch.is_grad_enabled()
        if record and self.weight.requires_grad and not self._b2s_backward:
            # The backward (upstream's indice_conv_backward) is opt-in: b2second.training.enable_sparse_backward(net).
            # Without it a training-mode call that autograd would record must fail instead of silently returning
            # gradient-free tensors.  (eval() with autograd enabled is the reference's own inference mode --
            # voxelnet.py:368-374 -- and runs; so does anything under torch.no_grad().)
            raise NotImplementedError("b2second spconv: autograd through sparse convolutions is opt-in: call "
                                      "b2second.training.enable_sparse_backward(net) to train, or net.eval() / "
                                      "torch.no_grad() for inference")
        lib = _lib.load()
        K = int(np.prod(self.kernel_size))
        # a 1x1x1 stride-1 conv keeps the active set (upstream short-circuits it to a plain mm)
        subm = self.subm or (self.conv1x1 and all(s == 1 for s in self.stride) and all(p == 0 for p in self.padding))
        if subm:
            out_shape = input.spatial_shape
        else:
            out_shape = ops.get_conv_output_size(input.spatial_shape, self.kernel_size, self.stride, self.padding,
                                                 self.dilation)
        datas = input.find_indice_pair(self.indice_key)
        if self.indice_key is not None and datas is not None:
            rb = datas
        else:
            rb = ops.build_rulebook(input, self.kernel_size, self.stride, self.padding, self.dilation, subm)
            input.indice_dict[self.indice_key] = rb
        n_out = rb.num_out
        dev = input.indices.device
        if _epilogue is not None:
            scale, shift, relu = _epilogue
        else:
            scale, shift, relu = None, (self.bias.detach().float().contiguous() if self.bias is not None else None), False
        out = SparseConvTensor(None, rb.out_indices, out_shape, input.batch_size)
        out._hash = rb.out_hash
        out.indice_dict = input.indice_dict
        out.grid = input.grid
        if record and self._b2s_backward:
            # training (opt-in): fp32 output rows recorded by autograd; BN / ReLU run as the torch modules that follow
            feats = input.features
            _lib.require_cuda(feats, "SparseConvTensor.features")
            out._features = _SparseConvFunction.apply(feats.contiguous().float(), self.weight, self.bias, self, rb)
            return out
        cin_tc = self._wgrad_tc_cin(lib, K)
        if cin_tc is not None:
            # tensor pipe (wgmma, 3xF16 split): fp16 hi/lo rows in, fp16 hi/lo rows out
            if input._hilo is not None and input._hilo[0].shape[1] == cin_tc:
                hi, lo, stride = input._hilo
            else:
                feats = input.features
                _lib.require_cuda(feats, "SparseConvTensor.features")
                feats = feats.contiguous().float()
                n_in = feats.shape[0]
                buf = torch.empty(max(n_in, 1), 2, cin_tc, dtype=torch.float16, device=dev)
                hi, lo, stride = buf[:, 0], buf[:, 1], 2 * cin_tc
                if n_in > 0:
                    _lib.check(lib.b2s_split_f16(_lib.ptr(feats), _lib.ptr(hi), _lib.ptr(lo), None, n_in,
                                                 self.in_channels, cin_tc, stride, _lib.stream()), "b2s_split_f16")
                input._hilo = (hi[:n_in], lo[:n_in], stride)
            w_hi, w_lo, ws, inv = self._tc_weights(cin_tc)
            scale_tc = inv if scale is None else (scale / ws).contiguous()
            obuf = torch.empty(max(n_out, 1), 2, self.out_channels, dtype=torch.float16, device=dev)
            o_hi, o_lo = obuf[:, 0], obuf[:, 1]
            # SubM rulebooks get a tile plan: K blocks no row of a tile needs are skipped
            out._status = _conv_tc((hi, lo, stride), (w_hi, w_lo), rb.nbr, K, rb.num_out_dev, n_out, ops.tile_plan(rb),
                                   scale_tc, shift, relu, o_hi, o_lo)
            out._hilo = (o_hi[:n_out], o_lo[:n_out], 2 * self.out_channels)
            out._keep = obuf
            return out
        feats = input.features
        _lib.require_cuda(feats, "SparseConvTensor.features")
        feats = feats.contiguous().float()
        out._features = torch.empty(n_out, self.out_channels, dtype=torch.float32, device=dev)
        w = self.weight.detach().float().contiguous().view(K, self.in_channels, self.out_channels)
        _conv_fma(feats, w, rb.nbr, rb.num_out_dev, n_out, scale, shift, relu, out._features)
        return out

    # ---- training (b2second.training.enable_sparse_backward sets _b2s_backward and _b2s_products) ---------------------
    _b2s_backward = False
    _b2s_products = 3       # tensor-pipe products per MAC in training: 3 (3xF16, fp32-grade) or 1 (the f16 mode)

    def _forward_rows(self, feats, rb, products=None):
        """(fp32 output rows [n_out, Cout] (+ bias) from fp32 input rows, the _GradSplit of X or None) on the kernel the
        inference path would pick (tensor pipe with fp32 output, or b2s_sparse_conv).  On the tensor pipe X is split
        under its own power-of-two scale, as in the backward: unscaled, an activation above 65504 would saturate and one
        below 2^-3 keep only 2^-25 absolute precision.  The split is kept for the weight gradient.  products: the
        tensor-pipe product count (None: the module's _b2s_products)."""
        products = self._b2s_products if products is None else products
        lib = _lib.load()
        K, n_out = rb.K, rb.num_out
        dev = feats.device
        shift = self.bias.detach().float().contiguous() if self.bias is not None else None
        out = torch.empty(n_out, self.out_channels, dtype=torch.float32, device=dev)
        if n_out == 0:
            return out, None
        cin_tc = self._wgrad_tc_cin(lib, K)
        if cin_tc is not None:
            split = _GradSplit(feats, cin_tc, products)
            hi, lo, stride, inv_x = split.planes()
            w_hi, w_lo, ws, inv = self._tc_weights(cin_tc, products)
            scale = inv * inv_x                                        # powers of two: exact, no host sync
            _conv_tc((hi, lo, stride), (w_hi, w_lo), rb.nbr, K, rb.num_out_dev, n_out, ops.tile_plan(rb), scale, shift,
                     False, out, products=products)
            return out, split
        w = self.weight.detach().float().contiguous().view(K, self.in_channels, self.out_channels)
        _conv_fma(feats, w, rb.nbr, rb.num_out_dev, n_out, None, shift, False, out)
        return out, None

    def _wgrad_tc_cin(self, lib, K):
        """channel count of the tensor-pipe forward / weight gradient (the input padded to 8, tc.sparse_tc_channels), or
        None: fp32 kernels"""
        from b2second import tc as _tc
        return _tc.sparse_tc_channels(lib, self.in_channels, self.out_channels, K) if USE_TENSOR_CORES else None

    def _dgrad_weights(self, w, flip, products=3):
        """packed fp16 hi/lo planes of W'[k] = W[k]^T (flip: W[K-1-k]^T) for the tensor-pipe input gradient, with their
        power-of-two scale as a [1] device tensor; cached until the weight or the product count changes (one scale
        measurement per weight version; products = 1: the hi plane only, lo None)."""
        key = (w.data_ptr(), w._version, str(w.device), flip, products)
        cached = getattr(self, "_b2s_tc_wt", None)
        if cached is None or cached[0] != key:
            K = int(np.prod(self.kernel_size))
            with torch.no_grad():
                wk = w.detach().float().contiguous().view(K, self.in_channels, self.out_channels)
                hi, lo, ws, _ = (_pack_tc_weights(wk, transpose=True, flip=flip) if products == 3 else
                                 _pack_tc_weights(wk, transpose=True, flip=flip, products=products))
            cached = (key, hi, lo, ws)
            self._b2s_tc_wt = cached
        return cached[1:]

    def _dgrad(self, dy, weight, rb, n_in, split=None, products=None):
        """input gradient [n_in, Cin] = the forward contraction of dY [n_out, Cout] over the transposed table with
        W'[k] = W[k]^T.  A SubM table with odd kernel sizes is its own transpose under k <-> K-1-k (same table, same tile
        plan, W'[k] = W[K-1-k]^T); any other table is transposed once (ops.transpose_rulebook)."""
        from b2second import tc as _tc
        products = self._b2s_products if products is None else products
        lib = _lib.load()
        K, cin, cout, n_out = rb.K, self.in_channels, self.out_channels, rb.num_out
        dev = dy.device
        if n_in == 0 or n_out == 0:
            return torch.zeros(n_in, cin, dtype=torch.float32, device=dev)
        flip = rb.subm and all(k % 2 == 1 for k in rb.ksize)
        if flip:
            table, n_dev, plan = rb.nbr, rb.num_out_dev, ops.tile_plan(rb)
        else:
            table, plan = ops.transpose_rulebook(rb, n_in), (None, None)
            n_dev = rb.nbrT_rows_dev                    # cached with the table: no host copy, the backward can be captured
        dx = torch.empty(n_in, cin, dtype=torch.float32, device=dev)
        # the contraction runs Cout -> Cin; dY is not padded, so it takes the tensor pipe only at an unpadded width
        if USE_TENSOR_CORES and _tc.sparse_tc_channels(lib, cout, cin, K) == cout:
            # dY goes onto the tensor pipe scaled by a power of two picked on the device (gradients are often far below
            # the fp16 normal range); the kernel's epilogue scale undoes both that and the weights' scale
            w_hi, w_lo, ws = self._dgrad_weights(weight, flip, products)
            g_hi, g_lo, g_stride, inv = (split or _GradSplit(dy, products=products)).planes()
            scale = (inv / ws).expand(cin).contiguous()
            _conv_tc((g_hi, g_lo, g_stride), (w_hi, w_lo), table, K, n_dev, n_in, plan, scale, None, False, dx,
                     products=products)
            return dx
        w = weight.detach().float().reshape(K, cin, cout)
        wt = (w.flip(0) if flip else w).transpose(1, 2).contiguous()        # [K, Cout, Cin]
        _conv_fma(dy, wt, table, n_dev, n_in, None, None, False, dx)
        return dx

    def _wgrad(self, feats, dy, rb, split=None, x_split=None, products=None):
        """weight gradient [K, Cin, Cout] = sum over output rows of X[nbr[o,k]]^T dY[o]: b2s_sparse_conv_wgrad_tc on the
        tensor pipe, b2s_sparse_conv_wgrad (fp32 FMA) otherwise.  On the tensor pipe both operands are split under their
        own power-of-two scale (b2s_split_f16_autoscale; X's split is the forward's when given): unscaled, a small
        activation would keep only 2^-25 absolute precision, which a weight gradient of few pairs would see; rows are
        reduced in the forward's tile-plan order.  products = 1 (the f16 mode): b2s_sparse_conv_wgrad_tc_ex on the hi
        planes."""
        products = self._b2s_products if products is None else products
        lib = _lib.load()
        K, cin, cout, n_out = rb.K, self.in_channels, self.out_channels, rb.num_out
        dev = dy.device
        cin_tc = self._wgrad_tc_cin(lib, K)
        if cin_tc is not None and n_out > 0 and feats.shape[0] > 0:
            x_hi, x_lo, x_stride, inv_x = (x_split or _GradSplit(feats, cin_tc, products)).planes()
            g_hi, g_lo, g_stride, inv_g = (split or _GradSplit(dy, products=products)).planes()
            scale = inv_x * inv_g                                      # powers of two: exact
            perm, tmask = ops.tile_plan(rb)
            dw = torch.empty(K, cin_tc, cout, dtype=torch.float32, device=dev)
            ws_bytes = lib.b2s_sparse_conv_wgrad_tc_workspace_bytes(n_out, K, cin_tc, cout)
            work = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
            if products == 1:
                _lib.check(lib.b2s_sparse_conv_wgrad_tc_ex(
                    _lib.ptr(x_hi), None, x_stride, x_hi.shape[0], cin_tc, _lib.ptr(g_hi), None, g_stride, cout,
                    _lib.ptr(rb.nbr.contiguous()), K, _lib.ptr(rb.num_out_dev), n_out, _lib.ptr(perm), _lib.ptr(tmask),
                    _lib.ptr(scale), _lib.ptr(dw), _lib.ptr(work), ws_bytes, 1, _lib.stream()),
                    "b2s_sparse_conv_wgrad_tc_ex")
                return dw if cin_tc == cin else dw[:, :cin].contiguous()
            _lib.check(lib.b2s_sparse_conv_wgrad_tc(
                _lib.ptr(x_hi), _lib.ptr(x_lo), x_stride, x_hi.shape[0], cin_tc, _lib.ptr(g_hi), _lib.ptr(g_lo), g_stride,
                cout, _lib.ptr(rb.nbr.contiguous()), K, _lib.ptr(rb.num_out_dev), n_out, _lib.ptr(perm), _lib.ptr(tmask),
                _lib.ptr(scale), _lib.ptr(dw), _lib.ptr(work), ws_bytes, _lib.stream()), "b2s_sparse_conv_wgrad_tc")
            return dw if cin_tc == cin else dw[:, :cin].contiguous()
        dw = torch.empty(K, cin, cout, dtype=torch.float32, device=dev)
        ws_bytes = lib.b2s_sparse_conv_wgrad_workspace_bytes(n_out, K, cin, cout)
        work = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        _lib.check(lib.b2s_sparse_conv_wgrad(_lib.ptr(feats), cin, _lib.ptr(dy), cout, _lib.ptr(rb.nbr.contiguous()), K,
                                             _lib.ptr(rb.num_out_dev), n_out, None, _lib.ptr(dw), _lib.ptr(work), ws_bytes,
                                             _lib.stream()), "b2s_sparse_conv_wgrad")
        return dw


class SparseConv3d(SparseConvolution):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, indice_key=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         indice_key=indice_key)


class SubMConv3d(SparseConvolution):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, indice_key=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         True, indice_key=indice_key)


class ToDense(SparseModule):
    def forward(self, x):
        return x.dense()
