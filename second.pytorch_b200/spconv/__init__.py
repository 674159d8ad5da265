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
        lib = _lib.load()
        feats = feats.contiguous().float()
        idx = self.indices.contiguous()
        n, C = feats.shape
        D, H, W = self.spatial_shape
        B = self.batch_size
        dev = feats.device
        n_dev = torch.tensor([n], dtype=torch.int32, device=dev)
        if channels_first:
            out = torch.empty(B, C, D, H, W, dtype=torch.float32, device=dev)
            layout = 0
        else:
            out = torch.empty(B, D, H, W, C, dtype=torch.float32, device=dev)
            layout = 1
        if channels_first or D == 1:
            _lib.check(lib.b2s_to_bev(_lib.ptr(feats), _lib.ptr(idx), _lib.ptr(n_dev), n, C, B, D, H, W,
                                      _lib.ptr(out), layout, _lib.stream()), "b2s_to_bev")
            return out
        # channels_last with D>1: [B,D,H,W,C] is not a BEV layout; go through NCDHW once
        return self.dense(True).permute(0, 2, 3, 4, 1).contiguous()

    @property
    def sparity(self):
        return self.indices.shape[0] / np.prod(self.spatial_shape) / self.batch_size


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

    def _tc_weights(self, cin_tc):
        """fp16 hi/lo planes of the (power-of-two scaled) weight in the tensor-core kernel's layout; cached until the
        parameter changes."""
        from b2second import tc as _tc
        w = self.weight
        key = (w.data_ptr(), w._version, str(w.device))
        cached = getattr(self, "_b2s_tc_w", None)
        if cached is None or cached[0] != key:
            K = int(np.prod(self.kernel_size))
            with torch.no_grad():
                wp = _tc.pack_sparse_weights(w.detach().float().contiguous().view(K, self.in_channels,
                                                                                 self.out_channels))
                ws = _tc.pow2_scale(wp)
                hi, lo = _tc.split_f16(wp, ws)
                inv = torch.full((self.out_channels,), 1.0 / ws, dtype=torch.float32, device=w.device)
            cached = (key, hi, lo, ws, inv)
            self._b2s_tc_w = cached
        return cached[1:]

    def forward(self, input, _epilogue=None):
        assert isinstance(input, SparseConvTensor)
        if self.training and torch.is_grad_enabled() and self.weight.requires_grad:
            # upstream implements indice_conv_backward; this drop-in covers the inference path only (SURVEY.md §8(f)4).
            # A training-mode call that autograd would record must fail instead of silently returning gradient-free
            # tensors.  (eval() with autograd enabled is the reference's own inference mode -- voxelnet.py:368-374 --
            # and runs; so does anything under torch.no_grad().)
            raise NotImplementedError("b2second spconv: training / autograd through sparse convolutions is not "
                                      "implemented (inference drop-in); call net.eval() and run under torch.no_grad()")
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
        from b2second import tc as _tc
        cin_tc = _tc.sparse_tc_cin(self.in_channels)
        use_tc = (USE_TENSOR_CORES and cin_tc is not None
                  and bool(lib.b2s_sparse_conv_tc_supported(cin_tc, self.out_channels)))
        if use_tc:
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
            if n_out > 0:
                status = torch.zeros(1, dtype=torch.int32, device=dev)
                perm, tmask = ops.tile_plan(rb)        # SubM rulebooks: K blocks no row of a tile needs are skipped
                _lib.check(lib.b2s_sparse_conv_tc_plan(
                    _lib.ptr(hi), _lib.ptr(lo), stride, hi.shape[0], cin_tc, _lib.ptr(w_hi), _lib.ptr(w_lo),
                    _lib.ptr(rb.nbr), K, _lib.ptr(rb.num_out_dev), n_out, _lib.ptr(perm), _lib.ptr(tmask),
                    _lib.ptr(scale_tc), _lib.ptr(shift), 1 if relu else 0, _lib.ptr(o_hi), _lib.ptr(o_lo),
                    2 * self.out_channels, self.out_channels, _lib.ptr(status), _lib.stream()), "b2s_sparse_conv_tc_plan")
                out._status = status
            out._hilo = (o_hi[:n_out], o_lo[:n_out], 2 * self.out_channels)
            out._keep = obuf
            return out
        feats = input.features
        _lib.require_cuda(feats, "SparseConvTensor.features")
        feats = feats.contiguous().float()
        out_feats = torch.empty(n_out, self.out_channels, dtype=torch.float32, device=dev)
        w = self.weight.detach().float().contiguous().view(K, self.in_channels, self.out_channels)
        if n_out > 0:
            _lib.check(lib.b2s_sparse_conv(_lib.ptr(feats), self.in_channels, _lib.ptr(w), _lib.ptr(rb.nbr), K,
                                           _lib.ptr(rb.num_out_dev), n_out, _lib.ptr(scale), _lib.ptr(shift),
                                           1 if relu else 0, _lib.ptr(out_feats), self.out_channels,
                                           _lib.stream()), "b2s_sparse_conv")
        out._features = out_feats
        return out


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
