"""Host-only description of a SECOND inference network, read off a module tree by duck typing.

The fused engine (``b2second.engine``) must sit behind the *reference's own* ``VoxelNet`` -- the object
``second/pytorch/builder/second_builder.py:22-133`` returns -- as well as behind the mirror classes in
``b2second.models``.  So nothing here looks at classes or at a ``ModelConfig``: only at the attribute names
the reference defines:

  VoxelNet            second/pytorch/models/voxelnet.py:104-158 (``_use_rotate_nms``, ``_multiclass_nms``,
                      ``_nms_*``, ``_post_center_range``, ``_dir_offset`` ..., ``voxel_generator``, ``target_assigner``)
  SimpleVoxel(/Radius) second/pytorch/models/voxel_encoder.py:206-255 (``num_input_features``)
  PillarFeatureNet    second/pytorch/models/pointpillars.py:153-201 (``pfn_layers[i].linear/.norm``, ``vx vy x_offset y_offset``)
  PillarFeatureNetRadius pointpillars.py:240-325 (same attributes; recognised, like every PFN, by its class name)
  SpMiddleFHD*        second/pytorch/models/middle.py:110-210 (``middle_conv`` = SparseSequential, ``sparse_shape``)
  PointPillarsScatter pointpillars.py:420-442 (``ny nx nchannels``)
  RPNV2               second/pytorch/models/rpn.py:202-420 (``blocks deblocks conv_box conv_cls conv_dir_cls _upsample_start_idx``)
  VoxelNetNuscenesMultiHead  second/pytorch/models/net_multi_head.py:121-176 (``small_head.net/.conv_*``,
                      ``large_head.conv_*``, an RPNNoHead ``rpn`` with ``blocks deblocks`` and no ``conv_box``)

``spec_from_module`` needs no CUDA and no ``spconv`` import: sparse conv layers are recognised by their
attributes (``subm kernel_size stride padding dilation indice_key weight``), so a network built on ANY spconv
package (the CUDA drop-in, the CPU oracle) yields the same spec -- tests/test_reference_dropin.py checks that the
spec of the unmodified reference network equals the spec of the mirror for all five BASELINE configs.
"""
import hashlib

import numpy as np
import torch
from torch import nn


class UnsupportedNetwork(ValueError):
    """the module tree has a layer pattern the fused engine does not cover (callers fall back to the
    module-by-module path on the CUDA spconv drop-in)."""


def fold_bn(bn):
    """eval-mode BatchNorm -> per-channel (scale, shift), fp32."""
    w = bn.weight if bn.weight is not None else torch.ones_like(bn.running_mean)
    b = bn.bias if bn.bias is not None else torch.zeros_like(bn.running_mean)
    scale = (w / torch.sqrt(bn.running_var + bn.eps)).detach().float().contiguous()
    shift = (b - bn.running_mean * scale).detach().float().contiguous()
    return scale, shift


def _is_sparse_conv(m):
    return all(hasattr(m, a) for a in ("subm", "kernel_size", "stride", "padding", "dilation", "indice_key", "weight",
                                       "in_channels", "out_channels"))


def _triple(v):
    if isinstance(v, (list, tuple, np.ndarray)):
        return [int(x) for x in v]
    return [int(v)] * 3


class NetSpec:
    """plain attribute bag; see spec_from_module."""

    def signature(self):
        """hashable summary (structure + sha1 of every weight) used to compare two specs."""
        def h(t):
            if t is None:
                return None
            return hashlib.sha1(np.ascontiguousarray(t.detach().cpu().float().numpy()).tobytes()).hexdigest()

        sig = {k: getattr(self, k) for k in (
            "voxel_size", "point_cloud_range", "grid_size", "max_points_per_voxel", "max_voxels", "num_point_features",
            "vfe_kind", "vfe_num_features", "is_pillars", "sparse_shape", "bev_channels", "num_class", "box_code_size",
            "num_anchors_per_loc", "use_direction_classifier", "num_direction_bins", "direction_offset",
            "direction_limit_offset", "use_rotate_nms", "multiclass_nms", "nms_class_agnostic", "nms_score_thresholds",
            "nms_pre_max_sizes", "nms_post_max_sizes", "nms_iou_thresholds", "post_center_range")}
        sig["layers"] = [{k: (h(v) if isinstance(v, torch.Tensor) else v) for k, v in lyr.items()}
                         for lyr in self.layers]
        if self.pfn is not None:
            sig["pfn"] = {k: (h(v) if isinstance(v, torch.Tensor) else v) for k, v in self.pfn.items()}
        sig["rpn"] = {k: h(v) for k, v in self.rpn.state_dict().items() if v.dtype.is_floating_point}
        # keys only the radius PFN / the multi-head network have (the signature of every other network is unchanged)
        if getattr(self, "pfn_decoration", 0):
            sig["pfn_decoration"] = self.pfn_decoration
        if getattr(self, "heads", None) is not None:
            sig["heads"] = {name: {k: h(v) for k, v in m.state_dict().items() if v.dtype.is_floating_point}
                            for name, m in self.heads}
            sig["head_feature_map_sizes"] = self.head_feature_map_sizes
        return sig


def _f(v):
    """list of floats at float32 precision: protobuf configs hold float32 (0.30000001...), hand-written ones Python
    floats (0.3); every consumer is a C `float` parameter, so float32 is the value that counts."""
    return [float(np.float32(x)) for x in v]


def spec_from_module(net, max_voxels=None):
    """VoxelNet-like module tree (reference-built or mirror) -> NetSpec.  Raises UnsupportedNetwork."""
    s = NetSpec()
    s.device = next(net.parameters()).device
    # ---- voxel generator (spconv.utils.VoxelGeneratorV2 attributes, voxel_builder.py:23-32)
    vg = net.voxel_generator
    s.voxel_size = _f(vg.voxel_size)
    s.point_cloud_range = _f(vg.point_cloud_range)
    s.grid_size = [int(x) for x in vg.grid_size]                  # xyz
    T = getattr(vg, "max_num_points_per_voxel", None)
    if T is None:
        T = getattr(vg, "_max_num_points")
    s.max_points_per_voxel = int(T)
    s.max_voxels = int(max_voxels or getattr(vg, "_max_voxels", 20000))
    # ---- VFE
    vfe = net.voxel_feature_extractor
    s.pfn = None
    s.pfn_decoration = 0          # 0: PillarFeatureNet ([x, y, z, r, ...]), 1: PillarFeatureNetRadius ([|xy|, z, r, ...])
    if hasattr(vfe, "pfn_layers"):
        name = type(vfe).__name__
        # PillarFeatureNetRadiusHeight and PillarFeatureNetOld decorate differently (the latter overwrites x/y in place
        # through a view, so its Linear sees the centre offsets twice): same attributes, other numbers
        if name not in ("PillarFeatureNet", "PillarFeatureNetRadius"):
            raise UnsupportedNetwork("voxel feature extractor %s (PillarFeatureNet and PillarFeatureNetRadius are "
                                     "covered)" % name)
        s.pfn_decoration = 1 if name == "PillarFeatureNetRadius" else 0
        s.vfe_kind = "pfn"
        if len(vfe.pfn_layers) != 1:
            raise UnsupportedNetwork("multi-layer PillarFeatureNet (every BASELINE config has num_filters=[64])")
        lyr = vfe.pfn_layers[0]
        if not isinstance(lyr.norm, nn.BatchNorm1d) or lyr.linear.bias is not None:
            raise UnsupportedNetwork("PFNLayer without BatchNorm (use_norm=False)")
        sc, sh = fold_bn(lyr.norm)
        s.pfn = {"w": lyr.linear.weight.detach().float().contiguous(), "scale": sc, "shift": sh,
                 "cout": int(lyr.linear.weight.shape[0]), "vx": float(vfe.vx), "vy": float(vfe.vy),
                 "x_offset": float(vfe.x_offset), "y_offset": float(vfe.y_offset),
                 "with_distance": bool(getattr(vfe, "_with_distance", False))}
        s.num_point_features = int(lyr.linear.weight.shape[1]) - (4 if s.pfn_decoration else 5) - \
            (1 if s.pfn["with_distance"] else 0)
        s.vfe_num_features = s.num_point_features
    elif hasattr(vfe, "num_input_features") and not any(True for _ in vfe.parameters()):
        name = type(vfe).__name__
        if name not in ("SimpleVoxel", "SimpleVoxelRadius"):
            raise UnsupportedNetwork("voxel feature extractor %s" % name)
        s.vfe_kind = "mean" if name == "SimpleVoxel" else "mean_radius"
        s.vfe_num_features = int(vfe.num_input_features)
        s.num_point_features = int(getattr(net, "_num_input_features", s.vfe_num_features))
    else:
        raise UnsupportedNetwork("voxel feature extractor %s" % type(vfe).__name__)
    # ---- middle
    mid = net.middle_feature_extractor
    s.layers = []
    if hasattr(mid, "middle_conv") and hasattr(mid, "sparse_shape"):
        s.is_pillars = False
        s.sparse_shape = [int(x) for x in mid.sparse_shape]
        mods = list(mid.middle_conv._modules.values())
        i = 0
        while i < len(mods):
            m = mods[i]
            if not _is_sparse_conv(m):
                raise UnsupportedNetwork("middle_conv[%d] is %s, expected a sparse conv" % (i, type(m).__name__))
            bn = mods[i + 1] if i + 1 < len(mods) and isinstance(mods[i + 1], nn.BatchNorm1d) else None
            relu = i + 1 + (bn is not None) < len(mods) and isinstance(mods[i + 1 + (bn is not None)], nn.ReLU)
            ks = _triple(m.kernel_size)
            K = int(np.prod(ks))
            if K > 27 or getattr(m, "transposed", False) or getattr(m, "inverse", False) or \
                    getattr(m, "groups", 1) != 1:
                raise UnsupportedNetwork("sparse conv with K > 27 / transposed / groups")
            lyr = {"K": K, "kernel_size": ks, "stride": _triple(m.stride), "padding": _triple(m.padding),
                   "dilation": _triple(m.dilation), "subm": bool(m.subm), "indice_key": m.indice_key,
                   "cin": int(m.in_channels), "cout": int(m.out_channels), "relu": bool(relu),
                   "w": m.weight.detach().float().contiguous().view(K, m.in_channels, m.out_channels)}
            bias = m.bias.detach().float() if getattr(m, "bias", None) is not None else None
            if bn is not None:
                lyr["scale"], lyr["shift"] = fold_bn(bn)
                if bias is not None:                       # conv bias ahead of a BN: BN(x + b) = scale*x + (shift + scale*b)
                    lyr["shift"] = (lyr["shift"] + lyr["scale"] * bias).contiguous()
            else:
                lyr["scale"], lyr["shift"] = None, (bias.contiguous() if bias is not None else None)
            s.layers.append(lyr)
            i += 1 + (bn is not None) + (1 if relu else 0)
        if not s.layers:
            raise UnsupportedNetwork("empty middle_conv")
        s.bev_channels = None                                  # = last cout * final depth, known after planning
    elif all(hasattr(mid, a) for a in ("nx", "ny", "nchannels")):
        s.is_pillars = True
        s.sparse_shape = [1, int(mid.ny), int(mid.nx)]
        s.bev_channels = int(mid.nchannels)
        if s.vfe_kind != "pfn":
            raise UnsupportedNetwork("PointPillarsScatter without a PillarFeatureNet")
    else:
        raise UnsupportedNetwork("middle feature extractor %s" % type(mid).__name__)
    if not s.is_pillars and s.vfe_kind == "pfn":
        raise UnsupportedNetwork("PillarFeatureNet in front of a sparse middle extractor")
    # ---- RPN (layer plan is made by b2second.tc.plan_rpn from the module itself)
    rpn = net.rpn
    s.heads = None
    s.head_feature_map_sizes = None
    if hasattr(net, "small_head") or hasattr(net, "large_head"):
        _multi_head(net, s)
    else:
        for a in ("blocks", "deblocks", "conv_box", "conv_cls", "_upsample_start_idx", "_num_anchor_per_loc",
                  "_box_code_size", "_num_class"):
            if not hasattr(rpn, a):
                raise UnsupportedNetwork("RPN %s lacks attribute %s" % (type(rpn).__name__, a))
        s.num_class = int(rpn._num_class)
        s.box_code_size = int(rpn._box_code_size)
        s.num_anchors_per_loc = int(rpn._num_anchor_per_loc)
        s.use_direction_classifier = bool(getattr(rpn, "_use_direction_classifier", False))
        s.num_direction_bins = int(getattr(rpn, "_num_direction_bins", 2))
    s.rpn = rpn
    # ---- predict() parameters (voxelnet.py:104-143)
    if not getattr(net, "_encode_background_as_zeros", True) or not getattr(net, "_use_sigmoid_score", True):
        raise UnsupportedNetwork("softmax scores / background class (every BASELINE config: sigmoid, background as zeros)")
    s.use_rotate_nms = bool(net._use_rotate_nms)
    s.multiclass_nms = bool(net._multiclass_nms)
    s.nms_class_agnostic = bool(getattr(net, "_nms_class_agnostic", False))
    s.nms_score_thresholds = _f(net._nms_score_thresholds)
    s.nms_pre_max_sizes = [int(x) for x in net._nms_pre_max_sizes]
    s.nms_post_max_sizes = [int(x) for x in net._nms_post_max_sizes]
    s.nms_iou_thresholds = _f(net._nms_iou_thresholds)
    s.post_center_range = _f(getattr(net, "_post_center_range", None) or [])
    s.direction_offset = float(np.float32(getattr(net, "_dir_offset", 0.0)))
    s.direction_limit_offset = float(np.float32(getattr(net, "_dir_limit_offset", 0.0)))
    # per-class anchor index ranges (target_assigner.anchors_range, used by the per-class NMS branch)
    s.class_anchor_counts = None
    ta = getattr(net, "target_assigner", None)
    if ta is not None and hasattr(ta, "_anchor_generators"):
        s.class_anchor_counts = [int(g.num_anchors_per_localization) for g in ta._anchor_generators]
    if s.heads is not None:
        if s.multiclass_nms:
            raise UnsupportedNetwork("the per-class NMS branch on the multi-head network")
        _check_head_feature_maps(net, s)
    s.anchor_source = net
    s.layout = structure(s)          # as read now: the RPN and head modules are live, so refresh compares to this
    return s


STRUCTURE_KEYS = ("device", "vfe_kind", "vfe_num_features", "num_point_features", "is_pillars", "sparse_shape",
                  "pfn_decoration", "num_class", "box_code_size", "num_anchors_per_loc", "use_direction_classifier",
                  "num_direction_bins", "head_feature_map_sizes")


def structure(s):
    """what an engine's layout depends on: the spec with every weight tensor replaced by its shape (the predict()
    parameters and the voxel generator are left out: refresh does not re-read them)"""
    def layout(d):
        return None if d is None else {k: tuple(v.shape) if isinstance(v, torch.Tensor) else v for k, v in d.items()}

    def shapes(m):
        return {k: tuple(v.shape) for k, v in m.state_dict().items()}

    st = {k: getattr(s, k) for k in STRUCTURE_KEYS}
    st["layers"] = [layout(lyr) for lyr in s.layers]
    st["pfn"] = layout(s.pfn)
    st["rpn"] = shapes(s.rpn)
    st["heads"] = None if s.heads is None else [(name, shapes(m)) for name, m in s.heads]
    return st


def refresh(s, net):
    """re-read the weights of ``net`` (the module ``s`` was read from) into the spec ``s``: the sparse layers' weights
    and folded BatchNorm, the PFN's, and the RPN / head modules the engine plans from.  Raises UnsupportedNetwork, and
    leaves ``s`` as it was, when the network no longer has the structure of ``s`` (layers, shapes, head layout) or a
    parameter or BatchNorm buffer has left the spec's device."""
    new = spec_from_module(net, s.max_voxels)
    old_st, new_st = s.layout, new.layout
    if old_st != new_st:
        changed = sorted(k for k in old_st if old_st[k] != new_st[k])
        raise UnsupportedNetwork("the network's structure changed since it was accelerated (%s); accelerate a newly "
                                 "built network instead" % ", ".join(changed))
    tensors = list(net.parameters())
    for m in net.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            tensors += [t for t in (m.running_mean, m.running_var) if t is not None]
    if any(t.device != s.device for t in tensors):
        raise UnsupportedNetwork("a parameter or BatchNorm buffer is no longer on %s, the device the network was "
                                 "accelerated on" % s.device)
    s.layers, s.pfn, s.rpn, s.heads = new.layers, new.pfn, new.rpn, new.heads


def _head_module(m, what, with_net):
    for a in ("conv_box", "conv_cls", "_num_anchor_per_loc", "_box_code_size", "_num_class") + (("net",) if with_net else ()):
        if not hasattr(m, a):
            raise UnsupportedNetwork("%s %s lacks attribute %s" % (what, type(m).__name__, a))
    return m


def _multi_head(net, s):
    """VoxelNetNuscenesMultiHead (net_multi_head.py:121-176): large head (1x1 convs) on the RPN's concatenated map,
    small head (3 x Conv3x3+BN+ReLU, then 1x1 convs) on stage 0 cropped by round(0.1 H); predictions concatenated
    large first.  Any other arrangement is refused."""
    rpn = net.rpn
    if not (hasattr(net, "small_head") and hasattr(net, "large_head")):
        raise UnsupportedNetwork("a multi-head network needs both small_head and large_head")
    for a in ("blocks", "deblocks", "_upsample_start_idx"):
        if not hasattr(rpn, a):
            raise UnsupportedNetwork("RPN %s lacks attribute %s" % (type(rpn).__name__, a))
    if hasattr(rpn, "conv_box") or hasattr(rpn, "conv_cls"):
        raise UnsupportedNetwork("multi-head network whose RPN has heads of its own")
    large = _head_module(net.large_head, "large_head", False)
    small = _head_module(net.small_head, "small_head", True)
    if hasattr(large, "net"):
        raise UnsupportedNetwork("large_head with convolutions ahead of its 1x1 heads")
    for a in ("_num_class", "_box_code_size", "_use_direction_classifier", "_num_direction_bins"):
        if getattr(large, a, None) != getattr(small, a, None):
            raise UnsupportedNetwork("the two heads disagree on %s" % a)
    s.heads = [("large", large), ("small", small)]
    s.num_class = int(large._num_class)
    s.box_code_size = int(large._box_code_size)
    s.num_anchors_per_loc = int(large._num_anchor_per_loc) + int(small._num_anchor_per_loc)
    s.use_direction_classifier = bool(getattr(large, "_use_direction_classifier", False))
    s.num_direction_bins = int(getattr(large, "_num_direction_bins", 2))


def _check_head_feature_maps(net, s):
    """the anchors of the target assigner's classes, in order, must be the large head's a_loc on one feature map followed
    by the small head's on another (target_assigner.generate_anchors concatenates classes in config order)."""
    ta = getattr(net, "target_assigner", None)
    sizes = getattr(ta, "_feature_map_sizes", None)
    counts = s.class_anchor_counts
    if sizes is None or counts is None or len(sizes) != len(counts):
        raise UnsupportedNetwork("multi-head network without per-class feature map sizes")
    out, i = [], 0
    for _, m in s.heads:
        need, fs = int(m._num_anchor_per_loc), None
        while need > 0 and i < len(counts):
            f = [int(x) for x in sizes[i]]
            if len(f) != 3 or f[0] != 1 or (fs is not None and f != fs):
                raise UnsupportedNetwork("classes of one head on different feature maps (%s vs %s)" % (fs, f))
            fs, need, i = f, need - counts[i], i + 1
        if need != 0 or fs is None:
            raise UnsupportedNetwork("per-class anchor counts do not add up to the heads' anchors per location")
        out.append(fs[1:])
    if i != len(counts):
        raise UnsupportedNetwork("classes beyond the two heads' anchors")
    s.head_feature_map_sizes = out


def anchors_for(spec, feature_hw):
    """[A, code] float32 anchors of the network for an H x W RPN output map.

    mirror: ``net.anchors()``; reference: ``net.target_assigner.generate_anchors([1, H, W])``
    (second/core/target_assigner.py:169-207; feature-map rule second/builder/dataset_builder.py:58,66-67)."""
    net = spec.anchor_source
    H, W = feature_hw
    if hasattr(net, "anchors") and callable(net.anchors):
        a = net.anchors()
    else:
        ret = net.target_assigner.generate_anchors([1, int(H), int(W)])
        a = ret["anchors"]
    a = np.asarray(a, dtype=np.float32).reshape(-1, spec.box_code_size)
    return a
