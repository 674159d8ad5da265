"""Host-side mirror of second.pytorch's inference network (``VoxelNet.forward(example)``).

The GPU box has no copy of the reference, so the operator-level interface of the hot path is
mirrored here -- same class names, constructor meaning, ``forward(example)`` dict-in / list-out
contract and *state-dict keys*, so reference checkpoints load unchanged:

  VoxelNet.forward / network_forward / predict   second/pytorch/models/voxelnet.py:314-645
  SimpleVoxel / SimpleVoxelRadius                second/pytorch/models/voxel_encoder.py:206-255
  PillarFeatureNet / PFNLayer                    second/pytorch/models/pointpillars.py:22-65,153-237
  PillarFeatureNetRadius                         second/pytorch/models/pointpillars.py:240-325
  PointPillarsScatter                            second/pytorch/models/pointpillars.py:420-476
  SpMiddleFHD / SpMiddleFHDLite                  second/pytorch/models/middle.py:110-210,417-483
  RPNV2 (RPNBase/RPNNoHeadBase)                  second/pytorch/models/rpn.py:202-420,467-497
  RPNNoHead                                      second/pytorch/models/rpn.py:202-331,500-529
  VoxelNetNuscenesMultiHead, SmallObjectHead,
  DefaultHead                                    second/pytorch/models/net_multi_head.py:14-176

Every module takes the ``spconv`` *backend module* it should build on: the product backend is
``second.pytorch_b200/spconv`` (CUDA, fails loudly without the extension); tests and the CPU
baseline pass the oracle package instead.  Only the inference path is mirrored; the training loss is b2second.loss.
"""
from enum import Enum

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import box_ops
from .anchors import generate_anchors
from .config import ModelConfig


def _bn1d(c):
    return nn.BatchNorm1d(c, eps=1e-3, momentum=0.01)


def _bn2d(c):
    return nn.BatchNorm2d(c, eps=1e-3, momentum=0.01)


# ---------------------------------------------------------------------------------- VFE
class SimpleVoxel(nn.Module):
    def __init__(self, num_input_features=4, **kw):
        super().__init__()
        self.num_input_features = num_input_features

    def forward(self, features, num_voxels, coors):
        points_mean = features[:, :, :self.num_input_features].sum(dim=1, keepdim=False) \
            / num_voxels.type_as(features).view(-1, 1)
        return points_mean.contiguous()


class SimpleVoxelRadius(nn.Module):
    def __init__(self, num_input_features=4, **kw):
        super().__init__()
        self.num_input_features = num_input_features

    def forward(self, features, num_voxels, coors):
        points_mean = features[:, :, :self.num_input_features].sum(dim=1, keepdim=False) \
            / num_voxels.type_as(features).view(-1, 1)
        radius = torch.norm(points_mean[:, :2], p=2, dim=1, keepdim=True)
        return torch.cat([radius, points_mean[:, 2:self.num_input_features]], dim=1)


class PFNLayer(nn.Module):
    def __init__(self, in_channels, out_channels, last_layer=False):
        super().__init__()
        self.last_vfe = last_layer
        if not last_layer:
            out_channels = out_channels // 2
        self.units = out_channels
        self.linear = nn.Linear(in_channels, self.units, bias=False)
        self.norm = _bn1d(self.units)

    def forward(self, inputs):
        x = self.linear(inputs)
        x = self.norm(x.permute(0, 2, 1).contiguous()).permute(0, 2, 1).contiguous()
        x = F.relu(x)
        x_max = torch.max(x, dim=1, keepdim=True)[0]
        if self.last_vfe:
            return x_max
        return torch.cat([x, x_max.repeat(1, inputs.shape[1], 1)], dim=2)


class PillarFeatureNet(nn.Module):
    def __init__(self, num_input_features=4, num_filters=(64,), with_distance=False,
                 voxel_size=(0.2, 0.2, 4), pc_range=(0, -40, -3, 70.4, 40, 1), **kw):
        super().__init__()
        assert len(num_filters) > 0
        cin = num_input_features + 5 + (1 if with_distance else 0)
        self._with_distance = with_distance
        filters = [cin] + list(num_filters)
        self.pfn_layers = nn.ModuleList([
            PFNLayer(filters[i], filters[i + 1], last_layer=(i == len(filters) - 2))
            for i in range(len(filters) - 1)])
        self.vx = voxel_size[0]
        self.vy = voxel_size[1]
        self.x_offset = self.vx / 2 + pc_range[0]
        self.y_offset = self.vy / 2 + pc_range[1]

    def forward(self, features, num_voxels, coors):
        dtype = features.dtype
        points_mean = features[:, :, :3].sum(dim=1, keepdim=True) / num_voxels.type_as(features).view(-1, 1, 1)
        f_cluster = features[:, :, :3] - points_mean
        f_center = torch.zeros_like(features[:, :, :2])
        f_center[:, :, 0] = features[:, :, 0] - (coors[:, 3].to(dtype).unsqueeze(1) * self.vx + self.x_offset)
        f_center[:, :, 1] = features[:, :, 1] - (coors[:, 2].to(dtype).unsqueeze(1) * self.vy + self.y_offset)
        parts = [features, f_cluster, f_center]
        if self._with_distance:
            parts.append(torch.norm(features[:, :, :3], 2, 2, keepdim=True))
        features = torch.cat(parts, dim=-1)
        T = features.shape[1]
        mask = (num_voxels.int().unsqueeze(1) > torch.arange(T, dtype=torch.int, device=features.device).view(1, -1))
        features = features * mask.unsqueeze(-1).type_as(features)
        for pfn in self.pfn_layers:
            features = pfn(features)
        return features.squeeze()


class PillarFeatureNetRadius(nn.Module):
    """PillarFeatureNet with the point's x, y replaced by its radius |xy|: F+4 Linear inputs."""

    def __init__(self, num_input_features=4, num_filters=(64,), with_distance=False,
                 voxel_size=(0.2, 0.2, 4), pc_range=(0, -40, -3, 70.4, 40, 1), **kw):
        super().__init__()
        assert len(num_filters) > 0
        cin = num_input_features + 4 + (1 if with_distance else 0)
        self._with_distance = with_distance
        filters = [cin] + list(num_filters)
        self.pfn_layers = nn.ModuleList([
            PFNLayer(filters[i], filters[i + 1], last_layer=(i == len(filters) - 2))
            for i in range(len(filters) - 1)])
        self.vx = voxel_size[0]
        self.vy = voxel_size[1]
        self.x_offset = self.vx / 2 + pc_range[0]
        self.y_offset = self.vy / 2 + pc_range[1]

    def forward(self, features, num_voxels, coors):
        dtype = features.dtype
        points_mean = features[:, :, :3].sum(dim=1, keepdim=True) / num_voxels.type_as(features).view(-1, 1, 1)
        f_cluster = features[:, :, :3] - points_mean
        f_center = torch.zeros_like(features[:, :, :2])
        f_center[:, :, 0] = features[:, :, 0] - (coors[:, 3].to(dtype).unsqueeze(1) * self.vx + self.x_offset)
        f_center[:, :, 1] = features[:, :, 1] - (coors[:, 2].to(dtype).unsqueeze(1) * self.vy + self.y_offset)
        radius = torch.norm(features[:, :, :2], p=2, dim=2, keepdim=True)
        parts = [torch.cat([radius, features[:, :, 2:]], dim=2), f_cluster, f_center]
        if self._with_distance:
            parts.append(torch.norm(features[:, :, :3], 2, 2, keepdim=True))
        features = torch.cat(parts, dim=-1)
        T = features.shape[1]
        mask = (num_voxels.int().unsqueeze(1) > torch.arange(T, dtype=torch.int, device=features.device).view(1, -1))
        features = features * mask.unsqueeze(-1).type_as(features)
        for pfn in self.pfn_layers:
            features = pfn(features)
        return features.squeeze()


VFE_CLASSES = {"SimpleVoxel": SimpleVoxel, "SimpleVoxelRadius": SimpleVoxelRadius,
               "PillarFeatureNet": PillarFeatureNet, "PillarFeatureNetRadius": PillarFeatureNetRadius}


# ------------------------------------------------------------------------------- middle
class _SparseMiddle(nn.Module):
    def __init__(self, backend, output_shape):
        super().__init__()
        self._sp = backend
        self.sparse_shape = np.array(output_shape[1:4]) + [1, 0, 0]   # middle.py:139
        self.voxel_output_shape = output_shape

    def forward(self, voxel_features, coors, batch_size):
        sp = self._sp
        coors = coors.int()
        ret = sp.SparseConvTensor(voxel_features, coors, self.sparse_shape, batch_size)
        ret = self.middle_conv(ret)
        ret = ret.dense()
        N, C, D, H, W = ret.shape
        return ret.view(N, C * D, H, W)


class SpMiddleFHD(_SparseMiddle):
    def __init__(self, backend, output_shape, num_input_features=128, **kw):
        super().__init__(backend, output_shape)
        sp = backend

        def subm(cin, cout, key):
            return [sp.SubMConv3d(cin, cout, 3, bias=False, indice_key=key), _bn1d(cout), nn.ReLU()]

        def down(cin, cout, k, s, p):
            return [sp.SparseConv3d(cin, cout, k, s, padding=p, bias=False), _bn1d(cout), nn.ReLU()]

        layers = []
        layers += subm(num_input_features, 16, "subm0") + subm(16, 16, "subm0")
        layers += down(16, 32, 3, 2, 1)
        layers += subm(32, 32, "subm1") + subm(32, 32, "subm1")
        layers += down(32, 64, 3, 2, 1)
        layers += subm(64, 64, "subm2") + subm(64, 64, "subm2") + subm(64, 64, "subm2")
        layers += down(64, 64, 3, 2, [0, 1, 1])
        layers += subm(64, 64, "subm3") + subm(64, 64, "subm3") + subm(64, 64, "subm3")
        layers += down(64, 64, (3, 1, 1), (2, 1, 1), 0)
        self.middle_conv = sp.SparseSequential(*layers)


class SpMiddleFHDLite(_SparseMiddle):
    def __init__(self, backend, output_shape, num_input_features=128, **kw):
        super().__init__(backend, output_shape)
        sp = backend

        def down(cin, cout, k, s, p):
            return [sp.SparseConv3d(cin, cout, k, s, padding=p, bias=False), _bn1d(cout), nn.ReLU()]

        layers = down(num_input_features, 16, 3, 2, 1) + down(16, 32, 3, 2, 1) \
            + down(32, 64, 3, 2, [0, 1, 1]) + down(64, 64, (3, 1, 1), (2, 1, 1), 0)
        self.middle_conv = sp.SparseSequential(*layers)


class PointPillarsScatter(nn.Module):
    def __init__(self, backend, output_shape, num_input_features=64, **kw):
        super().__init__()
        self.output_shape = output_shape
        self.ny = output_shape[2]
        self.nx = output_shape[3]
        self.nchannels = num_input_features

    def forward(self, voxel_features, coords, batch_size):
        canvas = torch.zeros(batch_size, self.nchannels, self.ny * self.nx, dtype=voxel_features.dtype,
                             device=voxel_features.device)
        idx = (coords[:, 2] * self.nx + coords[:, 3]).long()
        canvas[coords[:, 0].long(), :, idx] = voxel_features
        return canvas.view(batch_size, self.nchannels, self.ny, self.nx)


MIDDLE_CLASSES = {"SpMiddleFHD": SpMiddleFHD, "SpMiddleFHDLite": SpMiddleFHDLite,
                  "PointPillarsScatter": PointPillarsScatter}


# ---------------------------------------------------------------------------------- RPN
class RPNNoHead(nn.Module):
    """the RPN backbone without heads; forward returns ``stage{i}`` (block outputs), ``up{i}`` (deblock outputs) and
    ``out`` (their concatenation), like RPNNoHeadBase.forward."""

    def __init__(self, num_class=2, layer_nums=(3, 5, 5), layer_strides=(2, 2, 2), num_filters=(128, 128, 256),
                 upsample_strides=(1, 2, 4), num_upsample_filters=(256, 256, 256), num_input_features=128,
                 num_anchor_per_loc=2, encode_background_as_zeros=True, use_direction_classifier=True,
                 box_code_size=7, num_direction_bins=2):
        super().__init__()
        assert len(layer_strides) == len(layer_nums) == len(num_filters)
        assert len(num_upsample_filters) == len(upsample_strides)
        self._upsample_start_idx = len(layer_nums) - len(upsample_strides)
        ratios = [upsample_strides[i] / np.prod(layer_strides[:i + self._upsample_start_idx + 1])
                  for i in range(len(upsample_strides))]
        assert all(r == ratios[0] for r in ratios)
        self._num_filters = list(num_filters)
        self._num_upsample_filters = list(num_upsample_filters)
        self._num_anchor_per_loc = num_anchor_per_loc
        self._num_direction_bins = num_direction_bins
        self._num_class = num_class
        self._use_direction_classifier = use_direction_classifier
        self._box_code_size = box_code_size
        in_filters = [num_input_features, *num_filters[:-1]]
        blocks, deblocks = [], []
        for i, layer_num in enumerate(layer_nums):
            mods = [nn.ZeroPad2d(1), nn.Conv2d(in_filters[i], num_filters[i], 3, stride=layer_strides[i], bias=False),
                    _bn2d(num_filters[i]), nn.ReLU()]
            for _ in range(layer_num):
                mods += [nn.Conv2d(num_filters[i], num_filters[i], 3, padding=1, bias=False),
                         _bn2d(num_filters[i]), nn.ReLU()]
            blocks.append(nn.Sequential(*mods))
            j = i - self._upsample_start_idx
            if j >= 0:
                stride = upsample_strides[j]
                if stride >= 1:
                    s = int(np.round(stride))
                    up = nn.ConvTranspose2d(num_filters[i], num_upsample_filters[j], s, stride=s, bias=False)
                else:
                    s = int(np.round(1 / stride))
                    up = nn.Conv2d(num_filters[i], num_upsample_filters[j], s, stride=s, bias=False)
                deblocks.append(nn.Sequential(up, _bn2d(num_upsample_filters[j]), nn.ReLU()))
        self.blocks = nn.ModuleList(blocks)
        self.deblocks = nn.ModuleList(deblocks)

    def forward(self, x):
        ups, res = [], {}
        for i in range(len(self.blocks)):
            x = self.blocks[i](x)
            res["stage%d" % i] = x
            if i - self._upsample_start_idx >= 0:
                ups.append(self.deblocks[i - self._upsample_start_idx](x))
        if len(ups) > 0:
            x = torch.cat(ups, dim=1)
        for i, up in enumerate(ups):
            res["up%d" % i] = up
        res["out"] = x
        return res


class RPNV2(RPNNoHead):
    def __init__(self, num_class=2, layer_nums=(3, 5, 5), layer_strides=(2, 2, 2), num_filters=(128, 128, 256),
                 upsample_strides=(1, 2, 4), num_upsample_filters=(256, 256, 256), num_input_features=128,
                 num_anchor_per_loc=2, encode_background_as_zeros=True, use_direction_classifier=True,
                 box_code_size=7, num_direction_bins=2):
        super().__init__(num_class, layer_nums, layer_strides, num_filters, upsample_strides, num_upsample_filters,
                         num_input_features, num_anchor_per_loc, encode_background_as_zeros, use_direction_classifier,
                         box_code_size, num_direction_bins)
        final = sum(num_upsample_filters) if len(num_upsample_filters) else num_filters[-1]
        num_cls = num_anchor_per_loc * (num_class if encode_background_as_zeros else num_class + 1)
        self.conv_cls = nn.Conv2d(final, num_cls, 1)
        self.conv_box = nn.Conv2d(final, num_anchor_per_loc * box_code_size, 1)
        if use_direction_classifier:
            self.conv_dir_cls = nn.Conv2d(final, num_anchor_per_loc * num_direction_bins, 1)

    def backbone(self, x):
        ups = []
        for i in range(len(self.blocks)):
            x = self.blocks[i](x)
            if i - self._upsample_start_idx >= 0:
                ups.append(self.deblocks[i - self._upsample_start_idx](x))
        if len(ups) > 0:
            x = torch.cat(ups, dim=1)
        return x

    def forward(self, x):
        x = self.backbone(x)
        box_preds = self.conv_box(x)
        cls_preds = self.conv_cls(x)
        C, H, W = box_preds.shape[1:]
        A = self._num_anchor_per_loc
        box_preds = box_preds.view(-1, A, self._box_code_size, H, W).permute(0, 1, 3, 4, 2).contiguous()
        cls_preds = cls_preds.view(-1, A, self._num_class, H, W).permute(0, 1, 3, 4, 2).contiguous()
        ret = {"box_preds": box_preds, "cls_preds": cls_preds}
        if self._use_direction_classifier:
            d = self.conv_dir_cls(x)
            ret["dir_cls_preds"] = d.view(-1, A, self._num_direction_bins, H, W).permute(0, 1, 3, 4, 2).contiguous()
        return ret


RPN_CLASSES = {"RPNV2": RPNV2, "RPNNoHead": RPNNoHead}


class DefaultHead(nn.Module):
    """1x1 box / cls / dir convs; predictions flattened to [B, A_loc*H*W, k] in (a_loc, y, x) order."""

    def __init__(self, num_filters, num_class, num_anchor_per_loc, box_code_size, num_direction_bins,
                 use_direction_classifier, encode_background_as_zeros):
        super().__init__()
        self._num_anchor_per_loc = num_anchor_per_loc
        self._num_direction_bins = num_direction_bins
        self._num_class = num_class
        self._use_direction_classifier = use_direction_classifier
        self._box_code_size = box_code_size
        num_cls = num_anchor_per_loc * (num_class if encode_background_as_zeros else num_class + 1)
        self.conv_cls = nn.Conv2d(num_filters, num_cls, 1)
        self.conv_box = nn.Conv2d(num_filters, num_anchor_per_loc * box_code_size, 1)
        if use_direction_classifier:
            self.conv_dir_cls = nn.Conv2d(num_filters, num_anchor_per_loc * num_direction_bins, 1)

    def forward(self, x):
        B = x.shape[0]
        box_preds = self.conv_box(x)
        cls_preds = self.conv_cls(x)
        C, H, W = box_preds.shape[1:]
        A = self._num_anchor_per_loc
        box_preds = box_preds.view(-1, A, self._box_code_size, H, W).permute(0, 1, 3, 4, 2).contiguous()
        cls_preds = cls_preds.view(-1, A, self._num_class, H, W).permute(0, 1, 3, 4, 2).contiguous()
        ret = {"box_preds": box_preds.view(B, -1, self._box_code_size), "cls_preds": cls_preds.view(B, -1, self._num_class)}
        if self._use_direction_classifier:
            d = self.conv_dir_cls(x)
            d = d.view(-1, A, self._num_direction_bins, H, W).permute(0, 1, 3, 4, 2).contiguous()
            ret["dir_cls_preds"] = d.view(B, -1, self._num_direction_bins)
        return ret


class SmallObjectHead(DefaultHead):
    """three Conv3x3 64 -> 64 (+BN, eps 1e-5, +ReLU) ahead of the 1x1 heads."""

    def __init__(self, num_filters, num_class, num_anchor_per_loc, box_code_size, num_direction_bins,
                 use_direction_classifier, encode_background_as_zeros):
        super().__init__(64, num_class, num_anchor_per_loc, box_code_size, num_direction_bins,
                         use_direction_classifier, encode_background_as_zeros)
        self.net = nn.Sequential(
            nn.Conv2d(num_filters, 64, 3, bias=False, padding=1), nn.BatchNorm2d(64), nn.ReLU(),
            nn.Conv2d(64, 64, 3, bias=False, padding=1), nn.BatchNorm2d(64), nn.ReLU(),
            nn.Conv2d(64, 64, 3, bias=False, padding=1), nn.BatchNorm2d(64), nn.ReLU())

    def forward(self, x):
        return super().forward(self.net(x))


# ------------------------------------------------------------------------------ VoxelNet
class _AnchorGeneratorInfo:
    def __init__(self, ac, ts):
        self.class_name = ac.class_name
        self.num_anchors_per_localization = ac.num_anchors_per_loc
        self.match_threshold = ts.matched_threshold if ts is not None else None
        self.unmatch_threshold = ts.unmatched_threshold if ts is not None else None
        self.custom_ndim = len(ac.custom_values)
        self.ndim = 7 + self.custom_ndim


# the region similarity calculators and box coders of second/core/region_similarity.py and box_coders.py, by the
# class names and attributes b2second.targets reads
class NearestIouSimilarity:
    pass


class RotateIouSimilarity:
    pass


class DistanceSimilarity:
    def __init__(self, distance_norm, with_rotation=False, rotation_alpha=0.5):
        self._distance_norm = distance_norm
        self._with_rotation = with_rotation
        self._rotation_alpha = rotation_alpha


class GroundBox3dCoder:
    def __init__(self, linear_dim=False, vec_encode=False, custom_ndim=0):
        self.linear_dim = linear_dim
        self.vec_encode = vec_encode
        self.custom_ndim = custom_ndim

    @property
    def code_size(self):
        return self.custom_ndim + (8 if self.vec_encode else 7)


class BevBoxCoder(GroundBox3dCoder):
    pass


def _similarity(ts):
    if ts.similarity == "distance":
        return DistanceSimilarity(ts.distance_norm, ts.with_rotation)
    return RotateIouSimilarity() if ts.similarity == "rotate_iou" else NearestIouSimilarity()


class MirrorTargetAssigner:
    """the slice of second/core/target_assigner.py ``TargetAssigner`` that inference and b2second.targets read: anchors
    per location, per-class anchor ranges (``anchors_range``, :269-278), ``generate_anchors`` (:169-207) and the
    assignment settings (thresholds, similarity calculators, box coder, positive fraction, per-class mode)."""

    def __init__(self, cfg):
        self._cfg = cfg
        ta = getattr(cfg, "target_assigner", None)
        tcs = ta.classes if ta is not None else [None] * len(cfg.classes)
        self._anchor_generators = [_AnchorGeneratorInfo(ac, ts) for ac, ts in zip(cfg.classes, tcs)]
        self._classes = [ac.class_name for ac in cfg.classes]
        # per-class anchor feature maps (class_settings.feature_map_size); None: every class on cfg.feature_map_size
        self._feature_map_sizes = [list(f) for f in cfg.class_feature_map_sizes] \
            if getattr(cfg, "class_feature_map_sizes", None) else None
        if ta is not None:
            self._sim_calcs = [_similarity(ts) for ts in ta.classes]
            coder = BevBoxCoder if ta.box_coder == "bev" else GroundBox3dCoder
            self._box_coder = coder(ta.linear_dim, ta.encode_angle_vector, self._anchor_generators[0].custom_ndim)
            self._positive_fraction = ta.sample_positive_fraction if ta.sample_positive_fraction >= 0 else None
            self._assign_per_class = ta.assign_per_class

    @property
    def classes(self):
        return self._classes

    @property
    def num_anchors_per_location(self):
        return self._cfg.num_anchors_per_loc

    def generate_anchors(self, feature_map_size):
        a = generate_anchors(self._cfg)
        fm = [int(x) for x in feature_map_size]
        if self._feature_map_sizes is None:
            assert a.shape[0] == self._cfg.num_anchors_per_loc * int(np.prod(fm)), \
                "feature map size does not match the config"
        return {"anchors": a}

    def _class_hw(self, c):
        fs = self._feature_map_sizes[c] if self._feature_map_sizes is not None else None
        return int(np.prod(fs if fs else self._cfg.feature_map_size))

    def anchors_range(self, class_idx):
        start = sum(g.num_anchors_per_localization * self._class_hw(c)
                    for c, g in enumerate(self._anchor_generators[:class_idx]))
        return start, start + self._anchor_generators[class_idx].num_anchors_per_localization * self._class_hw(class_idx)


class LossNormType(Enum):
    """voxelnet.py:51-55"""
    NormByNumPositives = "norm_by_num_positives"
    NormByNumExamples = "norm_by_num_examples"
    NormByNumPosNeg = "norm_by_num_pos_neg"
    DontNorm = "dont_norm"


class SigmoidFocalClassificationLoss:
    """the settings of second/pytorch/core/losses.py:236-253 under the reference's attribute names"""

    def __init__(self, gamma=2.0, alpha=0.25):
        self._alpha = alpha
        self._gamma = gamma


class WeightedSmoothL1LocalizationLoss:
    """the settings of losses.py:135-151 under the reference's attribute names"""

    def __init__(self, sigma=3.0, code_weights=None):
        self._sigma = sigma
        self._code_weights = torch.from_numpy(np.array(code_weights, dtype=np.float32)) \
            if code_weights is not None else None


class _UnsupportedLoss:
    """a loss block b2second.loss does not cover; ``kind`` is its protobuf name"""

    def __init__(self, kind):
        self.kind = kind


class VoxelNet(nn.Module):
    """Inference network with the reference's ``forward(example)`` contract.

    example keys (SURVEY.md App. E): ``voxels [N,T,F] f32``, ``num_points [N] i32``,
    ``coordinates [N,4] i32 (b,z,y,x)``, ``anchors [B,A,7] f32`` (+ optional ``anchors_mask``,
    ``metadata``, ``num_voxels``).  Returns a list of dicts ``box3d_lidar [n,7]``, ``scores [n]``,
    ``label_preds [n]``, ``metadata``.
    """

    def __init__(self, cfg: ModelConfig, backend):
        super().__init__()
        assert cfg.use_sigmoid_score and cfg.encode_background_as_zeros
        self.cfg = cfg
        self._sp = backend
        self.name = "voxelnet"
        self.voxel_generator = backend.utils.VoxelGeneratorV2(
            voxel_size=list(cfg.voxel_size), point_cloud_range=list(cfg.point_cloud_range),
            max_num_points=cfg.max_points_per_voxel, max_voxels=20000)
        self.voxel_feature_extractor = VFE_CLASSES[cfg.vfe_class](
            num_input_features=cfg.num_point_features, num_filters=cfg.vfe_num_filters,
            with_distance=cfg.vfe_with_distance, voxel_size=self.voxel_generator.voxel_size,
            pc_range=self.voxel_generator.point_cloud_range)
        self.middle_feature_extractor = MIDDLE_CLASSES[cfg.middle_class](
            backend, cfg.dense_shape, num_input_features=cfg.middle_num_input_features)
        self.rpn = RPN_CLASSES[cfg.rpn_class](
            num_class=cfg.num_class, layer_nums=cfg.rpn_layer_nums, layer_strides=cfg.rpn_layer_strides,
            num_filters=cfg.rpn_num_filters, upsample_strides=cfg.rpn_upsample_strides,
            num_upsample_filters=cfg.rpn_num_upsample_filters, num_input_features=cfg.rpn_num_input_features,
            num_anchor_per_loc=cfg.num_anchors_per_loc, encode_background_as_zeros=cfg.encode_background_as_zeros,
            use_direction_classifier=cfg.use_direction_classifier, box_code_size=cfg.box_code_size,
            num_direction_bins=cfg.num_direction_bins)
        self.register_buffer("global_step", torch.LongTensor(1).zero_())
        self._anchors_np = None
        # the reference's own attribute names (voxelnet.py:104-143): b2second.spec reads a network through these,
        # so the fused engine plans identically from this mirror and from the reference-built VoxelNet
        self._num_class = cfg.num_class
        self._num_input_features = cfg.num_point_features
        self._use_rotate_nms = cfg.use_rotate_nms
        self._multiclass_nms = cfg.use_multi_class_nms
        self._nms_class_agnostic = cfg.nms_class_agnostic
        nrep = cfg.num_class          # second_builder.py:47-62 passes one entry per class (equal unless multi-class NMS)
        self._nms_score_thresholds = [cfg.nms_score_threshold] * nrep
        self._nms_pre_max_sizes = [cfg.nms_pre_max_size] * nrep
        self._nms_post_max_sizes = [cfg.nms_post_max_size] * nrep
        self._nms_iou_thresholds = [cfg.nms_iou_threshold] * nrep
        self._use_sigmoid_score = cfg.use_sigmoid_score
        self._encode_background_as_zeros = cfg.encode_background_as_zeros
        self._use_direction_classifier = cfg.use_direction_classifier
        self._num_direction_bins = cfg.num_direction_bins
        self._post_center_range = list(cfg.post_center_limit_range)
        self._dir_offset = cfg.direction_offset
        self._dir_limit_offset = cfg.direction_limit_offset
        self.target_assigner = MirrorTargetAssigner(cfg)
        self._box_coder = getattr(self.target_assigner, "_box_coder", None)
        ls = getattr(cfg, "loss", None)
        if ls is not None:
            # the loss settings as second_builder.py:46-62 hands them to VoxelNet (voxelnet.py:110-141); what
            # b2second.loss.plan reads.  ``loss`` itself exists only after b2second.loss.enable_gpu_loss(net).
            self._cls_loss_ftor = SigmoidFocalClassificationLoss(ls.gamma, ls.alpha) \
                if ls.classification_loss == "weighted_sigmoid_focal" else _UnsupportedLoss(ls.classification_loss)
            self._loc_loss_ftor = WeightedSmoothL1LocalizationLoss(ls.sigma, ls.code_weight or None) \
                if ls.localization_loss == "weighted_smooth_l1" else _UnsupportedLoss(ls.localization_loss)
            self._loss_norm_type = LossNormType[ls.loss_norm_type]
            self._pos_cls_weight = ls.pos_class_weight
            self._neg_cls_weight = ls.neg_class_weight
            self._loc_loss_weight = ls.localization_weight
            self._cls_loss_weight = ls.classification_weight
            self._direction_loss_weight = ls.direction_loss_weight
            self._encode_rad_error_by_sin = ls.encode_rad_error_by_sin
            self._sin_error_factor = ls.sin_error_factor

    # -- helpers --------------------------------------------------------------------------
    def anchors(self):
        if self._anchors_np is None:
            self._anchors_np = generate_anchors(self.cfg)
        return self._anchors_np

    def update_global_step(self):
        """voxelnet.py:230-237"""
        self.global_step += 1

    def get_global_step(self):
        return int(self.global_step.cpu().numpy()[0])

    def clear_global_step(self):
        self.global_step.zero_()

    def load_reference_state_dict(self, sd):
        """load a reference checkpoint; training-metric buffers (rpn_acc.*, rpn_metrics.* ...) load once
        b2second.metrics.enable_gpu_metrics(net) has added them, and are skipped before."""
        own = self.state_dict()
        missing = [k for k in own if k not in sd]
        if missing:
            raise KeyError("checkpoint lacks keys: %s" % missing[:5])
        self.load_state_dict({k: sd[k] for k in own}, strict=True)

    # -- forward --------------------------------------------------------------------------
    def network_forward(self, voxels, num_points, coors, batch_size):
        voxel_features = self.voxel_feature_extractor(voxels, num_points, coors)
        spatial_features = self.middle_feature_extractor(voxel_features, coors, batch_size)
        return self.rpn(spatial_features)

    def forward(self, example):
        if "points" in example and not self.training:
            # raw clouds instead of voxels: only the fused engine takes those (b2second.fastpath); bind it once
            from . import fastpath
            fastpath.accelerate(self)
            return self.forward(example)
        voxels = example["voxels"]
        num_points = example["num_points"]
        coors = example["coordinates"]
        if len(num_points.shape) == 2:  # DataParallel padded layout (voxelnet.py:345-357)
            nv = example["num_voxels"].cpu().numpy().reshape(-1)
            voxels = torch.cat([voxels[i, :n] for i, n in enumerate(nv)], dim=0)
            num_points = torch.cat([num_points[i, :n] for i, n in enumerate(nv)], dim=0)
            coors = torch.cat([coors[i, :n] for i, n in enumerate(nv)], dim=0)
        batch_anchors = example["anchors"]
        batch_size_dev = batch_anchors.shape[0]
        preds_dict = self.network_forward(voxels, num_points, coors, batch_size_dev)
        box_preds = preds_dict["box_preds"].view(batch_size_dev, -1, self.cfg.box_code_size)
        assert batch_anchors.shape[1] == box_preds.shape[1], \
            f"num_anchors={batch_anchors.shape[1]}, but num_output={box_preds.shape[1]}. please check size"
        if self.training:
            if getattr(self, "b2s_loss", None) is None:
                raise NotImplementedError("only the inference path is mirrored (losses are out of scope)")
            # b2second.loss.enable_gpu_loss(net) bound ``loss`` to the CUDA loss (voxelnet.py:367-368)
            return self.loss(example, preds_dict)
        with torch.no_grad():
            return self.predict(example, preds_dict)

    def predict(self, example, preds_dict):
        cfg = self.cfg
        batch_size = example["anchors"].shape[0]
        meta_list = example.get("metadata") or [None] * batch_size
        batch_anchors = example["anchors"].view(batch_size, -1, example["anchors"].shape[-1])
        if "anchors_mask" in example:
            batch_anchors_mask = example["anchors_mask"].view(batch_size, -1)
        else:
            batch_anchors_mask = [None] * batch_size
        batch_box_preds = preds_dict["box_preds"].view(batch_size, -1, cfg.box_code_size)
        batch_cls_preds = preds_dict["cls_preds"].view(batch_size, -1, cfg.num_class)
        batch_box_preds = box_ops.second_box_decode(batch_box_preds, batch_anchors)
        if cfg.use_direction_classifier:
            batch_dir_preds = preds_dict["dir_cls_preds"].view(batch_size, -1, cfg.num_direction_bins)
        else:
            batch_dir_preds = [None] * batch_size
        post_center_range = None
        if len(cfg.post_center_limit_range) > 0:
            post_center_range = torch.tensor(cfg.post_center_limit_range, dtype=batch_box_preds.dtype,
                                             device=batch_box_preds.device).float()
        out = []
        for box_preds, cls_preds, dir_preds, a_mask, meta in zip(
                batch_box_preds, batch_cls_preds, batch_dir_preds, batch_anchors_mask, meta_list):
            if a_mask is not None:
                a_mask = a_mask.bool()
                box_preds = box_preds[a_mask]
                cls_preds = cls_preds[a_mask]
            box_preds = box_preds.float()
            cls_preds = cls_preds.float()
            dir_labels = None
            if cfg.use_direction_classifier:
                if a_mask is not None:
                    dir_preds = dir_preds[a_mask]
                dir_labels = torch.max(dir_preds, dim=-1)[1]
            total_scores = torch.sigmoid(cls_preds)
            if cfg.use_multi_class_nms:
                # per-class NMS branch (voxelnet.py:458-547)
                sel = self._predict_multiclass(box_preds, total_scores, dir_labels, a_mask)
                sel_boxes, sel_labels, sel_scores, sel_dir = sel
                out.append(self._finish_frame(sel_boxes, sel_scores, sel_labels, sel_dir, post_center_range, meta,
                                              batch_box_preds))
                continue
            if cfg.num_class == 1:
                top_scores = total_scores.squeeze(-1)
                top_labels = torch.zeros(total_scores.shape[0], device=total_scores.device, dtype=torch.long)
            else:
                top_scores, top_labels = torch.max(total_scores, dim=-1)
            thr = cfg.nms_score_threshold
            if thr > 0.0:
                keep_mask = top_scores >= thr
                top_scores = top_scores[keep_mask]
            if top_scores.shape[0] != 0:
                if thr > 0.0:
                    box_preds = box_preds[keep_mask]
                    if dir_labels is not None:
                        dir_labels = dir_labels[keep_mask]
                    top_labels = top_labels[keep_mask]
                boxes_for_nms = box_preds[:, [0, 1, 3, 4, 6]]
                selected = self._nms(boxes_for_nms, top_scores, cfg.nms_pre_max_size, cfg.nms_post_max_size,
                                     cfg.nms_iou_threshold)
            else:
                selected = torch.zeros([0], dtype=torch.long, device=box_preds.device)
            sel_dir = dir_labels[selected] if dir_labels is not None else None
            out.append(self._finish_frame(box_preds[selected], top_scores[selected], top_labels[selected], sel_dir,
                                          post_center_range, meta, batch_box_preds))
        return out


def _voxelnet_nms(self, boxes_for_nms, scores, pre_max, post_max, iou_thr):
    """rotate_nms / nms on BEV boxes (x, y, w, l, r) (voxelnet.py:449-456,571-584)."""
    if self.cfg.use_rotate_nms:
        return box_ops.rotate_nms(self._sp, boxes_for_nms, scores, pre_max, post_max, iou_thr)
    corners = box_ops.corners_2d_torch(boxes_for_nms[:, :2], boxes_for_nms[:, 2:4], boxes_for_nms[:, 4])
    return box_ops.aligned_nms(self._sp, box_ops.standup_torch(corners), scores, pre_max, post_max, iou_thr)


def _voxelnet_predict_multiclass(self, box_preds, total_scores, dir_labels, a_mask):
    """voxelnet.py:458-547: one NMS per class over that class's anchors (``target_assigner.anchors_range``) or, with
    ``nms_class_agnostic``, over all anchors; results concatenated in class order."""
    cfg = self.cfg
    assert a_mask is None or cfg.nms_class_agnostic, "anchors_mask + per-class anchor ranges is ill-defined upstream"
    boxes_for_nms = box_preds[:, [0, 1, 3, 4, 6]]
    A = box_preds.shape[0]
    hw = A // cfg.num_anchors_per_loc
    sel_boxes, sel_labels, sel_scores, sel_dir = [], [], [], []
    start = 0
    for c, ac in enumerate(cfg.classes):
        n_c = ac.num_anchors_per_loc
        if cfg.nms_class_agnostic:
            r0, r1 = 0, A
        else:
            r0, r1 = start * hw, (start + n_c) * hw
        start += n_c
        scores = total_scores[r0:r1, c].contiguous()
        cb, cbn = box_preds[r0:r1], boxes_for_nms[r0:r1]
        cd = dir_labels[r0:r1] if dir_labels is not None else None
        thr = self._nms_score_thresholds[c]
        if thr > 0.0:
            m = scores >= thr
            scores, cb, cbn = scores[m], cb[m], cbn[m]
            cd = cd[m] if cd is not None else None
        if scores.shape[0] == 0:
            continue
        keep = self._nms(cbn, scores, self._nms_pre_max_sizes[c], self._nms_post_max_sizes[c],
                         self._nms_iou_thresholds[c])
        if keep.shape[0] == 0:
            continue
        sel_boxes.append(cb[keep])
        sel_labels.append(torch.full([keep.shape[0]], c, dtype=torch.int64, device=box_preds.device))
        sel_scores.append(scores[keep])
        if cd is not None:
            sel_dir.append(cd[keep])
    if not sel_boxes:
        z = torch.zeros([0], dtype=torch.long, device=box_preds.device)
        return box_preds[z], z, total_scores[z, 0], (z if dir_labels is not None else None)
    return (torch.cat(sel_boxes), torch.cat(sel_labels), torch.cat(sel_scores),
            torch.cat(sel_dir) if dir_labels is not None else None)


def _voxelnet_finish_frame(self, sel_boxes, sel_scores, sel_labels, sel_dir, post_center_range, meta, like):
    """direction fix-up + post_center_range test + result dict (voxelnet.py:594-645)."""
    cfg = self.cfg
    if sel_boxes.shape[0] != 0:
        sel_boxes = sel_boxes.clone()
        if cfg.use_direction_classifier:
            period = 2 * np.pi / cfg.num_direction_bins
            dir_rot = box_ops.limit_period(sel_boxes[..., 6] - cfg.direction_offset, cfg.direction_limit_offset, period)
            sel_boxes[..., 6] = dir_rot + cfg.direction_offset + period * sel_dir.to(sel_boxes.dtype)
        if post_center_range is not None:
            m = (sel_boxes[:, :3] >= post_center_range[:3]).all(1)
            m &= (sel_boxes[:, :3] <= post_center_range[3:]).all(1)
            sel_boxes, sel_scores, sel_labels = sel_boxes[m], sel_scores[m], sel_labels[m]
        return {"box3d_lidar": sel_boxes, "scores": sel_scores, "label_preds": sel_labels, "metadata": meta}
    dev, dt = like.device, like.dtype
    return {"box3d_lidar": torch.zeros([0, cfg.box_code_size], dtype=dt, device=dev),
            "scores": torch.zeros([0], dtype=dt, device=dev),
            "label_preds": torch.zeros([0], dtype=torch.long, device=dev), "metadata": meta}


class VoxelNetNuscenesMultiHead(VoxelNet):
    """RPNNoHead backbone; a DefaultHead on the concatenated map for the large classes and a SmallObjectHead on the
    stage-0 map cropped by round(0.1 H) on every side for the small ones.  The predictions are concatenated
    (large first), which is the anchor order of the config (large classes listed first)."""
    small_classes = ["pedestrian", "traffic_cone", "bicycle", "motorcycle", "barrier"]
    large_classes = ["car", "truck", "trailer", "bus", "construction_vehicle"]

    def __init__(self, cfg, backend):
        super().__init__(cfg, backend)
        assert cfg.num_class == 10 and isinstance(self.rpn, RPNNoHead) and not isinstance(self.rpn, RPNV2)
        per_loc = {c.class_name: c.num_anchors_per_loc for c in cfg.classes}
        head_kw = dict(num_class=cfg.num_class, encode_background_as_zeros=cfg.encode_background_as_zeros,
                       use_direction_classifier=cfg.use_direction_classifier, box_code_size=cfg.box_code_size,
                       num_direction_bins=cfg.num_direction_bins)
        self.small_head = SmallObjectHead(num_filters=cfg.rpn_num_filters[0],
                                          num_anchor_per_loc=sum(per_loc[c] for c in self.small_classes), **head_kw)
        self.large_head = DefaultHead(num_filters=int(np.sum(cfg.rpn_num_upsample_filters)),
                                      num_anchor_per_loc=sum(per_loc[c] for c in self.large_classes), **head_kw)

    def network_forward(self, voxels, num_points, coors, batch_size):
        voxel_features = self.voxel_feature_extractor(voxels, num_points, coors)
        spatial_features = self.middle_feature_extractor(voxel_features, coors, batch_size)
        rpn_out = self.rpn(spatial_features)
        r1 = rpn_out["stage0"]
        c = int(np.round(r1.shape[2] * 0.1))
        small = self.small_head(r1[:, :, c:-c, c:-c])
        large = self.large_head(rpn_out["out"])
        res = {k: torch.cat([large[k], small[k]], dim=1) for k in ("box_preds", "cls_preds")}
        if self._use_direction_classifier:
            res["dir_cls_preds"] = torch.cat([large["dir_cls_preds"], small["dir_cls_preds"]], dim=1)
        return res


NETWORK_CLASSES = {"VoxelNet": VoxelNet, "VoxelNetNuscenesMultiHead": VoxelNetNuscenesMultiHead}


VoxelNet._nms = _voxelnet_nms
VoxelNet._predict_multiclass = _voxelnet_predict_multiclass
VoxelNet._finish_frame = _voxelnet_finish_frame


def build_network(cfg, backend):
    """counterpart of second/pytorch/train.py:58-68 ``build_network``."""
    if isinstance(cfg, str):
        from .config import get_config
        cfg = get_config(cfg)
    return NETWORK_CLASSES[getattr(cfg, "network_class", "VoxelNet")](cfg, backend)


# per-config constants for synthetic weights: head gain keeps box residuals O(0.3) (exp() stays finite),
# cls bias lets ~2 % of the anchors pass the score threshold on a seed-0 synthetic cloud, so top-k and
# NMS run at realistic sizes (SURVEY.md §8d).  Constants, not data-dependent: weights must be
# bit-identical wherever they are generated (golden fixtures, GPU box).
SYNTH_INIT = {
    # cls_sign=-1 for car.fhd: with +1 the constant "empty receptive field" logit lands in the top 2 %, i.e.
    # hundreds of exactly tied scores at the top-k boundary, where torch.topk's order is unspecified.
    "car.fhd": dict(cls_bias=-1.893, head_gain=1.0, cls_sign=-1.0),
    "car.lite": dict(cls_bias=-0.890, head_gain=0.5),
    "all.fhd": dict(cls_bias=-1.526, head_gain=1.0),
    "pointpillars.car.xyres_16": dict(cls_bias=-3.421, head_gain=0.15),
    "nuscenes.all.pp.largea": dict(cls_bias=-3.888, head_gain=0.02),
    "nuscenes.all.pp.mhead": dict(cls_bias=-3.9, head_gain=0.02),
}


def synthetic_weights_(net, name, seed=0):
    """seeded_init_ with the per-config constants of SYNTH_INIT."""
    return seeded_init_(net, seed, **SYNTH_INIT.get(name, {}))


def seeded_init_(net, seed=0, cls_bias=None, head_gain=1.0, cls_sign=1.0):
    """Deterministic synthetic weights (no checkpoints offline), reproducible on any host:
    every float entry of the state dict, in key order, is drawn from one CPU generator --
    conv/linear weights U(-b,b) with b = sqrt(6/fan_in), BN weight U(.5,1.5), bias N(0,.1),
    running_mean N(0,.1), running_var U(.5,1.5) (SURVEY.md §8(d) 'Weights').  The same function
    applied to the reference VoxelNet (same keys/shapes) yields identical parameters."""
    g = torch.Generator().manual_seed(seed)
    sd = net.state_dict()
    new = {}
    for k in sorted(sd.keys()):
        v = sd[k]
        if not v.dtype.is_floating_point or k.split(".")[0] in (
                "rpn_acc", "rpn_precision", "rpn_recall", "rpn_metrics", "rpn_cls_loss", "rpn_loc_loss",
                "rpn_total_loss"):
            continue
        leaf = k.split(".")[-1]
        if v.dim() >= 2:
            if "middle_conv" in k:          # spconv layout [kD,kH,kW,Cin,Cout]
                fan_in = int(np.prod(v.shape[:-1]))
            else:                            # conv2d [Cout,Cin,kh,kw] / linear [out,in] / convT [Cin,Cout,k,k]
                fan_in = int(np.prod(v.shape[1:]))
            b = float(np.sqrt(6.0 / max(fan_in, 1)))   # He-uniform: keeps activation scale through ReLU
            t = (torch.rand(v.shape, generator=g) * 2 - 1) * b
        elif leaf == "running_var":
            t = torch.rand(v.shape, generator=g) + 0.5
        elif leaf == "running_mean":
            t = torch.randn(v.shape, generator=g) * 0.1
        elif leaf == "weight":
            t = torch.rand(v.shape, generator=g) + 0.5
        elif leaf == "bias":
            t = torch.randn(v.shape, generator=g) * 0.1
        else:
            continue
        new[k] = t.to(v.dtype)
    for head in ("rpn", "small_head", "large_head"):      # the multi-head network's heads live beside the RPN
        cls_w = head + ".conv_cls.weight"
        for hk in (head + ".conv_cls.weight", head + ".conv_box.weight", head + ".conv_dir_cls.weight"):
            if hk in new:
                new[hk] = new[hk] * float(head_gain) * (float(cls_sign) if hk == cls_w else 1.0)
        if cls_bias is not None and head + ".conv_cls.bias" in new:
            new[head + ".conv_cls.bias"] = torch.full_like(new[head + ".conv_cls.bias"], float(cls_bias))
    merged = dict(sd)
    merged.update(new)
    net.load_state_dict(merged, strict=True)
    return net
