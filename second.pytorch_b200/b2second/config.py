"""Model configuration for the SECOND inference hot path.

The reference describes a model with protobuf text configs (second/protos/second.proto,
second/configs/*.config) turned into objects by second/pytorch/builder/second_builder.py:22-133 and
second/pytorch/train.py:58-68.  Here the same information is a plain dataclass so that the host
side needs neither protobuf nor the reference tree:

* ``parse_prototxt`` / ``ModelConfig.from_prototxt`` read a reference-format ``.config`` file
  (only the ``model.second`` and ``eval_input_reader`` blocks are interpreted);
* ``BUILTIN`` holds the five BASELINE.json configurations, written out by hand from the values in
  SURVEY.md App. B (car.fhd, car.lite, all.fhd, pointpillars/car/xyres_16, nuscenes/all.pp.largea);
  ``EXTRA`` the further ones ``get_config`` knows (nuscenes/all.pp.mhead, a ``MultiHeadModelConfig``);
* ``TargetAssignerSettings`` (what training target assignment reads: thresholds, similarity, box coder) rides along
  as the ``target_assigner`` attribute of a config -- parsed from the file, or written out in ``TARGET_ASSIGNERS`` for
  the builtins.  It is not a dataclass field, so the inference fields above keep their shape.
* ``AugmentSettings`` (``train_input_reader.preprocess``'s augmentation fields, what b2second.augment reads) rides
  along the same way as the ``augment`` attribute, written out in ``AUGMENTS`` for the builtins.
* ``DatabaseSamplerSettings`` (``train_input_reader.preprocess.database_sampler`` and the two preprocess fields that go
  with it, what b2second.dbsample reads) rides along as the ``db_sampler`` attribute (None without a sampler), written
  out in ``DB_SAMPLERS`` for the builtins.
* ``LossSettings`` (``model.second.loss`` and the loss fields of ``model.second``, what VoxelNet.loss and
  b2second.loss read) rides along as the ``loss`` attribute, written out in ``LOSSES`` for the builtins.
"""
import re
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np


@dataclass
class AnchorClass:
    class_name: str
    sizes: List[float] = field(default_factory=list)          # flat [w,l,h]*n ; empty = no_anchor
    rotations: List[float] = field(default_factory=lambda: [0.0, 1.57])
    anchor_ranges: Optional[List[float]] = None               # range generator (x0,y0,z0,x1,y1,z1)
    strides: Optional[List[float]] = None                     # stride generator
    offsets: Optional[List[float]] = None
    custom_values: List[float] = field(default_factory=list)

    @property
    def num_anchors_per_loc(self):
        if not self.sizes:
            return 0
        return (len(self.sizes) // 3) * len(self.rotations)


@dataclass
class ModelConfig:
    name: str
    point_cloud_range: List[float]
    voxel_size: List[float]
    max_points_per_voxel: int
    max_voxels: int                         # eval_input_reader.preprocess.max_number_of_voxels
    num_point_features: int
    vfe_class: str
    vfe_num_filters: List[int]
    vfe_with_distance: bool
    middle_class: str
    middle_num_input_features: int
    middle_downsample_factor: int
    rpn_class: str
    rpn_layer_nums: List[int]
    rpn_layer_strides: List[int]
    rpn_num_filters: List[int]
    rpn_upsample_strides: List[float]
    rpn_num_upsample_filters: List[int]
    rpn_num_input_features: int
    classes: List[AnchorClass]
    use_rotate_nms: bool
    use_multi_class_nms: bool
    nms_pre_max_size: int
    nms_post_max_size: int
    nms_score_threshold: float
    nms_iou_threshold: float
    post_center_limit_range: List[float]
    use_sigmoid_score: bool = True
    encode_background_as_zeros: bool = True
    use_direction_classifier: bool = True
    num_direction_bins: int = 2
    direction_limit_offset: float = 0.0
    direction_offset: float = 0.0
    nms_class_agnostic: bool = False
    eval_batch_size: int = 1
    anchor_area_threshold: float = -1.0
    box_code_size: int = 7

    # ---- derived quantities (mirrors of reference helpers) -------------------------------
    @property
    def grid_size(self):
        """xyz int64, as VoxelGeneratorV2.grid_size (round((hi-lo)/vs))."""
        r = np.array(self.point_cloud_range, dtype=np.float32)
        vs = np.array(self.voxel_size, dtype=np.float32)
        return np.round((r[3:] - r[:3]) / vs).astype(np.int64)

    @property
    def num_class(self):
        return len(self.classes)

    @property
    def num_anchors_per_loc(self):
        return sum(c.num_anchors_per_loc for c in self.classes)

    @property
    def downsample_factor(self):
        """second/utils/config_tool/__init__.py:45-52."""
        f = float(np.prod(self.rpn_layer_strides))
        if len(self.rpn_upsample_strides) > 0:
            f /= self.rpn_upsample_strides[-1]
        f *= self.middle_downsample_factor
        f = int(np.round(f))
        assert f > 0
        return f

    @property
    def feature_map_size(self):
        """[1, H, W] -- second/builder/dataset_builder.py:58,66-67."""
        fm = self.grid_size[:2] // self.downsample_factor
        return [1, int(fm[1]), int(fm[0])]

    @property
    def dense_shape(self):
        """[1, D, H, W, C] as second_builder.py:31."""
        g = self.grid_size
        return [1, int(g[2]), int(g[1]), int(g[0]), self.vfe_num_filters[-1]]

    # ---- prototxt -----------------------------------------------------------------------
    @staticmethod
    def from_prototxt(text, name="custom"):
        tree = parse_prototxt(text)
        m = _one(_one(tree["model"])["second"])
        ev = _one(tree["eval_input_reader"]) if "eval_input_reader" in tree else {}
        prep = _one(ev["preprocess"]) if "preprocess" in ev else {}
        vg = _one(m["voxel_generator"])
        vfe = _one(m["voxel_feature_extractor"])
        mid = _one(m["middle_feature_extractor"])
        rpn = _one(m["rpn"])
        ta = _one(m["target_assigner"])
        classes = []
        for cs in ta.get("class_settings", []):
            ac = AnchorClass(class_name=_one(cs.get("class_name", [""])))
            if "anchor_generator_range" in cs:
                g = _one(cs["anchor_generator_range"])
                ac.sizes = [float(v) for v in g["sizes"]]
                ac.rotations = [float(v) for v in g["rotations"]]
                ac.anchor_ranges = [float(v) for v in g["anchor_ranges"]]
                ac.custom_values = [float(v) for v in g.get("custom_values", [])]
            elif "anchor_generator_stride" in cs:
                g = _one(cs["anchor_generator_stride"])
                ac.sizes = [float(v) for v in g["sizes"]]
                ac.rotations = [float(v) for v in g["rotations"]]
                ac.strides = [float(v) for v in g["strides"]]
                ac.offsets = [float(v) for v in g["offsets"]]
                ac.custom_values = [float(v) for v in g.get("custom_values", [])]
            classes.append((ac, cs))
        first = classes[0][1]

        def cls_val(key, default):
            vals = [c[1].get(key, [default])[-1] for c in classes]
            assert all(v == vals[0] for v in vals), "per-class %s must agree (second_builder.py:55-59)" % key
            return vals[0]

        kw = {}
        cls = ModelConfig
        if _one(m.get("network_class_name", ["VoxelNet"])) == "VoxelNetNuscenesMultiHead":
            cls = MultiHeadModelConfig
            kw["class_feature_map_sizes"] = [[int(v) for v in c[1].get("feature_map_size", [])] for c in classes]
        cfg = cls(
            **kw,
            name=name,
            point_cloud_range=[float(v) for v in vg["point_cloud_range"]],
            voxel_size=[float(v) for v in vg["voxel_size"]],
            max_points_per_voxel=int(_one(vg["max_number_of_points_per_voxel"])),
            max_voxels=int(_one(prep.get("max_number_of_voxels", [20000]))),
            num_point_features=int(_one(m.get("num_point_features", [4]))),
            vfe_class=_one(vfe["module_class_name"]),
            vfe_num_filters=[int(v) for v in vfe.get("num_filters", [])],
            vfe_with_distance=bool(_one(vfe.get("with_distance", [False]))),
            middle_class=_one(mid["module_class_name"]),
            middle_num_input_features=int(_one(mid.get("num_input_features", [-1]))),
            middle_downsample_factor=int(_one(mid.get("downsample_factor", [1]))),
            rpn_class=_one(rpn["module_class_name"]),
            rpn_layer_nums=[int(v) for v in rpn["layer_nums"]],
            rpn_layer_strides=[int(v) for v in rpn["layer_strides"]],
            rpn_num_filters=[int(v) for v in rpn["num_filters"]],
            rpn_upsample_strides=[float(v) for v in rpn["upsample_strides"]],
            rpn_num_upsample_filters=[int(v) for v in rpn["num_upsample_filters"]],
            rpn_num_input_features=int(_one(rpn["num_input_features"])),
            classes=[c[0] for c in classes],
            use_rotate_nms=bool(cls_val("use_rotate_nms", False)),
            use_multi_class_nms=bool(cls_val("use_multi_class_nms", False)),
            nms_pre_max_size=int(cls_val("nms_pre_max_size", 1000)),
            nms_post_max_size=int(cls_val("nms_post_max_size", 100)),
            nms_score_threshold=float(cls_val("nms_score_threshold", 0.0)),
            nms_iou_threshold=float(cls_val("nms_iou_threshold", 0.5)),
            post_center_limit_range=[float(v) for v in m.get("post_center_limit_range", [])],
            use_sigmoid_score=bool(_one(m.get("use_sigmoid_score", [False]))),
            encode_background_as_zeros=bool(_one(m.get("encode_background_as_zeros", [False]))),
            use_direction_classifier=bool(_one(m.get("use_direction_classifier", [False]))),
            num_direction_bins=int(_one(m.get("num_direction_bins", [2]))),
            direction_limit_offset=float(_one(m.get("direction_limit_offset", [0.0]))),
            direction_offset=float(_one(m.get("direction_offset", [0.0]))),
            nms_class_agnostic=bool(_one(m.get("nms_class_agnostic", [False]))),
            eval_batch_size=int(_one(ev.get("batch_size", [1]))),
            anchor_area_threshold=float(_one(prep.get("anchor_area_threshold", [-1]))),
            box_code_size=7 + len(classes[0][0].custom_values),
        )
        cfg.target_assigner = _target_assigner_settings(m, ta)
        tr = _one(tree["train_input_reader"]) if "train_input_reader" in tree else {}
        cfg.augment = _augment_settings(_one(tr["preprocess"]) if "preprocess" in tr else {})
        cfg.db_sampler = _db_sampler_settings(_one(tr["preprocess"]) if "preprocess" in tr else {})
        cfg.loss = _loss_settings(m)
        return cfg

    @staticmethod
    def from_file(path, name=None):
        with open(path) as f:
            return ModelConfig.from_prototxt(f.read(), name or path)


@dataclass
class MultiHeadModelConfig(ModelConfig):
    """``network_class_name: "VoxelNetNuscenesMultiHead"`` (second/pytorch/models/net_multi_head.py:121-176): an
    RPNNoHead backbone with a DefaultHead on the concatenated map and a SmallObjectHead on the cropped stage-0 map.
    Each class has its own anchor feature map (``class_settings.feature_map_size``, [1, H, W]); the classes of the
    large head come first in the config."""
    network_class: str = "VoxelNetNuscenesMultiHead"
    class_feature_map_sizes: List[List[int]] = field(default_factory=list)


@dataclass
class ClassTargetSettings:
    """one ``class_settings`` entry's target-assignment part (second/protos/target.proto, similarity.proto).  Floats are
    the float32 values protobuf stores, widened to Python floats as the reference's builders read them."""
    matched_threshold: float
    unmatched_threshold: float
    similarity: str = "nearest_iou"            # nearest_iou | distance | rotate_iou
    distance_norm: float = 0.0
    with_rotation: bool = False


@dataclass
class TargetAssignerSettings:
    """``target_assigner`` and ``box_coder`` settings behind TargetAssigner.assign (proto3 defaults where absent)."""
    classes: List[ClassTargetSettings]
    assign_per_class: bool = False
    sample_positive_fraction: float = 0.0
    box_coder: str = "ground_box3d"            # ground_box3d | bev
    linear_dim: bool = False
    encode_angle_vector: bool = False


def _f32(v):
    return float(np.float32(v))


def _target_assigner_settings(m, ta):
    classes = []
    for cs in ta.get("class_settings", []):
        sim = _one(cs.get("region_similarity_calculator", [{}]))
        c = ClassTargetSettings(_f32(_one(cs.get("matched_threshold", [0.0]))),
                                _f32(_one(cs.get("unmatched_threshold", [0.0]))))
        if "distance_similarity" in sim:
            d = _one(sim["distance_similarity"])
            c.similarity = "distance"
            c.distance_norm = _f32(_one(d.get("distance_norm", [0.0])))
            c.with_rotation = bool(_one(d.get("with_rotation", [False])))
        elif "rotate_iou_similarity" in sim:
            c.similarity = "rotate_iou"
        classes.append(c)
    coder = _one(m.get("box_coder", [{"ground_box3d_coder": [{}]}]))
    kind = "bev" if "bev_box_coder" in coder else "ground_box3d"
    cc = _one(coder.get("bev_box_coder" if kind == "bev" else "ground_box3d_coder", [{}]))
    return TargetAssignerSettings(
        classes=classes, assign_per_class=bool(_one(ta.get("assign_per_class", [False]))),
        sample_positive_fraction=_f32(_one(ta.get("sample_positive_fraction", [0.0]))), box_coder=kind,
        linear_dim=bool(_one(cc.get("linear_dim", [False]))),
        encode_angle_vector=bool(_one(cc.get("encode_angle_vector", [False]))))


@dataclass
class AugmentSettings:
    """``train_input_reader.preprocess``'s augmentation fields (second/protos/input_reader.proto), as
    second/builder/dataset_builder.py:84-103 hands them to prep_pointcloud.  Floats are the float32 values protobuf
    stores, widened to Python floats; absent fields take proto3's defaults (empty lists, false)."""
    shuffle_points: bool = False
    groundtruth_localization_noise_std: List[float] = field(default_factory=list)
    groundtruth_rotation_uniform_noise: List[float] = field(default_factory=list)
    global_rotation_uniform_noise: List[float] = field(default_factory=list)
    global_scaling_uniform_noise: List[float] = field(default_factory=list)
    global_random_rotation_range_per_object: List[float] = field(default_factory=list)
    global_translate_noise_std: List[float] = field(default_factory=list)
    random_flip_x: bool = False
    random_flip_y: bool = False
    use_group_id: bool = False


def _augment_settings(prep):
    def floats(key):
        return [_f32(v) for v in prep.get(key, [])]

    def flag(key):
        return bool(_one(prep.get(key, [False])))

    return AugmentSettings(
        shuffle_points=flag("shuffle_points"),
        groundtruth_localization_noise_std=floats("groundtruth_localization_noise_std"),
        groundtruth_rotation_uniform_noise=floats("groundtruth_rotation_uniform_noise"),
        global_rotation_uniform_noise=floats("global_rotation_uniform_noise"),
        global_scaling_uniform_noise=floats("global_scaling_uniform_noise"),
        global_random_rotation_range_per_object=floats("global_random_rotation_range_per_object"),
        global_translate_noise_std=floats("global_translate_noise_std"),
        random_flip_x=flag("random_flip_x"), random_flip_y=flag("random_flip_y"), use_group_id=flag("use_group_id"))


@dataclass
class DatabaseSamplerSettings:
    """``train_input_reader.preprocess.database_sampler`` (second/protos/sampler.proto) as
    second/builder/dbsampler_builder.py hands it to DataBaseSamplerV2, with the two preprocess fields prep_pointcloud
    uses with it (second/protos/input_reader.proto).  sample_groups: one ``{name: max_num}`` per group, in file order;
    database_prep_steps: ``("filter_by_min_num_points", [(name, min_num), ...])`` or
    ``("filter_by_difficulty", [difficulty, ...])``, in file order.  Floats are protobuf's float32 values widened;
    absent fields take proto3's defaults."""
    sample_groups: List[dict] = field(default_factory=list)
    database_prep_steps: List[tuple] = field(default_factory=list)
    rate: float = 0.0
    global_random_rotation_range_per_object: List[float] = field(default_factory=list)
    database_info_path: str = ""
    remove_points_after_sample: bool = False
    sample_importance: float = 0.0


def _db_sampler_settings(prep):
    """None when the block enables no sampler (second/builder/dataset_builder.py:61-64)"""
    ds = _one(prep["database_sampler"]) if "database_sampler" in prep else {}
    groups = [{_one(kv["key"]): int(_one(kv["value"])) for kv in g.get("name_to_max_num", [])}
              for g in ds.get("sample_groups", [])]
    path = _one(ds.get("database_info_path", [""]))
    if not groups and path == "":
        return None
    steps = []
    for st in ds.get("database_prep_steps", []):
        if "filter_by_min_num_points" in st:
            pairs = _one(st["filter_by_min_num_points"]).get("min_num_point_pairs", [])
            steps.append(("filter_by_min_num_points", [(_one(kv["key"]), int(_one(kv["value"]))) for kv in pairs]))
        elif "filter_by_difficulty" in st:
            steps.append(("filter_by_difficulty",
                          [int(v) for v in _one(st["filter_by_difficulty"]).get("removed_difficulties", [])]))
        else:
            raise ValueError("unknown database prep step %r" % (sorted(st),))
    return DatabaseSamplerSettings(
        sample_groups=groups, database_prep_steps=steps, rate=_f32(_one(ds.get("rate", [0.0]))),
        global_random_rotation_range_per_object=[_f32(v) for v in ds.get("global_random_rotation_range_per_object", [])],
        database_info_path=path, remove_points_after_sample=bool(_one(prep.get("remove_points_after_sample", [False]))),
        sample_importance=_f32(_one(prep.get("sample_importance", [0.0]))))


@dataclass
class LossSettings:
    """``model.second.loss`` (second/protos/losses.proto) and the loss fields of ``model.second`` (second.proto), as
    second/pytorch/builder/second_builder.py:46-62 and losses_builder.py hand them to VoxelNet.  Floats are protobuf's
    float32 values widened; absent fields take proto3's defaults, except sin_error_factor, where the builder turns 0
    into 1.  code_weight empty: none (the loss applies no code weights)."""
    classification_loss: str = ""                 # weighted_sigmoid_focal | weighted_sigmoid | weighted_softmax ...
    alpha: float = 0.0
    gamma: float = 0.0
    localization_loss: str = ""                   # weighted_smooth_l1 | weighted_l2 ...
    sigma: float = 0.0
    code_weight: List[float] = field(default_factory=list)
    classification_weight: float = 0.0
    localization_weight: float = 0.0
    loss_norm_type: str = "NormByNumExamples"
    pos_class_weight: float = 0.0
    neg_class_weight: float = 0.0
    encode_rad_error_by_sin: bool = False
    sin_error_factor: float = 1.0
    direction_loss_weight: float = 0.0


def _loss_settings(m):
    loss = _one(m.get("loss", [{}]))
    cl = _one(loss.get("classification_loss", [{}]))
    ll = _one(loss.get("localization_loss", [{}]))
    ckind = next(iter(cl), "")
    lkind = next(iter(ll), "")
    cc = _one(cl[ckind]) if ckind else {}
    lc = _one(ll[lkind]) if lkind else {}
    sin_factor = _f32(_one(m.get("sin_error_factor", [0.0])))
    return LossSettings(
        classification_loss=ckind, alpha=_f32(_one(cc.get("alpha", [0.0]))), gamma=_f32(_one(cc.get("gamma", [0.0]))),
        localization_loss=lkind, sigma=_f32(_one(lc.get("sigma", [0.0]))),
        code_weight=[_f32(v) for v in lc.get("code_weight", [])],
        classification_weight=_f32(_one(loss.get("classification_weight", [0.0]))),
        localization_weight=_f32(_one(loss.get("localization_weight", [0.0]))),
        loss_norm_type=str(_one(m.get("loss_norm_type", ["NormByNumExamples"]))),
        pos_class_weight=_f32(_one(m.get("pos_class_weight", [0.0]))),
        neg_class_weight=_f32(_one(m.get("neg_class_weight", [0.0]))),
        encode_rad_error_by_sin=bool(_one(m.get("encode_rad_error_by_sin", [False]))),
        sin_error_factor=sin_factor if sin_factor != 0 else 1.0,
        direction_loss_weight=_f32(_one(m.get("direction_loss_weight", [0.0]))))


def _one(v):
    assert isinstance(v, list) and len(v) >= 1
    return v[-1]


_TOKEN = re.compile(r'\s*(?:(#[^\n]*)|([{}\[\]:,])|"((?:[^"\\]|\\.)*)"|([^\s{}\[\]:,#"]+))')


def parse_prototxt(text):
    """Minimal protobuf text-format reader: -> dict name -> list of values (scalars or dicts)."""
    toks = []
    pos = 0
    while pos < len(text):
        m = _TOKEN.match(text, pos)
        if m is None:
            if text[pos:].strip() == "":
                break
            raise ValueError("prototxt: cannot tokenise at %d: %r" % (pos, text[pos:pos + 20]))
        pos = m.end()
        if m.group(1) is not None:
            continue
        if m.group(2) is not None:
            toks.append(("p", m.group(2)))
        elif m.group(3) is not None:
            toks.append(("s", m.group(3)))
        else:
            toks.append(("w", m.group(4)))

    def scalar(kind, tok):
        if kind == "s":
            return tok
        if tok in ("true", "True"):
            return True
        if tok in ("false", "False"):
            return False
        try:
            if re.fullmatch(r"[-+]?\d+", tok):
                return int(tok)
            return float(tok)
        except ValueError:
            return tok  # enum identifier

    def block(i, closing):
        out = {}
        while i < len(toks):
            kind, tok = toks[i]
            if kind == "p" and tok == closing:
                return out, i + 1
            if kind != "w":
                raise ValueError("prototxt: expected field name, got %r" % (tok,))
            name = tok
            i += 1
            if i < len(toks) and toks[i] == ("p", ":"):
                i += 1
            kind, tok = toks[i]
            if kind == "p" and tok == "{":
                val, i = block(i + 1, "}")
                out.setdefault(name, []).append(val)
            elif kind == "p" and tok == "[":
                i += 1
                while toks[i] != ("p", "]"):
                    if toks[i] == ("p", ","):
                        i += 1
                        continue
                    out.setdefault(name, []).append(scalar(*toks[i]))
                    i += 1
                out.setdefault(name, [])
                i += 1
            else:
                out.setdefault(name, []).append(scalar(kind, tok))
                i += 1
        if closing is not None:
            raise ValueError("prototxt: unbalanced braces")
        return out, i

    tree, _ = block(0, None)
    return tree


# ------------------------------------------------------------------------------------------
# The five BASELINE.json configurations (values: SURVEY.md App. B and the cited config lines)
# ------------------------------------------------------------------------------------------
def _car_fhd():
    # second/configs/car.fhd.config:1-110,205-217
    return ModelConfig(
        name="car.fhd", point_cloud_range=[0, -40, -3, 70.4, 40, 1], voxel_size=[0.05, 0.05, 0.1],
        max_points_per_voxel=5, max_voxels=40000, num_point_features=4,
        vfe_class="SimpleVoxel", vfe_num_filters=[16], vfe_with_distance=False,
        middle_class="SpMiddleFHD", middle_num_input_features=4, middle_downsample_factor=8,
        rpn_class="RPNV2", rpn_layer_nums=[5], rpn_layer_strides=[1], rpn_num_filters=[128],
        rpn_upsample_strides=[1], rpn_num_upsample_filters=[128], rpn_num_input_features=128,
        classes=[AnchorClass("Car", [1.6, 3.9, 1.56], [0, 1.57], anchor_ranges=[0, -40.0, -1.0, 70.4, 40.0, -1.0])],
        use_rotate_nms=True, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=100,
        nms_score_threshold=0.3, nms_iou_threshold=0.01,
        post_center_limit_range=[0, -40, -2.2, 70.4, 40, 0.8], direction_limit_offset=1.0,
        eval_batch_size=8)


def _car_lite():
    # second/configs/car.lite.config
    return ModelConfig(
        name="car.lite", point_cloud_range=[0, -32.0, -3, 52.8, 32.0, 1], voxel_size=[0.05, 0.05, 0.1],
        max_points_per_voxel=1, max_voxels=30000, num_point_features=4,
        vfe_class="SimpleVoxelRadius", vfe_num_filters=[16], vfe_with_distance=False,
        middle_class="SpMiddleFHDLite", middle_num_input_features=3, middle_downsample_factor=8,
        rpn_class="RPNV2", rpn_layer_nums=[5], rpn_layer_strides=[1], rpn_num_filters=[128],
        rpn_upsample_strides=[1], rpn_num_upsample_filters=[128], rpn_num_input_features=128,
        classes=[AnchorClass("Car", [1.6, 3.9, 1.56], [0, 1.57], anchor_ranges=[0, -32.0, -1.0, 52.8, 32.0, -1.0])],
        use_rotate_nms=True, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=100,
        nms_score_threshold=0.3, nms_iou_threshold=0.01,
        post_center_limit_range=[0, -40, -2.2, 70.4, 40, 0.8], direction_limit_offset=1.0,
        eval_batch_size=12)


def _all_fhd():
    # second/configs/all.fhd.config
    def rng(z):
        return [0, -32.0, z, 52.8, 32.0, z]
    return ModelConfig(
        name="all.fhd", point_cloud_range=[0, -32.0, -3, 52.8, 32.0, 1], voxel_size=[0.05, 0.05, 0.1],
        max_points_per_voxel=5, max_voxels=60000, num_point_features=4,
        vfe_class="SimpleVoxelRadius", vfe_num_filters=[16], vfe_with_distance=False,
        middle_class="SpMiddleFHD", middle_num_input_features=3, middle_downsample_factor=8,
        rpn_class="RPNV2", rpn_layer_nums=[5, 5], rpn_layer_strides=[1, 2], rpn_num_filters=[64, 128],
        rpn_upsample_strides=[1, 2], rpn_num_upsample_filters=[128, 128], rpn_num_input_features=128,
        classes=[
            AnchorClass("Car", [1.6, 3.9, 1.56], [0, 1.57], anchor_ranges=rng(-1.0)),
            AnchorClass("Cyclist", [0.6, 1.76, 1.73], [0, 1.57], anchor_ranges=rng(-0.6)),
            AnchorClass("Pedestrian", [0.6, 0.8, 1.73], [0, 1.57], anchor_ranges=rng(-0.6)),
            AnchorClass("Van", [1.87103749, 5.02808195, 2.20964255], [0, 1.57], anchor_ranges=rng(-1.41)),
        ],
        use_rotate_nms=True, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=100,
        nms_score_threshold=0.3, nms_iou_threshold=0.1,
        post_center_limit_range=[0, -40, -2.2, 70.4, 40, 0.8], direction_limit_offset=1.0,
        eval_batch_size=3)


def _pp_xyres16():
    # second/configs/pointpillars/car/xyres_16.config
    return ModelConfig(
        name="pointpillars.car.xyres_16", point_cloud_range=[0, -39.68, -3, 69.12, 39.68, 1],
        voxel_size=[0.16, 0.16, 4], max_points_per_voxel=100, max_voxels=12000, num_point_features=4,
        vfe_class="PillarFeatureNet", vfe_num_filters=[64], vfe_with_distance=False,
        middle_class="PointPillarsScatter", middle_num_input_features=64, middle_downsample_factor=1,
        rpn_class="RPNV2", rpn_layer_nums=[3, 5, 5], rpn_layer_strides=[2, 2, 2],
        rpn_num_filters=[64, 128, 256], rpn_upsample_strides=[1, 2, 4],
        rpn_num_upsample_filters=[128, 128, 128], rpn_num_input_features=64,
        classes=[AnchorClass("Car", [1.6, 3.9, 1.56], [0, 1.57], strides=[0.32, 0.32, 0.0],
                             offsets=[0.16, -39.52, -1.78])],
        use_rotate_nms=False, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=300,
        nms_score_threshold=0.05, nms_iou_threshold=0.5,
        post_center_limit_range=[0, -39.68, -5, 69.12, 39.68, 5], direction_limit_offset=1.0,
        eval_batch_size=2, anchor_area_threshold=1.0)


def _nusc_largea():
    # second/configs/nuscenes/all.pp.largea.config
    def rng(z):
        return [-50, -50, z, 50, 50, z]
    return ModelConfig(
        name="nuscenes.all.pp.largea", point_cloud_range=[-50, -50, -10, 50, 50, 10],
        voxel_size=[0.25, 0.25, 20], max_points_per_voxel=60, max_voxels=30000, num_point_features=4,
        vfe_class="PillarFeatureNet", vfe_num_filters=[64], vfe_with_distance=False,
        middle_class="PointPillarsScatter", middle_num_input_features=64, middle_downsample_factor=1,
        rpn_class="RPNV2", rpn_layer_nums=[3, 5, 5], rpn_layer_strides=[2, 2, 2],
        rpn_num_filters=[64, 128, 256], rpn_upsample_strides=[0.25, 0.5, 1],
        rpn_num_upsample_filters=[128, 128, 128], rpn_num_input_features=64,
        classes=[
            AnchorClass("car", [1.95017717, 4.60718145, 1.72270761], [0, 1.57], anchor_ranges=rng(-0.93897414)),
            AnchorClass("bus", [2.94046906, 11.1885991, 3.47030982], [0, 1.57], anchor_ranges=rng(-0.0715754)),
            AnchorClass("construction_vehicle", [2.73050468, 6.38352896, 3.13312415], [0, 1.57],
                        anchor_ranges=rng(-0.08168083)),
            AnchorClass("trailer", [3, 15, 3.8, 2, 3, 3.8], [0, 1.57], anchor_ranges=rng(0.22228277)),
            AnchorClass("truck", [2.4560939, 6.73778078, 2.73004906], [0, 1.57], anchor_ranges=rng(-0.37937912)),
            AnchorClass("bicycle"), AnchorClass("motorcycle"), AnchorClass("pedestrian"),
            AnchorClass("traffic_cone"), AnchorClass("barrier"),
        ],
        use_rotate_nms=False, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=300,
        nms_score_threshold=0.05, nms_iou_threshold=0.5,
        post_center_limit_range=[-59.6, -59.6, -10, 59.6, 59.6, 10], direction_limit_offset=0.0,
        direction_offset=0.78, nms_class_agnostic=True, eval_batch_size=1)


def _nusc_mhead():
    # second/configs/nuscenes/all.pp.mhead.config
    def rng(z, r=50):
        return [-r, -r, z, r, r, z]
    big, small = [1, 100, 100], [1, 160, 160]
    return MultiHeadModelConfig(
        name="nuscenes.all.pp.mhead", point_cloud_range=[-50, -50, -5, 50, 50, 3],
        voxel_size=[0.25, 0.25, 8], max_points_per_voxel=60, max_voxels=30000, num_point_features=4,
        vfe_class="PillarFeatureNetRadius", vfe_num_filters=[64], vfe_with_distance=False,
        middle_class="PointPillarsScatter", middle_num_input_features=64, middle_downsample_factor=1,
        rpn_class="RPNNoHead", rpn_layer_nums=[3, 5, 5], rpn_layer_strides=[2, 2, 2],
        rpn_num_filters=[64, 128, 256], rpn_upsample_strides=[0.5, 1, 2],
        rpn_num_upsample_filters=[128, 128, 128], rpn_num_input_features=64,
        classes=[
            AnchorClass("bus", [2.94046906, 11.1885991, 3.47030982], [0, 1.57], anchor_ranges=rng(-0.0715754)),
            AnchorClass("car", [1.95017717, 4.60718145, 1.72270761], [0, 1.57], anchor_ranges=rng(-0.93897414)),
            AnchorClass("construction_vehicle", [2.73050468, 6.38352896, 3.13312415], [0, 1.57],
                        anchor_ranges=rng(-0.08168083)),
            AnchorClass("trailer", [3, 15, 3.8, 2, 3, 3.8], [0, 1.57], anchor_ranges=rng(0.22228277)),
            AnchorClass("truck", [2.4560939, 6.73778078, 2.73004906], [0, 1.57], anchor_ranges=rng(-0.37937912)),
            AnchorClass("barrier", [2.49008838, 0.48578221, 0.98297065], [0, 1.57], anchor_ranges=rng(-1.27247968, 40)),
            AnchorClass("bicycle", [0.60058911, 1.68452161, 1.27192197], [0, 1.57], anchor_ranges=rng(-1.03743013, 40)),
            AnchorClass("motorcycle", [0.76279481, 2.09973778, 1.44403034], [0, 1.57],
                        anchor_ranges=rng(-0.99194854, 40)),
            AnchorClass("pedestrian", [0.66344886, 0.7256437, 1.75748069], [0], anchor_ranges=rng(-0.73911038, 40)),
            AnchorClass("traffic_cone", [0.39694519, 0.40359262, 1.06232151], [0], anchor_ranges=rng(-1.27868911, 40)),
        ],
        use_rotate_nms=False, use_multi_class_nms=False, nms_pre_max_size=1000, nms_post_max_size=300,
        nms_score_threshold=0.05, nms_iou_threshold=0.5,
        post_center_limit_range=[-59.6, -59.6, -10, 59.6, 59.6, 10], direction_limit_offset=0.0,
        direction_offset=0.78, nms_class_agnostic=False, eval_batch_size=1,
        class_feature_map_sizes=[big] * 5 + [small] * 5)


BUILTIN = {
    "car.fhd": _car_fhd,
    "car.lite": _car_lite,
    "all.fhd": _all_fhd,
    "pointpillars.car.xyres_16": _pp_xyres16,
    "nuscenes.all.pp.largea": _nusc_largea,
}

# reference config file (relative to second/configs) for each builtin -- used by the container-only
# drop-in tests to check the hand-written dataclasses against the parsed reference files.
REFERENCE_FILES = {
    "car.fhd": "car.fhd.config",
    "car.lite": "car.lite.config",
    "all.fhd": "all.fhd.config",
    "pointpillars.car.xyres_16": "pointpillars/car/xyres_16.config",
    "nuscenes.all.pp.largea": "nuscenes/all.pp.largea.config",
}


# configs beyond the five BASELINE ones: get_config knows them, BUILTIN (what the BASELINE suites iterate) does not
EXTRA = {
    "nuscenes.all.pp.mhead": _nusc_mhead,
}
EXTRA_REFERENCE_FILES = {
    "nuscenes.all.pp.mhead": "nuscenes/all.pp.mhead.config",
}


def _ta(per_class, *classes):
    """classes: (matched, unmatched) or (matched, unmatched, distance_norm) for a DistanceSimilarity without rotation"""
    return TargetAssignerSettings(
        classes=[ClassTargetSettings(_f32(c[0]), _f32(c[1])) if len(c) == 2 else
                 ClassTargetSettings(_f32(c[0]), _f32(c[1]), "distance", _f32(c[2])) for c in classes],
        assign_per_class=per_class, sample_positive_fraction=-1.0)


# target-assignment settings of the builtins (the target_assigner / box_coder blocks of the cited config files; every
# one uses ground_box3d_coder with linear_dim and encode_angle_vector false)
TARGET_ASSIGNERS = {
    "car.fhd": lambda: _ta(True, (0.6, 0.45)),
    "car.lite": lambda: _ta(True, (0.6, 0.45)),
    "all.fhd": lambda: _ta(True, (0.6, 0.45), (0.35, 0.2), (0.35, 0.2), (0.6, 0.45)),
    "pointpillars.car.xyres_16": lambda: _ta(True, (0.6, 0.45)),
    "nuscenes.all.pp.largea": lambda: _ta(False, (0.4, 0.3), (0.5, 0.35), (0.5, 0.35), (0.5, 0.35), (0.5, 0.35),
                                          (0.2, 0.15), (0.2, 0.15), (0.5, 0.35, 1.414), (0.5, 0.35, 1.414),
                                          (0.3, 0.2)),
    "nuscenes.all.pp.mhead": lambda: _ta(True, (0.5, 0.35), (0.4, 0.3), (0.4, 0.3), (0.5, 0.35), (0.5, 0.35),
                                         (0.3, 0.2), (0.3, 0.2), (0.3, 0.2), (0.2, 0.1), (0.5, 0.35, 1.0)),
}


def _aug(loc, rot, grot, scale, translate, flip_x, shuffle):
    return AugmentSettings(
        shuffle_points=shuffle, groundtruth_localization_noise_std=[_f32(v) for v in loc],
        groundtruth_rotation_uniform_noise=[_f32(v) for v in rot], global_rotation_uniform_noise=[_f32(v) for v in grot],
        global_scaling_uniform_noise=[_f32(v) for v in scale], global_random_rotation_range_per_object=[0.0, 0.0],
        global_translate_noise_std=[_f32(v) for v in translate], random_flip_x=flip_x, random_flip_y=True)


_KITTI_AUG = ([1.0, 1.0, 0.5], [-0.78539816, 0.78539816], [-0.78539816, 0.78539816], [0.95, 1.05], [0, 0, 0])
_NUSC_AUG = ([0, 0, 0], [0, 0], [0, 0], [1.0, 1.0], [0, 0, 0])
# augmentation settings of the builtins (the train_input_reader.preprocess blocks of the cited config files)
AUGMENTS = {
    "car.fhd": lambda: _aug(*_KITTI_AUG, flip_x=False, shuffle=True),
    "car.lite": lambda: _aug(*_KITTI_AUG, flip_x=False, shuffle=True),
    "all.fhd": lambda: _aug(*_KITTI_AUG, flip_x=False, shuffle=True),
    "pointpillars.car.xyres_16": lambda: _aug([0.25, 0.25, 0.25], [-0.15707963267, 0.15707963267],
                                              [-0.78539816, 0.78539816], [0.95, 1.05], [0.2, 0.2, 0.2], flip_x=False,
                                              shuffle=True),
    "nuscenes.all.pp.largea": lambda: _aug(*_NUSC_AUG, flip_x=True, shuffle=False),
    "nuscenes.all.pp.mhead": lambda: _aug(*_NUSC_AUG, flip_x=True, shuffle=False),
}


_KITTI_DB = "/media/yy/960evo/datasets/kitti/kitti_dbinfos_train.pkl"
_KITTI_DB_PASSPORT = "/media/yy/My Passport/datasets/kitti/kitti_dbinfos_train.pkl"
_NUSC_DB = "/media/yy/960evo/datasets/nuscene/v1.0-trainval/kitti_dbinfos_train.pkl"


def _dbs(groups, min_points, path, remove, importance=1.0, difficulties=(-1,)):
    """groups: [(name, max_num)]; min_points: [(name, min_num)] or None (no prep steps at all)"""
    steps = [] if min_points is None else [("filter_by_min_num_points", list(min_points)),
                                           ("filter_by_difficulty", list(difficulties))]
    return DatabaseSamplerSettings(
        sample_groups=[{n: m} for n, m in groups], database_prep_steps=steps, rate=1.0,
        global_random_rotation_range_per_object=[0.0, 0.0], database_info_path=path,
        remove_points_after_sample=remove, sample_importance=_f32(importance))


_NUSC_GROUPS = [("bus", 4), ("trailer", 4), ("truck", 4)]
# database-sampler settings of the builtins (the train_input_reader.preprocess.database_sampler blocks of the cited
# config files)
DB_SAMPLERS = {
    "car.fhd": lambda: _dbs([("Car", 15)], [("Car", 5)], _KITTI_DB, True),
    "car.lite": lambda: _dbs([("Car", 15)], [("Car", 5)], _KITTI_DB_PASSPORT, False),
    "all.fhd": lambda: _dbs([("Car", 11), ("Pedestrian", 6), ("Cyclist", 6), ("Van", 4)],
                            [("Car", 5), ("Pedestrian", 10), ("Cyclist", 10), ("Van", 8)], _KITTI_DB, True),
    "pointpillars.car.xyres_16": lambda: _dbs([("Car", 15)], [("Car", 5)], _KITTI_DB_PASSPORT, False),
    "nuscenes.all.pp.largea": lambda: _dbs(_NUSC_GROUPS, None, _NUSC_DB, True),
    "nuscenes.all.pp.mhead": lambda: _dbs(_NUSC_GROUPS, None, _NUSC_DB, True, importance=0.5),
}


def _loss():
    """the loss every builtin config sets (the loss blocks and fields of the cited config files agree)"""
    return LossSettings(
        classification_loss="weighted_sigmoid_focal", alpha=0.25, gamma=2.0, localization_loss="weighted_smooth_l1",
        sigma=3.0, code_weight=[1.0] * 7, classification_weight=1.0, localization_weight=2.0,
        loss_norm_type="NormByNumPositives", pos_class_weight=1.0, neg_class_weight=1.0, encode_rad_error_by_sin=True,
        sin_error_factor=1.0, direction_loss_weight=_f32(0.2))


LOSSES = {name: _loss for name in list(TARGET_ASSIGNERS)}


def get_config(name):
    if name in BUILTIN:
        cfg = BUILTIN[name]()
    elif name in EXTRA:
        cfg = EXTRA[name]()
    else:
        raise KeyError("unknown config %r (have %s)" % (name, sorted(BUILTIN) + sorted(EXTRA)))
    cfg.target_assigner = TARGET_ASSIGNERS[name]()
    cfg.augment = AUGMENTS[name]()
    cfg.db_sampler = DB_SAMPLERS[name]()
    cfg.loss = LOSSES[name]()
    return cfg
