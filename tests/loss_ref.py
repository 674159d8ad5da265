"""A dtype-generic torch restatement of VoxelNet.loss (second/pytorch/models/voxelnet.py:239-312) for the settings
b2second.loss covers, and the seeded synthetic loss inputs the fixtures of tests/golden/make_loss_golden.py use.

``loss(s, example, preds)`` follows the reference's own op sequence (prepare_loss_weights, one-hot, add_sin_difference,
the smooth-L1 and focal functors, _get_pos_neg_loss, get_direction_target and the softmax cross-entropy), so in float64
it is an oracle that needs no reference tree, and autograd gives its backward.  In float32 it is the torch chain the
CUDA loss replaces (what tools/loss_times.py times, and the stand-in loss of the end-to-end test).

``make_case(case, B, A, C, nb, dir_offset, seed)`` builds one batch of loss inputs on the CPU (float32, int64 labels):
  a  a realistic mix: mostly background, some ignored, a few positives; importance in [0.5, 2]
  b  no positives (both normalizers clamp to 1)
  c  every anchor ignored
  d  logits up to |x| = 80
  e  ``rot - dir_offset`` on 0, 2 pi k / nb and 2 pi and one and two float32 steps beside them; anchors whose float32
     and float64 bins differ are made background, so both arithmetics weigh the same direction targets
"""
import os

import numpy as np
import torch

CASES = "abcde"
CONFIGS = ["car.fhd", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea", "nuscenes.all.pp.mhead"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss")
# the bounds of the loss checks (tests/test_gpu_loss.py docstring): scalars within 1e-5 relative, every element of
# the per-anchor outputs and gradients within C_REL eps32 |v64| + C_MAX eps32 max|v64|
EPS32 = float(np.finfo(np.float32).eps)
C_REL, C_MAX = 8.0, 1.0
SCALARS = ["loss", "cls_loss_reduced", "loc_loss_reduced", "dir_loss_reduced", "cls_pos_loss", "cls_neg_loss"]


def anchors_per_frame(num_class):
    """a few thousand (anchor, class) logits per frame, and fixtures under 1 MB"""
    return 2048 if num_class == 1 else 512


def limit_period(val, offset=0.5, period=np.pi):
    return val - torch.floor(val / period + offset) * period


def direction_target(anchors, reg_targets, dir_offset, num_bins):
    """get_direction_target (voxelnet.py:814-828) without the one-hot: int64 bins"""
    rot = reg_targets[..., 6] + anchors[..., 6]
    off = limit_period(rot - dir_offset, 0, 2 * np.pi)
    return torch.clamp(torch.floor(off / (2 * np.pi / num_bins)).long(), min=0, max=num_bins - 1)


def loss(s, example, preds):
    """VoxelNet.loss for LossSettings ``s`` (b2second.loss); preds' dtype sets the arithmetic.  -> the reference's dict"""
    box_preds, cls_preds = preds["box_preds"], preds["cls_preds"]
    B = cls_preds.shape[0]
    dt = box_preds.dtype
    labels = example["labels"]
    importance = example["importance"].to(dt)
    reg_targets = example["reg_targets"].to(dt)
    # prepare_loss_weights, NormByNumPositives
    cared = labels >= 0
    positives = labels > 0
    negatives = labels == 0
    cls_weights = negatives.type(dt) * s.neg_cls_weight + s.pos_cls_weight * positives.type(dt)
    reg_weights = positives.type(dt)
    pos_normalizer = positives.sum(1, keepdim=True).type(dt)
    reg_weights = reg_weights / torch.clamp(pos_normalizer, min=1.0)
    cls_weights = cls_weights / torch.clamp(pos_normalizer, min=1.0)
    cls_targets = labels * cared.type_as(labels)
    # create_loss
    box_preds = box_preds.view(B, -1, 7)
    cls_preds = cls_preds.view(B, -1, s.num_class)
    one_hot = torch.zeros(*cls_targets.shape, s.num_class + 1, dtype=dt, device=labels.device)
    one_hot.scatter_(-1, cls_targets.unsqueeze(-1).long(), 1.0)
    one_hot = one_hot[..., 1:]
    f = s.sin_factor
    p_rot, t_rot = box_preds[..., 6:7], reg_targets[..., 6:7]
    if f != 1.0:
        p_rot, t_rot = f * p_rot, f * t_rot
    bp = torch.cat([box_preds[..., :6], torch.sin(p_rot) * torch.cos(t_rot), box_preds[..., 7:]], dim=-1)
    bt = torch.cat([reg_targets[..., :6], torch.cos(p_rot) * torch.sin(t_rot), reg_targets[..., 7:]], dim=-1)
    # WeightedSmoothL1LocalizationLoss
    diff = bp - bt
    diff = torch.tensor(s.code_weight, dtype=dt, device=diff.device).view(1, 1, -1) * diff
    abs_diff = torch.abs(diff)
    lt = torch.le(abs_diff, 1 / (s.sigma ** 2)).type_as(abs_diff)
    loc_loss = lt * 0.5 * torch.pow(abs_diff * s.sigma, 2) + (abs_diff - 0.5 / (s.sigma ** 2)) * (1. - lt)
    loc_loss = loc_loss * (reg_weights * importance).unsqueeze(-1)
    # SigmoidFocalClassificationLoss
    x, z = cls_preds, one_hot
    ce = torch.clamp(x, min=0) - x * z
    ce = ce + torch.log1p(torch.exp(-torch.abs(x)))
    p = torch.sigmoid(x)
    p_t = z * p + (1 - z) * (1 - p)
    m = torch.pow(1.0 - p_t, s.gamma) if s.gamma else 1.0
    a = z * s.alpha + (1 - z) * (1 - s.alpha)
    cls_loss = m * a * ce * (cls_weights * importance).unsqueeze(2)
    # reductions
    loc_loss_reduced = loc_loss.sum() / B * s.loc_weight
    if s.num_class == 1:
        cls_pos_loss = ((labels > 0).type_as(cls_loss) * cls_loss.view(B, -1)).sum() / B
        cls_neg_loss = ((labels == 0).type_as(cls_loss) * cls_loss.view(B, -1)).sum() / B
    else:
        cls_pos_loss = cls_loss[..., 1:].sum() / B
        cls_neg_loss = cls_loss[..., 0].sum() / B
    cls_pos_loss = cls_pos_loss / s.pos_cls_weight
    cls_neg_loss = cls_neg_loss / s.neg_cls_weight
    cls_loss_reduced = cls_loss.sum() / B * s.cls_weight
    total = loc_loss_reduced + cls_loss_reduced
    # direction
    anchors = example["anchors"].to(dt).view(B, -1, example["anchors"].shape[-1])
    bins = direction_target(anchors, reg_targets, s.dir_offset, s.num_dir_bins)
    logits = preds["dir_cls_preds"].view(B, -1, s.num_dir_bins)
    w = positives.type(dt) * importance
    w = w / torch.clamp(w.sum(-1, keepdim=True), min=1.0)
    dir_ce = torch.nn.functional.cross_entropy(logits.reshape(-1, s.num_dir_bins), bins.reshape(-1), reduction="none")
    dir_loss = (dir_ce.view(w.shape) * w).sum() / B
    total = total + dir_loss * s.dir_weight
    return {"loss": total, "cls_loss": cls_loss, "loc_loss": loc_loss, "cls_pos_loss": cls_pos_loss,
            "cls_neg_loss": cls_neg_loss, "cls_preds": preds["cls_preds"], "cls_loss_reduced": cls_loss_reduced,
            "loc_loss_reduced": loc_loss_reduced, "cared": cared, "dir_loss_reduced": dir_loss, "dir_bins": bins}


# ------------------------------------------------------------------------------------------------ synthetic inputs
def _boundary_rots(nb, dir_offset):
    """float32 values of rot (= reg_targets[..., 6] + anchors[..., 6] with a zero anchor yaw) that put
    rot - dir_offset on 0, 2 pi k / nb, 2 pi and -2 pi, and one and two float32 steps to either side"""
    off = np.float32(dir_offset)
    out = []
    for k in range(-nb, nb + 1):
        v = np.float32(np.float32(2 * np.pi * k / nb) + off)
        for step in (-2, -1, 0, 1, 2):
            u = v
            for _ in range(abs(step)):
                u = np.nextafter(u, np.float32(np.inf if step > 0 else -np.inf), dtype=np.float32)
            out.append(u)
    return np.array(out, np.float32)


def make_case(case, B, A, C, nb, dir_offset, seed):
    """-> (example, preds): float32 CPU tensors, int64 labels (the reference collate's dtype)"""
    rng = np.random.default_rng(seed)
    labels = np.zeros((B, A), np.int64)
    imp = rng.uniform(0.5, 2.0, (B, A)).astype(np.float32)
    anchors = np.zeros((B, A, 7), np.float32)
    anchors[..., 3:6] = rng.uniform(0.5, 4.0, (B, A, 3))
    anchors[..., 6] = np.where(rng.random((B, A)) < 0.5, np.float32(0), np.float32(np.pi / 2))
    box = (rng.standard_normal((B, A, 7)) * 0.4).astype(np.float32)
    cls = (rng.standard_normal((B, A, C)) * 2.0 - 2.0).astype(np.float32)
    dirp = rng.standard_normal((B, A, nb)).astype(np.float32)
    u = rng.random((B, A))
    if case in "ad":
        labels[u < 0.1] = -1
        pos = u > 0.95
        labels[pos] = rng.integers(1, C + 1, int(pos.sum()))
    elif case == "b":
        labels[u < 0.2] = -1
    elif case == "c":
        labels[:] = -1
    elif case == "e":
        labels[u < 0.1] = -1
        rots = _boundary_rots(nb, dir_offset)
        n = len(rots)
        for b in range(B):
            labels[b, :n] = rng.integers(1, C + 1, n)
            anchors[b, :n, 6] = 0
        dirp[:, :rots.shape[0]] = 0                           # softmax 1/nb: the gradient's sign gives the bin
    reg = np.zeros((B, A, 7), np.float32)
    posm = labels > 0
    reg[posm] = (rng.standard_normal((int(posm.sum()), 7)) * 0.3).astype(np.float32)
    reg[..., 6][posm] = rng.uniform(-np.pi, np.pi, int(posm.sum())).astype(np.float32)
    if case == "d":
        cls = rng.uniform(-80, 80, (B, A, C)).astype(np.float32)
        cls[:, :8] = np.array([-80, -60, -20, -1e-3, 0, 1e-3, 20, 80], np.float32)[:, None]
        dirp = rng.uniform(-80, 80, (B, A, nb)).astype(np.float32)
        box[posm] += rng.uniform(-3, 3, (int(posm.sum()), 7)).astype(np.float32)
    if case == "e":
        n = len(rots)
        reg[:, :n, 6] = rots
        # keep the anchors whose float32 and float64 bins agree positive
        t = torch.from_numpy(reg)
        a = torch.from_numpy(anchors)
        b32 = direction_target(a, t, dir_offset, nb)
        b64 = direction_target(a.double(), t.double(), dir_offset, nb)
        labels[(b32 != b64).numpy() & posm] = 0
        reg[labels <= 0] = 0
    example = {"labels": torch.from_numpy(labels), "reg_targets": torch.from_numpy(reg),
               "importance": torch.from_numpy(imp), "anchors": torch.from_numpy(anchors)}
    preds = {"box_preds": torch.from_numpy(box), "cls_preds": torch.from_numpy(cls),
             "dir_cls_preds": torch.from_numpy(dirp)}
    return example, preds


def case_inputs(name, case, settings):
    """the inputs of fixture (name, case): B = 2 frames"""
    ci = CONFIGS.index(name) if name in CONFIGS else 0
    A = anchors_per_frame(settings.num_class)
    return make_case(case, 2, A, settings.num_class, settings.num_dir_bins, settings.dir_offset,
                     seed=9000 + 10 * ci + CASES.index(case))


def mirror_settings(name):
    from b2second import config, loss, models, loader
    cfg = config.get_config(name)
    net = models.build_network(cfg, loader.oracle_spconv())
    return loss.plan(net).settings


def load_fixture(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def reference_run(s, example, preds, dtype):
    """loss + autograd gradients of ``loss`` through this restatement in ``dtype`` -> (dict of numpy, grads)"""
    pr = {k: v.to(dtype).clone().requires_grad_() for k, v in preds.items()}
    ex = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in example.items()}
    r = loss(s, ex, pr)
    r["loss"].backward()
    out = {k: r[k].detach().numpy() for k in SCALARS + ["cls_loss", "loc_loss", "cared", "dir_bins"]}
    grads = {k: pr[k].grad.numpy() for k in pr}
    return out, grads


def check_scalars(got, want64, what):
    """the six scalars (SCALARS order) within 1e-5 relative of float64, within 1e-7 absolute where that is 0"""
    got = np.asarray(got, np.float64)
    for k, g, w in zip(SCALARS, got, want64):
        if w == 0:
            assert abs(g) <= 1e-7, (what, k, g)
        else:
            assert abs(g - w) <= 1e-5 * abs(w), (what, k, g, w)
