"""Anchor grid for the SECOND head (constant per model; generated once, cached on device).

Mirrors, without importing the reference:
* range generator  second/core/box_np_ops.py:602-638 (``linspace`` centres incl. both range ends)
* stride generator second/core/box_np_ops.py:561-599 (``arange*stride+offset``)
* per-class layout and concatenation second/core/target_assigner.py:169-207:
  each class contributes ``[(size,rot), z, y, x, 7]`` flattened, classes concatenated.
Box element order ``[x, y, z, w, l, h, r]`` (+ custom values).
"""
import numpy as np


def _class_anchors(feature_size, cls, dtype=np.float32):
    """feature_size = [D, H, W] (zyx) -> [n_size*n_rot, D, H, W, 7+custom]."""
    D, H, W = (int(v) for v in feature_size)
    sizes = np.reshape(np.array(cls.sizes, dtype=dtype), [-1, 3])
    rots = np.array(cls.rotations, dtype=dtype)
    if cls.anchor_ranges is not None:
        ar = np.array(cls.anchor_ranges, dtype)
        zc = np.linspace(ar[2], ar[5], D, dtype=dtype)
        yc = np.linspace(ar[1], ar[4], H, dtype=dtype)
        xc = np.linspace(ar[0], ar[3], W, dtype=dtype)
    else:
        xs, ys, zs = cls.strides
        xo, yo, zo = cls.offsets
        zc = np.arange(D, dtype=dtype) * zs + zo
        yc = np.arange(H, dtype=dtype) * ys + yo
        xc = np.arange(W, dtype=dtype) * xs + xo
    ns, nr = sizes.shape[0], rots.shape[0]
    ncode = 7 + len(cls.custom_values)
    out = np.zeros([ns, nr, D, H, W, ncode], dtype=dtype)
    out[..., 0] = xc[None, None, None, None, :]
    out[..., 1] = yc[None, None, None, :, None]
    out[..., 2] = zc[None, None, :, None, None]
    out[..., 3:6] = sizes[:, None, None, None, None, :]
    out[..., 6] = rots[None, :, None, None, None]
    for i, v in enumerate(cls.custom_values):
        out[..., 7 + i] = v
    return out.reshape(ns * nr, D, H, W, ncode)


def generate_anchors(cfg):
    """-> float32 [A, 7+custom] for ``cfg.feature_map_size`` in the reference's order.  A class with its own
    ``feature_map_size`` (``cfg.class_feature_map_sizes``, the multi-head network) is laid out on that map."""
    fsize = cfg.feature_map_size
    per_class = getattr(cfg, "class_feature_map_sizes", None) or [None] * len(cfg.classes)
    parts = []
    for cls, fs in zip(cfg.classes, per_class):
        if cls.num_anchors_per_loc == 0:
            continue
        a = _class_anchors(fs if fs else fsize, cls)
        parts.append(a.reshape(-1, a.shape[-1]))
    return np.concatenate(parts, axis=0)
