"""Integer BEV boxes of the anchors for the anchor-area mask (second/data/preprocess.py:345-357).

The reference derives each anchor's box in two steps:

  rbbox2d_to_near_bbox     box_np_ops.py:286-298  (axis-aligned box of the anchor, dims swapped past 45 degrees)
  fused_get_anchors_area   box_np_ops.py:925-946  floor((bv - pc_range[0|1]) / voxel_size[0|1]), x0/y0 clamped below
                                                  at 0, x1/y1 clamped above at grid - 1

Both run in float32 (float32 anchors, the voxel generator's float32 voxel_size / point_cloud_range), and about half of
the bounds lie within 1e-3 of a cell edge: the same floors in float64 change ~30 % of the boxes.  So the statements
below keep the reference's dtypes and operation order.  The boxes do not depend on the data: the engine derives them
once per anchor set and the device kernel (csrc/anchor_mask.cu) only does integer loads.
"""
import numpy as np


def near_bboxes(anchors):
    """anchors [A, >=7] (x, y, z, w, l, h, yaw, ...) -> float32 [A, 4] (xmin, ymin, xmax, ymax):
    rbbox2d_to_near_bbox(anchors[:, [0, 1, 3, 4, 6]]) with limit_period and center_to_minmax_2d inlined."""
    a = np.asarray(anchors, dtype=np.float32)
    a = a.reshape(-1, a.shape[-1])
    rbboxes = a[:, [0, 1, 3, 4, 6]]
    rots = rbboxes[..., -1]
    rots_0_pi_div_2 = np.abs(rots - np.floor(rots / np.pi + 0.5) * np.pi)
    cond = (rots_0_pi_div_2 > np.pi / 4)[..., np.newaxis]
    c = np.where(cond, rbboxes[:, [0, 1, 3, 2]], rbboxes[:, :4])
    centers, dims = c[:, :2], c[:, 2:]
    return np.concatenate([centers - dims / 2, centers + dims / 2], axis=-1)


def anchor_boxes(anchors, voxel_size, point_cloud_range, grid_size):
    """-> int32 [A, 4] (x0, y0, x1, y1) cell indices of fused_get_anchors_area; asserts every clamped box lies inside
    the grid and is not inverted (the reference's numba loop would read outside its map without a word)."""
    bv = near_bboxes(anchors)
    stride = np.asarray(voxel_size, dtype=np.float32)
    offset = np.asarray(point_cloud_range, dtype=np.float32)
    gx, gy = int(grid_size[0]) - 1, int(grid_size[1]) - 1
    x0 = np.floor((bv[:, 0] - offset[0]) / stride[0])
    y0 = np.floor((bv[:, 1] - offset[1]) / stride[1])
    x1 = np.floor((bv[:, 2] - offset[0]) / stride[0])
    y1 = np.floor((bv[:, 3] - offset[1]) / stride[1])
    assert x0.dtype == np.float32 and x1.dtype == np.float32, "the floors must be taken in float32"
    out = np.stack([np.maximum(x0, 0), np.maximum(y0, 0), np.minimum(x1, gx), np.minimum(y1, gy)], axis=1)
    out = out.astype(np.int32)
    bad = ~((0 <= out[:, 0]) & (out[:, 0] <= out[:, 2]) & (out[:, 2] <= gx) &
            (0 <= out[:, 1]) & (out[:, 1] <= out[:, 3]) & (out[:, 3] <= gy))
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError("anchor %d: BEV box %s lies outside the %dx%d voxel grid or is inverted (%d such anchors)"
                         % (i, out[i].tolist(), gx + 1, gy + 1, int(bad.sum())))
    return np.ascontiguousarray(out)


def enabled(threshold):
    """None or a negative threshold: no mask (the reference's `anchor_area_threshold >= 0` test)."""
    return threshold is not None and float(threshold) >= 0
