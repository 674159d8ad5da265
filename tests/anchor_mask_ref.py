"""TEST INFRASTRUCTURE (oracle): numpy restatement of the reference's anchor-area mask (second/data/preprocess.py:345-357)
with the map in float32, as the reference holds it:

  sparse_sum_for_anchors_mask   box_np_ops.py:917-922   one +1 per voxel at (coors[i, 1], coors[i, 2]) = (y, x)
  cumsum(0).cumsum(1)           preprocess.py:351-352
  fused_get_anchors_area        box_np_ops.py:925-946   ID - IB - IC + IA over the integer boxes
  area > threshold              preprocess.py:355

The integer boxes come from b2second.anchor_mask.anchor_boxes (checked against the reference's own arithmetic in
tests/test_anchor_mask.py).  Coordinates here carry the batch column: (b, z, y, x).
"""
import numpy as np


def summed_area(coors, batch_size, ny, nx):
    """-> float32 [B, ny, nx] summed-area tables of the per-frame voxel counts."""
    m = np.zeros((batch_size, ny, nx), np.float32)
    c = np.asarray(coors).reshape(-1, 4)
    np.add.at(m, (c[:, 0], c[:, 2], c[:, 3]), np.float32(1))
    return m.cumsum(1).cumsum(2)


def anchor_area_mask_np(coors, batch_size, boxes, grid_size, threshold):
    """-> bool [B, A]"""
    S = summed_area(coors, batch_size, int(grid_size[1]), int(grid_size[0]))
    x0, y0, x1, y1 = (np.asarray(boxes)[:, k] for k in range(4))
    ID = S[:, y1, x1]
    IA = S[:, y0, x0]
    IB = S[:, y1, x0]
    IC = S[:, y0, x1]
    area = ID - IB - IC + IA
    return area > np.float32(threshold)
