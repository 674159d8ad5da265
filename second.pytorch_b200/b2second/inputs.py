"""On-GPU input path in front of the voxelizer (SURVEY.md §8(f)1): raw sweeps / raw KITTI clouds -> the engine's point
buffer, without the DataLoader-worker numpy code and without a host round trip.

  merge_sweeps      second/data/nuscenes_dataset.py:166-185  (key frame + N sweeps -> [x, y, z, dt] rows)
  frustum_planes    second/core/box_np_ops.py:682-690 (``remove_outside_points``: camera frustum of the image in lidar
                    coordinates) + second/core/geometry.py:332-355 (plane equations) -- host side, 6 planes
  crop_convex       box_np_ops.py:691-692 -> geometry.py:149-172,358-395 (points strictly inside all planes, in order)

The calibration algebra (a handful of 3x3 / 4x4 float64 operations per frame) stays on the host, where the reference
does it; everything that touches the points runs in csrc/inputs.cu.
"""
import ctypes

import numpy as np
import torch


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


# ------------------------------------------------------------------------------------------------ host: calibration
def projection_matrix_to_CRT_kitti(proj):
    """P = C @ [R|T] with C upper triangular (box_np_ops.py:507-518)."""
    CR = proj[0:3, 0:3]
    CT = proj[0:3, 3]
    RinvCinv = np.linalg.inv(CR)
    Rinv, Cinv = np.linalg.qr(RinvCinv)
    C = np.linalg.inv(Cinv)
    R = np.linalg.inv(Rinv)
    T = Cinv @ CT
    return C, R, T


def get_frustum(bbox_image, C, near_clip=0.001, far_clip=100):
    """8 corners of the camera frustum behind an image box (box_np_ops.py:521-538)."""
    fku, fkv = C[0, 0], -C[1, 1]
    u0v0 = C[0:2, 2]
    z_points = np.array([near_clip] * 4 + [far_clip] * 4, dtype=C.dtype)[:, np.newaxis]
    b = bbox_image
    box_corners = np.array([[b[0], b[1]], [b[0], b[3]], [b[2], b[3]], [b[2], b[1]]], dtype=C.dtype)
    near = (box_corners - u0v0) / np.array([fku / near_clip, -fkv / near_clip], dtype=C.dtype)
    far = (box_corners - u0v0) / np.array([fku / far_clip, -fkv / far_clip], dtype=C.dtype)
    return np.concatenate([np.concatenate([near, far], axis=0), z_points], axis=1)


_SURFACE_CORNERS = np.array([0, 1, 2, 3, 7, 6, 5, 4, 0, 3, 7, 4, 1, 5, 6, 2, 0, 4, 5, 1, 3, 2, 6, 7]).reshape(6, 4)


def planes_of_box_corners(corners):
    """corners [8,3] (corner order of the reference's corner functions) -> planes [6,4] (a,b,c,d) with inward normals:
    corner_to_surfaces_3d_jit (box_np_ops.py:764-783) + surface_equ_3d_jitv2 (geometry.py:332-355)."""
    s = corners[_SURFACE_CORNERS]                       # [6, 4, 3]
    sv0 = s[:, 0] - s[:, 1]
    sv1 = s[:, 1] - s[:, 2]
    n = np.stack([sv0[:, 1] * sv1[:, 2] - sv0[:, 2] * sv1[:, 1], sv0[:, 2] * sv1[:, 0] - sv0[:, 0] * sv1[:, 2],
                  sv0[:, 0] * sv1[:, 1] - sv0[:, 1] * sv1[:, 0]], axis=1)
    d = -s[:, 0, 0] * n[:, 0] - s[:, 0, 1] * n[:, 1] - s[:, 0, 2] * n[:, 2]
    return np.ascontiguousarray(np.concatenate([n, d[:, None]], axis=1), dtype=np.float64)


def frustum_planes(rect, Trv2c, P2, image_shape):
    """the 6 planes ``remove_outside_points(points, rect, Trv2c, P2, image_shape)`` tests against (box_np_ops.py:682-690)."""
    C, R, T = projection_matrix_to_CRT_kitti(P2)
    image_bbox = [0, 0, image_shape[1], image_shape[0]]
    frustum = get_frustum(image_bbox, C)
    frustum = frustum - T
    frustum = np.linalg.inv(R) @ frustum.T
    pts = frustum.T
    pts = np.concatenate([pts, np.ones([pts.shape[0], 1])], axis=-1)
    lidar = (pts @ np.linalg.inv((rect @ Trv2c).T))[..., :3]          # camera_to_lidar (box_np_ops.py:650-655)
    return planes_of_box_corners(lidar)


# ------------------------------------------------------------------------------------------------ device
def merge_sweeps(sweeps, rotations, translations, time_lags, out=None):
    """sweeps: list of CUDA float32 [P_i, F>=3] tensors, key frame first (its rotation/translation are ignored, its
    time lag is 0); rotations [3,3] / translations [3] float64 (``sweep2lidar_*``); time_lags = ts - sweep_ts.
    -> CUDA float32 [sum P_i, 4] = [x, y, z, dt] in sweep order (nuscenes_dataset.py:166-185)."""
    L, lib = _lib()
    total = sum(int(s.shape[0]) for s in sweeps)
    dev = sweeps[0].device
    if out is None:
        out = torch.empty(total, 4, dtype=torch.float32, device=dev)
    assert out.shape[0] >= total and out.shape[1] == 4 and out.is_contiguous()
    off = 0
    for i, s in enumerate(sweeps):
        L.require_cuda(s, "sweep")
        s = s.contiguous().float()
        n = int(s.shape[0])
        if i == 0:
            rot, tr, lag = None, None, 0.0
        else:
            rot = np.ascontiguousarray(rotations[i], dtype=np.float64).ctypes.data_as(ctypes.c_void_p)
            tr = np.ascontiguousarray(translations[i], dtype=np.float64).ctypes.data_as(ctypes.c_void_p)
            lag = float(np.float32(time_lags[i]))
        L.check(lib.b2s_transform_sweep(L.ptr(s), n, int(s.shape[1]), rot, tr, lag,
                                        ctypes.c_void_p(out.data_ptr() + 16 * off), L.stream()), "b2s_transform_sweep")
        off += n
    return out[:total]


class ConvexCrop:
    """order-preserving crop of frames into a shared point buffer (see b2s_crop_convex)."""

    def __init__(self, max_points, device):
        L, lib = _lib()
        self.ws_bytes = lib.b2s_crop_workspace_bytes(int(max_points))
        self.ws = torch.empty(max(self.ws_bytes, 1), dtype=torch.uint8, device=device)
        self.max_points = int(max_points)

    def crop_into(self, points, planes, out_points, offsets_dev, slot, status=None):
        """keep the rows of CUDA ``points`` [P,F] inside ``planes`` [n,4] (float64, host); append them to ``out_points``
        at row offsets_dev[slot] and set offsets_dev[slot+1].  No host sync."""
        L, lib = _lib()
        L.require_cuda(points, "points")
        p = points.contiguous().float()
        assert p.shape[0] <= self.max_points and p.shape[1] == out_points.shape[1]
        pl = np.ascontiguousarray(planes, dtype=np.float64)
        L.check(lib.b2s_crop_convex(L.ptr(p), int(p.shape[0]), int(p.shape[1]), pl.ctypes.data_as(ctypes.c_void_p),
                                    int(pl.shape[0]), L.ptr(out_points), int(out_points.shape[0]),
                                    ctypes.c_void_p(offsets_dev.data_ptr() + 4 * slot), L.ptr(self.ws), self.ws_bytes,
                                    L.ptr(status), L.stream()), "b2s_crop_convex")
        return p          # keep the (possibly converted) input alive until the stream has consumed it


def crop_convex(points, planes):
    """stand-alone form: CUDA [P,F] -> (CUDA [P,F] buffer, device int32 [2] offsets); rows [0, offsets[1]) are kept."""
    out = torch.empty_like(points, dtype=torch.float32)
    offs = torch.zeros(2, dtype=torch.int32, device=points.device)
    ConvexCrop(points.shape[0], points.device).crop_into(points, planes, out, offs, 0)
    return out, offs


def anchor_area_mask(coordinates, batch_size, anchors, voxel_size, point_cloud_range, grid_size, threshold):
    """the reference preprocessing's ``anchors_mask`` (second/data/preprocess.py:345-357) on the GPU, for callers who
    build examples themselves: coordinates CUDA int [N, 4] (b, z, y, x) of the voxels that survived max_voxels;
    anchors [A, >=7] (host or device; read on the host once to derive the integer boxes, b2second.anchor_mask);
    grid_size (x, y, z).  -> CUDA bool [batch_size, A]: the anchor's BEV box holds more than ``threshold`` voxels."""
    from . import anchor_mask
    L, lib = _lib()
    L.require_cuda(coordinates, "coordinates")
    dev = coordinates.device
    a = anchors.detach().cpu().numpy() if isinstance(anchors, torch.Tensor) else np.asarray(anchors)
    boxes = torch.from_numpy(anchor_mask.anchor_boxes(a.reshape(-1, a.shape[-1]), voxel_size, point_cloud_range,
                                                      grid_size)).to(dev)
    B, A = int(batch_size), int(boxes.shape[0])
    ny, nx = int(grid_size[1]), int(grid_size[0])
    coors = coordinates.to(torch.int32).contiguous()
    n = int(coors.shape[0])
    n_dev = torch.tensor([n], dtype=torch.int32).to(dev)
    ws_bytes = lib.b2s_anchor_area_mask_workspace_bytes(B, ny, nx)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    mask = torch.empty(B, A, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.b2s_anchor_area_mask(L.ptr(coors) if n else None, L.ptr(n_dev), n, B, ny, nx, L.ptr(boxes), A,
                                         float(threshold), L.ptr(ws), ws_bytes, L.ptr(mask), L.stream()),
                "b2s_anchor_area_mask")
    return mask.bool()
