"""``spconv.ops`` on libb2second.so: rulebooks and the nms op.

upstream: ``torch.ops.spconv.get_indice_pairs`` / ``indice_conv`` / ``nms`` -- call sites
second/pytorch/models/middle.py:146-189 (through SubMConv3d / SparseConv3d) and
second/pytorch/core/box_torch_ops.py:488 (``spconv.ops.nms``, used by ``nms_v2`` only).
"""
import numpy as np
import torch

from . import _lib


def get_conv_output_size(input_size, kernel_size, stride, padding, dilation):
    out = []
    for i in range(len(input_size)):
        size = (input_size[i] + 2 * padding[i] - dilation[i] * (kernel_size[i] - 1) - 1) // stride[i] + 1
        out.append(int(size))
    return out


def _pow2_at_least(n):
    c = 1024
    while c < n:
        c <<= 1
    return c


class Rulebook:
    """output-stationary rulebook: ``nbr[o,k]`` = input row feeding output row ``o`` via offset ``k`` (-1: none)."""
    __slots__ = ("out_indices", "nbr", "num_out", "num_out_dev", "out_hash", "K", "out_shape", "subm", "row_mask", "ksize", "plan",
                 "nbrT", "nbrT_rows_dev")

    # tuple-style access keeps code written against upstream's (outids, indices, pairs, pair_num, shape) working
    def __iter__(self):
        pairs, pair_num = pairs_from_nbr(self)
        return iter((self.out_indices, None, pairs, pair_num, self.out_shape))


def build_rulebook(x, ksize, stride, padding, dilation, subm):
    """x: SparseConvTensor (CUDA).  Synchronises once for a strided conv (to size the output exactly,
    as upstream does per layer); the fused engine path (b2second.engine) never does."""
    lib = _lib.load()
    _lib.require_cuda(x.indices, "indices")
    idx = x.indices.contiguous()
    dev = idx.device
    n_in = idx.shape[0]
    K = int(np.prod(ksize))
    n_in_dev = torch.tensor([n_in], dtype=torch.int32, device=dev)
    rb = Rulebook()
    rb.K = K
    rb.subm = bool(subm)
    rb.ksize = [int(k) for k in ksize]
    rb.plan = None
    rb.nbrT = None
    rb.nbrT_rows_dev = None
    if subm:
        keys, vals, cap = x._locator()
        nbr = torch.empty(max(n_in, 1), K, dtype=torch.int32, device=dev)
        rb.row_mask = torch.empty(max(n_in, 1), dtype=torch.int32, device=dev)      # bit k: nbr[row][k] exists
        _lib.check(lib.b2s_rulebook_subm(_lib.ptr(idx), _lib.ptr(n_in_dev), n_in, _lib.i3(x.spatial_shape),
                                         _lib.i3(ksize), _lib.i3(dilation), _lib.ptr(keys), _lib.ptr(vals), cap,
                                         _lib.ptr(nbr), _lib.ptr(rb.row_mask), _lib.stream()), "b2s_rulebook_subm")
        rb.out_indices = idx
        rb.nbr = nbr[:n_in]
        rb.num_out = n_in
        rb.num_out_dev = n_in_dev
        rb.out_hash = (keys, vals, cap)
        rb.out_shape = list(x.spatial_shape)
        return rb
    out_shape = get_conv_output_size(x.spatial_shape, ksize, stride, padding, dilation)
    cells = int(np.prod(out_shape)) * x.batch_size
    fan = int(np.prod([-(-k // s) for k, s in zip(ksize, stride)]))   # outputs one input can touch
    cap_out = max(1, min(cells, n_in * fan))
    hash_cap_out = _pow2_at_least(2 * cap_out)
    coors_out = torch.empty(cap_out, 4, dtype=torch.int32, device=dev)
    nbr = torch.empty(cap_out, K, dtype=torch.int32, device=dev)
    row_mask = torch.empty(cap_out, dtype=torch.int32, device=dev)                  # bit k: nbr[row][k] exists
    num_out_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    keys_out = torch.empty(hash_cap_out, dtype=torch.int64, device=dev)
    vals_out = torch.empty(hash_cap_out, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    oshape = _lib.i3(out_shape)
    ws_bytes = lib.b2s_rulebook_conv_workspace_bytes(x.batch_size, oshape)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.b2s_rulebook_conv(
        _lib.ptr(idx), _lib.ptr(n_in_dev), n_in, x.batch_size, _lib.i3(x.spatial_shape), oshape, _lib.i3(ksize),
        _lib.i3(stride), _lib.i3(padding), _lib.i3(dilation), _lib.ptr(coors_out), _lib.ptr(num_out_dev), cap_out,
        _lib.ptr(nbr), _lib.ptr(keys_out), _lib.ptr(vals_out), hash_cap_out, _lib.ptr(ws), ws_bytes, _lib.ptr(row_mask), _lib.ptr(status), _lib.stream()), "b2s_rulebook_conv")
    n_out, st = int(num_out_dev.item()), int(status.item())   # the one sync of the module-by-module path
    if st:
        raise RuntimeError("b2s_rulebook_conv: " + _lib.status_message(st))
    rb.out_indices = coors_out[:n_out]
    rb.nbr = nbr[:n_out]
    rb.row_mask = row_mask
    rb.num_out = n_out
    rb.num_out_dev = num_out_dev
    rb.out_hash = (keys_out, vals_out, hash_cap_out)
    rb.out_shape = out_shape
    return rb


def tile_plan(rb):
    """tile plan of a rulebook for b2s_sparse_conv_tc_plan: (perm, tile_mask), built once per rulebook from the row masks
    the builder wrote, or (None, None) where b2second.tc.wants_tile_plan says the rulebook gets none."""
    from b2second import tc as _tc
    if rb.plan is None:
        if not _tc.wants_tile_plan(rb.subm, rb.K) or rb.num_out <= 0 or getattr(rb, "row_mask", None) is None:
            rb.plan = (None, None)
        else:
            lib = _lib.load()
            dev = rb.nbr.device
            perm = torch.empty(rb.num_out, dtype=torch.int32, device=dev)
            tmask = torch.empty((rb.num_out + 127) // 128, dtype=torch.int32, device=dev)
            _lib.check(lib.b2s_sparse_tile_plan(None, _lib.ptr(rb.row_mask), rb.K, _lib.i3(rb.ksize), _lib.ptr(rb.num_out_dev),
                                                rb.num_out, 1, _lib.ptr(perm), _lib.ptr(tmask), _lib.stream()),
                       "b2s_sparse_tile_plan")
            rb.plan = (perm, tmask)
    return rb.plan


def transpose_rulebook(rb, n_in):
    """input-side table of a rulebook, ``nbrT [n_in, K]``: ``nbrT[i, k] = o`` where ``nbr[o, k] = i`` (-1: none) --
    what the input gradient of a strided conv gathers through.  Built on first use and cached on the rulebook, with its
    row count n_in as a [1] device tensor (``rb.nbrT_rows_dev``), so a backward makes no host copy and can be captured."""
    if rb.nbrT is None or rb.nbrT.shape[0] != n_in:
        lib = _lib.load()
        nbrT = torch.empty(max(n_in, 1), rb.K, dtype=torch.int32, device=rb.nbr.device)
        _lib.check(lib.b2s_rulebook_transpose(_lib.ptr(rb.nbr.contiguous()), _lib.ptr(rb.num_out_dev), rb.num_out, rb.K,
                                              _lib.ptr(nbrT), n_in, None, _lib.stream()), "b2s_rulebook_transpose")
        rb.nbrT = nbrT[:n_in]
        rb.nbrT_rows_dev = torch.tensor([n_in], dtype=torch.int32, device=rb.nbr.device)
    return rb.nbrT


def pairs_from_nbr(rb, length=None):
    """spconv-format view of a rulebook: (indice_pairs [K,2,L] i32 (-1 filled), indice_pair_num [K])."""
    lib = _lib.load()
    dev = rb.nbr.device
    L = int(length if length is not None else max(rb.num_out, 1))
    pairs = torch.full((rb.K, 2, L), -1, dtype=torch.int32, device=dev)
    pair_num = torch.zeros(rb.K, dtype=torch.int32, device=dev)
    if rb.num_out > 0:
        _lib.check(lib.b2s_rulebook_pairs(_lib.ptr(rb.nbr.contiguous()), _lib.ptr(rb.num_out_dev), rb.num_out, rb.K,
                                          L, _lib.ptr(pairs), _lib.ptr(pair_num), _lib.stream()),
                   "b2s_rulebook_pairs")
    return pairs, pair_num


def get_indice_pairs(indices, batch_size, spatial_shape, ksize=3, stride=1, padding=0, dilation=1, out_padding=0,
                     subm=False, transpose=False, grid=None, use_hash=False):
    """upstream signature; returns (out_indices, indice_pairs [K,2,L], indice_pair_num [K])."""
    from . import SparseConvTensor
    assert not transpose, "transposed sparse conv is not on the SECOND inference path"

    def t3(v):
        return [int(x) for x in v] if isinstance(v, (list, tuple, np.ndarray)) else [int(v)] * 3

    ksize, stride, padding, dilation = t3(ksize), t3(stride), t3(padding), t3(dilation)
    x = SparseConvTensor(torch.empty(indices.shape[0], 1, device=indices.device), indices, spatial_shape, batch_size)
    rb = build_rulebook(x, ksize, stride, padding, dilation, subm)
    L = indices.shape[0] if not subm else rb.num_out
    # an output row can appear once per offset, an input row once per offset: L = max(n_in, n_out) is safe
    L = max(L, rb.num_out, 1)
    pairs, pair_num = pairs_from_nbr(rb, L)
    return rb.out_indices, pairs, pair_num


def nms(boxes, scores, pre_max_size, post_max_size, thresh, eps):
    """``spconv.ops.nms`` (box_torch_ops.py:479-489 ``nms_v2``): CPU tensors in, LongTensor out.
    eps-style IoU (``w = x2-x1+eps``), suppress when ``>= thresh``: same predicate as
    ``non_max_suppression_cpu``; runs the device bitmask kernel on the eps-padded boxes."""
    from .utils import non_max_suppression_cpu
    scores_np = scores.detach().cpu().numpy()
    boxes_np = boxes.detach().cpu().numpy().astype(np.float32)
    order = np.argsort(-scores_np, kind="stable").astype(np.int32)
    if pre_max_size > 0:
        order = order[:pre_max_size]
    dets = np.concatenate([boxes_np, scores_np[:, None].astype(np.float32)], axis=1)
    keep = non_max_suppression_cpu(dets, order, thresh, eps)
    if post_max_size > 0:
        keep = keep[:post_max_size]
    return torch.tensor(keep, dtype=torch.long)
