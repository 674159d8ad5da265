"""Fused device pipeline for ``VoxelNet`` inference: points in HBM -> detections in HBM, no host sync.

This is the fast path behind the ``VoxelNet.forward(example)`` contract (SURVEY.md §8b; reached through
``b2second.fastpath.accelerate(net)`` for a reference-built network and through ``models.VoxelNet.forward`` for
the mirror).  Where the module-by-module path mirrors the reference call by call -- one rulebook sync per
strided conv, a D2H -> CPU NMS -> H2D round trip per frame (second/pytorch/core/box_torch_ops.py:503,512) -- the
engine keeps every data-dependent count in device memory and runs a fixed launch sequence over capacity-sized
buffers, so the whole frame batch is ONE CUDA graph:

  b2s_voxelize (+ fused SimpleVoxel mean)                     voxelnet.py:325-328, preprocess.py:303-315
     or, for an example that arrives already voxelised (the reference's own dict):
     b2s_hash_build + b2s_vfe_mean over the caller's voxels   voxel_encoder.py:220-225,246-255
  b2s_anchor_area_mask (only with anchor_area_threshold >= 0 and no example mask)   preprocess.py:345-357
  per sparse layer: b2s_rulebook_{subm,conv} (cached per indice_key) + b2s_sparse_conv_tc (wgmma, fp16 hi/lo
      planes flow from layer to layer) with BatchNorm1d/ReLU folded into the epilogue      middle.py:145-192
  b2s_pfn_ex (PointPillars: plain decoration, PillarFeatureNetRadius: radius)   pointpillars.py:203-237,240-325
  b2s_to_bev_tc_ex (NHWC + halo, fp16 hi/lo)                   middle.py:206-209 / pointpillars.py:444-476
  RPN as a program of b2s_conv2d_tc_ex2 launches (tc.plan_rpn) rpn.py:314-331,393-420,467-497
      (rpn_impl="cudnn" keeps the torch modules as a cross-check: fp32, TF32 off)
  b2s_decode_filter_strided + b2s_nms (+ direction/range epilogue)   voxelnet.py:377-645

precision="f16" is the half-precision mode: every tensor-pipe operand (sparse rows, BEV and RPN planes, weights) is ONE
fp16 plane instead of a hi/lo pair, and each MMA is one f16 wgmma with fp32 accumulation (the ``*_ex`` entry points
with products = 1).  Everything off the tensor pipe (voxelizer, VFE / PFN, the scatter's index work, decode, the anchor
mask, NMS) is the fp32 code of the default mode, and the head outputs and detections stay float32.

VoxelNetNuscenesMultiHead (net_multi_head.py:121-176) runs the same way with two head "segments": the large head's
packed 1x1 convs on the concatenated map, and b2s_crop_nhwc of stage 0 -> three 3x3 convs -> the small head's packed
1x1 convs; b2s_decode_filter_segments reads both records into ONE candidate list per frame, with global anchor ids.

The network is read through ``b2second.spec.spec_from_module`` (attribute names of the reference), never through
``b2second.models`` classes or a ``ModelConfig``.

Output per batch: ``det [B, post_max, code+2]`` (box, score, label) + ``det_count [B]`` -- the fixed-stride
record the multi-GPU path all-gathers (SURVEY.md §8e); ``det`` and ``det_count`` live in ONE buffer
(``det_record [B, post_max*(code+2) + 1]``) so the all-gather needs no packing step.
"""
import contextlib
import ctypes
import gc

import numpy as np
import torch

from . import anchor_mask as _anchor_mask
from . import spec as _spec
from . import tc as _tc

# height of the RPN background strips (8 pixels wide; csrc/rpn_bg.cu, csrc/conv_tc2.cu): two 8x4 strips make one
# consumer warpgroup's 64-pixel tile.  k_conv3x3_tc2 is bound by the bytes it streams from L2 (weights 4.5 KB per
# computed pixel, activation windows 1.9 / 2.25 / 3 KB at 8 / 4 / 2 rows), not by its MMAs: 8x4 moves the fewest
# bytes per step, 8x2 computes 16 % fewer pixels than 8x8 but moves as many bytes and runs slower (DESIGN.md §7).
# For the same reason background strips inside the field's constant interior (_field_margin) are stored from a value
# the fill warps hold in registers instead of being copied from the field
BG_ROWS = 4

# one head map as the decode kernels read it: b2s_decode_filter_strided's leading arguments, in order, and the leading
# fields of b2s_head_segment
_HEAD_VIEW = ("box", "cls", "dir", "box_batch_stride", "cls_batch_stride", "dir_batch_stride", "ch_stride",
              "pix_stride")


def _field_margin(hi, lo):
    """the smallest m such that a layer's empty-frame response (halo-padded hi/lo planes [H+2, W+2, C]; lo None in the
    f16 mode) holds, bit for bit, its value at pixel (m, m) wherever it is at least m pixels from every border; -1 when
    no such interior exists.  The conv kernel stores that value into the background strips there instead of copying
    the field."""
    H, W = hi.shape[0] - 2, hi.shape[1] - 2
    planes = [hi] if lo is None else [hi, lo]
    return _bits_margin(torch.cat([t[1:H + 1, 1:W + 1] for t in planes], -1).view(torch.int16))


@contextlib.contextmanager
def no_cyclic_gc():
    """the block runs with Python's cyclic garbage collector off (restored after, also on an exception).  Used around a
    CUDA graph capture: torch does not collect before capturing, and a CUDAGraph the collector frees inside the capture
    (one of an engine dropped earlier and kept alive by a reference cycle) is destroyed mid-capture, which invalidates
    the capture."""
    on = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if on:
            gc.enable()


# arithmetic modes of the tensor-pipe kernels: precision -> wgmma products per K step (the kernels' `products`)
PRECISIONS = {"fp32": 3, "f16": 1}


def check_precision(precision, sparse_impl="tc", rpn_impl="auto"):
    """-> the kernels' product count for ``precision``; raises ValueError for an unknown precision and for the f16 mode
    with the fp32 reference paths (sparse_impl="fma", rpn_impl="cudnn")"""
    if precision not in PRECISIONS:
        raise ValueError("precision must be one of %s, got %r" % (sorted(PRECISIONS), precision))
    if precision == "f16" and (sparse_impl == "fma" or rpn_impl == "cudnn"):
        raise ValueError("precision='f16' runs on the tensor pipe only: sparse_impl='fma' and rpn_impl='cudnn' are the "
                         "fp32 reference paths")
    return PRECISIONS[precision]


def _record_margin(rec, n):
    """_field_margin for the fused tail's empty-frame head records [H, W, stride] (fp32, the first n channels)."""
    return _bits_margin(rec[:, :, :n].contiguous().view(torch.int32))


def _bits_margin(f):
    """f [H, W, K] integer bits (+0 and -0 differ) -> the margin of _field_margin."""
    H, W = f.shape[0], f.shape[1]
    diff = (f != f[H // 2, W // 2]).any(-1)
    ys, xs = torch.arange(H, device=f.device), torch.arange(W, device=f.device)
    dist = torch.minimum(torch.minimum(ys, H - 1 - ys)[:, None], torch.minimum(xs, W - 1 - xs)[None, :])
    m = int(dist[diff].max().item()) + 1 if bool(diff.any()) else 0
    return m if 2 * m < H and 2 * m < W else -1


def _pow2_at_least(n):
    c = 1024
    while c < n:
        c <<= 1
    return c


def ctypes_ptr(addr):
    return ctypes.c_void_p(int(addr))


class _Level:
    """one active-site set: coordinates, device count, coordinate->row hash, row capacity."""
    __slots__ = ("coors", "n_dev", "keys", "vals", "hcap", "cap", "shape")


class _Streamed:
    """what streamed batches add to an engine, allocated on the first streamed call: slot 1's input buffers (slot 0's
    are the engine's own ``points`` / ``offsets``), the copy stream, and per slot the free / ready / done events and
    the pinned read-back buffers."""

    def __init__(self, eng):
        self.points = torch.zeros_like(eng.points)
        self.offsets = torch.zeros_like(eng.offsets)
        self.copy = torch.cuda.Stream(eng.dev)
        self.free = [torch.cuda.Event(), torch.cuda.Event()]
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.done = [torch.cuda.Event(), torch.cuda.Event()]
        self.rec_host = [torch.empty(eng.B, eng.rec_width, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.status_host = [torch.zeros(1, dtype=torch.int32).pin_memory() for _ in range(2)]
        self.next_slot = 0


class InferenceEngine:
    def __init__(self, net, batch_size=1, max_points=None, max_voxels=None, row_cap_factor=2.0,
                 cand_cap=None, use_cuda_graph=True, rpn_impl="auto", sparse_impl="tc", device=None,
                 anchor_area_threshold=None, precision="fp32"):
        import spconv as sp                      # the CUDA drop-in: fails loudly if the library is missing
        assert not getattr(sp, "__oracle__", False), "the engine is the product path; it never runs on the oracle"
        self.sp = sp
        self.lib = sp._lib.load()
        self._L = sp._lib
        # "fp32": 3xF16 (fp32-grade) tensor-pipe products; "f16": one fp16 plane per operand, one product
        self.products = check_precision(precision, sparse_impl, rpn_impl)
        self.precision = precision
        self.spec = s = net if isinstance(net, _spec.NetSpec) else _spec.spec_from_module(net, max_voxels)
        if max_voxels:
            s.max_voxels = int(max_voxels)
        self.B = int(batch_size)
        dev = torch.device(device) if device is not None else s.device
        assert dev.type == "cuda", "InferenceEngine needs the network on a CUDA device"
        self.dev = dev
        # parity bar is fp32: keep cuDNN/cuBLAS off TF32 (torch allows TF32 convs by default)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.benchmark = True
        self.F = s.num_point_features
        self.T = s.max_points_per_voxel
        self.max_voxels = s.max_voxels
        self.P_cap = int(max_points or 40000) * self.B
        self.grid = s.grid_size
        self.code = s.box_code_size
        self.use_graph = use_cuda_graph
        self._graphs = {}
        # RPN: "tc" = hand-written wgmma implicit GEMM (csrc/conv_tc.cu, 3xF16), "cudnn" = torch/cuDNN fp32.
        if rpn_impl == "auto":
            rpn_impl = "tc" if _tc.supported(s.rpn, s.heads) else "cudnn"
        assert rpn_impl in ("tc", "cudnn")
        if rpn_impl == "cudnn" and self.products == 1:
            raise ValueError("precision='f16': this RPN has a layer b2s_conv2d_tc_ex3 does not cover, and rpn_impl="
                             "'cudnn' is the fp32 reference path")
        if rpn_impl == "tc" and not _tc.supported(s.rpn, s.heads):
            raise ValueError("rpn_impl='tc': this RPN has a layer b2s_conv2d_tc_ex2 does not cover (channels % 64, "
                             "kernel > 4)")
        self.rpn_impl = rpn_impl
        assert sparse_impl in ("tc", "fma")       # sparse-conv inner product: wgmma 3xF16 | fp32 FMA tiles
        self.sparse_impl = sparse_impl
        # anchor-area mask of the reference's eval preprocessing (preprocess.py:345-357): None / negative = off
        self.area_threshold = float(anchor_area_threshold) if _anchor_mask.enabled(anchor_area_threshold) else None
        # every operand derived from the weights is allocated by its first fill (_fill) while the engine is built;
        # refresh() runs the same fills again into the same tensors
        self._allocating = True
        with torch.cuda.device(dev):
            self.status = torch.zeros(1, dtype=torch.int32, device=dev)
            self._plan_middle(row_cap_factor)
            self._alloc_voxel_buffers()
            if rpn_impl == "tc":
                self._alloc_tc_rpn()
            else:
                self._module_ptrs = self._rpn_module_ptrs()
            self._alloc_detect_buffers(cand_cap)
            if self.area_threshold is not None:
                self._alloc_area_mask()
        self._allocating = False

    # ---------------------------------------------------------------- weight-derived operands
    def _fill(self, dst, key, value):
        """store the weight-derived operand ``value`` as ``dst[key]``: allocated while the engine is built, written in
        place by a refresh, so the addresses the captured graphs hold stay valid"""
        if value is None:
            assert dst.get(key) is None, "operand %s appeared or vanished" % key
            dst[key] = None
            return
        if self._allocating:
            dst[key] = torch.empty(value.shape, dtype=value.dtype, device=self.dev)
        t = dst[key]
        if t is None or t.shape != value.shape or t.dtype != value.dtype:
            raise _spec.UnsupportedNetwork("operand %s changed shape or type since the engine was built" % key)
        t.copy_(value)

    def _fill_middle(self):
        """the PFN's weight and folded BatchNorm, or every sparse layer's weight, folded BatchNorm and, on the tensor
        pipe, its packed fp16 hi/lo weight planes and epilogue scale -- from the spec"""
        s = self.spec
        if self.is_pillars:
            p = s.pfn
            for key, v in (("pfn_w", p["w"]), ("pfn_scale", p["scale"]), ("pfn_shift", p["shift"])):
                self._fill(vars(self), key, v)
            return
        for lyr, ls in zip(self.layers, s.layers):
            for key in ("w", "scale", "shift"):
                self._fill(lyr, key, ls[key])
            if lyr["tc"]:
                wp = _tc.pack_sparse_weights(lyr["w"])
                ws = _tc.pow2_scale(wp)
                hi, lo = _tc.weight_planes(wp, ws, self.products)
                base = lyr["scale"] if lyr["scale"] is not None else torch.ones(lyr["cout"], device=self.dev)
                self._fill(lyr, "w_hi", hi)
                self._fill(lyr, "w_lo", lo)
                self._fill(lyr, "scale_tc", (base.float() / ws).contiguous())

    def _rpn_plan(self):
        D, H, W = self.final_level.shape
        rpn, heads = self.spec.rpn, getattr(self.spec, "heads", None)
        if heads is None:
            return _tc.plan_rpn(rpn, H, W, products=self.products)
        return _tc.plan_rpn_multihead(rpn, dict(heads), H, W, products=self.products)

    def _fill_tc_rpn(self):
        """every tensor-core RPN op's weight planes, epilogue scale and shift -- blocks, deblock sub-grids, packed head
        records, the multi-head network's crop-branch convs -- from the live modules through tc.plan_rpn*"""
        plan = self._rpn_plan()
        if self._allocating:
            self.tc_prog, self.tc_plan = plan, plan["ops"]
        elif _tc.plan_layout(plan) != _tc.plan_layout(self.tc_prog):
            raise _spec.UnsupportedNetwork("the RPN's layer plan changed since the engine was built")
        for op, new in zip(self.tc_plan, plan["ops"]):
            for key in _tc.OP_OPERANDS:
                self._fill(op, key, new.get(key))
            if "w_scale" in new:
                op["w_scale"] = new["w_scale"]

    def _fill_background(self):
        """the background-tracked layers' empty-frame responses, the fused tail's empty-frame records and their margins;
        -> whether a margin (a host-side launch argument of the captured graphs) changed"""
        fields, records = self._empty_frame_response()
        if self._allocating:
            self.bg_field, self.tail_field = fields, records
        else:
            for old, new in zip(self.bg_field, fields):
                for o, n in zip(old, new):
                    if o is not None:
                        o.copy_(n)
            self.tail_field.copy_(records)
        margins = ([_field_margin(hi, lo) for hi, lo in self.bg_field],
                   _record_margin(self.tail_field, self.tc_plan[-1]["cout"]))
        changed = margins != (getattr(self, "bg_margin", None), getattr(self, "tail_margin", None))
        self.bg_margin, self.tail_margin = margins
        return changed

    def _rpn_module_ptrs(self):
        """addresses of the RPN / head modules' tensors, which the rpn_impl="cudnn" graphs read directly"""
        mods = [self.spec.rpn] + [m for _, m in (getattr(self.spec, "heads", None) or [])]
        return [t.data_ptr() for m in mods for t in list(m.parameters()) + list(m.buffers())]

    def refresh(self):
        """re-derive every weight-derived operand from the spec (``b2second.spec.refresh`` re-reads the network into
        it) by the fills that built them, into the same tensors; bit for bit what a newly built engine holds.  The
        work is enqueued on the current stream, after whatever is already there, so batches enqueued before finish with
        the weights they were enqueued with.  The captured graphs stay valid unless a host-side launch argument changed
        (a background margin; for rpn_impl="cudnn" the address of a module tensor): then they are dropped and
        re-captured on the next run.  -> whether they were dropped."""
        with torch.cuda.device(self.dev), torch.no_grad():
            self._fill_middle()
            if self.rpn_impl == "tc":
                self._fill_tc_rpn()
                drop = bool(self.bg_idx) and self._fill_background()
            else:
                ptrs = self._rpn_module_ptrs()
                drop, self._module_ptrs = ptrs != self._module_ptrs, ptrs
            if drop and self._graphs:
                torch.cuda.synchronize(self.dev)        # no replay of a graph in flight when it is destroyed
                self._graphs = {}
        return drop

    # ---------------------------------------------------------------- planning / allocation
    def _new_level(self, cap, shape, with_storage=True):
        lv = _Level()
        lv.cap = int(cap)
        lv.shape = [int(x) for x in shape]
        lv.hcap = _pow2_at_least(2 * lv.cap)
        if with_storage:
            lv.coors = torch.zeros(lv.cap, 4, dtype=torch.int32, device=self.dev)
            lv.n_dev = torch.zeros(1, dtype=torch.int32, device=self.dev)
            lv.keys = torch.empty(lv.hcap, dtype=torch.int64, device=self.dev)
            lv.vals = torch.empty(lv.hcap, dtype=torch.int32, device=self.dev)
        return lv

    def _hilo_rows(self, cap, c):
        """interleaved fp16 rows [cap][hi c | lo c] -> (buffer, hi view, lo view, row stride in halves); in the f16 mode
        rows [cap][c] of one plane, lo None."""
        if self.products == 1:
            buf = torch.zeros(cap, c, dtype=torch.float16, device=self.dev)
            return buf, buf, None, c
        buf = torch.zeros(cap, 2, c, dtype=torch.float16, device=self.dev)
        return buf, buf[:, 0], buf[:, 1], 2 * c

    def _plan_middle(self, row_cap_factor):
        s, sp, dev = self.spec, self.sp, self.dev
        self.is_pillars = s.is_pillars
        self.layers = []
        self.rb_ws = None
        cap0 = self.B * self.max_voxels
        if self.is_pillars:
            self.level0 = self._new_level(cap0, s.sparse_shape, with_storage=False)
            p = s.pfn
            self.pfn_cout = p["cout"]
            if p["with_distance"]:
                raise _spec.UnsupportedNetwork("PillarFeatureNet with_distance (off in every BASELINE config)")
            self._fill_middle()                                          # pfn_w, pfn_scale, pfn_shift
            self.pfn_geom = (p["vx"], p["vy"], p["x_offset"], p["y_offset"])
            self.pfn_deco = int(getattr(s, "pfn_decoration", 0))      # B2S_PFN_PLAIN / B2S_PFN_RADIUS
            self.feat_final_c = self.pfn_cout
            self.final_level = self.level0
            self.pfn_out = torch.zeros(cap0, self.pfn_cout, dtype=torch.float32, device=dev)
            return
        self.level0 = self._new_level(cap0, s.sparse_shape, with_storage=False)   # storage = voxelizer outputs
        level = self.level0
        rulebooks = {}
        max_ws = 0
        for j, ls in enumerate(s.layers):
            K = ls["K"]
            lyr = {k: v for k, v in ls.items() if not isinstance(v, torch.Tensor)}    # operands: _fill_middle
            lyr["index"] = j
            if ls["subm"]:
                key = ("subm", ls["indice_key"], id(level)) if ls["indice_key"] is not None else ("subm", j)
                if key not in rulebooks:
                    rulebooks[key] = {"nbr": torch.empty(level.cap, K, dtype=torch.int32, device=dev)}
                    lyr["build_rb"] = True
                    # the strided conv right before this layer produced `level`: its occupancy bitmap is still in the
                    # rulebook workspace, so this SubM table is built by rank lookups (b2s_rulebook_subm_ranked, up
                    # to 27 kernel offsets) and the level needs no hash table
                    prev = self.layers[-1] if self.layers else None
                    lyr["ranked"] = bool(prev is not None and not prev["subm"] and prev["out_level"] is level and K <= 27)
                else:
                    lyr["build_rb"] = False
                lyr["rb"] = rulebooks[key]
                lyr["in_level"], lyr["out_level"] = level, level
            else:
                out_shape = sp.ops.get_conv_output_size(level.shape, ls["kernel_size"], ls["stride"], ls["padding"],
                                                        ls["dilation"])
                cells = int(np.prod(out_shape))
                fan = int(np.prod([-(-k // st) for k, st in zip(ls["kernel_size"], ls["stride"])]))
                per_frame = min(cells, int(self.max_voxels * row_cap_factor), level.cap // self.B * fan)
                new = self._new_level(self.B * per_frame, out_shape)
                lyr["rb"] = {"nbr": torch.empty(new.cap, K, dtype=torch.int32, device=dev)}
                lyr["build_rb"] = True
                lyr["in_level"], lyr["out_level"] = level, new
                max_ws = max(max_ws, self.lib.b2s_rulebook_conv_workspace_bytes(self.B, self._L.i3(out_shape)))
                level = new
            # tile plan of the rulebook (csrc/sparse_plan.cu): which kernel offsets each 128-row tile needs, and an order
            # of the rows that makes that set small
            rb = lyr["rb"]
            if "tile_mask" not in rb and _tc.wants_tile_plan(ls["subm"], K):
                cap_rb = lyr["out_level"].cap
                rb["tile_mask"] = torch.zeros((cap_rb + 127) // 128, dtype=torch.int32, device=dev)
                rb["row_mask"] = torch.zeros(cap_rb, dtype=torch.int32, device=dev)    # written by the rulebook builder
                rb["perm"] = torch.zeros(cap_rb, dtype=torch.int32, device=dev)
            # tensor-pipe core (csrc/sparse_conv_tc.cu) where tc.sparse_tc_channels allows; else fp32 FMA core
            cin_tc = _tc.sparse_tc_channels(self.lib, ls["cin"], ls["cout"], K) if self.sparse_impl == "tc" else None
            lyr["cin_tc"] = cin_tc
            lyr["tc"] = cin_tc is not None
            self.layers.append(lyr)
        # a level's coordinate hash is only built when some SubM rulebook still looks rows up by hash
        for lyr in self.layers:
            if not lyr["subm"]:
                lyr["want_hash"] = any(l["subm"] and l.get("build_rb") and l["in_level"] is lyr["out_level"]
                                       and not l.get("ranked") for l in self.layers)
        # once a layer runs on the tensor pipe all later ones must too (hi/lo planes flow forward)
        seen_tc = False
        for lyr in self.layers:
            if seen_tc and not lyr["tc"]:
                for l2 in self.layers:
                    l2["tc"] = False
                break
            seen_tc = seen_tc or lyr["tc"]
        for j, lyr in enumerate(self.layers):
            cap = lyr["out_level"].cap
            if lyr["tc"]:
                lyr["out_buf"], lyr["out_hi"], lyr["out_lo"], lyr["out_stride"] = self._hilo_rows(cap, lyr["cout"])
                if j == 0 or not self.layers[j - 1]["tc"]:
                    # first tensor-pipe layer: its fp32 input rows are split into fp16 hi/lo planes first
                    lyr["in_split"] = self._hilo_rows(lyr["in_level"].cap, lyr["cin_tc"])
            else:
                lyr["out"] = torch.zeros(cap, lyr["cout"], dtype=torch.float32, device=dev)
        self._fill_middle()
        self.any_sparse_tc = any(l["tc"] for l in self.layers)
        self.rb_ws = torch.empty(max(max_ws, 1), dtype=torch.uint8, device=dev)
        self.rb_ws_bytes = max_ws
        self.final_level = level
        self.feat_final_c = self.layers[-1]["cout"]

    def _alloc_voxel_buffers(self):
        lib, dev, s = self.lib, self.dev, self.spec
        cap = self.B * self.max_voxels
        self.points = torch.zeros(self.P_cap, self.F, dtype=torch.float32, device=dev)
        self.offsets = torch.zeros(self.B + 1, dtype=torch.int32, device=dev)
        self.vox_coors = torch.zeros(cap, 4, dtype=torch.int32, device=dev)
        self.vox_num = torch.zeros(cap, dtype=torch.int32, device=dev)
        self.vox_slots = torch.zeros(cap, self.T, dtype=torch.int32, device=dev)
        self.num_voxels = torch.zeros(1 + self.B, dtype=torch.int32, device=dev)
        # the voxelizer's hash doubles as level 0's coordinate->row locator: sized for the points it must absorb AND
        # (pre-voxelised entry, b2s_hash_build) for 2x the voxel rows
        self.vox_hcap = max(lib.b2s_voxelize_hash_capacity(self.P_cap), _pow2_at_least(2 * cap))
        self.vox_keys = torch.empty(self.vox_hcap, dtype=torch.int64, device=dev)
        self.vox_vals = torch.empty(self.vox_hcap, dtype=torch.int32, device=dev)
        # the workspace holds one int per hash slot: query it for a point count whose own hash capacity is vox_hcap
        self.vox_ws_bytes = lib.b2s_voxelize_workspace_bytes(max(self.P_cap, self.vox_hcap // 2), self.B,
                                                             self.max_voxels, self.T)
        self.vox_ws = torch.empty(max(self.vox_ws_bytes, 1), dtype=torch.uint8, device=dev)
        if s.vfe_kind == "mean":
            self.vfe_mode, self.vfe_nf, c = 1, s.vfe_num_features, s.vfe_num_features
        elif s.vfe_kind == "mean_radius":
            self.vfe_mode, self.vfe_nf, c = 2, s.vfe_num_features, s.vfe_num_features - 1
        else:
            self.vfe_mode, self.vfe_nf, c = 0, self.F, 0
        self.vfe_out = torch.zeros(cap, c, dtype=torch.float32, device=dev) if c else None
        # level 0 aliases the voxelizer outputs
        lv = self.level0
        lv.coors, lv.n_dev, lv.keys, lv.vals, lv.hcap = (self.vox_coors, self.num_voxels, self.vox_keys,
                                                         self.vox_vals, self.vox_hcap)
        C = self.feat_final_c
        D, H, W = self.final_level.shape
        self.bev_cd = C * D
        if self.spec.bev_channels is None:
            self.spec.bev_channels = C * D
        if self.rpn_impl == "cudnn":
            self.bev = torch.zeros(self.B, C * D, H, W, dtype=torch.float32, device=dev)
        # pre-voxelised entry (the reference's own example dict): the caller's voxels land here
        self.in_voxels = None

    # tensor-pipe entry points: the 3xF16 call of the default mode -> (its products-taking form, how many trailing
    # arguments -- status, stream -- follow the inserted products arguments)
    _F16_FORMS = {"b2s_conv2d_tc_ex2": ("b2s_conv2d_tc_ex3", 2),
                  "b2s_sparse_conv_tc_plan": ("b2s_sparse_conv_tc_plan_ex", 2),
                  "b2s_rpn_tail_tc_ex": ("b2s_rpn_tail_tc_ex2", 2), "b2s_to_bev_tc_ex": ("b2s_to_bev_tc_ex2", 1),
                  "b2s_crop_nhwc": ("b2s_crop_nhwc_ex", 1), "b2s_split_f16": ("b2s_split_f16_ex", 1)}

    def _tc_call(self, name, *args, f16=(), what=""):
        """one tensor-pipe library call: ``name`` with ``args`` in the default mode, exactly as it has always been
        called; in the f16 mode its products-taking form with products = 1 and then ``f16`` inserted before the
        trailing status / stream arguments.  ``what`` follows the entry point's name in an error message."""
        if self.products == 3:
            return self._L.check(getattr(self.lib, name)(*args), name + what)
        name1, tail = self._F16_FORMS[name]
        args = args[:-tail] + (1,) + tuple(f16) + args[-tail:]
        return self._L.check(getattr(self.lib, name1)(*args), name1 + what)

    @property
    def n_planes(self):
        """fp16 planes per tensor-pipe operand: 2 (hi, lo) for precision "fp32", 1 for "f16"."""
        return 2 if self.products == 3 else 1

    def _alloc_tc_rpn(self):
        """buffers of the tensor-core RPN: NHWC halo-padded fp16 hi/lo planes (halo zero-filled once, never written);
        (hi, None) in the f16 mode."""
        dev, B = self.dev, self.B
        D, H, W = self.final_level.shape
        C = self.feat_final_c * D
        rpn = self.spec.rpn
        if next(rpn.parameters()).device != dev:
            raise ValueError("the RPN's parameters must live on the engine's device")
        heads = getattr(self.spec, "heads", None)
        self._fill_tc_rpn()                                 # tc_prog, tc_plan and the ops' operands
        plan = self.tc_prog
        # single-scale tail (one k = s = 1 deblock 128 -> 128 feeding the heads): one fused kernel, the deblock output
        # never goes to HBM (csrc/rpn_tail.cu; bit-identical to the two launches)
        self.tc_tail_fused = _tc.fusable_tail(plan)
        assert plan["in_channels"] == C, "BEV channels %d != RPN input %d" % (C, plan["in_channels"])

        def plane(h, w, c):
            return tuple(torch.zeros(B, h + 2, w + 2, c, dtype=torch.float16, device=dev) if i < self.n_planes else None
                         for i in range(2))
        # the BEV planes are zero except at the pixels flagged in bev_occ (b2s_to_bev_tc_ex keeps that so from step
        # to step); nothing else writes them
        self.tc_bev = plane(H, W, C)
        self.bev_occ = torch.zeros(B, H, W, dtype=torch.uint8, device=dev)
        self.tc_bufs = {"in": self.tc_bev}
        for name, (h, w, c) in plan["buffers"].items():
            self.tc_bufs[name] = plane(h, w, c)
        if heads is not None:
            # one packed fp32 record map per head segment [B, H, W, stride]
            self.tc_seg_heads = {}
            for sg in plan["segments"]:
                t = torch.zeros(B, sg["H"], sg["W"], sg["stride"], dtype=torch.float32, device=dev)
                self.tc_seg_heads[sg["name"]] = t
                self.tc_bufs[sg["buffer"]] = (t, None)
        else:
            hd = plan["heads"]
            self.tc_head_stride = hd["stride"]
            self.tc_heads = torch.zeros(B, hd["H"], hd["W"], self.tc_head_stride, dtype=torch.float32, device=dev)
            self.tc_bufs["heads"] = (self.tc_heads, None)
        self.tc_hw = (H, W)
        # background strips (csrc/rpn_bg.cu): through the leading chain of 3x3 stride-1 layers, output strips 8 pixels
        # wide and BG_ROWS high whose whole receptive field is empty BEV are not computed but copied from the layer's
        # response to an empty frame.  Only the strips a later launch reads need that response (b2s_rpn_strip_bands):
        # the next layer's windows, and for the last layer the fused tail's computed 8 x 16 tiles; the tail writes the
        # records of its other tiles from the records of an empty frame.  So the chain must end in the fused tail.
        self.bg_idx = _tc.background_layers(plan)
        if self.bg_idx:
            assert (self.tc_tail_fused and len(plan["ops"]) == len(self.bg_idx) + 2
                    and plan["ops"][-2]["src"] == plan["ops"][self.bg_idx[-1]]["dst"]), \
                "background strips are tracked only through a 3x3 chain whose last layer feeds the fused tail"
            nl = len(self.bg_idx)
            self.bg_tiles = B * (-(-H // BG_ROWS)) * (-(-W // 8))    # strips per layer
            self.bg_scratch = torch.zeros(2, B, H, W, dtype=torch.uint8, device=dev)
            self.bg_flags = torch.zeros(nl, self.bg_tiles, dtype=torch.int32, device=dev)
            self.bg_work = torch.zeros(nl, self.bg_tiles, dtype=torch.int32, device=dev)
            self.bg_list = torch.zeros(nl, self.bg_tiles, dtype=torch.int32, device=dev)
            self.bg_counts = torch.zeros(nl, 2, dtype=torch.int32, device=dev)
            self.bg_bands = torch.zeros(nl, self.bg_tiles, dtype=torch.int32, device=dev)
            self.bg_band_counts = torch.zeros(nl, dtype=torch.int32, device=dev)
            self.tail_tiles = B * (-(-H // 8)) * (-(-W // 16))         # fused-tail tiles of 8 x 16 pixels
            self.tail_work = torch.zeros(self.tail_tiles, dtype=torch.int32, device=dev)
            self.tail_bg = torch.zeros(self.tail_tiles, dtype=torch.int32, device=dev)
            self.tail_counts = torch.zeros(2, dtype=torch.int32, device=dev)
            self._fill_background()                         # bg_field, tail_field, bg_margin, tail_margin

    def _empty_frame_response(self):
        """per background-tracked layer: what the layer's own kernel produces for an empty frame, as one halo-padded
        frame [H+2, W+2, C] of fp16 hi/lo planes; and the fused tail's head records [H, W, stride] for an empty frame,
        from the tail kernel on the last layer's response.  Computed in one-frame zero planes of its own, so the
        engine's activation buffers, BEV planes, bev_occ and strip state -- which the next batch reads -- are not
        touched."""
        st = self._L.stream()
        shapes = dict(self.tc_prog["buffers"], **{"in": self.tc_hw + (self.tc_bev[0].shape[-1],)})
        planes = {}

        def plane(name):
            if name not in planes:
                h, w, c = shapes[name]
                planes[name] = tuple(torch.zeros(1, h + 2, w + 2, c, dtype=torch.float16, device=self.dev)
                                     if i < self.n_planes else None for i in range(2))
            return planes[name]
        fields = []
        for oi in self.bg_idx:
            op = self.tc_plan[oi]
            src, dst = plane(op["src"]), plane(op["dst"])
            self._launch_conv(op, src, dst, 1, None, None, -1, st)
            fields.append(tuple(t[0, :, :, :op["cout"]].clone().contiguous() if t is not None else None for t in dst))
        d = self.tc_plan[-2]
        records = torch.zeros(1, d["Hin"], d["Win"], self.tc_head_stride, dtype=torch.float32, device=self.dev)
        self._launch_fused_tail(plane(d["src"]), records, 1, None, None, None, None, None, -1, st)
        return fields, records[0]

    def _launch_conv(self, op, src, dst, batch, lists, field, margin, st):
        """one b2s_conv2d_tc_ex2 (f16 mode: _ex3) launch of the tc_plan op ``op``: hi/lo planes ``src`` -> planes
        ``dst`` from the op's channel offset on (fp32 records for a "planes": 1 op; lo planes None in the f16 mode).
        ``lists``: (strip work list, its count, background strip list, its count), or None for a dense launch;
        ``field``: the (hi, lo) empty-frame response the background strips are stored from, or None."""
        L = self._L
        cdst = dst[0].shape[-1]                                   # channels per pixel of the destination map
        esz = dst[0].element_size()
        o_hi = ctypes_ptr(dst[0].data_ptr() + esz * op["dst_coff"])
        o_lo = None if op["planes"] == 1 or dst[1] is None else ctypes_ptr(dst[1].data_ptr() + esz * op["dst_coff"])
        work, work_n, bgl, bgn = lists or (None,) * 4
        bhi, blo = (L.ptr(field[0]), L.ptr(field[1])) if field is not None else (None, None)
        self._tc_call(
            "b2s_conv2d_tc_ex2", L.ptr(src[0]), L.ptr(src[1]), batch, op["Hin"], op["Win"], op["cin"],
            L.ptr(op["w_hi"]), L.ptr(op["w_lo"]), op["kh"], op["kw"], op["stride"], op["pad"], op["cout"], op["n_pad"],
            L.ptr(op["scale"]), L.ptr(op["shift"]), 1 if op["relu"] else 0, op["Hg"], op["Wg"], o_hi, o_lo,
            op["Hout"], op["Wout"], 1 if op["padded"] else 0, cdst, op["out_mul"], op["off_h"], op["off_w"],
            work, work_n, bgl, bgn, bhi, blo, margin, BG_ROWS, L.ptr(self.status), st,
            f16=(1 if op["planes"] == 1 else 0,), what="(%s)" % op["kind"])    # f16: out_fp32 for the head records

    def _launch_fused_tail(self, src, out, batch, work, work_n, bgl, bgn, field, margin, st):
        L, lib = self._L, self.lib
        d, h = self.tc_plan[-2], self.tc_plan[-1]
        self._tc_call(
            "b2s_rpn_tail_tc_ex", L.ptr(src[0]), L.ptr(src[1]), batch, d["Hin"], d["Win"], d["cin"], L.ptr(d["w_hi"]),
            L.ptr(d["w_lo"]), d["cout"], L.ptr(d["scale"]), L.ptr(d["shift"]), L.ptr(h["w_hi"]), L.ptr(h["w_lo"]),
            h["cout"], h["n_pad"], L.ptr(h["scale"]), L.ptr(h["shift"]), L.ptr(out), self.tc_head_stride, work, work_n,
            bgl, bgn, L.ptr(field), margin, L.ptr(self.status), st)

    def _feature_hw(self):
        if self.rpn_impl == "tc":
            return self.tc_prog["heads"]["H"], self.tc_prog["heads"]["W"]
        D, H, W = self.final_level.shape
        with torch.no_grad():
            y = self.spec.rpn.conv_box(self._rpn_backbone(torch.zeros(1, self.bev_cd, H, W, device=self.dev))[0])
        return int(y.shape[2]), int(y.shape[3])

    def _head_segments(self):
        """multi-head network: [{"name", "H", "W", "a_loc", "base"}] in anchor order (large head first)."""
        if self.rpn_impl == "tc":
            segs = [{"name": g["name"], "H": g["H"], "W": g["W"], "a_loc": g["a_loc"]} for g in self.tc_prog["segments"]]
        else:
            D, H, W = self.final_level.shape
            with torch.no_grad():
                outs = self._rpn_multihead(torch.zeros(1, self.bev_cd, H, W, device=self.dev))
            segs = [{"name": name, "H": int(o[0].shape[2]), "W": int(o[0].shape[3]), "a_loc": int(m._num_anchor_per_loc)}
                    for (name, m), o in zip(self.spec.heads, outs)]
        base = 0
        for g in segs:
            g["base"] = base
            base += g["a_loc"] * g["H"] * g["W"]
        want = self.spec.head_feature_map_sizes
        got = [[g["H"], g["W"]] for g in segs]
        if want is not None and got != [list(x) for x in want]:
            raise _spec.UnsupportedNetwork("head maps %s do not match the per-class feature map sizes %s" % (got, want))
        return segs

    def _rpn_multihead(self, x):
        """VoxelNetNuscenesMultiHead.network_forward after the scatter (net_multi_head.py:155-161) on the torch modules:
        cuDNN cross-check path.  -> [(box, cls, dir) NCHW conv outputs] per head, large first."""
        x, stage0 = self._rpn_backbone(x)
        c = int(np.round(stage0.shape[2] * 0.1))
        hd = dict(self.spec.heads)
        small = hd["small"].net(stage0[:, :, c:-c, c:-c])
        return [self._conv_heads(hd["large"], x), self._conv_heads(hd["small"], small)]

    def _rpn_backbone(self, x):
        """RPNNoHeadBase.forward (rpn.py:314-331) on the torch modules: cuDNN cross-check path only.  -> (the
        concatenated map, stage 0's output)"""
        rpn = self.spec.rpn
        ups, stage0 = [], None
        for i in range(len(rpn.blocks)):
            x = rpn.blocks[i](x)
            if i == 0:
                stage0 = x
            if i - rpn._upsample_start_idx >= 0:
                ups.append(rpn.deblocks[i - rpn._upsample_start_idx](x))
        if len(ups) > 0:
            x = torch.cat(ups, dim=1)
        return x, stage0

    def _conv_heads(self, m, x):
        """a head module's box / cls / dir 1x1 convs on the torch modules -> (box, cls, dir or None), NCHW"""
        return (m.conv_box(x).contiguous(), m.conv_cls(x).contiguous(),
                m.conv_dir_cls(x).contiguous() if self.spec.use_direction_classifier else None)

    def _alloc_detect_buffers(self, cand_cap):
        s, dev = self.spec, self.dev
        self.segments = None
        if getattr(s, "heads", None) is None:
            self.fH, self.fW = self._feature_hw()
            self.a_loc = s.num_anchors_per_loc
            self.A = self.a_loc * self.fH * self.fW
        else:
            self.segments = self._head_segments()
            self.fH, self.fW = self.segments[0]["H"], self.segments[0]["W"]
            self.a_loc = s.num_anchors_per_loc
            self.A = sum(g["a_loc"] * g["H"] * g["W"] for g in self.segments)
        self.anchors = torch.zeros(self.A, self.code, dtype=torch.float32, device=dev)
        self._anchors_key = None
        try:
            a = _spec.anchors_for(s, (self.fH, self.fW))
        except Exception:
            a = None                                  # anchors then come with the first example (set_anchors)
        if a is not None:
            assert a.shape[0] == self.A, "anchor count %d != RPN output %d" % (a.shape[0], self.A)
            self.anchors.copy_(torch.from_numpy(a))
            self._anchors_key = "generated"
        self.anchors_mask = None                      # [B, A] uint8, allocated on first use
        self.use_mask = False
        self._mask_src = None                         # None | "given" (the example's anchors_mask) | "area" (computed)
        self.cand_cap = int(cand_cap or min(self.A, 32768))
        B, cc, code = self.B, self.cand_cap, self.code
        # per-class NMS branch (voxelnet.py:458-547): one candidate list and one NMS per (class, frame) -- "virtual
        # frames" v = c*B + b -- then the per-class results are concatenated in class order
        self.mc = bool(s.multiclass_nms)
        self.ncls = s.num_class
        V = self.ncls * B if self.mc else B
        self.cand_box = torch.zeros(V, cc, code, dtype=torch.float32, device=dev)
        self.cand_score = torch.zeros(V, cc, dtype=torch.float32, device=dev)
        self.cand_label = torch.zeros(V, cc, dtype=torch.int32, device=dev)
        self.cand_dir = torch.zeros(V, cc, dtype=torch.int32, device=dev)
        self.cand_anchor = torch.zeros(V, cc, dtype=torch.int32, device=dev)
        self.cand_count = torch.zeros(V, dtype=torch.int32, device=dev)
        self.score_thresh = float(s.nms_score_thresholds[0])
        self.pre_max, self.post_max = int(s.nms_pre_max_sizes[0]), int(s.nms_post_max_sizes[0])
        self.iou_thresh = float(s.nms_iou_thresholds[0])
        if self.mc:
            n = self.ncls
            assert n <= 16 and all(len(x) >= n for x in (s.nms_score_thresholds, s.nms_pre_max_sizes,
                                                         s.nms_post_max_sizes, s.nms_iou_thresholds))
            self.mc_thresh = (ctypes.c_float * n)(*s.nms_score_thresholds[:n])
            self.mc_pre = [int(x) for x in s.nms_pre_max_sizes[:n]]
            self.mc_post = [int(x) for x in s.nms_post_max_sizes[:n]]
            self.mc_iou = [float(x) for x in s.nms_iou_thresholds[:n]]
            self.mc_uniform = len(set(self.mc_pre)) == 1 and len(set(self.mc_post)) == 1 and len(set(self.mc_iou)) == 1
            self.pre_max, self.post_max_class = max(self.mc_pre), max(self.mc_post)
            self.post_max = n * self.post_max_class               # rows of a frame's record
            if s.nms_class_agnostic:
                self.mc_lo = self.mc_hi = None
            else:
                counts = s.class_anchor_counts
                if counts is None or len(counts) != n or sum(counts) != self.a_loc:
                    raise _spec.UnsupportedNetwork("per-class NMS needs target_assigner anchor counts per class")
                lo = np.cumsum([0] + counts[:-1]).tolist()
                self.mc_lo = (ctypes.c_int * n)(*lo)
                self.mc_hi = (ctypes.c_int * n)(*[a + c for a, c in zip(lo, counts)])
            self.det_mc = torch.zeros(V, self.post_max_class, code + 2, dtype=torch.float32, device=dev)
            self.cnt_mc = torch.zeros(V, dtype=torch.int32, device=dev)
        self.nms_ws_bytes = self.lib.b2s_nms_workspace_bytes(V, cc, self.pre_max)
        self.nms_ws = torch.empty(max(self.nms_ws_bytes, 1), dtype=torch.uint8, device=dev)
        # one record per frame: post_max*(code+2) detection floats followed by the count (as a float: < 2^24) --
        # exactly the all-gather payload (b2second/dist.py), written in place by the NMS epilogue
        self.rec_width = self.post_max * (code + 2) + 1
        self.det_record = torch.zeros(B, self.rec_width, dtype=torch.float32, device=dev)
        self.det_count = torch.zeros(B, dtype=torch.int32, device=dev)
        rng = s.post_center_range
        self.range_host = self._L.f6(rng) if len(rng) == 6 else None

    def _alloc_area_mask(self):
        """buffers of the computed anchor-area mask: the per-frame count map at voxel-grid resolution, the anchors'
        integer BEV boxes (derived on the host whenever the anchor set changes) and the [B, A] mask decode reads."""
        s = self.spec
        self.am_ny, self.am_nx = int(s.grid_size[1]), int(s.grid_size[0])
        self.am_ws_bytes = self.lib.b2s_anchor_area_mask_workspace_bytes(self.B, self.am_ny, self.am_nx)
        self.am_ws = torch.empty(max(self.am_ws_bytes, 1), dtype=torch.uint8, device=self.dev)
        self.am_boxes = torch.zeros(self.A, 4, dtype=torch.int32, device=self.dev)
        if self.anchors_mask is None:
            self.anchors_mask = torch.zeros(self.B, self.A, dtype=torch.uint8, device=self.dev)
        self._mask_src, self.use_mask = "area", True
        if self._anchors_key is not None:
            self._set_area_boxes(self.anchors)

    def _set_area_boxes(self, anchors):
        """float32 host derivation of the boxes (b2second.anchor_mask); reads the anchors back once per anchor set."""
        a = anchors.detach().reshape(-1, anchors.shape[-1]).float().cpu().numpy()
        s = self.spec
        boxes = _anchor_mask.anchor_boxes(a, s.voxel_size, s.point_cloud_range, s.grid_size)
        self.am_boxes.copy_(torch.from_numpy(boxes))

    def _launch_area_mask(self, st):
        """count map of level 0's voxels -> summed-area table -> anchors_mask [B, A] (one memset, four kernels)."""
        L, lv = self._L, self.level0
        self._mark("anchor_mask")
        L.check(self.lib.b2s_anchor_area_mask(
            L.ptr(lv.coors), L.ptr(lv.n_dev), lv.cap, self.B, self.am_ny, self.am_nx, L.ptr(self.am_boxes), self.A,
            self.area_threshold, L.ptr(self.am_ws), self.am_ws_bytes, L.ptr(self.anchors_mask), st),
            "b2s_anchor_area_mask")

    @property
    def det(self):
        """[B, post_max, code+2] view of the detection records."""
        return self.det_record[:, :self.rec_width - 1].view(self.B, self.post_max, self.code + 2)

    # ---------------------------------------------------------------- the launch sequence
    def _launch(self, mode="points", slot=0):
        L, lib, s = self._L, self.lib, self.spec
        st = L.stream()
        self.status.zero_()
        if mode == "points":
            points, offsets = self._inputs(slot)
            self._mark("voxelize")
            L.check(lib.b2s_voxelize(
                L.ptr(points), L.ptr(offsets), self.P_cap, self.F, self.B,
                L.f3(s.point_cloud_range[:3]), L.f3(s.voxel_size), L.i3(self.grid), self.T, self.max_voxels,
                L.ptr(self.vox_coors), L.ptr(self.vox_num), L.ptr(self.vox_slots), None, self.vfe_mode, self.vfe_nf,
                L.ptr(self.vfe_out), L.ptr(self.num_voxels), L.ptr(self.vox_keys), L.ptr(self.vox_vals), self.vox_hcap,
                int(self.level0.shape[0]),       # hash keys in the middle encoder's shape (grid_z + 1, middle.py:139)
                L.ptr(self.vox_ws), self.vox_ws_bytes, L.ptr(self.status), st), "b2s_voxelize")
            pfn_points, pfn_slots = points, self.vox_slots
        else:
            # the caller's voxels / num_points / coordinates are already in in_voxels / vox_num / vox_coors and
            # num_voxels[0] holds their count: build level 0's locator and the voxel features from them
            self._mark("voxelize")
            lv = self.level0
            if not self.is_pillars:
                L.check(lib.b2s_hash_build(L.ptr(lv.coors), L.ptr(lv.n_dev), lv.cap, L.i3(lv.shape), L.ptr(lv.keys),
                                           L.ptr(lv.vals), lv.hcap, L.ptr(self.status), st), "b2s_hash_build")
                L.check(lib.b2s_vfe_mean(L.ptr(self.in_voxels), L.ptr(self.vox_num), L.ptr(lv.n_dev), lv.cap, self.T,
                                         self.F, self.vfe_mode, self.vfe_nf, L.ptr(self.vfe_out), st), "b2s_vfe_mean")
            pfn_points, pfn_slots = self.in_voxels, self.in_slots
        if self._mask_src == "area":
            self._launch_area_mask(st)
        if self.is_pillars:
            vx, vy, xo, yo = self.pfn_geom
            self._mark("pfn")
            L.check(lib.b2s_pfn_ex(L.ptr(pfn_points), self.F, L.ptr(pfn_slots), L.ptr(self.vox_num),
                                   L.ptr(self.vox_coors), L.ptr(self.num_voxels), self.level0.cap, self.T,
                                   L.ptr(self.pfn_w), L.ptr(self.pfn_scale), L.ptr(self.pfn_shift), self.pfn_cout,
                                   vx, vy, xo, yo, self.pfn_deco, L.ptr(self.pfn_out), st), "b2s_pfn_ex")
            feats, hilo = self.pfn_out, None
        else:
            feats, hilo = self.vfe_out, None          # hilo = (hi, lo, stride) once on the tensor pipe
            for lyr in self.layers:
                lin, lout = lyr["in_level"], lyr["out_level"]
                if lyr["build_rb"]:
                    self._mark("rulebook%d" % lyr["index"])
                    if lyr["subm"] and lyr.get("ranked"):
                        L.check(lib.b2s_rulebook_subm_ranked(
                            L.ptr(lin.coors), L.ptr(lin.n_dev), lin.cap, self.B, L.i3(lin.shape),
                            L.i3(lyr["kernel_size"]), L.i3(lyr["dilation"]), L.ptr(self.rb_ws), self.rb_ws_bytes,
                            L.ptr(lyr["rb"]["nbr"]), L.ptr(lyr["rb"].get("row_mask")), st), "b2s_rulebook_subm_ranked")
                    elif lyr["subm"]:
                        L.check(lib.b2s_rulebook_subm(L.ptr(lin.coors), L.ptr(lin.n_dev), lin.cap, L.i3(lin.shape),
                                                      L.i3(lyr["kernel_size"]), L.i3(lyr["dilation"]), L.ptr(lin.keys),
                                                      L.ptr(lin.vals), lin.hcap, L.ptr(lyr["rb"]["nbr"]),
                                                      L.ptr(lyr["rb"].get("row_mask")), st), "b2s_rulebook_subm")
                    else:
                        L.check(lib.b2s_rulebook_conv(
                            L.ptr(lin.coors), L.ptr(lin.n_dev), lin.cap, self.B, L.i3(lin.shape), L.i3(lout.shape),
                            L.i3(lyr["kernel_size"]), L.i3(lyr["stride"]), L.i3(lyr["padding"]), L.i3(lyr["dilation"]),
                            L.ptr(lout.coors), L.ptr(lout.n_dev), lout.cap,
                            L.ptr(lyr["rb"]["nbr"]), L.ptr(lout.keys) if lyr["want_hash"] else None,
                            L.ptr(lout.vals) if lyr["want_hash"] else None, lout.hcap,
                            L.ptr(self.rb_ws), self.rb_ws_bytes, L.ptr(lyr["rb"].get("row_mask")), L.ptr(self.status), st),
                            "b2s_rulebook_conv")
                    if lyr["tc"] and "tile_mask" in lyr["rb"]:
                        rb = lyr["rb"]
                        L.check(lib.b2s_sparse_tile_plan(
                            L.ptr(rb["nbr"]), L.ptr(rb["row_mask"]), lyr["K"], L.i3(lyr["kernel_size"]), L.ptr(lout.n_dev), lout.cap,
                            1, L.ptr(rb["perm"]), L.ptr(rb["tile_mask"]), st),
                            "b2s_sparse_tile_plan")
                self._mark("sparse_conv%d" % lyr["index"])
                if lyr["tc"]:
                    if "in_split" in lyr:
                        _, hi, lo, stride = lyr["in_split"]
                        self._tc_call("b2s_split_f16", L.ptr(feats), L.ptr(hi), L.ptr(lo), L.ptr(lin.n_dev), lin.cap,
                                      lyr["cin"], lyr["cin_tc"], stride, st)
                        hilo = (hi, lo, stride)
                    self._tc_call(
                        "b2s_sparse_conv_tc_plan", L.ptr(hilo[0]), L.ptr(hilo[1]), hilo[2], lin.cap, lyr["cin_tc"],
                        L.ptr(lyr["w_hi"]), L.ptr(lyr["w_lo"]), L.ptr(lyr["rb"]["nbr"]), lyr["K"], L.ptr(lout.n_dev),
                        lout.cap, L.ptr(lyr["rb"].get("perm")), L.ptr(lyr["rb"].get("tile_mask")),
                        L.ptr(lyr["scale_tc"]), L.ptr(lyr["shift"]), 1 if lyr["relu"] else 0, L.ptr(lyr["out_hi"]),
                        L.ptr(lyr["out_lo"]), lyr["out_stride"], lyr["cout"], L.ptr(self.status), st)
                    feats, hilo = None, (lyr["out_hi"], lyr["out_lo"], lyr["out_stride"])
                else:
                    L.check(lib.b2s_sparse_conv(L.ptr(feats), lyr["cin"], L.ptr(lyr["w"]), L.ptr(lyr["rb"]["nbr"]),
                                                lyr["K"], L.ptr(lout.n_dev), lout.cap, L.ptr(lyr["scale"]),
                                                L.ptr(lyr["shift"]), 1 if lyr["relu"] else 0, L.ptr(lyr["out"]),
                                                lyr["cout"], st), "b2s_sparse_conv")
                    feats, hilo = lyr["out"], None
        if self.rpn_impl == "tc":
            heads = self._launch_tc_rpn(feats, hilo, st)
        else:
            heads = self._launch_cudnn_rpn(feats, hilo, st)
        self._launch_detect(heads, st)

    def _launch_cudnn_rpn(self, feats, hilo, st):
        """sparse rows -> NCHW BEV -> the torch RPN modules (cuDNN cross-check) -> one _head_view per head."""
        L, lib = self._L, self.lib
        fl = self.final_level
        D, H, W = fl.shape
        if hilo is not None:          # back to plain fp32 rows for the NCHW scatter (hi + lo is exact)
            if getattr(self, "merged_out", None) is None:
                self.merged_out = torch.zeros(fl.cap, self.feat_final_c, dtype=torch.float32, device=self.dev)
            L.check(lib.b2s_merge_f16(L.ptr(hilo[0]), L.ptr(hilo[1]), L.ptr(self.merged_out), L.ptr(fl.n_dev),
                                      fl.cap, self.feat_final_c, hilo[2], st), "b2s_merge_f16")
            feats = self.merged_out
        self._mark("to_bev")
        L.check(lib.b2s_to_bev(L.ptr(feats), L.ptr(fl.coors), L.ptr(fl.n_dev), fl.cap, self.feat_final_c, self.B,
                               D, H, W, L.ptr(self.bev), 0, st), "b2s_to_bev")
        self._mark("rpn")
        if self.segments is not None:
            self._keep = self._rpn_multihead(self.bev)
            return [self._head_view(o, g["H"], g["W"], g["a_loc"]) for g, o in zip(self.segments, self._keep)]
        x, _ = self._rpn_backbone(self.bev)
        self._keep = (x,) + self._conv_heads(self.spec.rpn, x)
        return [self._head_view(self._keep[1:], self.fH, self.fW, self.a_loc)]

    def _launch_tc_rpn(self, feats, hilo, st):
        """sparse rows -> BEV (NHWC, halo, fp16 hi/lo) -> wgmma RPN layers -> packed head records -> one _head_view
        per head."""
        L, lib = self._L, self.lib
        fl = self.final_level
        D, H, W = fl.shape
        self._mark("to_bev")
        feat, f_hi, f_lo, f_stride = (feats, None, None, 0) if hilo is None else (None,) + hilo
        self._tc_call("b2s_to_bev_tc_ex", L.ptr(feat), L.ptr(f_hi), L.ptr(f_lo), f_stride, L.ptr(fl.coors),
                      L.ptr(fl.n_dev), fl.cap, self.feat_final_c, self.B, D, H, W, L.ptr(self.tc_bev[0]),
                      L.ptr(self.tc_bev[1]), L.ptr(self.bev_occ), st)
        self._mark("rpn")
        nl = len(self.bg_idx)
        if nl:
            L.check(lib.b2s_rpn_strip_plan(L.ptr(self.bev_occ), self.B, H, W, nl, BG_ROWS,
                                           L.ptr(self.bg_scratch), L.ptr(self.bg_flags), L.ptr(self.bg_work),
                                           L.ptr(self.bg_list), L.ptr(self.bg_counts), st), "b2s_rpn_strip_plan")
            L.check(lib.b2s_rpn_strip_bands(L.ptr(self.bg_flags), self.B, H, W, nl, BG_ROWS, L.ptr(self.bg_bands),
                                            L.ptr(self.bg_band_counts), L.ptr(self.tail_work), L.ptr(self.tail_bg),
                                            L.ptr(self.tail_counts), st), "b2s_rpn_strip_bands")
        marked_tail = False
        n_ops = len(self.tc_plan) - (2 if self.tc_tail_fused else 0)
        for oi, op in enumerate(self.tc_plan[:n_ops]):
            if not op["v2"] and op["kind"] != "block" and not marked_tail:
                self._mark("rpn_1x1")          # the 3x3 stack (k_conv3x3_tc2) is timed apart from the deblock/heads tail
                marked_tail = True
            src, dst = self.tc_bufs[op["src"]], self.tc_bufs[op["dst"]]
            if op["kind"] == "crop":                                  # small head input: stage 0 inside a zero halo
                self._tc_call("b2s_crop_nhwc", L.ptr(src[0]), L.ptr(src[1]), self.B, op["Hin"], op["Win"], op["cin"],
                              op["crop"], L.ptr(dst[0]), L.ptr(dst[1]), st)
                continue
            lists, field, margin = None, None, -1
            if oi in self.bg_idx:
                bl = self.bg_idx.index(oi)
                # the conv kernel's fill warps store the empty-frame response into the background strips a later
                # launch reads
                lists = (L.ptr(self.bg_work[bl]), L.ptr(self.bg_counts[bl, 0:]), L.ptr(self.bg_bands[bl]),
                         L.ptr(self.bg_band_counts[bl:]))
                field, margin = self.bg_field[bl], self.bg_margin[bl]
            self._launch_conv(op, src, dst, self.B, lists, field, margin, st)
        if not marked_tail:
            self._mark("rpn_1x1")
        if self.tc_tail_fused:
            src = self.tc_bufs[self.tc_plan[-2]["src"]]
            if nl:          # computed tiles only; background tiles' records from the empty frame's records
                self._launch_fused_tail(src, self.tc_heads, self.B, L.ptr(self.tail_work), L.ptr(self.tail_counts[0:]),
                                        L.ptr(self.tail_bg), L.ptr(self.tail_counts[1:]), self.tail_field,
                                        self.tail_margin, st)
            else:
                self._launch_fused_tail(src, self.tc_heads, self.B, None, None, None, None, None, -1, st)
        if self.segments is not None:
            return [self._head_view(self.tc_seg_heads[g["name"]], g["H"], g["W"], offsets=pg["offsets"])
                    for g, pg in zip(self.segments, self.tc_prog["segments"])]
        return [self._head_view(self.tc_heads, self.fH, self.fW, offsets=self.tc_prog["heads"]["offsets"])]

    def _head_view(self, heads, H, W, a_loc=None, offsets=None):
        """one head map as the decode kernels read it: a tuple in _HEAD_VIEW order.  ``heads``: the (box, cls, dir or
        None) NCHW conv outputs [B, a_loc * n, H, W]; or, with ``offsets``, a packed record map [B, H, W, S] whose box,
        cls and dir channels start at offsets[0], [1] and [2]."""
        s, HW = self.spec, H * W
        if offsets is None:
            box, cls, dirp = heads
            return (box.data_ptr(), cls.data_ptr(), dirp.data_ptr() if dirp is not None else None,
                    a_loc * self.code * HW, a_loc * s.num_class * HW, a_loc * s.num_direction_bins * HW, HW, 1)
        S, esz = heads.shape[-1], heads.element_size()
        box, cls, dirp = (heads.data_ptr() + o * esz for o in offsets[:3])
        return (box, cls, dirp if s.use_direction_classifier else None, HW * S, HW * S, HW * S, 1, S)

    def _launch_detect(self, heads, st):
        """the head maps (one _head_view each, in anchor order) -> sigmoid + score threshold + box decode over all
        anchors -> candidate lists (per frame, or per (class, frame)) -> NMS."""
        L, lib, s = self._L, self.lib, self.spec
        self._mark("decode_filter")
        if self.segments is not None:
            # several head maps -> one candidate list per frame (global anchor ids; the single-class NMS branch)
            segs = [dict(zip(_HEAD_VIEW, v), a_loc=g["a_loc"], H=g["H"], W=g["W"], anchor_base=g["base"])
                    for v, g in zip(heads, self.segments)]
            L.check(lib.b2s_decode_filter_segments(
                L.head_segments(segs), len(segs), L.ptr(self.anchors),
                L.ptr(self.anchors_mask) if self.use_mask else None, self.A, self.B, self.code, s.num_class,
                s.num_direction_bins, self.score_thresh, L.ptr(self.cand_box), L.ptr(self.cand_score),
                L.ptr(self.cand_label), L.ptr(self.cand_dir), L.ptr(self.cand_anchor), L.ptr(self.cand_count),
                self.cand_cap, L.ptr(self.status), st), "b2s_decode_filter_segments")
        elif self.mc:
            if self.use_mask:
                raise RuntimeError("anchors_mask with the per-class NMS branch is ill-defined upstream (masking shifts "
                                   "the anchors_range indices, voxelnet.py:432-439,492-501)")
            L.check(lib.b2s_decode_filter_multiclass(
                *heads[0], L.ptr(self.anchors), self.B, self.a_loc, self.fH, self.fW, self.code, s.num_class,
                s.num_direction_bins, self.mc_lo, self.mc_hi, self.mc_thresh, L.ptr(self.cand_box),
                L.ptr(self.cand_score), L.ptr(self.cand_label), L.ptr(self.cand_dir), L.ptr(self.cand_anchor),
                L.ptr(self.cand_count), self.cand_cap, L.ptr(self.status), st), "b2s_decode_filter_multiclass")
        else:
            L.check(lib.b2s_decode_filter_strided(
                *heads[0], L.ptr(self.anchors), L.ptr(self.anchors_mask) if self.use_mask else None, self.B,
                self.a_loc, self.fH, self.fW, self.code, s.num_class, s.num_direction_bins, self.score_thresh,
                L.ptr(self.cand_box), L.ptr(self.cand_score), L.ptr(self.cand_label), L.ptr(self.cand_dir),
                L.ptr(self.cand_anchor), L.ptr(self.cand_count), self.cand_cap, L.ptr(self.status), st),
                "b2s_decode_filter_strided")
        self._launch_nms(st)

    def _launch_nms(self, st):
        L, lib, s = self._L, self.lib, self.spec
        self._mark("nms")
        if self.mc:
            B, cc, code, n = self.B, self.cand_cap, self.code, self.ncls
            groups = [(0, n * B, self.mc_pre[0], self.mc_post[0], self.mc_iou[0])] if self.mc_uniform else \
                [(c * B, B, self.mc_pre[c], self.mc_post[c], self.mc_iou[c]) for c in range(n)]
            for v0, nv, pre, post, iou in groups:         # class-major virtual frames: one class = B contiguous lists
                L.check(lib.b2s_nms(
                    L.ptr(self.cand_box[v0:]), L.ptr(self.cand_score[v0:]), L.ptr(self.cand_label[v0:]),
                    L.ptr(self.cand_dir[v0:]), L.ptr(self.cand_anchor[v0:]), L.ptr(self.cand_count[v0:]), nv, cc, code,
                    1 if s.use_rotate_nms else 0, pre, post, iou, 1 if s.use_direction_classifier else 0,
                    float(s.direction_offset), float(s.direction_limit_offset), s.num_direction_bins, self.range_host,
                    L.ptr(self.det_mc[v0:]), self.post_max_class * (code + 2), L.ptr(self.cnt_mc[v0:]),
                    L.ptr(self.nms_ws), self.nms_ws_bytes, st), "b2s_nms")
            L.check(lib.b2s_concat_class_detections(L.ptr(self.det_mc), L.ptr(self.cnt_mc), B, n, self.post_max_class,
                                                    code, L.ptr(self.det_record), self.rec_width, L.ptr(self.det_count),
                                                    st), "b2s_concat_class_detections")
            self._mark("end")
            return
        L.check(lib.b2s_nms(
            L.ptr(self.cand_box), L.ptr(self.cand_score), L.ptr(self.cand_label), L.ptr(self.cand_dir),
            L.ptr(self.cand_anchor), L.ptr(self.cand_count), self.B, self.cand_cap, self.code,
            1 if s.use_rotate_nms else 0, self.pre_max, self.post_max, self.iou_thresh,
            1 if s.use_direction_classifier else 0, float(s.direction_offset),
            float(s.direction_limit_offset), s.num_direction_bins, self.range_host, L.ptr(self.det_record),
            self.rec_width, L.ptr(self.det_count), L.ptr(self.nms_ws), self.nms_ws_bytes, st), "b2s_nms")
        self._mark("end")

    # ---------------------------------------------------------------- instrumentation
    _marks = None

    def _mark(self, name):
        if self._marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._marks.append((name, ev))

    def run_timed(self, iters=5, mode="points"):
        """eager (no graph) replay with a CUDA event before every stage; returns {stage: mean ms}."""
        acc = {}
        with torch.no_grad(), torch.cuda.device(self.dev):
            self._launch(mode)     # warm
            for _ in range(iters):
                self._marks = []
                self._launch(mode)
                torch.cuda.synchronize()
                for (name, ev), (_, nxt) in zip(self._marks[:-1], self._marks[1:]):
                    acc[name] = acc.get(name, 0.0) + ev.elapsed_time(nxt)
                self._marks = None
        return {k: v / iters for k, v in acc.items()}

    def kernel_launches_per_step(self):
        """how many of OUR kernels one pipeline pass launches (memsets and cuDNN kernels not counted)."""
        n = 7                                    # b2s_voxelize: insert, flag_scan, scan_sums, assign, fill, gather, finish
        if self._mask_src == "area":
            n += 4                               # b2s_anchor_area_mask: scatter, scan_rows, scan_cols, lookup
        if self.is_pillars:
            n += 1                               # b2s_pfn_ex
        for lyr in self.layers:
            if lyr["build_rb"]:
                # subm_nbr / subm_ranked | mark, summary_scan, scan_sums, compact_words, nz_scan, scan_sums, emit,
                # (hash_build,) scatter_nbr
                n += 1 if lyr["subm"] else (8 + (1 if lyr.get("want_hash") else 0))
                if lyr["tc"] and "tile_mask" in lyr["rb"]:
                    n += 1                       # b2s_sparse_tile_plan
            n += 1                               # b2s_sparse_conv / b2s_sparse_conv_tc_plan
            if lyr.get("in_split") is not None:
                n += 1                           # b2s_split_f16
        if self.rpn_impl == "tc":
            # one tensor-core kernel per RPN layer (fused tail: 1 for 2); the multi-head crop op is one b2s_crop_nhwc kernel
            n += len(self.tc_plan) - (1 if self.tc_tail_fused else 0)
            n += 1                               # k_bev_clear (b2s_to_bev_tc_ex)
            if self.bg_idx:
                n += len(self.bg_idx) + 2        # k_bg_layer per layer, k_bg_compact, k_strip_bands
        elif getattr(self, "any_sparse_tc", False):
            n += 1                               # b2s_merge_f16
        if self.mc:
            return n + 1 + 1 + 3 * (1 if self.mc_uniform else self.ncls) + 1      # ... + k_concat_classes
        return n + 1 + 1 + 3                     # to_bev, decode_filter(_segments), nms: select_sort + iou_mask + reduce

    def fp16_plane_bytes(self):
        """bytes of the fp16 operand planes this engine holds -- activations, BEV, weights, background fields -- as
        {"hi": ..., "lo": ...}; the f16 mode allocates no lo planes, so an fp32-mode engine's "lo" is what it saves"""
        seen, out = set(), {"hi": 0, "lo": 0}

        def add(t, kind):
            if isinstance(t, torch.Tensor) and t.dtype == torch.float16:
                st = t.untyped_storage()
                key = (st.data_ptr(), t.storage_offset(), tuple(t.shape))
                if key not in seen:
                    seen.add(key)
                    out[kind] += t.numel() * 2
        for lyr in getattr(self, "layers", []):
            for split in (lyr.get("in_split"), (None, lyr.get("out_hi"), lyr.get("out_lo"))):
                if split is not None:
                    add(split[1], "hi")
                    add(split[2], "lo")
            add(lyr.get("w_hi"), "hi")
            add(lyr.get("w_lo"), "lo")
        if self.rpn_impl == "tc":
            for pl in list(self.tc_bufs.values()) + list(getattr(self, "bg_field", [])):
                add(pl[0], "hi")
                add(pl[1], "lo")
            for op in self.tc_plan:
                add(op.get("w_hi"), "hi")
                add(op.get("w_lo"), "lo")
        return out

    def sparse_layer_stats(self):
        """sync; per sparse layer: rows in/out, pairs, algorithmic bytes and flops (SURVEY.md §8d formulas)."""
        out = []
        for lyr in self.layers:
            n_out = int(lyr["out_level"].n_dev[0].item())
            n_in = int(lyr["in_level"].n_dev[0].item())
            pairs = int((lyr["rb"]["nbr"][:n_out] >= 0).sum().item())
            cin, cout, K = lyr["cin"], lyr["cout"], lyr["K"]
            out.append({"index": lyr["index"], "subm": bool(lyr["subm"]), "cin": cin, "cout": cout, "K": K,
                        "n_in": n_in, "n_out": n_out, "pairs": pairs,
                        "useful_mma_frac": pairs / max(1, K * n_out),
                        "bytes": 4 * (n_in * cin + n_out * cout) + 8 * pairs + 4 * K * cin * cout,
                        "flops": 2 * pairs * cin * cout})
        return out

    def rpn_layer_stats(self):
        """per tensor-core RPN layer: algorithmic fp32 flops (2*pixels*taps*cin*cout; the 3xF16 split issues 3x that on
        the tensor pipe) and bytes moved (fp16 hi/lo planes in and out + weights)."""
        if self.rpn_impl != "tc":
            return []
        out = []
        for i, op in enumerate(self.tc_plan):
            cin, cout, taps = op["cin"], op["cout"], op["taps"]
            px = self.B * op["Hg"] * op["Wg"]
            px_in = self.B * op["Hin"] * op["Win"]
            npl = self.n_planes
            out_b = npl * 2 * px * cout if op["planes"] == 2 else 4 * px * cout
            frac = 1.0                        # share of the 8 x BG_ROWS output strips actually computed (the rest: background)
            if getattr(self, "bg_idx", None) and i in self.bg_idx:
                frac = float(self.bg_counts[self.bg_idx.index(i), 0].item()) / self.bg_tiles
            out.append({"index": i, "kind": op["kind"], "v2": op["v2"], "cin": cin, "cout": cout, "taps": taps,
                        "tiles_computed_frac": frac,
                        "pixels": px, "flops": 2 * px * taps * cin * cout,
                        "bytes": npl * 2 * px_in * cin + out_b + npl * 2 * taps * cin * op["n_pad"],
                        "bytes_fp32_algorithmic": 4 * (px_in * cin + px * cout + taps * cin * cout)})
        return out

    # ---------------------------------------------------------------- public API
    def set_anchors(self, anchors):
        """anchors [A, code] or [B', A, code] (the example's ``anchors``; every frame shares one grid)."""
        a = anchors[0] if anchors.dim() == 3 else anchors
        key = (a.data_ptr(), tuple(a.shape), a._version, str(a.device))
        if key == self._anchors_key:
            return
        a = a.reshape(-1, a.shape[-1])
        assert a.shape[0] == self.A and a.shape[1] == self.code, \
            "num_anchors=%d, but num_output=%d. please check size" % (a.shape[0], self.A)
        self.anchors.copy_(a, non_blocking=True)
        self._anchors_key = key
        if self.area_threshold is not None:
            self._set_area_boxes(a)            # one read-back per anchor set; the steady state does not sync

    def set_anchors_mask(self, mask):
        """anchors_mask [B, A] (bool/uint8) or None (voxelnet.py:397-400,432-439).  With ``anchor_area_threshold``
        set, None means the engine computes the mask; a given mask wins, as in the reference's example dict.
        The three cases (no mask, given, computed) launch different sequences and keep separate CUDA graphs."""
        if mask is None:
            self._mask_src = "area" if self.area_threshold is not None else None
            self.use_mask = self._mask_src is not None
            return
        if self.anchors_mask is None:
            self.anchors_mask = torch.zeros(self.B, self.A, dtype=torch.uint8, device=self.dev)
        self._mask_src, self.use_mask = "given", True
        self.anchors_mask.copy_(mask.reshape(self.B, self.A).to(torch.uint8), non_blocking=True)

    def load_points(self, frames, slot=0):
        """frames: list of B CUDA (or pinned/CPU) float32 [P_i, F] tensors -> static input buffers (of input slot
        `slot`; slot 1 is streamed batches' second pair, see stream_load).  The copies go on the current stream."""
        assert len(frames) == self.B
        sizes = [int(f.shape[0]) for f in frames]
        total = sum(sizes)
        assert total <= self.P_cap, "more points (%d) than the engine's capacity (%d)" % (total, self.P_cap)
        points, offsets = self._inputs(slot)
        # frames that lie back to back in memory (views of one pinned slab, or of one device tensor) go over in ONE copy:
        # a serving loop that reads clouds into a pinned ring buffer pays one cudaMemcpyAsync per batch instead of B.
        # The run structure only depends on where the frames lie: a serving loop cycles through a few slabs, so it is
        # remembered per (pointers, sizes, strides) -- finding it anew is ~0.25 ms of Python per call for 32 frames.
        key = (tuple(f.data_ptr() for f in frames), tuple(sizes), tuple(f.stride(0) for f in frames),
               frames[0].dtype, frames[0].device) if frames else None
        cache = getattr(self, "_run_cache", None)
        if cache is None:
            cache = self._run_cache = {}
        runs = cache.get(key)
        if runs is not None:
            # (a remembered multi-frame run must still lie inside ONE storage: same addresses, different allocations)
            for i, off, run_rows, whole in runs:
                if whole and frames[i].untyped_storage().nbytes() < 4 * (frames[i].storage_offset() + run_rows * self.F):
                    runs = None
                    del cache[key]
                    break
        if runs is not None:
            for i, off, run_rows, whole in runs:
                if whole:
                    src = torch.as_strided(frames[i], (run_rows, self.F), (self.F, 1))
                    points[off:off + run_rows].copy_(src, non_blocking=True)
                else:
                    points[off:off + run_rows].copy_(frames[i], non_blocking=True)
            return self._load_offsets(sizes, total, offsets)
        runs = []
        off, i = 0, 0
        while i < len(frames):
            f = frames[i]
            run_rows, j = sizes[i], i + 1
            if f.is_contiguous() and f.dtype == torch.float32:
                end = f.data_ptr() + 4 * f.numel()
                # (same STORAGE, not just adjacent addresses: two separate allocations can end up back to back in the
                # caching allocator, and a strided view must stay inside its own storage)
                base = f.untyped_storage().data_ptr()
                while j < len(frames) and frames[j].dtype == torch.float32 and frames[j].device == f.device and \
                        frames[j].is_contiguous() and frames[j].data_ptr() == end and \
                        frames[j].untyped_storage().data_ptr() == base:
                    end += 4 * frames[j].numel()
                    run_rows += sizes[j]
                    j += 1
            if run_rows:
                if j - i > 1:
                    src = torch.as_strided(f, (run_rows, self.F), (self.F, 1))      # the whole run through frame i's storage
                    points[off:off + run_rows].copy_(src, non_blocking=True)
                else:
                    points[off:off + run_rows].copy_(f, non_blocking=True)
                runs.append((i, off, run_rows, j - i > 1))
            off += run_rows
            i = j
        if len(cache) < 16 and all(f.dtype == torch.float32 for f in frames):
            cache[key] = runs
        return self._load_offsets(sizes, total, offsets)

    def _load_offsets(self, sizes, total, offsets):
        # frame offsets through a pinned staging buffer that is allocated once (a fresh pin_memory() per call is a
        # cudaHostAlloc on the serving path); two slots, so the copy of the previous call is never overwritten in flight
        if getattr(self, "_offs_host", None) is None:
            self._offs_host = [torch.zeros(self.B + 1, dtype=torch.int32).pin_memory() for _ in range(2)]
            self._offs_evt = [torch.cuda.Event(), torch.cuda.Event()]
            self._offs_slot = 0
        slot = self._offs_slot
        self._offs_slot ^= 1
        self._offs_evt[slot].synchronize()                 # (no-op unless two calls ago is still copying)
        self._offs_host[slot].copy_(torch.from_numpy(np.cumsum([0] + sizes).astype(np.int32)))
        offsets.copy_(self._offs_host[slot], non_blocking=True)
        self._offs_evt[slot].record()
        return total

    def load_points_cropped(self, frames, planes):
        """frames: list of B CUDA float32 [P_i, F] raw clouds; planes: one [n,4] float64 array per frame (or one for
        all): the points strictly inside the convex region (``b2second.inputs.frustum_planes``: the KITTI camera-FOV
        crop, box_np_ops.py:682-693) are compacted on the device straight into the static point buffer, in input
        order, and ``offsets`` is filled on the device -- no host sync, no host copy of the cropped cloud."""
        from . import inputs
        assert len(frames) == self.B
        if not isinstance(planes, (list, tuple)):
            planes = [planes] * self.B
        if getattr(self, "_crop", None) is None:
            self._crop = inputs.ConvexCrop(self.P_cap, self.dev)
            self.in_status = torch.zeros(1, dtype=torch.int32, device=self.dev)
        with torch.cuda.device(self.dev):
            self.offsets.zero_()
            self._crop_keep = [self._crop.crop_into(f if f.is_cuda else f.to(self.dev, non_blocking=True), pl,
                                                    self.points, self.offsets, b, self.in_status)
                               for b, (f, pl) in enumerate(zip(frames, planes))]

    def load_sweeps(self, frames):
        """frames: list of B dicts {"sweeps": [CUDA float32 [P_i, F>=3], key frame first], "rotations": [..[3,3]..],
        "translations": [..[3]..], "time_lags": [..]} (the ``sweep2lidar_*`` fields of a NuScenes info record).  The
        merged [x, y, z, dt] cloud of every frame (nuscenes_dataset.py:166-185) is written straight into the static
        point buffer."""
        from . import inputs
        assert len(frames) == self.B and self.F == 4, "sweep merging produces [x, y, z, dt] rows"
        sizes = [sum(int(s.shape[0]) for s in fr["sweeps"]) for fr in frames]
        assert sum(sizes) <= self.P_cap, "more points (%d) than the engine's capacity (%d)" % (sum(sizes), self.P_cap)
        off = 0
        with torch.cuda.device(self.dev):
            for fr, n in zip(frames, sizes):
                sw = [s if s.is_cuda else s.to(self.dev, non_blocking=True) for s in fr["sweeps"]]
                inputs.merge_sweeps(sw, fr["rotations"], fr["translations"], fr["time_lags"], out=self.points[off:off + n])
                off += n
            offs = torch.tensor(np.cumsum([0] + sizes), dtype=torch.int32)
            self.offsets.copy_(offs.pin_memory(), non_blocking=True)
        return off

    def load_voxels(self, voxels, num_points, coordinates):
        """the reference's example tensors (voxels [N,T,F], num_points [N], coordinates [N,4] (b,z,y,x)), on any
        device, -> static buffers.  N is known on the host (a tensor shape): no sync."""
        n = int(voxels.shape[0])
        cap = self.level0.cap
        assert n <= cap, "more voxels (%d) than the engine's capacity (%d)" % (n, cap)
        assert tuple(voxels.shape[1:]) == (self.T, self.F), "voxels must be [N, %d, %d]" % (self.T, self.F)
        if self.in_voxels is None:
            self.in_voxels = torch.zeros(cap, self.T, self.F, dtype=torch.float32, device=self.dev)
            # PFN reads points through per-voxel slot indices: voxel v, slot t -> row v*T + t of in_voxels
            self.in_slots = torch.arange(cap * self.T, dtype=torch.int32, device=self.dev).view(cap, self.T)
            self._nvox_host = torch.zeros(1 + self.B, dtype=torch.int32).pin_memory()
        self.in_voxels[:n].copy_(voxels, non_blocking=True)
        self.vox_num[:n].copy_(num_points.to(torch.int32) if num_points.dtype != torch.int32 else num_points,
                               non_blocking=True)
        self.vox_coors[:n].copy_(coordinates.to(torch.int32) if coordinates.dtype != torch.int32 else coordinates,
                                 non_blocking=True)
        self._nvox_host[0] = n
        self.num_voxels.copy_(self._nvox_host, non_blocking=True)
        return n

    def run(self, mode="points", slot=0):
        """launch the pipeline on the data currently in the static buffers (of input slot `slot`) (async)."""
        # the grid sizes of the per-point kernels are fixed at capacity so one graph serves any frame mix
        with torch.cuda.device(self.dev):
            if not self.use_graph:
                with torch.no_grad():
                    self._launch(mode, slot)
                return self.det, self.det_count
            # a slot's graph reads that slot's input buffers; every other buffer is shared by the slots' graphs, which
            # replay in order on one stream
            key = (mode, self._mask_src) if slot == 0 else (mode, self._mask_src, slot)
            g = self._graphs.get(key)
            if g is None:
                with torch.no_grad():
                    side = torch.cuda.Stream()
                    side.wait_stream(torch.cuda.current_stream())
                    with torch.cuda.stream(side):
                        for _ in range(3):          # warm-up: cuDNN autotune, lazy module init, func attributes
                            self._launch(mode, slot)
                    torch.cuda.current_stream().wait_stream(side)
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with no_cyclic_gc(), torch.cuda.graph(g):
                        self._launch(mode, slot)
                    self._graphs[key] = g
            g.replay()
        return self.det, self.det_count

    def infer(self, frames):
        self.load_points(frames)
        return self.run("points")

    def infer_voxels(self, voxels, num_points, coordinates):
        self.load_voxels(voxels, num_points, coordinates)
        return self.run("voxels")

    # ---------------------------------------------------------------- streamed batches (FastPath.stream)
    # Two input slots: while the graph of one slot's batch runs on the compute stream (the current stream), the next
    # batch's clouds go over the copy stream into the other slot.  Per slot k: the copy stream waits on free[k]
    # (recorded after the last replay that read slot k) before writing the slot and records ready[k]; the compute
    # stream waits on ready[k] before replaying slot k's graph; done[k] follows slot k's read-back into its own pinned
    # buffers.  Every buffer after the inputs is shared: the graphs replay in order on the compute stream.
    _streamed = None

    def _inputs(self, slot):
        """(points, offsets) of input slot `slot`: slot 0 is the pair every entry point loads, slot 1 the second pair
        streamed batches alternate with"""
        if slot == 0:
            return self.points, self.offsets
        return self._streamed.points, self._streamed.offsets

    def _stream_state(self):
        s = self._streamed
        if s is None:
            with torch.cuda.device(self.dev):
                s = self._streamed = _Streamed(self)
        return s

    def stream_load(self, frames):
        """enqueue frames (a list of B float32 [P_i, F] clouds: pinned, pageable or CUDA) on the engine's copy stream
        into the input slot the previous streamed batch did not use; returns that slot.  Raises before any copy is
        enqueued when the batch exceeds the point capacity.  The copies overlap the current (compute) stream's work
        only from pinned memory; device clouds are copied once the compute stream has reached this call (they may
        still be being written there)."""
        s = self._stream_state()
        slot = s.next_slot
        compute = torch.cuda.current_stream(self.dev)
        with torch.cuda.device(self.dev), torch.cuda.stream(s.copy):
            s.copy.wait_event(s.free[slot])
            if any(f.is_cuda for f in frames):
                s.copy.wait_stream(compute)
            self.load_points(frames, slot)
            s.ready[slot].record(s.copy)
        s.next_slot ^= 1
        return slot

    def stream_run(self, slot, mode="points"):
        """replay slot `slot`'s graph on the current stream once stream_load's copies have landed"""
        s = self._streamed
        compute = torch.cuda.current_stream(self.dev)
        compute.wait_event(s.ready[slot])
        self.run(mode, slot)
        s.free[slot].record(compute)

    def stream_read_back(self, slot, output):
        """enqueue on the current stream the read-back of the batch just run from slot `slot` into the slot's pinned
        buffers (and, for output="device", the snapshot clone); returns what stream_results needs besides the slot"""
        s = self._streamed
        with torch.cuda.device(self.dev):
            snap = self._read_back(s.rec_host[slot], s.status_host[slot], output)
            s.done[slot].record(torch.cuda.current_stream(self.dev))
        return snap

    def stream_results(self, slot, snap, metadata, output):
        """wait for slot `slot`'s read-back and build its list of dicts, as detections() does"""
        s = self._streamed
        s.done[slot].synchronize()
        return self._results(s.rec_host[slot], s.status_host[slot], snap, metadata, output)

    def stream_wait(self):
        """wait for every streamed copy and read-back enqueued so far"""
        s = self._streamed
        if s is not None:
            s.copy.synchronize()
            for ev in s.done:
                ev.synchronize()

    def check_status(self):
        """sync + raise on data-dependent overflow (call when results are read back)."""
        st = int(self.status.item())
        if getattr(self, "in_status", None) is not None:
            if int(self.in_status.item()):
                raise RuntimeError("b2second engine: cropped clouds exceed the point buffer (max_points)")
        self._raise_on_status(st)
        return st

    def _raise_on_status(self, word):
        """raise on a status word with a bit other than voxel overflow (bit 1: the reference's own drop-extra-voxels
        behaviour)"""
        if word & ~1:
            raise RuntimeError("b2second engine: " + self._L.status_message(word))

    def detections(self, metadata=None, output="host"):
        """sync and convert to the reference's list-of-dicts (voxelnet.py:616-645).

        output="host": ONE pinned D2H copy of the detection records (counts ride in the records' last element) +
        one stream sync, sliced on the host into CPU tensors.  output="device": the tensors stay on the GPU like the
        reference's (one snapshot clone, per-frame views)."""
        if getattr(self, "_rec_host", None) is None:
            self._rec_host = torch.empty(self.B, self.rec_width, dtype=torch.float32).pin_memory()
            self._status_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        with torch.cuda.device(self.dev):
            snap = self._read_back(self._rec_host, self._status_host, output)
            torch.cuda.current_stream().synchronize()          # the one sync of the step
        return self._results(self._rec_host, self._status_host, snap, metadata, output)

    def _read_back(self, rec_host, status_host, output):
        """enqueue on the current stream the D2H of the detection records and the status word into the given pinned
        buffers, and for output="device" the snapshot clone; returns (snapshot, labels) or None"""
        rec_host.copy_(self.det_record, non_blocking=True)
        status_host.copy_(self.status, non_blocking=True)
        if output == "device":
            snap = self.det.clone()
            return snap, snap[..., self.code + 1].long()
        return None

    def _results(self, rec_host, status_host, snap, metadata, output):
        """the list of dicts from a read-back that has landed; raises on a status bit other than voxel overflow"""
        code, B = self.code, self.B
        meta = metadata if metadata is not None and len(metadata) > 0 else [None] * B
        self._raise_on_status(int(status_host[0]))
        cnt = rec_host[:, -1].round().to(torch.int64).tolist()
        out = []
        if output == "device":
            snap, labels = snap
            for b in range(B):
                n = cnt[b]
                out.append({"box3d_lidar": snap[b, :n, :code], "scores": snap[b, :n, code],
                            "label_preds": labels[b, :n], "metadata": meta[b]})
            return out
        # per-frame views through numpy: 3 B tensor views cost ~0.1 ms this way and ~0.8 ms as torch indexing ops (the
        # Python between two steps is GPU idle time on the serving path)
        host = rec_host.numpy()[:, :-1].reshape(B, self.post_max, code + 2).copy()
        labels = host[..., code + 1].astype(np.int64)
        fn = torch.from_numpy
        for b in range(B):
            n = cnt[b]
            out.append({"box3d_lidar": fn(host[b, :n, :code]), "scores": fn(host[b, :n, code]),
                        "label_preds": fn(labels[b, :n]), "metadata": meta[b]})
        return out
