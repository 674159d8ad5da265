"""The fused engine behind the reference's own call: ``net(example)``.

``accelerate(net)`` takes ANY VoxelNet-like module -- the object the reference's
``second.pytorch.builder.second_builder.build`` returns (running on this repository's ``spconv`` package), or the
mirror ``b2second.models.VoxelNet`` -- reads it through ``b2second.spec`` and re-binds ``net.forward`` so that an
eval-mode call

    preds = net(example)          # second/pytorch/models/voxelnet.py:339-375 contract: dict in, list of dicts out

runs as one CUDA graph per frame batch (``b2second.engine.InferenceEngine``).  Accepted examples:

* the reference's own dict (``voxels [N,T,F]``, ``num_points [N]``, ``coordinates [N,4] (b,z,y,x)``, ``anchors
  [B,A,7]``, optional ``anchors_mask``, ``metadata``) -- tensors on any device; the voxels are copied into the
  engine's static buffers and everything after the voxelizer is fused;
* the same dict with ``points`` (a list of B float32 ``[P_i, F]`` tensors: CUDA, pinned or plain host memory)
  instead of the three voxel keys -- then the voxelizer runs on the GPU as well (SURVEY.md §8b "a fast path may
  additionally accept example['points']"); with ``crop_planes`` (``b2second.inputs.frustum_planes``) the raw clouds
  are first cropped to the camera field of view on the GPU (the ``velodyne_reduced`` step, box_np_ops.py:682-693);
* ``sweeps``: per frame the NuScenes key-frame cloud + its sweeps with their ``sweep2lidar`` calibration, merged on
  the GPU (nuscenes_dataset.py:166-185) -- see ``InferenceEngine.load_sweeps``.

``accelerate(net, anchor_area_threshold=t)`` (an engine keyword, like every other one ``FastPath`` forwards) makes the
engine compute the reference preprocessing's ``anchors_mask`` (preprocess.py:345-357) on the GPU for any of these
inputs that carries no ``anchors_mask`` of its own; the default (None) computes none.

The list of result dicts holds GPU tensors like the reference's (``output="device"``); ``accelerate(net,
output="host")`` returns CPU tensors through ONE pinned device-to-host copy of the detection records instead of one
small copy per frame and field.

``net.b2s_fastpath.stream(examples)`` (``FastPath.stream``) serves an iterable of ``points`` examples: it yields what
``net(example)`` would return for each, while the next batch's clouds go over to the GPU during the current batch's
graph (two input slots per engine, ``InferenceEngine.stream_load``).

The engine holds copies of the weights in its own layouts (folded BatchNorm, packed fp16 planes, background fields).
``eval()`` / ``train(False)`` and ``load_state_dict`` on the accelerated network mark them stale, and the next call
re-derives them from the network's current parameters and buffers (``FastPath.refresh``), so a training loop can
evaluate on the engine between steps and a restored checkpoint is served as loaded.

Anything the engine does not cover (training mode, the DataParallel padded layout, a layer pattern
``spec_from_module`` rejects) falls through to the module's original ``forward`` -- which still computes on the CUDA
``spconv`` drop-in; there is no CPU path anywhere.
"""
import collections
import types

import torch

from . import spec as _spec


class FastPath:
    def __init__(self, net, max_points=40000, max_voxels=None, use_cuda_graph=True, output="device", **engine_kw):
        self.net = net
        assert output in ("device", "host")
        self.output = output         # "device": tensors stay on the GPU like the reference's; "host": CPU tensors
                                     # through one pinned D2H of the whole detection record buffer
        self.post_run = None         # optional hook(engine) between the launch and the read-back (e.g. the
                                     # multi-GPU all-gather of engine.det_record, b2second/dist.py)
        self.max_points = int(max_points)
        self.use_cuda_graph = use_cuda_graph
        self.engine_kw = engine_kw
        from .engine import check_precision         # an unknown or refused precision raises here, not at the first call
        check_precision(engine_kw.get("precision", "fp32"), engine_kw.get("sparse_impl", "tc"),
                        engine_kw.get("rpn_impl", "auto"))
        self.spec = _spec.spec_from_module(net, max_voxels)      # raises UnsupportedNetwork for foreign layer patterns
        self.engines = {}
        self.stale = False           # the network's weights may have changed since the engines' operands were derived
        self.refreshes = 0           # refresh() calls that completed

    def mark_stale(self):
        """note that the network's weights may have changed: the next call, streamed batch or engine build refreshes
        first (accelerate marks on every train(False) / eval() and after load_state_dict)"""
        self.stale = True

    def refresh(self):
        """re-derive every engine operand from the network's current parameters and buffers: the folded BatchNorm, the
        packed weight planes of the sparse layers, the PFN and every RPN op, and the background fields the RPN's
        empty strips are filled from.  Each operand then equals, bit for bit, what a newly built engine would hold.
        Every engine built so far is refreshed in place (same addresses: captured graphs stay valid, unless a
        background margin changed, when they are re-captured on their next run); engines built later read the refreshed
        spec.  The work is enqueued on the current stream after everything already enqueued there, so batches in
        flight finish with the weights they were enqueued with.  Idempotent.

        Raises ``b2second.spec.UnsupportedNetwork`` when the network's structure (layer list, shapes, head layout)
        changed since ``accelerate`` or a parameter moved to another device; the fast path then stays stale, so every
        later call raises too, rather than serving a different network.  Non-weight attributes (NMS thresholds, the
        anchor configuration, the voxel generator) are read once, at ``accelerate``, and not re-read here."""
        with torch.no_grad():
            _spec.refresh(self.spec, self.net)
            for eng in self.engines.values():
                eng.refresh()
        self.stale = False
        self.refreshes += 1

    def engine(self, batch_size):
        if self.stale:
            self.refresh()
        eng = self.engines.get(batch_size)
        if eng is None:
            from .engine import InferenceEngine
            eng = InferenceEngine(self.spec, batch_size=batch_size, max_points=self.max_points,
                                  use_cuda_graph=self.use_cuda_graph, **self.engine_kw)
            self.engines[batch_size] = eng
        return eng

    def applicable(self, example):
        if self.net.training:
            return False
        if "points" in example or "sweeps" in example:
            return True
        if not all(k in example for k in ("voxels", "num_points", "coordinates")):
            return False
        return example["num_points"].dim() == 1          # 2-D = DataParallel padded layout (voxelnet.py:345-357)

    def __call__(self, example):
        if "points" in example or "sweeps" in example:
            frames = example["points"] if "points" in example else example["sweeps"]
            B = len(frames)
        else:
            B = int(example["anchors"].shape[0])
        eng = self.engine(B)
        self._set_anchors(eng, example)
        if "sweeps" in example:
            eng.load_sweeps(list(frames))             # NuScenes: key frame + sweeps merged on the GPU
            eng.run("points")
        elif "points" in example and example.get("crop_planes") is not None:
            eng.load_points_cropped(list(frames), example["crop_planes"])    # KITTI: camera-FOV crop on the GPU
            eng.run("points")
        elif "points" in example:
            eng.infer(list(frames))
        else:
            eng.infer_voxels(example["voxels"], example["num_points"], example["coordinates"])
        if self.post_run is not None:
            self.post_run(eng)
        return eng.detections(metadata=example.get("metadata"), output=self.output)

    @staticmethod
    def _set_anchors(eng, example):
        if "anchors" in example and example["anchors"] is not None:
            anchors = example["anchors"]
            eng.set_anchors(anchors.reshape(anchors.shape[0], -1, anchors.shape[-1]))   # asserts the anchor count
        elif eng._anchors_key is None:
            raise KeyError("example has no 'anchors' and the network cannot generate them")
        eng.set_anchors_mask(example.get("anchors_mask"))

    def _stream_frames(self, example):
        """the clouds of a streamed example; raises for what stream() does not take"""
        if self.net.training:
            raise RuntimeError("stream() runs the fused engine, which serves eval() networks only")
        carried = [k for k in ("voxels", "sweeps", "crop_planes") if example.get(k) is not None]
        if carried or "points" not in example:
            raise ValueError("stream() takes examples of raw clouds under 'points' (without %s); other examples go "
                             "through net(example)" % "/".join(carried or ["voxels", "sweeps", "crop_planes"]))
        return list(example["points"])

    def stream(self, examples):
        """yield, in input order, what ``net(example)`` returns for each example of the iterable ``examples``, with the
        host-to-device copies of each batch overlapping the previous batch's graph.

        An example is a ``points`` dict as ``net(example)`` takes it: B float32 ``[P_i, F]`` clouds (pinned, pageable
        or CUDA), ``anchors`` unless the network generates them, optional ``anchors_mask`` and ``metadata``.  The
        batch size may change from example to example.  Only pinned clouds are copied while the previous batch
        computes; pageable and CUDA clouds give the same results with less overlap.  ``voxels``, ``sweeps`` and
        ``crop_planes`` examples raise ValueError (they go through ``net(example)``); a network in ``train()`` mode
        raises RuntimeError.  Neither enqueues anything.

        At most two batches are in flight: example k+1 is taken from the iterable and enqueued before the result of
        example k is built and yielded, so the host builds that result while batch k+1 computes.  The caller may
        reuse or overwrite an example's memory once that example's result has been yielded, and not before.

        Errors are raised at the failing batch's turn, after every earlier result has been yielded: a status error
        (anything but voxel overflow) raises the RuntimeError ``detections()`` raises; a batch over the point
        capacity raises load_points' AssertionError before its copy is enqueued; a refused example raises as above.
        Closing the generator early (``break``, ``close()``, an exception in the caller) waits for the work in flight;
        the engines are then ready for ``net(example)`` or a new stream.  ``post_run`` is called once per batch, on
        the stream that runs the graphs, after the batch's graph and before its read-back."""
        # (engine, slot, snapshot, example) of the batches in flight, in input order: holding the example keeps its
        # clouds alive until their copies are known to be done
        pending = collections.deque()
        compute = None
        try:
            for example in examples:
                try:
                    frames = self._stream_frames(example)
                    if self.stale and compute is not None:
                        with torch.cuda.stream(compute):       # after the replays of the batches in flight
                            self.refresh()
                    eng = self.engine(len(frames))
                    if compute is None:     # every engine's graphs replay on this one stream, so batches stay in order
                        compute = torch.cuda.current_stream(eng.dev)
                    with torch.no_grad(), torch.cuda.stream(compute):
                        slot = eng.stream_load(frames)
                        self._set_anchors(eng, example)
                        eng.stream_run(slot)
                        if self.post_run is not None:
                            self.post_run(eng)
                        snap = eng.stream_read_back(slot, self.output)
                except Exception:
                    while pending:
                        yield self._stream_result(pending.popleft())
                    raise
                pending.append((eng, slot, snap, example))
                if len(pending) == 2:
                    yield self._stream_result(pending.popleft())
            while pending:
                yield self._stream_result(pending.popleft())
        finally:
            pending.clear()
            for eng in self.engines.values():
                eng.stream_wait()

    def _stream_result(self, item):
        eng, slot, snap, example = item
        return eng.stream_results(slot, snap, example.get("metadata"), self.output)


def accelerate(net, **kw):
    """re-bind ``net.forward`` to the fused engine (see module docstring); returns ``net``.  The keywords go to
    ``FastPath`` and the engines it builds; ``precision="f16"`` selects the half-precision mode (one fp16 plane per
    tensor-pipe operand, b2second.engine) and is checked here: an unknown precision, or "f16" with sparse_impl="fma" or
    rpn_impl="cudnn", raises ValueError.
    ``net.b2s_fastpath`` is the FastPath object, ``net.b2s_reference_forward`` the original bound method.

    ``net.train`` is wrapped as well: ``train(False)`` / ``eval()`` set the modes exactly as before and then mark the
    fast path stale, and so does a ``load_state_dict`` on ``net`` (a post-hook).  A stale fast path refreshes
    (``FastPath.refresh``) at its next call, streamed batch or engine build; a call that is not stale does no refresh
    work.  So a training loop can evaluate on the engine between steps, and a restored checkpoint is served as
    loaded."""
    if getattr(net, "b2s_fastpath", None) is not None:
        return net
    fast = FastPath(net, **kw)
    original = net.forward
    original_train = net.train

    def train(self, mode=True):
        out = original_train(mode)
        if not mode:
            fast.mark_stale()
        return out

    def forward(self, example):
        if fast.applicable(example):
            with torch.no_grad():
                return fast(example)
        return original(example)

    net.b2s_fastpath = fast
    net.b2s_reference_forward = original
    net.forward = types.MethodType(forward, net)
    net.train = types.MethodType(train, net)
    net.register_load_state_dict_post_hook(lambda module, incompatible_keys: fast.mark_stale())
    return net
