"""data-parallel training step times (CUDA events) at 1, 2, 4 and 8 GPUs:
python -m torch.distributed.run --nproc-per-node N tools/dp_train_times.py [steps] [frames_per_rank] [--draws device]

One process per GPU, NCCL.  For every world size W in (1, 2, 4, 8) up to N, ranks 0 .. W-1 form a group and train
car.fhd and pointpillars xyres_16, in the fp32 and f16 training modes, with b2second.training.enable_data_parallel: the
whole GPU step on seeded synthetic frames, dbsample -> augment -> voxelize -> anchor-area mask -> targets -> forward /
backward -> optimizer step (with the gradient all-reduce) -> metrics (with the count all-reduce).  The host draws
(dbsample.draw, augment.draw) are made for the global batch of W * B frames in single-process order and each rank keeps
its frames' draws (dbsample.select, augment.select), so the data does not depend on W; the frames' box and point
counts the augmentation draws need are all-gathered (one small collective next to the pipeline's one host read).
With --draws device every configuration is also measured, right after the numpy path, with the augmentation's draws
made on the device (augment.DeviceDrawer): each rank draws only its own frames, with frame_base = rank * B, and reads
only its own counts, so that path has no all-gather.  The database sampler draws from its own numpy state in both
paths, so both see the same frames.

Rank 0 prints one JSON line: per configuration, mode and W the step time (ms, CUDA events over the timed steps, after
warm-up ones), frames/s over the global batch, the scaling efficiency (frames/s over W times the one-GPU frames/s), and
the gradient all-reduce's share of the step (CUDA events around it); with rank 0's card, its power limit and its SM
clock sampled during the run."""
import argparse
import contextlib
import os
import sys
import tempfile

import _measure
import numpy as np
import torch
import torch.distributed as dist

import db_sample_times as dbt
import optim_ref as orf
from b2second import augment, config, dbsample, inputs, loader, loss, metrics, models, optim, targets, training

CONFIGS = ("car.fhd", "pointpillars.car.xyres_16")
MODES = ("fp32", "f16")
WORLDS = (1, 2, 4, 8)
POINTS = 20000


def build(name, precision, dev):
    net = models.build_network(config.get_config(name), loader.product_spconv())
    models.synthetic_weights_(net, name, seed=0)
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(dev), precision=precision))
    net = training.enable_rpn_training(net, precision=precision)
    net = training.enable_bn_relu_training(training.enable_pfn_training(net))
    return metrics.enable_gpu_metrics(net).train()


class Pipeline:
    """the input side of one rank: the global batch's frames and ground truths (host), the object database"""

    def __init__(self, name, net, root, world, rank, B, dev, group, draws):
        self.cfg = cfg = config.get_config(name)
        self.net, self.world, self.rank, self.B, self.dev, self.group = net, world, rank, B, dev, group
        rng = np.random.default_rng(0)
        infos = dbt.database(cfg, root, rng)
        self.classes = [c.class_name for c in cfg.classes]
        self.ds = dbsample.sampler(cfg.db_sampler, infos, root, cfg.num_point_features, self.classes, dev,
                                   np.random.RandomState(0))
        self.ap = augment.plan(cfg.augment, cfg.point_cloud_range, self.classes)
        self.tp = targets.plan(net.target_assigner, cfg.feature_map_size)
        self.gen = loader.product_spconv().utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range,
                                                                 cfg.max_points_per_voxel, cfg.max_voxels)
        r = np.asarray(cfg.point_cloud_range)
        self.frames = []                                   # the whole global batch, as every rank sees it
        for g in range(world * B):
            fr = np.random.default_rng(100 + g)
            b = np.zeros((10, 7), np.float32)
            b[:, :2] = fr.uniform(r[:2] + 2, r[3:5] - 2, (10, 2))
            b[:, 2] = -1.5
            b[:, 3:6] = [1.6, 3.9, 1.5]
            b[:, 6] = fr.uniform(-np.pi, np.pi, 10)
            pts = np.concatenate([fr.uniform(r[:3], r[3:], (POINTS, 3)),
                                  fr.random((POINTS, cfg.num_point_features - 3))], 1).astype(np.float32)
            self.frames.append((pts, b, np.array([self.classes[0]] * 10)))
        lo, hi = rank * B, (rank + 1) * B
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        mine = self.frames[lo:hi]
        self.inputs = (t(np.concatenate([f[0] for f in mine])),
                       t(np.cumsum([0] + [len(f[0]) for f in mine]).astype(np.int32)),
                       t(np.concatenate([f[1] for f in mine])),
                       t(np.arange(0, 10 * B + 1, 10, dtype=np.int32)), t(np.ones(10 * B, bool)),
                       t(np.ones(10 * B, np.int32)), None)
        # one state per sampler, so both draw paths sample the same database objects and counts every step
        self.db_rs, self.aug_rs = np.random.RandomState(1), np.random.RandomState(2)
        self.anchors = torch.from_numpy(net.anchors().reshape(-1, 7)).to(dev)[None].repeat(B, 1, 1)
        self.counts = torch.zeros(world, 2 * B, dtype=torch.int64, device=dev)
        self.drawer = augment.DeviceDrawer(1, dev) if draws == "device" else None

    def example(self):
        cfg, B, lo = self.cfg, self.B, self.rank * self.B
        cand = dbsample.draw(self.db_rs, self.ds.state, [f[2] for f in self.frames])
        s = self.ds.sample_batch(*self.inputs, dbsample.select(cand, lo, lo + B))
        if self.drawer is not None:
            nb, npts = s.counts()                          # the pipeline's host read, this rank's frames only
            d = self.drawer.draw(cfg.augment, s["gt_offsets"], s["point_offsets"], sum(nb), sum(npts), frame_base=lo)
            return self.finish(s, self.ap.augment_batch(*s.augment_inputs(nb, npts), d))
        mine = torch.cat([torch.diff(s["gt_offsets"]), torch.diff(s["point_offsets"])]).to(torch.int64)
        if self.world > 1:
            dist.all_gather_into_tensor(self.counts, mine, group=self.group)
        else:
            self.counts[0].copy_(mine)
        c = self.counts.cpu().numpy()                      # the pipeline's host read
        nb, npts = c[:, :B].reshape(-1).tolist(), c[:, B:].reshape(-1).tolist()
        d = augment.select(augment.draw(self.aug_rs, cfg.augment, nb, npts), lo, lo + B)
        return self.finish(s, self.ap.augment_batch(*s.augment_inputs(nb[lo:lo + B], npts[lo:lo + B]), d))

    def finish(self, s, a):
        cfg, B = self.cfg, self.B
        res = self.gen.generate_device(a["points"], cfg.max_voxels, frame_offsets=s["point_offsets"], batch=B)
        n = int(res["num_voxels"][0].item())
        ex = {"voxels": res["voxels"][:n], "num_points": res["num_points_per_voxel"][:n],
              "coordinates": res["coordinates"][:n], "anchors": self.anchors}
        mask = None
        if cfg.anchor_area_threshold >= 0:
            mask = inputs.anchor_area_mask(ex["coordinates"], B, self.tp.anchors, cfg.voxel_size,
                                           cfg.point_cloud_range, cfg.grid_size, cfg.anchor_area_threshold)
        ex.update(self.tp.assign_batch(a["boxes"], a["gt_offsets"], a["classes"], a["importance"], mask))
        return ex, mask


def step(p, opt):
    net = p.net
    ex, mask = p.example()
    ret = net(dict(ex))
    ret["loss"].backward()
    opt.step()
    net.b2s_metrics.update_metrics_async(ret["cls_loss_reduced"], ret["loc_loss_reduced"], ret["cls_preds"],
                                         ex["labels"], ret["cared"], ret, mask)


def measure(name, precision, world, rank, B, steps, warmup, group, dev, root, draws):
    net = build(name, precision, dev)
    dp = training.enable_data_parallel(net, group)
    opt = optim.plan(net, orf.ONE_CYCLE, warmup + steps + 1, data_parallel=dp)
    p = Pipeline(name, net, root, world, rank, B, dev, group, draws)
    for _ in range(warmup):
        step(p, opt)
    torch.cuda.synchronize()
    dist.barrier(group=group)
    dp.timing = []                                          # CUDA event pairs around each gradient all-reduce
    ms = _measure.timed(lambda: step(p, opt), steps, warmup=0)
    ar = sum(a.elapsed_time(b) for a, b in dp.timing) / steps
    del net, opt, p, dp
    torch.cuda.empty_cache()
    return ms, ar


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("steps", type=int, nargs="?", default=10)
    ap.add_argument("frames_per_rank", type=int, nargs="?", default=2)
    ap.add_argument("--draws", choices=("numpy", "device"), default="numpy",
                    help="device: also measure every configuration with augment.DeviceDrawer, after the numpy path")
    args = ap.parse_args(sys.argv[1:])
    steps, B = args.steps, args.frames_per_rank
    sources = ("numpy", "device") if args.draws == "device" else ("numpy",)
    warmup = 3
    local = int(os.environ.get("LOCAL_RANK", "0"))
    _measure.require_gpu("dp_train_times")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rank, size = dist.get_rank(), dist.get_world_size()
    torch.backends.cudnn.benchmark = False
    worlds = [w for w in WORLDS if w <= size]
    groups = {w: dist.new_group(list(range(w))) for w in worlds}    # every rank creates every group, in one order
    rows = []
    # one clock sampler, on rank 0's device, whose summary goes into the report
    sampling = _measure.clocks() if rank == 0 else contextlib.nullcontext({})
    with tempfile.TemporaryDirectory() as root, sampling as clk:
        for name in CONFIGS:
            for precision in MODES:
                base = {}
                for w in worlds:
                    for src in sources:
                        if rank < w:
                            ms, ar = measure(name, precision, w, rank, B, steps, warmup, groups[w], dev, root, src)
                            fps = w * B * 1e3 / ms
                            if w == 1:                     # only rank 0 reads base: ranks > 0 never run W = 1
                                base[src] = fps
                            if rank == 0:
                                rows.append({"config": name, "precision": precision, "draws": src, "gpus": w,
                                             "frames_per_rank": B, "step_ms": round(ms, 3),
                                             "frames_per_s": round(fps, 2),
                                             "scaling_efficiency": round(fps / (w * base[src]), 3),
                                             "allreduce_ms": round(ar, 3), "allreduce_share": round(ar / ms, 4)})
                        dist.barrier()
    if rank == 0:
        _measure.report("dp_train_times", rows, clk, steps=steps, warmup=warmup, processes=size)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
