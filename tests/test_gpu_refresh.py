"""FastPath.refresh on the H100: after load_state_dict, after training steps and after a train-mode forward that only
moves BatchNorm's running statistics, net(example) on the fused engine returns, bit for bit, what a newly built engine
returns for a network loaded with the same state, and every weight-derived operand and margin of the refreshed engines
equals the new engine's, at the addresses it had before the refresh.

Seeded mirror networks of all six configs at B = 2 and 3 (two engines built before the load), with CUDA graphs on and
off; car.fhd also with sparse_impl="fma" and rpn_impl="cudnn".  Training runs car.fhd and pointpillars.car.xyres_16 on
the drop-in with the training opt-ins and optim.plan.  stream() after a refresh and with a refresh requested while it
runs; a no-op refresh keeps the captured graphs, a refresh that moves a background margin re-captures them."""
import numpy as np
import pytest
import torch

import golden_util as gu
import optim_ref as orf
import train_ref as tr
from b2second import config, fastpath, models

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAMES = ["car.fhd", "car.lite", "all.fhd", "pointpillars.car.xyres_16", "nuscenes.all.pp.largea",
         "nuscenes.all.pp.mhead"]
SIZES = (2, 3)
POINTS = 9000
FIELDS = ("box3d_lidar", "scores", "label_preds")


@pytest.fixture(autouse=True)
def _fp32_convs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.cuda.empty_cache()


def _plain(product, name, seed=0):
    net = models.build_network(config.get_config(name), product).eval()
    return models.synthetic_weights_(net, name, seed=seed).to(DEV)


def _accelerated(net, **kw):
    # a candidate list that holds every anchor: no weights, seeded or trained, can overflow it
    anchors = int(np.prod(net.anchors().shape[:-1]))
    return fastpath.accelerate(net, max_points=POINTS + 1000, cand_cap=anchors, **kw)


def _fresh(product, name, state, **kw):
    """a newly built network loaded with `state` (the keys it has), accelerated"""
    net = _plain(product, name)
    own = net.state_dict()
    net.load_state_dict({k: state[k] for k in own}, strict=True)
    return _accelerated(net, **kw)


def _example(net, name, B, seed):
    clouds = [torch.from_numpy(gu.make_cloud(name, seed + i, POINTS - 700 * i)).to(DEV) for i in range(B)]
    return {"points": clouds, "anchors": torch.from_numpy(net.anchors()[None]).to(DEV)}


def _bits(t):
    t = t.detach().contiguous()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _assert_same(got, want, what):
    assert len(got) == len(want), what
    for b, (g, w) in enumerate(zip(got, want)):
        for k in FIELDS:
            assert g[k].shape == w[k].shape and torch.equal(_bits(g[k]), _bits(w[k])), "%s: frame %d %s" % (what, b, k)


def _operands(eng):
    """name -> every weight-derived device operand of an engine"""
    out = {}
    if eng.is_pillars:
        out.update({k: getattr(eng, k) for k in ("pfn_w", "pfn_scale", "pfn_shift")})
    for lyr in eng.layers:
        for k in ("w", "scale", "shift", "w_hi", "w_lo", "scale_tc"):
            if lyr.get(k) is not None:
                out["layer%d.%s" % (lyr["index"], k)] = lyr[k]
    if eng.rpn_impl == "tc":
        for i, op in enumerate(eng.tc_plan):
            for k in ("w_hi", "w_lo", "scale", "shift"):
                if op.get(k) is not None:
                    out["op%d.%s" % (i, k)] = op[k]
        if eng.bg_idx:
            for j, (hi, lo) in enumerate(eng.bg_field):
                out["bg_field%d.hi" % j], out["bg_field%d.lo" % j] = hi, lo
            out["tail_field"] = eng.tail_field
    return out


def _host_args(eng):
    if eng.rpn_impl != "tc":
        return {}
    return {"w_scale": [op.get("w_scale") for op in eng.tc_plan], "bg_margin": getattr(eng, "bg_margin", None),
            "tail_margin": getattr(eng, "tail_margin", None)}


def _assert_operands(eng, fresh, ptrs=None):
    got, want = _operands(eng), _operands(fresh)
    assert got.keys() == want.keys()
    for k in got:
        assert torch.equal(_bits(got[k]), _bits(want[k])), "operand %s" % k
    assert _host_args(eng) == _host_args(fresh)
    if ptrs is not None:
        assert {k: t.data_ptr() for k, t in got.items()} == ptrs, "an operand moved"


def _ptrs(eng):
    return {k: t.data_ptr() for k, t in _operands(eng).items()}


# ---- 1. checkpoint load ----------------------------------------------------------------------------------------------
def _check_load(product, name, **kw):
    net = _accelerated(_plain(product, name, seed=0), **kw)
    fast = net.b2s_fastpath
    examples = {B: _example(net, name, B, 10 * B) for B in SIZES}
    for B in SIZES:
        net(examples[B])                                            # builds both engines
    ptrs = {B: _ptrs(fast.engine(B)) for B in SIZES}
    before = {k: _bits(t).clone() for k, t in _operands(fast.engine(SIZES[0])).items()}
    state = _plain(product, name, seed=1).state_dict()
    net.load_state_dict(state)
    assert fast.stale
    got = {B: net(examples[B]) for B in SIZES}
    assert not fast.stale and fast.refreshes == 1
    fresh = _fresh(product, name, state, **kw)
    for B in SIZES:
        _assert_same(got[B], fresh(examples[B]), "%s B=%d after load_state_dict" % (name, B))
        _assert_operands(fast.engine(B), fresh.b2s_fastpath.engine(B), ptrs[B])
    assert fast.refreshes == 1
    after = _operands(fast.engine(SIZES[0]))
    assert sum(not torch.equal(before[k], _bits(after[k])) for k in after) > len(after) // 2, \
        "the seed-1 weights must change most operands for this test to mean anything"


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "eager"])
@pytest.mark.parametrize("name", NAMES)
def test_load_state_dict_serves_the_loaded_weights(product, name, graphs):
    _check_load(product, name, use_cuda_graph=graphs)


@pytest.mark.parametrize("impl", [{"sparse_impl": "fma"}, {"rpn_impl": "cudnn"}], ids=["fma", "cudnn"])
def test_load_state_dict_on_the_other_implementations(product, impl):
    _check_load(product, "car.fhd", **impl)


# ---- 2. train -> eval -> train ---------------------------------------------------------------------------------------
def _trainable(product, name):
    from b2second import loss, optim, targets, training
    net = _plain(product, name)
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net))
    net = training.enable_bn_relu_training(training.enable_pfn_training(training.enable_rpn_training(net)))
    net = _accelerated(net)
    cfg = config.get_config(name)
    return net, cfg, optim.plan(net.train(), orf.ONE_CYCLE, 100), targets.plan(net.target_assigner, cfg.feature_map_size)


def _train_example(product, name, cfg, tplan, B, seed):
    clouds = [gu.make_cloud(name, 500 + seed + i, 12000) for i in range(B)]
    gen = product.utils.VoxelGeneratorV2(cfg.voxel_size, cfg.point_cloud_range, cfg.max_points_per_voxel,
                                         cfg.max_voxels)
    offs = np.cumsum([0] + [c.shape[0] for c in clouds]).astype(np.int32)
    res = gen.generate_device(torch.from_numpy(np.concatenate(clouds)).to(DEV), cfg.max_voxels,
                              frame_offsets=torch.from_numpy(offs).to(DEV), batch=B)
    n = int(res["num_voxels"][0].item())
    ex = {"voxels": res["voxels"][:n], "num_points": res["num_points_per_voxel"][:n],
          "coordinates": res["coordinates"][:n]}
    rng = np.random.default_rng(seed)
    frames = [tr.gt_boxes(tplan, rng, "ordinary") for _ in range(B)]
    goffs = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
    ex.update(tplan.assign_batch(torch.from_numpy(np.concatenate([f[0] for f in frames])).to(DEV),
                                 torch.from_numpy(goffs).to(DEV),
                                 torch.from_numpy(np.concatenate([f[1] for f in frames])).to(DEV),
                                 torch.from_numpy(np.concatenate([f[2] for f in frames])).to(DEV)))
    ex["anchors"] = torch.from_numpy(tplan.anchors[:, :7].copy()).to(DEV)[None].repeat(B, 1, 1)
    return ex


def _check_eval(product, name, net, example, what):
    fast = net.b2s_fastpath
    got = net(example)
    assert not fast.stale
    fresh = _fresh(product, name, net.state_dict())
    _assert_same(got, fresh(example), what)
    _assert_operands(fast.engine(len(example["points"])), fresh.b2s_fastpath.engine(len(example["points"])))
    return got


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16"])
def test_train_eval_train(product, name):
    net, cfg, opt, tplan = _trainable(product, name)
    B = 2
    evaluation = _example(net, name, B, 77)
    step = 0
    for rnd in range(2):
        net.train()
        for _ in range(2):
            ret = net(_train_example(product, name, cfg, tplan, B, step))
            ret["loss"].backward()
            opt.step()
            step += 1
        net.eval()
        _check_eval(product, name, net, evaluation, "%s after %d steps" % (name, step))
    # BatchNorm's running statistics alone: a train-mode forward with no step
    before = net.b2s_fastpath.refreshes
    net.train()
    net(_train_example(product, name, cfg, tplan, B, 99))
    net.eval()
    _check_eval(product, name, net, evaluation, "%s after a train-mode forward" % name)
    assert net.b2s_fastpath.refreshes == before + 1
    assert opt.status.item() == 0


# ---- 3. stream -------------------------------------------------------------------------------------------------------
def _stream_examples(net, name, n):
    anchors = torch.from_numpy(net.anchors()[None]).to(DEV)
    out = []
    for k in range(n):
        clouds = [torch.from_numpy(gu.make_cloud(name, 300 + 4 * k + i, POINTS - 900 * i)).pin_memory()
                  for i in range(4)]
        out.append({"points": clouds, "anchors": anchors})
    return out


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16"])
def test_stream_after_and_during_a_refresh(product, name):
    net = _accelerated(_plain(product, name, seed=0))
    fast = net.b2s_fastpath
    examples = _stream_examples(net, name, 6)
    state0 = {k: v.clone() for k, v in net.state_dict().items()}         # (state_dict() holds the live tensors)
    state1 = _plain(product, name, seed=1).state_dict()
    ref0, ref1 = _fresh(product, name, state0), _fresh(product, name, state1)
    want0, want1 = [ref0(ex) for ex in examples], [ref1(ex) for ex in examples]
    _assert_same(list(fast.stream(examples))[0], want0[0], "stream before the load")
    # after a refresh: the stream refreshes before its first batch
    net.load_state_dict(state1)
    got = list(fast.stream(examples))
    assert fast.refreshes == 1
    for k, g in enumerate(got):
        _assert_same(g, want1[k], "stream after the load, batch %d" % k)
        _assert_same(g, net(examples[k]), "stream against net(example), batch %d" % k)
    # requested while the stream runs: batches 0 and 1 are in flight when the first result is yielded; the refresh
    # runs before batch 2 is enqueued, after both their graphs
    net.load_state_dict(state0)
    fast.refresh()
    gen = fast.stream(examples)
    got = [next(gen)]
    net.load_state_dict(state1)
    got += list(gen)
    assert fast.refreshes == 3
    for k, g in enumerate(got):
        _assert_same(g, (want0 if k < 2 else want1)[k], "refresh during the stream, batch %d" % k)


# ---- 4. no-op refresh, margin change ---------------------------------------------------------------------------------
def test_noop_refresh_keeps_graphs_and_a_margin_change_recaptures(product):
    name = "car.fhd"
    net = _accelerated(_plain(product, name, seed=0))
    fast = net.b2s_fastpath
    ex = _example(net, name, 2, 5)
    want = net(ex)
    eng = fast.engine(2)
    assert eng.bg_idx, "car.fhd's RPN tracks background strips"
    graphs, ptrs = dict(eng._graphs), _ptrs(eng)
    assert graphs
    fast.refresh()
    fast.refresh()
    _assert_same(net(ex), want, "no-op refresh")
    assert eng._graphs == graphs and all(eng._graphs[k] is g for k, g in graphs.items()), "a graph was re-captured"
    _assert_operands(eng, _fresh(product, name, net.state_dict()).b2s_fastpath.engine(2), ptrs)
    # every RPN BatchNorm bias strongly negative: the empty-frame response is zero everywhere
    margins = (list(eng.bg_margin), eng.tail_margin)
    state = {k: (torch.full_like(v, -4.0) if k.startswith("rpn.") and k.endswith(".bias") and
                 not any(h in k for h in ("conv_box", "conv_cls", "conv_dir_cls")) else v)
             for k, v in net.state_dict().items()}
    net.load_state_dict(state)
    got = net(ex)
    assert (list(eng.bg_margin), eng.tail_margin) != margins, "the margins must move for this test to mean anything"
    assert eng._graphs and not any(eng._graphs.get(k) is g for k, g in graphs.items()), "graphs not re-captured"
    fresh = _fresh(product, name, state)
    _assert_same(got, fresh(ex), "after a margin change")
    _assert_operands(eng, fresh.b2s_fastpath.engine(2), ptrs)
