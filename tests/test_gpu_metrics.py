"""Training metrics (csrc/metrics.cu through b2second.metrics) and the device-side packing of the sparse conv weights
(b2s_pack_sparse_weights) on the GPU.

The metrics are integer counts and float32 sums in the reference's order, so the kernel equals tests/metrics_ref.py run
as torch ops on the same GPU bit for bit.  Against the fixtures the reference made on the CPU, only the sigmoid can
differ (the CPU's and the GPU's float32 expf): every difference must come from anchors whose two sigmoids fall on
either side of a threshold."""
import glob
import json
import os

import numpy as np
import pytest
import torch

import metrics_ref as mr
from b2second import config, loader, loss, metrics, models, tc, training
from conftest import REPO
from test_metrics_reference import same_dict, same_floats

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = sorted(glob.glob(os.path.join(REPO, "tests", "golden", "metrics", "*.npz")))
SIZES = {"car.fhd": (8, 70400 * 2, 1), "nuscenes.all.pp.mhead": (4, 30000, 10)}     # name: (batch, anchors, classes)


def _net(name):
    net = models.build_network(config.get_config(name), loader.product_spconv())
    return metrics.enable_gpu_metrics(net.to(DEV))


def _state(net):
    b = {"acc_total": net.rpn_acc.total, "acc_count": net.rpn_acc.count,
         "prec_total": net.rpn_metrics.prec_total, "prec_count": net.rpn_metrics.prec_count,
         "rec_total": net.rpn_metrics.rec_total, "rec_count": net.rpn_metrics.rec_count,
         "cls_total": net.rpn_cls_loss.total, "cls_count": net.rpn_cls_loss.count,
         "loc_total": net.rpn_loc_loss.total, "loc_count": net.rpn_loc_loss.count}
    return {k: v.detach().cpu().numpy().copy() for k, v in b.items()}


def _load(net, state):
    cur = {"acc_total": net.rpn_acc.total, "acc_count": net.rpn_acc.count,
           "prec_total": net.rpn_metrics.prec_total, "prec_count": net.rpn_metrics.prec_count,
           "rec_total": net.rpn_metrics.rec_total, "rec_count": net.rpn_metrics.rec_count,
           "cls_total": net.rpn_cls_loss.total, "cls_count": net.rpn_cls_loss.count,
           "loc_total": net.rpn_loc_loss.total, "loc_count": net.rpn_loc_loss.count}
    with torch.no_grad():
        for k, v in state.items():
            cur[k].copy_(torch.from_numpy(np.asarray(v, np.float32)))


def _run_sequence(name, seed, preset):
    B, A, C = SIZES[name]
    net = _net(name)
    ref = mr.MetricsRef(device=DEV)
    if preset:
        ref.load(mr.state0())
        _load(net, mr.state0())
    out = []
    for s, st in enumerate(mr.make_steps(seed, B, A // 8, C, steps=6)):
        args = mr.to_torch(st, DEV)
        got = net.update_metrics(*args)
        want = ref.update(*args, C)
        out.append((got, want, _state(net), ref.state()))
    return out


@pytest.mark.parametrize("name", list(SIZES))
@pytest.mark.parametrize("preset", [False, True])
def test_kernel_equals_restatement_on_gpu(name, preset):
    """running buffers and dict equal the torch restatement on the same GPU at every step; two runs give the same bits"""
    a = _run_sequence(name, 5, preset)
    b = _run_sequence(name, 5, preset)
    for s, ((got, want, sg, sw), (got2, _, sg2, _)) in enumerate(zip(a, b)):
        assert same_dict(got, want), (s, got, want)
        assert same_dict(got, got2), s
        for k in mr.BUFFERS:
            assert same_floats(sg[k], sw[k]), (s, k, sg[k], sw[k])
            assert same_floats(sg[k], sg2[k]), (s, k)


def _cpu_sigmoid(x):
    return torch.sigmoid(x.cpu()).to(x.device)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_kernel_against_reference_fixtures(path):
    """against the reference's CPU run: equal bits unless an anchor's CPU and GPU sigmoids straddle a threshold; those
    anchors are listed, and the restatement fed the GPU's sigmoid (which equals the kernel bit for bit) differs from the
    fixtures only through them"""
    g = np.load(path)
    C = int(g["num_class"])
    name = str(g["name"])
    net = _net(name)
    init = {k: g["init_" + k] for k in mr.BUFFERS}
    _load(net, init)
    gpu_ref = mr.MetricsRef(device=DEV)
    gpu_ref.load(init)
    straddle_total = 0
    for s in range(int(g["steps"])):
        st = {k: g["%d_%s" % (s, k)] for k in ("cls_preds", "labels", "cared", "cls_loss", "loc_loss")}
        args = mr.to_torch(st, DEV)
        got = net.update_metrics(*args)
        want = gpu_ref.update(*args, C)
        assert same_dict(got, want), s
        state = _state(net)
        x = args[2].view(args[2].shape[0], -1, C)
        s_gpu, s_cpu = torch.sigmoid(x), _cpu_sigmoid(x)
        ths = torch.tensor(mr.THRESHOLDS + (0.5,), device=DEV).view(-1, 1, 1, 1)
        flips = ((s_gpu.unsqueeze(0) > ths) != (s_cpu.unsqueeze(0) > ths)).any(0).any(-1)     # [B, A]
        straddle = torch.nonzero(flips).tolist()
        straddle_total += len(straddle)
        if not straddle:
            assert same_dict(got, json.loads(str(g["%d_dict_json" % s]))), (s, got)
            for k in mr.BUFFERS:
                assert same_floats(state[k], g["%d_%s" % (s, k)]), (s, k)
        else:
            # the listed anchors account for the whole difference: the restatement with the CPU sigmoid on the GPU
            # reproduces the fixtures, and the one with the GPU sigmoid reproduces the kernel
            cpu_ref = mr.MetricsRef(device=DEV)
            cpu_ref.load({k: g["%d_%s" % (s - 1, k)] if s else init[k] for k in mr.BUFFERS})
            d = cpu_ref.update(*args, C, sigmoid=_cpu_sigmoid)
            assert same_dict(d, json.loads(str(g["%d_dict_json" % s]))), (s, straddle)
            _load(net, {k: g["%d_%s" % (s, k)] for k in mr.BUFFERS})        # continue from the reference's state
            gpu_ref.load({k: g["%d_%s" % (s, k)] for k in mr.BUFFERS})
    print("%s: %d anchors with straddling sigmoids" % (name, straddle_total))


def test_async_captured_in_a_graph_equals_eager_calls():
    name = "nuscenes.all.pp.mhead"
    B, A, C = SIZES[name]
    steps = mr.make_steps(9, B, A // 8, C, steps=1)
    args = mr.to_torch(steps[0], DEV)
    eager = _net(name)
    for _ in range(5):
        want = eager.update_metrics(*args)
    graphed = _net(name)
    plan = graphed.b2s_metrics
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.update_metrics_async(*args)          # warm-up outside the graph
    torch.cuda.current_stream().wait_stream(s)
    graphed.clear_metrics()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        h = plan.update_metrics_async(*args)
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert same_dict(h.result(), want)
    se, sg = _state(eager), _state(graphed)
    for k in mr.BUFFERS:
        assert same_floats(se[k], sg[k]), k


def test_no_sync_in_async_and_one_copy_in_update_metrics():
    from torch.profiler import ProfilerActivity, profile
    name = "car.fhd"
    B, A, C = SIZES[name]
    args = mr.to_torch(mr.make_steps(4, B, A // 8, C, steps=1)[0], DEV)
    net = _net(name)
    net.update_metrics(*args)
    torch.cuda.synchronize()

    def calls(fn):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
        names = [e.name for e in prof.events()]
        # the profiler flushes with a cudaDeviceSynchronize of its own when it stops; nothing here calls that one
        return (sum(n.startswith("cudaMemcpy") for n in names),
                sum(n in ("cudaStreamSynchronize", "cudaEventSynchronize") for n in names))

    assert calls(lambda: net.b2s_metrics.update_metrics_async(*args)) == (0, 0)
    assert calls(lambda: net.update_metrics(*args)) == (1, 1)


def test_step_log_fields():
    name = "car.fhd"
    B, A, C = 2, 5000, 1
    st = mr.make_steps(6, B, A, C, steps=1)[0]
    args = mr.to_torch(st, DEV)
    g = torch.Generator(device=DEV).manual_seed(0)
    ret = {"loc_loss": torch.rand(B, A, 7, device=DEV, generator=g), "cls_pos_loss": torch.tensor(0.25, device=DEV),
           "cls_neg_loss": torch.tensor(0.5, device=DEV), "dir_loss_reduced": torch.tensor(0.75, device=DEV)}
    mask = torch.rand(B, A, device=DEV, generator=g) > 0.3
    net = _net(name)
    h = net.b2s_metrics.update_metrics_async(*args, ret_dict=ret, anchors_mask=mask)
    log = h.step_log()
    labels = args[3]
    assert log["misc"] == {"num_pos": int((labels > 0)[0].sum()), "num_neg": int((labels == 0)[0].sum()),
                           "num_anchors": int(mask[0].sum())}
    assert (log["loss"]["cls_pos_rt"], log["loss"]["cls_neg_rt"], log["loss"]["dir_rt"]) == (0.25, 0.5, 0.75)
    want = (ret["loc_loss"].double().sum((0, 1)) / B).tolist()
    assert np.allclose(log["loss"]["loc_elem"], want, rtol=1e-6, atol=0)
    assert h.result()["loss"]["cls_loss_rt"] == float(st["cls_loss"])


def test_bad_labels_raise_the_status_bit():
    net = _net("car.fhd")
    st = mr.make_steps(7, 2, 300, 1, steps=1)[0]
    args = list(mr.to_torch(st, DEV))
    net.update_metrics(*args)
    assert int(net.b2s_metrics.last_status) == 0
    args[3] = args[3].clone()
    args[3][1, 7] = 2                           # num_class is 1
    net.update_metrics(*args)
    assert int(net.b2s_metrics.last_status) & 32


# ---- weight packing ----------------------------------------------------------------------------------------------

def _host_pack(w, transpose=False, flip=False):
    """tc.pack_sparse_weights + pow2_scale + split_f16, the host path"""
    K = w.shape[0]
    wt = w
    if transpose:
        wt = (w.flip(0) if flip else w).transpose(1, 2).contiguous()
    wp = tc.pack_sparse_weights(wt)
    ws = tc.pow2_scale(wp)
    hi, lo = tc.split_f16(wp, ws)
    return hi, lo, torch.tensor([ws], dtype=torch.float32, device=w.device), \
        torch.tensor([1.0 / ws], dtype=torch.float32, device=w.device)


def _pairs():
    lib = loader.product_spconv()._lib.load()
    out = []
    for cin in (1, 3, 4, 5, 8, 16, 32, 64):
        for cout in (16, 32, 64):
            if lib.b2s_sparse_conv_tc_supported(tc.sparse_tc_cin(cin), cout):
                out.append((cin, cout))
    return out


@pytest.mark.parametrize("kind", ["random", "zero", "pow2", "tiny", "subnormal"])
def test_device_pack_equals_host_pack(kind):
    sp = loader.product_spconv()
    pairs = _pairs()
    assert len(pairs) >= 12
    g = torch.Generator(device=DEV).manual_seed(1)
    for cin, cout in pairs:
        for K in (27, 3, 1):
            w = torch.randn(K, cin, cout, device=DEV, generator=g) * 0.05
            if kind == "zero":
                w.zero_()
            elif kind == "pow2":
                w[K // 2, 0, cout - 1] = -0.125          # max |w| is exactly 2^-3
                w.clamp_(-0.125, 0.125)
            elif kind == "tiny":                          # max |w| = 2^-120: the scale clamps at 2^126
                w.mul_(2.0 ** -118).clamp_(-2.0 ** -120, 2.0 ** -120)[K // 2, 0, cout - 1] = 2.0 ** -120
            elif kind == "subnormal":                     # every weight an fp32 subnormal
                w.mul_(2.0 ** -128).clamp_(-2.0 ** -127, 2.0 ** -127)
            for transpose, flip in ((False, False), (True, False), (True, True)):
                if transpose and tc.sparse_tc_cin(cout) != cout:
                    continue
                got = sp._pack_tc_weights(w, transpose, flip)
                want = _host_pack(w, transpose, flip)
                for a, b, what in zip(got, want, ("hi", "lo", "s", "1/s")):
                    assert a.shape == b.shape and torch.equal(a.view(torch.int16 if a.dtype == torch.float16
                                                                      else torch.int32),
                                                              b.view(torch.int16 if b.dtype == torch.float16
                                                                     else torch.int32)), (cin, cout, K, transpose,
                                                                                          flip, what)
            if kind == "pow2":
                assert float(sp._pack_tc_weights(w)[2]) == 2.0 ** 16          # 2^-3 * 2^16 = 2^13
            if kind == "zero":
                assert float(sp._pack_tc_weights(w)[2]) == 1.0
            if kind in ("tiny", "subnormal"):
                assert float(sp._pack_tc_weights(w)[2]) == 2.0 ** 126


def _train_step(net, ex):
    for p in net.parameters():
        p.grad = None
    r = net(ex)
    r["loss"].backward()
    torch.cuda.synchronize()
    return float(r["loss"]), {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}


def test_training_step_same_bits_with_device_and_host_packing(monkeypatch):
    """a drop-in training step (enable_sparse_backward + enable_gpu_loss) gives the same loss and gradients bit for bit
    with the device packing as with the host packing, and the device packing reads nothing on the host"""
    from test_gpu_loss import _car_lite_example
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)     # the RPN's cuDNN weight gradients
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    sp = loader.product_spconv()
    name = "car.lite"
    cfg = config.get_config(name)
    net = models.build_network(cfg, sp)
    models.synthetic_weights_(net, name, seed=0)
    net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV))).train()
    ex = _car_lite_example(net, cfg)
    l_dev, g_dev = _train_step(net, ex)
    convs = [m for m in net.modules() if isinstance(m, sp.SparseConvolution)]
    assert any(getattr(m, "_b2s_tc_w", None) is not None for m in convs)
    assert any(getattr(m, "_b2s_tc_wt", None) is not None for m in convs)

    def no_host_read(*a, **k):
        raise AssertionError("host read while packing weights")

    for m in convs:
        m._b2s_tc_w = m._b2s_tc_wt = None
    with monkeypatch.context() as mp:
        mp.setattr(torch.Tensor, "item", no_host_read)
        mp.setattr(torch.Tensor, "__float__", no_host_read)
        mp.setattr(torch.Tensor, "tolist", no_host_read)
        for m in convs:
            if m._wgrad_tc_cin(sp._lib.load(), int(np.prod(m.kernel_size))):
                m._tc_weights(tc.sparse_tc_cin(m.in_channels))
                if tc.sparse_tc_cin(m.out_channels) == m.out_channels:
                    m._dgrad_weights(m.weight, True)
    for m in convs:
        m._b2s_tc_w = m._b2s_tc_wt = None
    monkeypatch.setattr(sp, "_pack_tc_weights", _host_pack)
    l_host, g_host = _train_step(net, ex)
    assert l_dev == l_host
    assert g_dev.keys() == g_host.keys()
    for k in g_dev:
        assert torch.equal(g_dev[k], g_host[k]), k
