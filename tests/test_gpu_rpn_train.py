"""GPU tests of the RPN's 3x3 convolutions in training (b2second.rpn_train over csrc/conv_train.cu and
b2s_conv2d_tc_ex): per layer against float64 with the per-element 3xF16 bounds of tests/tc_ref.py, equal bits run to
run for the weight gradient, whole car.fhd and xyres_16 RPNs in train() mode against float64 next to cuDNN fp32, and a
complete drop-in car.fhd training step against the all-torch fp32 step."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import optim_ref as orf
import tc_ref
from b2second import config, loader, loss, metrics, models, optim, rpn_train, training

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def fp32_torch():
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _dense_nbr(B, H, W):
    """[B*H*W, 9] input pixel of each output pixel and tap (ky * 3 + kx) of a pad-1 3x3 conv, -1 past the border"""
    b, h, w = torch.meshgrid(torch.arange(B, device=DEV), torch.arange(H, device=DEV), torch.arange(W, device=DEV),
                             indexing="ij")
    cols = []
    for ky in range(3):
        for kx in range(3):
            hh, ww = h + ky - 1, w + kx - 1
            ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
            cols.append(torch.where(ok, (b * H + hh.clamp(0, H - 1)) * W + ww.clamp(0, W - 1), -1).reshape(-1))
    return torch.stack(cols, 1).int()


def _layer(cin, cout, seed):
    g = torch.Generator().manual_seed(seed)
    conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False)
    with torch.no_grad():
        conv.weight.copy_((torch.rand(conv.weight.shape, generator=g) * 2 - 1) * (6.0 / (9 * cin)) ** 0.5)
    conv = conv.to(DEV).train()
    rpn_train.enable(nn.Sequential(conv))
    return conv, g


def _run_layer(conv, x, dy):
    x = x.detach().clone().requires_grad_(True)
    conv.weight.grad = None
    y = conv(x)
    y.backward(dy)
    return y.detach(), x.grad.detach(), conv.weight.grad.detach().clone()


# (B, Cin, Cout, H, W, channels_last input): xyres_16 block sizes (W not a multiple of 8), car.fhd's map, 256 channels,
# Cin != Cout both ways (one 64-channel dY block per CTA; two launches of 128 output channels)
CASES = [(2, 64, 64, 124, 108, False), (2, 128, 128, 200, 176, False), (1, 256, 256, 31, 27, True),
         (2, 128, 64, 20, 13, False), (1, 64, 256, 9, 7, True)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%dx%d_%dx%d_b%d%s" % (c[1], c[2], c[3], c[4], c[0],
                                                                            "_cl" if c[5] else ""))
def test_layer_against_float64(case):
    B, cin, cout, H, W, cl = case
    conv, g = _layer(cin, cout, 1)
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    # dY spans decades (2^-40 .. 2^-20): the automatic scale has to bring it into the fp16 range
    dy = (torch.randn(B, cout, H, W, generator=g) * torch.exp2(torch.randint(-40, -19, (B, cout, H, W), generator=g)
                                                               .float())).to(DEV)
    if cl:
        x, dy = x.contiguous(memory_format=torch.channels_last), dy.contiguous(memory_format=torch.channels_last)
    y, dx, dw = _run_layer(conv, x, dy)
    assert y.is_contiguous(memory_format=torch.channels_last) and y.shape == (B, cout, H, W)
    w = conv.weight.detach()
    ws = 1.0 / float(rpn_train.pack_weights(conv, False)[2])
    tc_ref.assert_accurate(y, tc_ref.dense_ref(x, w, padding=1), ws, "forward")
    tc_ref.assert_accurate(dx, tc_ref.dense_ref(dy, w.flip(2, 3).transpose(0, 1), padding=1), ws, "dX")
    g_ws = 1.0 / float(rpn_train.split_halo(dy)[2])
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])
    ref = tc_ref.wgrad_ref(rows(x), rows(dy), _dense_nbr(B, H, W))
    tc_ref.assert_accurate(dw.permute(2, 3, 1, 0).reshape(9, cin, cout), ref, g_ws, "dW")
    assert float(dw.abs().max()) > 0
    _, dx2, dw2 = _run_layer(conv, x, dy)
    assert torch.equal(dw2.view(torch.int32), dw.view(torch.int32)), "dW differs between two runs"
    assert torch.equal(dx2.view(torch.int32), dx.view(torch.int32))


@pytest.mark.timeout(600)
def test_layer_one_sign_against_float64():
    """car.fhd's 200 x 176 map at its training batch B = 8, 128 -> 128, X post-ReLU (every term of one sign) and dY of
    mostly one sign: the accumulator cuts toward zero add up instead of cancelling.  Forward and dX (k_conv_tc) meet
    the tc_ref bound plus engine_ref's accumulation-chain term, dW (b2s_conv2d_wgrad_tc) the bound plus the chain term
    in its strip and slab order (train_ref.wgrad_chain_term): the terms tc_ref's ALPHA, calibrated on random-sign data,
    leaves out"""
    import train_ref
    conv, g = _layer(128, 128, 3)
    B, H, W = 8, 200, 176
    x = torch.relu(torch.randn(B, 128, H, W, generator=g) + 0.5).to(DEV)
    dy = ((torch.randn(B, 128, H, W, generator=g) * 0.5 + 1.0) * 2.0 ** -20).to(DEV)
    y, dx, dw = _run_layer(conv, x, dy)
    ws = 1.0 / float(rpn_train.pack_weights(conv, False)[2])
    train_ref.check_conv3x3_train(x, dy, y, dx, dw, conv.weight.detach(), ws, "one-sign 128 -> 128")


def test_layer_scale_follows_the_input():
    """the same layer at input scales 2^-30 and 2^20: results scale exactly (the split picks a new 2^e each call)"""
    conv, g = _layer(128, 128, 2)
    x = torch.randn(1, 128, 24, 20, generator=g).to(DEV)
    dy = torch.randn(1, 128, 24, 20, generator=g).to(DEV)
    y, dx, dw = _run_layer(conv, x, dy)
    for e in (-30, 20):
        ys, dxs, dws = _run_layer(conv, x * 2.0 ** e, dy * 2.0 ** -e)
        assert torch.equal(ys, y * 2.0 ** e) and torch.equal(dxs, dx * 2.0 ** -e) and torch.equal(dws, dw)


def _rpn_input(name, B, seed):
    cfg = config.get_config(name)
    net = models.build_network(cfg, loader.product_spconv())
    models.synthetic_weights_(net, name, seed=0)
    rpn = net.rpn
    cin = rpn.blocks[0][1].in_channels
    H, W = (int(v) for v in cfg.feature_map_size[1:])
    H, W = H * rpn.blocks[0][1].stride[0], W * rpn.blocks[0][1].stride[0]
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, cin, H, W, generator=g)) * (torch.rand(B, 1, H, W, generator=g) < 0.15)
    return rpn, x.to(DEV)


def _rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b).abs().max()) / max(float(b.abs().max()), 1e-300)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name,B", [("car.fhd", 2), ("pointpillars.car.xyres_16", 2)])
def test_whole_rpn_train_mode_against_float64(name, B, fp32_torch):
    rpn, x = _rpn_input(name, B, 5)
    nets = {"f64": copy.deepcopy(rpn).double(), "cudnn": copy.deepcopy(rpn), "ours": copy.deepcopy(rpn)}
    rpn_train.enable(nets["ours"])
    assert sum(getattr(m, "_b2s_rpn_train", False) for m in nets["ours"].modules()) > 0
    res = {}
    gen = torch.Generator().manual_seed(6)
    G = None
    for k, net in nets.items():
        net = net.to(DEV).train()
        xi = (x.double() if k == "f64" else x).clone().requires_grad_(True)
        out = net(xi)
        if G is None:
            G = {o: torch.randn(out[o].shape, generator=gen).to(DEV) / out[o].numel() ** 0.5 for o in sorted(out)}
        sum((out[o] * G[o].to(out[o].dtype)).sum() for o in sorted(out)).backward()
        res[k] = (out, xi.grad, {n: p.grad for n, p in net.named_parameters()},
                  {n: b for n, b in net.named_buffers() if "running" in n})
    o64, x64, p64, _ = res["f64"]
    report = []
    for k in ("cudnn", "ours"):
        out, gx, gp, _ = res[k]
        errs = {("out", o): _rel(out[o], o64[o]) for o in o64}
        errs[("grad", "input")] = _rel(gx, x64)
        errs.update({("grad", n): _rel(gp[n], p64[n]) for n in p64})
        res[k] = res[k] + (errs,)
        report.append((k, max(errs.values())))
    print("%s B=%d worst error relative to the float64 maximum: %s" % (name, B, report))
    ours, cudnn = res["ours"][4], res["cudnn"][4]
    for key in ours:
        assert ours[key] <= max(8 * cudnn[key], 2e-5), (key, ours[key], cudnn[key])
    for n, b in res["cudnn"][3].items():
        got = res["ours"][3][n]
        assert float((got - b).abs().max()) <= 1e-5 * max(float(b.abs().max()), 1.0), n


@pytest.mark.timeout(900)
def test_drop_in_training_step_matches_torch(fp32_torch):
    """car.fhd with enable_sparse_backward, enable_gpu_loss, enable_gpu_metrics and enable_rpn_training, stepped by
    optim.plan, against the same network without enable_rpn_training (the RPN on cuDNN fp32)"""
    from test_gpu_loss import _car_lite_example
    name = "car.fhd"
    cfg = config.get_config(name)
    sp = loader.product_spconv()
    nets = []
    for rpn_tc in (True, False):
        net = models.build_network(cfg, sp)
        models.synthetic_weights_(net, name, seed=0)
        net = loss.enable_gpu_loss(training.enable_sparse_backward(net.to(DEV)))
        net = metrics.enable_gpu_metrics(net)
        if rpn_tc:
            net = training.enable_rpn_training(net)
        nets.append(net.train())
    ex = _car_lite_example(nets[0], cfg)
    s = orf.ONE_CYCLE
    losses, params = [], []
    for net in nets:
        opt = optim.plan(net, s, 100)
        r = net(ex)
        r["loss"].backward()
        losses.append(float(r["loss"].detach()))
        opt.step()
        params.append({k: p.detach().clone() for k, p in net.named_parameters()})
    assert np.isfinite(losses[0]) and abs(losses[0] - losses[1]) <= 1e-5 * abs(losses[1]), losses
    lr = float(opt.table[0, 0])
    inside = []
    for k, p in params[0].items():
        q = params[1][k]
        diff = (p - q).abs()
        tight = 6 * orf.EPS32 * q.abs() + 0.01 * lr
        inside.append((diff <= tight).flatten())
        assert float(diff.max()) <= 2.2 * lr + float(tight.max()), k      # Adam's first step: at most lr per element
    assert float(torch.cat(inside).float().mean()) >= 0.99
