"""The float64 walk of the engine's RPN programs (tests/engine_ref.py) on the CPU: op by op it names the module layer
each op of tc.plan_rpn / tc.plan_rpn_multihead implements, and chaining the per-op float64 references through the
program's buffers reproduces the torch modules' own float64 forward -- RPNV2 with its heads, and the multi-head
network's large and small heads."""
import pytest
import torch

import engine_ref as E
from b2second import config, models, spec, tc

# (config, BEV H, W): every stride and upsampling of the program divides the map
CASES = [("car.fhd", 21, 19), ("car.lite", 17, 24), ("pointpillars.car.xyres_16", 24, 32), ("all.fhd", 24, 20),
         ("nuscenes.all.pp.largea", 32, 24), ("nuscenes.all.pp.mhead", 40, 48)]


def build(oracle, name):
    net = models.build_network(config.get_config(name), oracle).eval()
    models.synthetic_weights_(net, name, seed=0)
    return net


@pytest.mark.parametrize("name,H,W", CASES)
def test_op_chain_reproduces_the_modules(oracle, name, H, W):
    net = build(oracle, name)
    s = spec.spec_from_module(net)
    heads = dict(s.heads) if s.heads is not None else None
    rpn = net.rpn
    plan = tc.plan_rpn(rpn, H, W) if heads is None else tc.plan_rpn_multihead(rpn, heads, H, W)
    refs = E.rpn_refs(rpn, heads)
    E.assert_matches_plan(refs, plan)
    g = torch.Generator().manual_seed(len(name))
    x = torch.rand(2, plan["in_channels"], H, W, generator=g, dtype=torch.float64)
    x[:, :, :H // 3] = 0.0                                              # an empty band, as a sparse BEV map has
    maps = E.run_chain(refs, plan, x.permute(0, 2, 3, 1).contiguous())
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    with torch.no_grad():
        rpn64 = rpn.double()
        if heads is None:
            feat = rpn64.backbone(x)
            want = {"heads": [rpn64.conv_box(feat), rpn64.conv_cls(feat)] +
                    ([rpn64.conv_dir_cls(feat)] if rpn64._use_direction_classifier else [])}
        else:
            res = rpn64(x)
            large, small = heads["large"].double(), heads["small"].double()
            r1 = res["stage0"]
            c = E.crop_size(r1.shape[2])
            sm = small.net(r1[:, :, c:-c, c:-c])
            want = {"heads_large": [large.conv_box(res["out"]), large.conv_cls(res["out"]), large.conv_dir_cls(res["out"])],
                    "heads_small": [small.conv_box(sm), small.conv_cls(sm), small.conv_dir_cls(sm)]}
    for buf, outs in want.items():
        w = torch.cat([nhwc(o) for o in outs], -1)
        got = maps[buf][..., :w.shape[-1]]
        assert got.shape == w.shape, (buf, got.shape, w.shape)
        torch.testing.assert_close(got, w, rtol=1e-12, atol=1e-12, msg=buf)
        assert float(w.abs().max()) > 0


def test_walk_rejects_a_wrong_mapping(oracle):
    """the plan check is not vacuous: a walk with one block's stride or one deblock's sub-grid moved fails it"""
    net = build(oracle, "all.fhd")
    plan = tc.plan_rpn(net.rpn, 24, 20)
    refs = E.rpn_refs(net.rpn)
    for i, key, val in ((0, "stride", 2), (next(i for i, r in enumerate(refs) if r["out_mul"] > 1), "off", (0, 1))):
        bad = [dict(r) for r in refs]
        bad[i][key] = val
        with pytest.raises(AssertionError):
            E.assert_matches_plan(bad, plan)


def test_chain_term_by_hand():
    """op_ref's accumulation-chain term of k_conv_tc on a sum whose terms share a sign: a 1x1 layer, 320 input channels
    of ones, weights of ones -> five K blocks, chains of 4 and 1, twenty 16-channel steps of partial sums 16 q.
    Chain 1: sum_(q=1..16) 2 (16 (q - 1) + 16) + 16 q = 48 * 136; chain 2 (P restarts): 48 * 10; drains |Q| = 256, 320."""
    r = {"w": torch.ones(1, 1, 320, dtype=torch.float64), "k": 1, "stride": 1, "pad": 0, "bn": None, "bias": None,
         "relu": False, "c0": 0, "c1": 1}
    x = torch.ones(1, 2, 3, 320, dtype=torch.float64)
    ref, extra = E.op_ref(x, r, chains=True)
    plain, none = E.op_ref(x, r)
    assert torch.equal(ref.y, plain.y) and bool((ref.y == 320).all()) and not bool(none.any())
    want = 2.0 ** -23 * 48 * (136 + 10) + 2.0 ** -24 * (256 + 320)
    assert torch.allclose(extra, torch.full_like(extra, want), rtol=1e-15, atol=0)
