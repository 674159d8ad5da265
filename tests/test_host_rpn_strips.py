"""The RPN background skip at the granularity the engine plans it (output strips 8 pixels wide and BG_ROWS high,
b2s_rpn_strip_plan), checked against the torch modules on the CPU: wherever the numpy restatement of the plan calls a
strip of layer l background, the dense fp32 computation on the data yields exactly the empty-frame response there."""
import numpy as np
import pytest
import torch

from b2second import config, loader, models, tc
from b2second.engine import BG_ROWS, _field_margin


def strip_plan_numpy(occ, num_layers, rows, width=8):
    """numpy restatement of b2s_rpn_strip_plan (csrc/rpn_bg.cu): per layer the [B, strips_h, strips_w] flags (1 = the
    strip has a pixel whose receptive field holds data) after dilating the data mask by one pixel per layer; strips
    are `width` pixels wide and `rows` high, partial at the bottom / right edge."""
    B, H, W = occ.shape
    sh, sw = -(-H // rows), -(-W // width)
    cur = occ.astype(bool)
    flags = []
    for _ in range(num_layers):
        pad = np.pad(cur, ((0, 0), (1, 1), (1, 1)), constant_values=False)
        out = np.zeros_like(cur)
        for dy in range(3):
            for dx in range(3):
                out |= pad[:, dy:dy + H, dx:dx + W]
        f = np.zeros((B, sh, sw), np.int32)
        for i in range(sh):
            for j in range(sw):
                f[:, i, j] = out[:, i * rows:(i + 1) * rows, j * width:(j + 1) * width].any(axis=(1, 2))
        flags.append(f)
        cur = out
    return flags


def test_strip_plan_restatement_nests():
    """a strip is computed exactly when its 8x8 block row-slice holds data: every computed 8x8 block contains a
    computed 8x2 strip, and no background block does (the finer plan only drops work)."""
    rng = np.random.default_rng(5)
    occ = (rng.random((2, 37, 45)) < 0.01).astype(np.uint8)
    for blocks, strips in zip(strip_plan_numpy(occ, 4, 8), strip_plan_numpy(occ, 4, 2)):
        pad = np.pad(strips, ((0, 0), (0, 4 * blocks.shape[1] - strips.shape[1]), (0, 0)))
        assert np.array_equal(pad.reshape(2, blocks.shape[1], 4, -1).any(axis=2), blocks.astype(bool))
        assert strips.mean() <= blocks.mean()


@pytest.mark.parametrize("name", ["car.fhd", "car.lite"])
def test_background_strips_hold_the_empty_frame_response(name):
    sp = loader.oracle_spconv()
    net = models.build_network(config.get_config(name), sp).eval()
    models.synthetic_weights_(net, name, seed=0)
    rpn = net.rpn
    H, W = 67, 84                                      # odd H: the last strip row is partial; W: partial column
    plan = tc.plan_rpn(rpn, H, W)
    idx = tc.background_layers(plan)
    assert len(idx) >= 4
    cin = plan["in_channels"]
    torch.manual_seed(3)
    occ = torch.zeros(2, H, W, dtype=torch.bool)
    occ[0, 20:30, 40:52] = True                       # a blob in the middle, far from the border
    occ[1, 0:5, 10:20] = True                         # blobs touching the border
    occ[1, 60:64, 0:3] = True
    occ[1, 35, 80] = True
    x = torch.relu(torch.randn(2, cin, H, W)) * occ[:, None].float()
    flags = strip_plan_numpy(occ.numpy(), len(idx), BG_ROWS)
    assert flags[0].shape[1:] == (-(-H // BG_ROWS), 11)
    mods = [m for m in rpn.blocks[0].children()]
    cur, empty, li, i = x, torch.zeros(1, cin, H, W), 0, 0
    with torch.no_grad():
        while i < len(mods) and li < len(idx):
            step = 4 if isinstance(mods[i], torch.nn.ZeroPad2d) else 3
            for mm in mods[i:i + step]:
                cur, empty = mm(cur), mm(empty)
            i += step
            f = flags[li]
            n_bg = n_bottom = n_right = 0
            for b in range(2):
                for sh in range(f.shape[1]):
                    for sw in range(f.shape[2]):
                        if f[b, sh, sw]:
                            continue
                        n_bg += 1
                        n_bottom += sh == f.shape[1] - 1
                        n_right += sw == f.shape[2] - 1
                        sl = (slice(None), slice(sh * BG_ROWS, (sh + 1) * BG_ROWS), slice(sw * 8, (sw + 1) * 8))
                        assert torch.equal(cur[b][sl], empty[0][sl]), (li, b, sh, sw)
            assert n_bg > 0 and n_bottom > 0 and n_right > 0    # incl. partial strips at the bottom / right edge
            assert int(f.sum()) > 0
            li += 1


def test_field_margin_is_the_width_of_the_non_constant_border():
    """the engine's margin for the conv kernel's constant fill: the smallest m such that every pixel at least m from
    every border holds the centre value bit for bit (-0 differs from +0); -1 when the field has no constant interior."""
    H, W, C = 13, 18, 8
    torch.manual_seed(4)
    hi = torch.randn(H + 2, W + 2, C).half()
    lo = torch.randn(H + 2, W + 2, C).half()
    for m in (0, 2, 5):
        h, l = hi.clone(), lo.clone()
        h[1 + m:H + 1 - m, 1 + m:W + 1 - m] = 0.5
        l[1 + m:H + 1 - m, 1 + m:W + 1 - m] = 0.0
        if m:
            h[1 + m - 1, 1 + W // 2] = 0.5                 # a border pixel that happens to match does not matter
            l[1 + m - 1, 1 + W // 2] = 0.0
        assert _field_margin(h, l) == m
        l[1 + m, 1 + m + 1] = -0.0                         # equal to +0 as a number, different bits
        assert _field_margin(h, l) == m + 1
    assert _field_margin(hi, lo) == -1                     # random everywhere: no constant interior
