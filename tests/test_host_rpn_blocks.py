"""The RPN background skip at the granularity the engine plans it (8x8 output blocks, b2s_rpn_block_plan), checked
against the torch modules on the CPU: wherever the numpy restatement of the plan calls a block of layer l background,
the dense fp32 computation on the data yields exactly the empty-frame response at those pixels."""
import pytest
import torch

from b2second import config, loader, models, tc
from test_host_rpn_plan import bg_plan_numpy


@pytest.mark.parametrize("name", ["car.fhd", "car.lite"])
def test_background_blocks_hold_the_empty_frame_response(name):
    sp = loader.oracle_spconv()
    net = models.build_network(config.get_config(name), sp).eval()
    models.synthetic_weights_(net, name, seed=0)
    rpn = net.rpn
    H, W = 68, 84                                      # partial 8x8 blocks along the bottom and right edges
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
    flags = bg_plan_numpy(occ.numpy(), len(idx), tile=8)
    mods = [m for m in rpn.blocks[0].children()]
    cur, empty, li, i = x, torch.zeros(1, cin, H, W), 0, 0
    with torch.no_grad():
        while i < len(mods) and li < len(idx):
            step = 4 if isinstance(mods[i], torch.nn.ZeroPad2d) else 3
            for mm in mods[i:i + step]:
                cur, empty = mm(cur), mm(empty)
            i += step
            f = flags[li]
            n_bg = n_edge = 0
            for b in range(2):
                for bh in range(f.shape[1]):
                    for bw in range(f.shape[2]):
                        if f[b, bh, bw]:
                            continue
                        n_bg += 1
                        n_edge += bh == f.shape[1] - 1 or bw == f.shape[2] - 1
                        sl = (slice(None), slice(bh * 8, (bh + 1) * 8), slice(bw * 8, (bw + 1) * 8))
                        assert torch.equal(cur[b][sl], empty[0][sl]), (li, b, bh, bw)
            assert n_bg > 0 and n_edge > 0                  # incl. partial blocks at the bottom / right edge
            assert int(f.sum()) > 0
            li += 1
