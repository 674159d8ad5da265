"""A drop-in sparse layer past the tensor-pipe kernel's 27 kernel offsets runs on the fp32 FMA kernel in eval as it does
in training, checked against the float64 reference and bound of tests/fp32_ref.py."""
import numpy as np
import pytest
import torch

import fp32_ref as R

pytestmark = pytest.mark.gpu


def test_eval_subm5_runs_on_the_fma_kernel(product, monkeypatch):
    """SubMConv3d(16, 16, 5): K = 125 at widths the tensor-pipe kernel covers, in eval under no_grad with the tensor
    pipe on"""
    monkeypatch.setattr(product, "USE_TENSOR_CORES", True)
    rng = np.random.default_rng(125)
    idx = R.surface_coords(rng, 3000)
    _, nbr = R.build_table(idx, R.SHAPE, (5, 5, 5), subm=True)
    x = torch.from_numpy(rng.standard_normal((idx.shape[0], 16)).astype(np.float32)).cuda()
    conv = product.SubMConv3d(16, 16, 5).cuda().eval()
    with torch.no_grad():
        y = conv(product.SparseConvTensor(x, torch.from_numpy(idx).cuda(), list(R.SHAPE), R.BATCH))
    assert torch.equal(y.indices.cpu(), torch.from_numpy(idx))
    ref = R.sparse_ref(x, conv.weight.detach().view(125, 16, 16), torch.from_numpy(nbr).cuda(), shift=conv.bias.detach())
    R.assert_accurate(y.features, ref, "SubMConv3d(16, 16, 5)")
