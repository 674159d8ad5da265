"""tc.sparse_tc_channels: the one rule that sends a sparse layer to the tensor-pipe kernel or to the fp32 FMA kernel, for
the spconv drop-in and the fused engine alike (no GPU needed: b2s_sparse_conv_tc_supported is a host query)."""
from b2second import tc


def test_sparse_tc_channels_table():
    from spconv import _lib
    lib = _lib.load()
    padded = {3: 8, 4: 8, 8: 8, 16: 16, 32: 32, 64: 64}          # Cin 128: no kernel instance
    for cin in (3, 4, 8, 16, 32, 64, 128):
        for cout in (16, 64, 128):                               # Cout 128: no kernel instance
            for K in (1, 27, 28, 125):                           # the tensor-pipe kernel takes K <= 27
                want = padded.get(cin) if cout != 128 and K <= 27 else None
                assert tc.sparse_tc_channels(lib, cin, cout, K) == want, (cin, cout, K)
