"""CPU emulation of the data layout of the EXPERIMENTAL conv1d_t6 kernel (csrc/encodec.cu): the staged input slab
[4-channel chunk][stride phase][row][4 channels], the tap = descriptor-start-address rule, and the packed weight operand
of `pack_conv_t6`.  This test pins the index arithmetic the kernel relies on against the oracle convolution without a
GPU, so that a failure of the GPU tests points at the tensor-core or barrier code, not at the layout."""
import math

import numpy as np
import pytest
import torch

from audiocraft_b200.encodec import conv_geometry, pack_conv_t6
from oracle import encodec_oracle as EO

M = 128


def emulate_t6(x, w, bias, k, s, d, causal, reflect=True, elu=False):
    """x [B, Cin, T] fp32, w [Cout, Cin, K]: the output the kernel's addressing produces (fp64 accumulation)."""
    B, cin, T = x.shape
    cout = w.shape[0]
    pad_left, t_virt, t_out = conv_geometry(T, k, s, d, causal, reflect)
    tile = 128 if cout % 128 == 0 else 64
    w6 = pack_conv_t6(w, tile).double().numpy()            # [tile, cg, k, term, c, n, j]
    w6 = w6[:, :, :, 0] + w6[:, :, :, 1]                    # hi + lo: the split is exact up to 2^-22, irrelevant here
    span = (M - 1) * s + (k - 1) * d + 1
    PL = math.ceil(span / s)
    lbo = s * PL * 16
    xin = x.double().numpy()
    if elu:
        xin = np.where(xin > 0, xin, np.exp(xin) - 1)
    y = np.zeros((B, cout, t_out))
    for b in range(B):
        for t0 in range(0, t_out, M):
            for cg in range(cin // 8):
                slab = np.zeros(2 * s * PL * 4)             # one term's slab, in floats (16 B = 4 floats)
                g0 = t0 * s - pad_left
                for c in range(2):
                    for j in range(span):
                        g = g0 + j
                        if reflect:
                            if g < 0:
                                g = -g
                            if g >= t_virt:
                                g = 2 * (t_virt - 1) - g
                        off = (((c * s + j % s) * PL + j // s) * 16) // 4
                        for q in range(4):
                            slab[off + q] = xin[b, cg * 8 + c * 4 + q, g] if 0 <= g < T else 0.0
                for kk in range(k):
                    kd = kk * d
                    a_off = ((kd % s) * PL + kd // s) * 16
                    # A[m][c*4 + q] = slab[(a_off + c*lbo + m*16) / 4 + q]
                    idx = (a_off + np.arange(2)[None, :, None] * lbo + np.arange(M)[:, None, None] * 16) // 4 + np.arange(4)[None, None, :]
                    A = slab[idx].reshape(M, 8)
                    for tl in range(cout // tile):
                        Bm = w6[tl, cg, kk].transpose(1, 0, 2)          # [n, c, j]
                        Bm = Bm.reshape(tile, 8)
                        rows = min(M, t_out - t0)
                        y[b, tl * tile:(tl + 1) * tile, t0:t0 + rows] += (A[:rows] @ Bm.T).T
    if bias is not None:
        y += bias.double().numpy()[None, :, None]
    return torch.from_numpy(y)


@pytest.mark.parametrize('cin,cout,k,s,d,causal,T', [(16, 64, 7, 1, 1, False, 300), (8, 128, 3, 1, 2, False, 200),
                                                      (16, 64, 8, 4, 1, False, 1000), (8, 64, 10, 5, 1, True, 700),
                                                      (8, 64, 16, 8, 1, False, 1100), (8, 64, 1, 1, 1, False, 130),
                                                      (8, 64, 7, 1, 1, False, 5)])
def test_t6_layout_reproduces_the_convolution(cin, cout, k, s, d, causal, T):
    g = torch.Generator().manual_seed(cin * 1000 + cout + k + s)
    x = torch.randn(2, cin, T, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / math.sqrt(cin * k)
    bias = torch.randn(cout, generator=g)
    want = EO.sconv1d(EO.elu(x), w, bias, stride=s, dilation=d, causal=causal, pad_mode='reflect').double()
    got = emulate_t6(x, w, bias, k, s, d, causal, reflect=True, elu=True)
    assert got.shape == want.shape
    torch.testing.assert_close(got, want, rtol=0, atol=2e-5)


def test_t6_shared_memory_budget_of_the_encodec_32k_layers():
    """The launcher requires the double-buffered slab + weight stages to fit 220 KB: true for every strided encoder conv."""
    for (cin, cout, k, s) in [(64, 128, 8, 4), (128, 256, 8, 4), (256, 512, 10, 5), (512, 1024, 16, 8), (1024, 128, 7, 1),
                              (128, 64, 3, 1), (256, 128, 3, 1), (512, 256, 3, 1)]:
        span = (M - 1) * s + (k - 1) + 1
        PL = math.ceil(span / s)
        n = 128 if cout % 128 == 0 else 64
        tb = min(k, 4)
        total = 2 * (2 * 2 * s * PL * 16) + 2 * (tb * 2 * 2 * n * 16) + 12 * 8 + 16
        assert total <= 220 * 1024 and 2 * span <= 128 * 20, (cin, cout, k, s, total)
