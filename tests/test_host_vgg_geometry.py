"""The zero-haloed buffer geometry of the VGG path (include/b200asr.h, ops.VGGFn), restated in numpy without a GPU:
tap rows, junk rows landing on the next buffer's halo, and the tap-major weight packings of ops (forward, the flipped
input-gradient weights, the weight-gradient unpacking) against float64 conv2d and its gradients."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vgg_ref as V


def _ops():
    import importlib
    return importlib.import_module("end-to-end-asr-pytorch_b200").ops


def _buffer(x):
    """[B, C, T, F] -> zero-haloed buffer [R + F + 3, C] (numpy), followed by the F + 3 rows of zeros that the tensor
    map's zero fill supplies to the reads of the last grid rows."""
    B, C, T, Fq = x.shape
    buf = np.zeros((V.grid_rows(B, T, Fq) + 2 * Fq + 6, C))
    for b in range(B):
        for t in range(T):
            for f in range(Fq):
                buf[V.data_row(b, t, f, T, Fq)] = x[b, :, t, f]
    return buf


def _implicit_gemm(buf, wm, B, T, Fq, C):
    """y[m + F + 3] = sum_tap buf[tap_rows(m, tap)] . wm[:, tap C:(tap + 1) C]^T over the grid, junk rows zeroed."""
    R = V.grid_rows(B, T, Fq)
    m = np.arange(R)
    y = np.zeros((R + Fq + 3, wm.shape[0]))
    acc = np.zeros((R, wm.shape[0]))
    for tap in range(9):
        acc += buf[V.tap_rows(m, tap, Fq)] @ wm[:, tap * C:(tap + 1) * C].T
    acc[V.junk_rows(B, T, Fq)] = 0
    y[Fq + 3:] = acc
    return y


@pytest.mark.parametrize("T,Fq", [(4, 13), (8, 40), (6, 6)])
def test_junk_rows_land_on_the_halo(T, Fq):
    B = 2
    R = V.grid_rows(B, T, Fq)
    halo = np.ones(R + Fq + 3, bool)
    for b in range(B):
        for t in range(T):
            for f in range(Fq):
                halo[V.data_row(b, t, f, T, Fq)] = False
    junk = V.junk_rows(B, T, Fq)
    assert np.array_equal(halo[Fq + 3:], junk)          # output grid row m is written to buffer row m + F + 3
    assert halo[:Fq + 3].all()                          # rows the GEMM never writes: the head of the first utterance
    # the reads of the last grid row stay within R + 2 F + 6 rows (past the buffer: the tensor map's zero fill)
    assert V.tap_rows(R - 1, 8, Fq) == R + 2 * Fq + 5


@pytest.mark.parametrize("C,O", [(32, 64), (64, 32)])
def test_tap_packings_reproduce_conv2d_and_its_gradients(C, O):
    ops = _ops()
    B, T, Fq = 2, 6, 5
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, C, T, Fq, generator=g, dtype=torch.float64)
    w = torch.randn(O, C, 3, 3, generator=g, dtype=torch.float64)
    dy = torch.randn(B, O, T, Fq, generator=g, dtype=torch.float64)
    y = _implicit_gemm(_buffer(x.numpy()), ops._vgg_taps(w).numpy(), B, T, Fq, C)
    assert np.allclose(V.unpad(torch.from_numpy(y), B, T, Fq), F.conv2d(x, w, padding=1), rtol=0, atol=1e-12)
    dx = _implicit_gemm(_buffer(dy.numpy()), ops._vgg_taps_t(w).numpy(), B, T, Fq, O)
    ref = torch.nn.grad.conv2d_input(x.shape, w, dy, padding=1)
    assert np.allclose(V.unpad(torch.from_numpy(dx), B, T, Fq), ref, rtol=0, atol=1e-12)
    # weight gradient: dw[o][tap C + c] = sum_m dy[m + F + 3][o] x[tap_rows(m, tap)][c]
    R = V.grid_rows(B, T, Fq)
    xb, dyb = _buffer(x.numpy()), _buffer(dy.numpy())
    m = np.arange(R)
    dwm = np.concatenate([dyb[m + Fq + 3].T @ xb[V.tap_rows(m, tap, Fq)] for tap in range(9)], 1)
    dw = ops._vgg_untaps(torch.from_numpy(dwm), C)
    assert np.allclose(dw, torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=1), rtol=0, atol=1e-10)


def test_first_layer_im2col_order_matches_the_packed_weights():
    """k = tap C_in + c: the order vgg_im2col writes (restated here) pairs with ops._vgg_taps of the first conv."""
    ops = _ops()
    B, cin, T, Fq = 2, 3, 4, 13
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, cin, T, Fq, generator=g, dtype=torch.float64)
    w = torch.randn(64, cin, 3, 3, generator=g, dtype=torch.float64)
    xp = F.pad(x, (1, 1, 1, 1))
    R = V.grid_rows(B, T, Fq)
    col = np.zeros((R, 32))
    for mm in np.flatnonzero(~V.junk_rows(B, T, Fq)):
        f = mm % (Fq + 2)
        t = (mm // (Fq + 2)) % (T + 2)
        b = mm // ((Fq + 2) * (T + 2))
        for tap in range(9):
            col[mm, tap * cin:(tap + 1) * cin] = xp[b, :, t + tap // 3, f + tap % 3]
    wm = np.zeros((64, 32))
    wm[:, :9 * cin] = ops._vgg_taps(w).numpy()
    y = np.zeros((R + Fq + 3, 64))
    y[Fq + 3:] = col @ wm.T
    assert np.allclose(V.unpad(torch.from_numpy(y), B, T, Fq), F.conv2d(x, w, padding=1), rtol=0, atol=1e-12)
