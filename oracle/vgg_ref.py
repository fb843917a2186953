"""Float64 restatement of VGGExtractor (src/module.py:7-66) on plain torch ops, and the zero-haloed buffer geometry of the
GPU path (include/b200asr.h), for tests/test_gpu_vgg.py and tests/test_host_vgg_geometry.py.

Layout conventions here: activations [B, C, T, F] (NCHW, as the reference's nn.Conv2d sees them); params = the 8
tensors (w1, b1, ..., w4, b4) of extractor[0], [2], [5], [7]."""
import numpy as np
import torch
import torch.nn.functional as F


def view_input(feature, cin):
    """[B, T_in, cin * F] -> [B, cin, T, F] with T = T_in cropped to a multiple of 4 (view_input of the reference)."""
    B, T_in, D = feature.shape
    T = T_in - T_in % 4
    return feature[:, :T].reshape(B, T, cin, D // cin).transpose(1, 2)


def flatten_output(y):
    """[B, C, T', F'] -> [B, T', C F'] with index c F' + f."""
    B, C, T, Fq = y.shape
    return y.transpose(1, 2).reshape(B, T, C * Fq)


def forward(feature, cin, params, device="cpu"):
    """Every pre-activation a1..a4, activation y1..y4, pool output and the prenet output, in float64 on `device`."""
    w = [p.detach().double().to(device) for p in params]
    x = view_input(feature.detach().double().to(device), cin)
    r = {"x": x}
    r["a1"] = F.conv2d(x, w[0], w[1], padding=1)
    r["y1"] = torch.relu(r["a1"])
    r["a2"] = F.conv2d(r["y1"], w[2], w[3], padding=1)
    r["y2"] = torch.relu(r["a2"])
    r["p1"] = F.max_pool2d(r["y2"], 2, 2)
    r["a3"] = F.conv2d(r["p1"], w[4], w[5], padding=1)
    r["y3"] = torch.relu(r["a3"])
    r["a4"] = F.conv2d(r["y3"], w[6], w[7], padding=1)
    r["y4"] = torch.relu(r["a4"])
    r["p2"] = F.max_pool2d(r["y4"], 2, 2)
    r["out"] = flatten_output(r["p2"])
    return r


def pool_route(dp, idx, shape):
    """Max-pool backward routed by window indices idx (0..3 = 2 dt + df) [B, C, T/2, F/2] into a zero [B, C, T, F]."""
    g = torch.zeros(shape, dtype=dp.dtype, device=dp.device)
    T2, F2 = idx.shape[2], idx.shape[3]
    for k in range(4):
        g[:, :, k // 2:2 * T2:2, k % 2:2 * F2:2] += dp * (idx == k)
    return g


def routed_backward(inputs, masks, idx, params, dout, need_dx=True):
    """Float64 backward of the prenet that takes the ReLU masks (True = the gradient passes) and the max-pool window
    indices as given (the GPU's own), and the conv inputs [x, y1, p1, y3] as given (float64, on their device);
    returns the gradients of the 8 params and of x ([B, cin, T, F])."""
    x, y1, p1, y3 = inputs
    w = [p.detach().double().to(x.device) for p in params]
    m1, m2, m3, m4 = masks
    B, C4, T4, F4 = idx[1].shape
    dp2 = dout.double().to(x.device).reshape(B, T4, C4, F4).transpose(1, 2)
    d4 = pool_route(dp2, idx[1], m4.shape) * m4
    d3 = torch.nn.grad.conv2d_input(y3.shape, w[6], d4, padding=1) * m3
    dp1 = torch.nn.grad.conv2d_input(p1.shape, w[4], d3, padding=1)
    d2 = pool_route(dp1, idx[0], m2.shape) * m2
    d1 = torch.nn.grad.conv2d_input(y1.shape, w[2], d2, padding=1) * m1
    grads = []
    for inp, wt, d in ((x, w[0], d1), (y1, w[2], d2), (p1, w[4], d3), (y3, w[6], d4)):
        grads += [torch.nn.grad.conv2d_weight(inp, wt.shape, d, padding=1), d.sum((0, 2, 3))]
    dx = torch.nn.grad.conv2d_input(x.shape, w[0], d1, padding=1) if need_dx else None
    return grads, dx


# ---- geometry of the zero-haloed channels-last buffers (include/b200asr.h) -------------------------------------------
def grid_rows(B, T, Fq):
    return B * (T + 2) * (Fq + 2)


def junk_rows(B, T, Fq):
    """Boolean [R]: grid rows whose (t, f) is not a data position (t >= T or f >= F)."""
    m = np.arange(grid_rows(B, T, Fq))
    t = (m // (Fq + 2)) % (T + 2)
    f = m % (Fq + 2)
    return (t >= T) | (f >= Fq)


def tap_rows(m, tap, Fq):
    """Row of the input buffer that tap (3 dt + df) of output grid row m reads."""
    return m + (tap // 3) * (Fq + 2) + tap % 3


def data_row(b, t, f, T, Fq):
    """Buffer row of data position (b, t, f)."""
    return (b * (T + 2) + t + 1) * (Fq + 2) + f + 1


def unpad(buf, B, T, Fq):
    """Zero-haloed buffer [R + F + 3, C] -> [B, C, T, F]."""
    R = grid_rows(B, T, Fq)
    return buf[:R].reshape(B, T + 2, Fq + 2, -1)[:, 1:T + 1, 1:Fq + 1].permute(0, 3, 1, 2)
