"""torch.autograd wrappers around the C-ABI kernels (host-side plumbing; the arithmetic is in csrc/)."""
import ctypes
import os

import torch
from torch.autograd import Function

from . import lib as L


def _f32c(t):
    if t.dtype != torch.float32:
        raise L.B200AsrError("b200asr kernels compute in fp32 (got %s)" % t.dtype)
    return t if t.is_contiguous() else t.contiguous()


def _gemm_exact():
    """Plain library GEMMs (cuBLAS through torch) must run in true fp32 for the 1e-4 parity budget."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


_gemm_exact()

_perm_cache = {}


def gate_perm(H, device):
    """Row permutation from PyTorch's gate-major [i|f|g|o] layout to the kernels' unit-major layout:
    new row j*4+g  <-  old row g*H+j."""
    key = (H, str(device))
    p = _perm_cache.get(key)
    if p is None:
        p = torch.arange(4 * H, device=device).view(4, H).t().reshape(-1).contiguous()
        _perm_cache[key] = p
    return p


# ----------------------------------------------------------------------------------------------------------
# Dense contractions of the step (K6 / K9 / K11 and their autograd backward).  fp32 parity (1e-4 on logits after 4
# recurrent layers) rules out single-pass TF32/BF16, so every product is error-compensated (fp32 class).  Which
# implementation runs follows from the shapes alone:
# - The four contractions of a BiLSTM layer (input projection, dX, dW_ih, dW_hh) run on scaled fp16 hi/lo images
#   (f16_split / f16_split_t + gemm_f16x3: three fp16 tensor-core products, twice the 3xTF32 rate) when the input width
#   is a multiple of 4, else as three cuBLAS TF32 GEMMs on operands split by b200asr_split_tf32 (Split + mm3).
# - Every other dense contraction (Conv1d prenet, Linear3xFn, CTC head, decoder step, tied LM projection) runs on this
#   library's own 3xTF32 wgmma kernel (csrc/gemm.cu) in its three operand forms -
#   gemm_tn  x . W^T (+ bias)   forward;   gemm_nn  dY . W   input gradient (W in place);   gemm_nt  dY^T . X   weight
#   gradient (contraction over the B*T rows, h_prev read shifted from the layer output, gate permutation in the epilogue).
#   A is split into hi / lo in registers (wgmma with A from registers); B's raw fp32 tile is its TF32 hi operand and
#   its residual is made on the fly in shared memory, and the MMA accumulation chain is cut every 128 k and summed in
#   a second fp32 register tile.
#   The K-major w of gemm_tn may bring its residual pre-computed (tf32_residual: the weights, once per
#   step); an MN-major B (w of gemm_nn, b of gemm_nt) passes through the kernel's transposing pass, which makes its
#   residual anyway, and gemm_nt's a is gathered into registers with transposed addressing, so those forms take none.
#   Shapes the kernel does not take (a row pitch that is not a multiple of 4 floats) go through Split + mm3.


def tf32_residual(w):
    """w - trunc_tf32(w): the part of a weight matrix the tensor core does not see in the raw fp32 bit pattern.  Computed
    once per step and weight (instead of once per tile by every CTA) for the pre-split forms of gemm_tn."""
    lib = L.load()
    w = _f32c(w)
    lo = torch.empty_like(w)
    with L.timed("tf32_residual", 8 * w.numel()):
        L.check(lib.b200asr_tf32_residual(L.ptr(w), L.ptr(lo), w.numel(), L.stream()), "tf32_residual")
    return lo


def gemm_tn(a, w, bias=None, out=None, accumulate=False, w_lo=None):
    """out[M,N] (= or +=) a[M,K] @ w[N,K]^T (+ bias[N]) on the tensor cores at fp32-class accuracy (csrc/gemm.cu).
    w_lo = tf32_residual(w) selects the pre-split form."""
    lib = L.load()
    a, w = _f32c(a), _f32c(w)
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=torch.float32)
        accumulate = False
    assert out.stride(1) == 1 and out.shape == (M, N)
    b = _f32c(bias) if bias is not None else None
    ws, ws_bytes = None, 0
    # split-K over all SMs for a small tile grid: pre-split calls and skinny ones (the decoder's per-step products)
    if w_lo is not None or M <= 256:
        ws_bytes = lib.b200asr_gemm3x_workspace_bytes(M, N)
        ws = torch.empty(max(ws_bytes, 16), device=a.device, dtype=torch.uint8)
    # algorithmic bytes: both operands and the result once; flops 2*M*N*K (x3 tensor-core products)
    with L.timed("gemm3x_tn", 4 * (M * K + N * K + M * N * (2 if accumulate else 1))):
        L.check(lib.b200asr_gemm3x_tn(L.ptr(a), K, L.ptr(w), L.ptr(w_lo), L.ptr(b), L.ptr(out), M, N, K, out.stride(0),
                                      int(bool(accumulate)), L.ptr(ws), ws_bytes, L.stream()), "gemm3x_tn")
    return out


def gemm_tn_ld(a_base, lda, M, K, w, bias=None):
    """Like gemm_tn but A is given as (base tensor, row pitch lda in floats, M rows of K floats): rows may overlap."""
    lib = L.load()
    w = _f32c(w)
    N = w.shape[0]
    out = torch.empty((M, N), device=w.device, dtype=torch.float32)
    b = _f32c(bias) if bias is not None else None
    with L.timed("gemm3x_tn", 4 * (M * lda + N * K + M * N)):
        L.check(lib.b200asr_gemm3x_tn(L.ptr(a_base), lda, L.ptr(w), None, L.ptr(b), L.ptr(out), M, N, K, N, 0, None, 0,
                                      L.stream()), "gemm3x_tn")
    return out


def gemm_nn(a, w, out=None, accumulate=False):
    """out[M,N] (= or +=) a[M,K] @ w[K,N]: the input gradient dY . W with W read in place (MN-major operand)."""
    lib = L.load()
    a, w = _f32c(a), _f32c(w)
    M, K = a.shape
    N = w.shape[1]
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=torch.float32)
        accumulate = False
    assert out.stride(1) == 1 and out.shape == (M, N)
    ws, ws_bytes = None, 0
    if M <= 256:                        # skinny: split-K as in gemm_tn
        ws_bytes = lib.b200asr_gemm3x_workspace_bytes(M, N)
        ws = torch.empty(max(ws_bytes, 16), device=a.device, dtype=torch.uint8)
    with L.timed("gemm3x_nn", 4 * (M * K + N * K + M * N * (2 if accumulate else 1))):
        L.check(lib.b200asr_gemm3x_nn(L.ptr(a), K, L.ptr(w), N, None, L.ptr(out), M, N, K, out.stride(0),
                                      int(bool(accumulate)), L.ptr(ws), ws_bytes, L.stream()), "gemm3x_nn")
    return out


def gemm_nt(a, b, M, N, T, batches=1, lda=None, a_bstride=0, ldb=None, b_bstride=0, b_shift=0, permute_rows=False,
            out=None, accumulate=False):
    """out[M,N] (= or +=) sum over (batch, t) of a[batch, t, :M]^T b[batch, t + b_shift, :N]: the weight gradient
    dY^T . X.  `a` / `b` are tensors whose data pointer is element (0, 0, 0); pitches are in floats (default: dense
    [T, M] / [T, N]).  A given `out` must be a contiguous [M, N] fp32 tensor (e.g. a parameter's gradient view)."""
    lib = L.load()
    lda = M if lda is None else lda
    ldb = N if ldb is None else ldb
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=torch.float32)
        accumulate = False
    assert out.is_contiguous() and out.dtype == torch.float32 and out.numel() == M * N
    ws_bytes = lib.b200asr_gemm3x_workspace_bytes(M, N)
    ws = torch.empty(max(ws_bytes, 16), device=a.device, dtype=torch.uint8)
    with L.timed("gemm3x_nt", 4 * (batches * T * (M + N) + M * N * (2 if accumulate else 1))):
        L.check(lib.b200asr_gemm3x_nt(L.ptr(a), lda, a_bstride, 0, L.ptr(b), ldb, b_bstride, b_shift, L.ptr(out), M, N,
                                      T, batches, N, int(bool(accumulate)), int(bool(permute_rows)), L.ptr(ws),
                                      ws_bytes, L.stream()),
                "gemm3x_nt")
    return out


def f16_split(x, rows, K, ld=None):
    """K-major fp32 operand x[rows, K] (row pitch ld) -> f16x3 operand (img, sinv): img[0] / img[1] = the hi / lo fp16
    images [rows, Kp] (K zero-padded to the 128-k scale chunk), sinv[Kp // 128, rows] = the inverse chunk scales."""
    lib = L.load()
    ld = K if ld is None else ld
    Kp = lib.b200asr_f16x3_padded_k(K)
    img = torch.empty((2, rows, Kp), device=x.device, dtype=torch.float16)
    sinv = torch.empty((Kp // 128, rows), device=x.device, dtype=torch.float32)
    with L.timed("f16_split", 4 * rows * K + 4 * rows * Kp):
        L.check(lib.b200asr_f16x3_split_rows(L.ptr(x), ld, rows, K, L.ptr(img[0]), L.ptr(img[1]), L.ptr(sinv),
                                             L.stream()), "f16x3_split_rows")
    return img, sinv


def f16_split_t(x, cols, T, batches=1, ld=None, bstride=0, shift=0):
    """MN-major fp32 operand (element (b, t, c) at x[b*bstride + (t+shift)*ld + c], zero where t+shift is outside
    [0, T); `x`'s data pointer is element (0, 0, 0)) -> f16x3 operand of its transpose: images [2, cols, Rp] over the
    R = batches*T contraction rows, sinv[Rp // 128, cols]."""
    lib = L.load()
    ld = cols if ld is None else ld
    Rp = lib.b200asr_f16x3_padded_k(batches * T)
    img = torch.empty((2, cols, Rp), device=x.device, dtype=torch.float16)
    sinv = torch.empty((Rp // 128, cols), device=x.device, dtype=torch.float32)
    with L.timed("f16_split", 4 * batches * T * cols + 4 * cols * Rp):
        L.check(lib.b200asr_f16x3_split_cols(L.ptr(x), ld, bstride, shift, T, batches, cols, L.ptr(img[0]),
                                             L.ptr(img[1]), L.ptr(sinv), L.stream()), "f16x3_split_cols")
    return img, sinv


def f16_split_dg(g, row_images=True):
    """Gate gradient g[ndir, R, C] (contiguous) read once -> (per direction d the f16_split_t operand of g[d], the
    f16_split operand of all directions side by side or None, column sums [ndir, C]).  The row operand's images are
    [2, R, ndir * Kp] with direction d in columns [d * Kp, (d + 1) * Kp) (Kp = C padded to the scale chunk) and its
    sinv [ndir * Kp // 128, R]; the column sums add per-128-row-tile partial sums in a fixed order (no atomics)."""
    lib = L.load()
    assert g.is_contiguous() and g.dim() == 3
    ndir, R, C = g.shape
    Rp, Kp = lib.b200asr_f16x3_padded_k(R), lib.b200asr_f16x3_padded_k(C)
    timg = torch.empty((2, ndir, C, Rp), device=g.device, dtype=torch.float16)
    tsinv = torch.empty((ndir, Rp // 128, C), device=g.device, dtype=torch.float32)
    rimg = rsinv = None
    if row_images:
        rimg = torch.empty((2, R, ndir * Kp), device=g.device, dtype=torch.float16)
        rsinv = torch.empty((ndir * Kp // 128, R), device=g.device, dtype=torch.float32)
    part = torch.empty((Rp // 128, ndir * C), device=g.device, dtype=torch.float32)
    nbytes = 4 * ndir * (R * C + C * Rp + (R * Kp if row_images else 0)) + 4 * part.numel()
    with L.timed("f16_split_dg", nbytes):
        L.check(lib.b200asr_f16x3_split_dg(L.ptr(g), ndir, R, C, L.ptr(timg[0]), L.ptr(timg[1]), L.ptr(tsinv),
                                           L.ptr(rimg[0] if row_images else None),
                                           L.ptr(rimg[1] if row_images else None), L.ptr(rsinv), L.ptr(part),
                                           L.stream()), "f16x3_split_dg")
    return ([(timg[:, d], tsinv[d]) for d in range(ndir)], (rimg, rsinv) if row_images else None,
            part.sum(0).view(ndir, C))


def f16_split_cat_t(ws, Kp):
    """f16_split operand of [w_0^T | w_1^T | ...] (w_d [C, N]) with each block's C columns zero-padded to Kp: the B
    operand that pairs with f16_split_dg's row images, so that sum_d g_d . w_d is one contraction over all blocks."""
    C, N = ws[0].shape
    wt = torch.zeros((N, len(ws), Kp), device=ws[0].device, dtype=torch.float32)
    for d, w in enumerate(ws):
        wt[:, d, :C] = w.t()
    return f16_split(wt.view(N, len(ws) * Kp), N, len(ws) * Kp)


def gemm_f16x3(a, b, bias=None, out=None, accumulate=False, permute_rows=False, name="gemm_f16_tn"):
    """out[M,N] (= or +=) A . B^T (+ bias[N]) for two f16x3 operands (f16_split / f16_split_t with the same Kp):
    fp32-class products on the fp16 tensor cores (csrc/gemm.cu).  permute_rows writes row m to (m%4)*(M/4) + m/4."""
    lib = L.load()
    (aimg, asinv), (bimg, bsinv) = a, b
    M, Kp = aimg.shape[1], aimg.shape[2]
    N = bimg.shape[1]
    assert bimg.shape[2] == Kp
    if out is None:
        out = torch.empty((M, N), device=aimg.device, dtype=torch.float32)
        accumulate = False
    assert out.dtype == torch.float32 and out.stride(1) == 1 and out.shape == (M, N)
    ws_bytes = lib.b200asr_gemm3x_workspace_bytes(M, N)
    ws = torch.empty(max(ws_bytes, 16), device=aimg.device, dtype=torch.uint8)
    bb = _f32c(bias) if bias is not None else None
    with L.timed(name, 4 * Kp * (M + N) + 4 * M * N * (2 if accumulate else 1)):
        L.check(lib.b200asr_gemm_f16x3(L.ptr(aimg[0]), L.ptr(aimg[1]), L.ptr(asinv), L.ptr(bimg[0]), L.ptr(bimg[1]),
                                       L.ptr(bsinv), L.ptr(bb), L.ptr(out), M, N, Kp, out.stride(0),
                                       int(bool(accumulate)), int(bool(permute_rows)), L.ptr(ws), ws_bytes,
                                       L.stream()), "gemm_f16x3")
    return out


class Conv1dK4S2Fn(Function):
    """Conv1d(C -> O, kernel 4, stride 2, padding 1) over [B, T, C] (CNNExtractor, src/module.py:75-78) as ONE
    tensor-core GEMM: with one zero row in front of every utterance, output frame t reads the 4*C CONTIGUOUS floats that
    start at padded row 2t, so the im2col matrix is just the padded buffer viewed with row pitch 2*C (overlapping rows)
    and the TMA tensor map reads it in place.  Input gradient = GEMM + an overlap-add of the two window halves."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x = _f32c(x)
        B, T, C = x.shape
        O = weight.shape[0]
        Tout = T // 2
        Tp = 2 * (Tout + 1)                                   # padded rows per utterance (even)
        xp = torch.zeros((B, Tp, C), device=x.device, dtype=torch.float32)
        xp[:, 1:T + 1] = x
        wm = weight.detach().permute(0, 2, 1).reshape(O, 4 * C).contiguous()    # K index = tap * C + channel
        M = B * (Tp // 2) - 1                                 # the last row of the view would read past the buffer
        yf = torch.empty((B * (Tp // 2), O), device=x.device, dtype=torch.float32)
        yf[M:] = 0
        yf[:M] = gemm_tn_ld(xp, 2 * C, M, 4 * C, wm, bias.detach() if bias is not None else None)
        ctx.save_for_backward(xp, wm)
        ctx.dims = (B, T, C, O, Tout, Tp, M)
        ctx.has_bias = bias is not None
        return yf.view(B, Tp // 2, O)[:, :Tout]

    @staticmethod
    def backward(ctx, dy):
        xp, wm = ctx.saved_tensors
        B, T, C, O, Tout, Tp, M = ctx.dims
        half = Tp // 2
        dyf = torch.zeros((B, half, O), device=dy.device, dtype=torch.float32)
        dyf[:, :Tout] = dy
        dy2 = dyf.view(B * half, O)
        dx = None
        if ctx.needs_input_grad[0]:
            dcols = gemm_nn(dy2, wm).view(B, half, 2, 2 * C)      # [.., 0]: rows 2t,2t+1  [.., 1]: 2t+2,2t+3
            dxp = torch.zeros((B, half + 1, 2 * C), device=dy.device, dtype=torch.float32)
            dxp[:, :half] += dcols[:, :, 0]
            dxp[:, 1:] += dcols[:, :, 1]
            dx = dxp.view(B, Tp + 2, C)[:, 1:T + 1].contiguous()
        dw = db = None
        if ctx.needs_input_grad[1]:
            dwm = gemm_nt(dy2, xp, O, 4 * C, M, ldb=2 * C)                          # [O, 4C], windows read in place
            dw = dwm.view(O, 4, C).permute(0, 2, 1).contiguous()
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.reshape(-1, O).sum(0)
        return dx, dw, db


def conv1d_k4s2p1(x, conv):
    """[B,T,C] -> [B,T//2,O] through the tensor-core GEMM when available, else the library convolution."""
    C = x.shape[-1]
    if (x.is_cuda and conv.kernel_size == (4,) and conv.stride == (2,) and conv.padding == (1,) and x.shape[1] >= 2
            and (2 * C) % 4 == 0):
        return Conv1dK4S2Fn.apply(x, conv.weight, conv.bias)
    return conv(x.transpose(1, 2)).transpose(1, 2)


def _vgg_buffer(B, T, F, C, device, zero_head=False):
    """Zero-haloed channels-last buffer of a (T, F) activation: R = B (T+2) (F+2) grid rows plus F + 3 trailing rows
    (include/b200asr.h).  zero_head zeroes the F + 3 rows in front of the first position, which a conv3x3_fwd output
    does not write."""
    buf = torch.empty((B * (T + 2) * (F + 2) + F + 3, C), device=device, dtype=torch.float32)
    if zero_head:
        buf[:F + 3].zero_()
    return buf


def conv3x3(x, C, taps, w, B, T, F, bias=None, mask=None, relu=False):
    """3x3 convolution (padding 1) of the zero-haloed buffer x of (T, F) -> a new buffer of w.shape[0] channels: one
    implicit-GEMM launch (b200asr_conv3x3_fwd); taps = 1 reads x as the first layer's [R, 32] im2col."""
    lib = L.load()
    O = w.shape[0]
    y = _vgg_buffer(B, T, F, O, w.device, zero_head=True)
    with L.timed("conv3x3_fwd", 4 * (x.numel() + w.numel() + y.numel() * (2 if mask is not None else 1))):
        L.check(lib.b200asr_conv3x3_fwd(L.ptr(x), C, taps, L.ptr(w), L.ptr(bias), L.ptr(mask), int(relu), L.ptr(y), B,
                                        T, F, O, L.stream()), "conv3x3_fwd")
    return y


def conv3x3_wgrad(dy, x, C, taps, B, T, F):
    """dW [O, taps * C] (tap-major K) of a 3x3 convolution from the padded dY and its input buffer (b200asr_conv3x3_wgrad,
    split-K over the grid rows)."""
    lib = L.load()
    O = dy.shape[1]
    dw = torch.empty((O, taps * C), device=dy.device, dtype=torch.float32)
    ws_bytes = lib.b200asr_gemm3x_workspace_bytes(O, taps * C)
    ws = torch.empty(max(ws_bytes, 16), device=dy.device, dtype=torch.uint8)
    with L.timed("conv3x3_wgrad", 4 * (dy.numel() + x.numel() + dw.numel())):
        L.check(lib.b200asr_conv3x3_wgrad(L.ptr(dy), L.ptr(x), C, taps, L.ptr(dw), B, T, F, O, L.ptr(ws), ws_bytes,
                                          L.stream()), "conv3x3_wgrad")
    return dw


def _vgg_taps(w):
    """[O, C, 3, 3] -> [O, 9 C] with K = tap * C + c."""
    return w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def _vgg_taps_t(w):
    """Weights of the input gradient: [O, C, 3, 3] -> [C, 9 O], flipped taps (w'[c][tap' O + o] = w[o][c][2-dt'][2-df'])."""
    return w.detach().flip(2, 3).permute(1, 2, 3, 0).reshape(w.shape[1], -1).contiguous()


def _vgg_untaps(dw, C):
    """[O, 9 C] tap-major -> [O, C, 3, 3]."""
    return dw.view(dw.shape[0], 3, 3, C).permute(0, 3, 1, 2).contiguous()


class VGGFn(Function):
    """VGGExtractor.extractor (src/module.py:7-66) on [B, T_in, Cin * F] features: T = T_in cropped to a multiple of 4,
    2 x (conv3x3 -> ReLU -> conv3x3 -> ReLU -> MaxPool 2x2), output [B, T / 4, 128 * (F / 2 / 2)] with index c F' + f.
    Each convolution, its input gradient and its weight gradient is one launch of the conv-mode 3xTF32 GEMM over
    zero-haloed channels-last buffers (csrc/gemm.cu); bias + ReLU, the ReLU backward mask and the halo zeros are in its
    epilogue.  The first conv (Cin <= 3) reads a staged [R, 32] im2col; max-pool forward / backward and the feature
    gradient are csrc/vgg.cu; the bias gradients are column sums of the padded dY (zeros off the data)."""

    @staticmethod
    def forward(ctx, feature, Cin, w1, b1, w2, b2, w3, b3, w4, b4):
        lib = L.load()
        feature = _f32c(feature)
        B, T_in, D = feature.shape
        F = D // Cin
        T = T_in - T_in % 4
        T2, F2 = T // 2, F // 2
        dev = feature.device
        x0 = torch.empty((B * (T + 2) * (F + 2), 32), device=dev, dtype=torch.float32)
        with L.timed("vgg_im2col", 4 * (B * T * D + x0.numel())):
            L.check(lib.b200asr_vgg_im2col(L.ptr(feature), T_in * D, B, T, Cin, F, L.ptr(x0), L.stream()), "vgg_im2col")
        wm1 = torch.zeros((w1.shape[0], 32), device=dev, dtype=torch.float32)
        wm1[:, :9 * Cin] = _vgg_taps(w1)
        y1 = conv3x3(x0, 32, 1, wm1, B, T, F, bias=_f32c(b1.detach()), relu=True)
        y2 = conv3x3(y1, y1.shape[1], 9, _vgg_taps(w2), B, T, F, bias=_f32c(b2.detach()), relu=True)
        p1 = _vgg_buffer(B, T2, F2, y2.shape[1], dev)
        i1 = torch.empty((B, T2, F2, y2.shape[1]), device=dev, dtype=torch.uint8)
        with L.timed("vgg_pool_fwd", 4 * (y2.numel() + p1.numel()) + i1.numel()):
            L.check(lib.b200asr_vgg_pool_fwd(L.ptr(y2), B, T, F, y2.shape[1], L.ptr(p1), L.ptr(i1), 0, L.stream()),
                    "vgg_pool_fwd")
        y3 = conv3x3(p1, p1.shape[1], 9, _vgg_taps(w3), B, T2, F2, bias=_f32c(b3.detach()), relu=True)
        y4 = conv3x3(y3, y3.shape[1], 9, _vgg_taps(w4), B, T2, F2, bias=_f32c(b4.detach()), relu=True)
        C4 = y4.shape[1]
        out = torch.empty((B, T2 // 2, C4 * (F2 // 2)), device=dev, dtype=torch.float32)
        i2 = torch.empty((B, T2 // 2, F2 // 2, C4), device=dev, dtype=torch.uint8)
        with L.timed("vgg_pool_fwd", 4 * (y4.numel() + out.numel()) + i2.numel()):
            L.check(lib.b200asr_vgg_pool_fwd(L.ptr(y4), B, T2, F2, C4, L.ptr(out), L.ptr(i2), 1, L.stream()),
                    "vgg_pool_fwd")
        ctx.save_for_backward(x0, y1, y2, p1, y3, y4, i1, i2, w1, w2, w3, w4)
        ctx.dims = (B, T_in, T, F, Cin)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.load()
        x0, y1, y2, p1, y3, y4, i1, i2, w1, w2, w3, w4 = ctx.saved_tensors
        B, T_in, T, F, Cin = ctx.dims
        T2, F2 = T // 2, F // 2
        dout = _f32c(dout)
        dev = dout.device

        def pool_bwd(dsrc, idx, y, T_, F_, flat):
            dy = torch.empty_like(y)
            with L.timed("vgg_pool_bwd", 4 * (dsrc.numel() + 2 * y.numel()) + idx.numel()):
                L.check(lib.b200asr_vgg_pool_bwd(L.ptr(dsrc), L.ptr(idx), L.ptr(y), B, T_, F_, y.shape[1], L.ptr(dy),
                                                 flat, L.stream()), "vgg_pool_bwd")
            return dy

        dy4 = pool_bwd(dout, i2, y4, T2, F2, 1)
        dw4 = _vgg_untaps(conv3x3_wgrad(dy4, y3, y3.shape[1], 9, B, T2, F2), y3.shape[1])
        dy3 = conv3x3(dy4, dy4.shape[1], 9, _vgg_taps_t(w4), B, T2, F2, mask=y3)
        dw3 = _vgg_untaps(conv3x3_wgrad(dy3, p1, p1.shape[1], 9, B, T2, F2), p1.shape[1])
        dp1 = conv3x3(dy3, dy3.shape[1], 9, _vgg_taps_t(w3), B, T2, F2)
        dy2 = pool_bwd(dp1, i1, y2, T, F, 0)
        dw2 = _vgg_untaps(conv3x3_wgrad(dy2, y1, y1.shape[1], 9, B, T, F), y1.shape[1])
        dy1 = conv3x3(dy2, dy2.shape[1], 9, _vgg_taps_t(w2), B, T, F, mask=y1)
        dw1 = conv3x3_wgrad(dy1, x0, 32, 1, B, T, F)[:, :9 * Cin]
        dw1 = dw1.reshape(dw1.shape[0], 3, 3, Cin).permute(0, 3, 1, 2).contiguous()
        dfeat = None
        if ctx.needs_input_grad[0]:
            dfeat = torch.empty((B, T_in, Cin * F), device=dev, dtype=torch.float32)
            with L.timed("vgg_feat_grad", 4 * (dy1.numel() + dfeat.numel())):
                L.check(lib.b200asr_vgg_feat_grad(L.ptr(dy1), L.ptr(_f32c(w1.detach())), B, T, T_in, Cin, F,
                                                  w1.shape[0], L.ptr(dfeat), L.stream()), "vgg_feat_grad")
        return (dfeat, None, dw1, dy1.sum(0), dw2, dy2.sum(0), dw3, dy3.sum(0), dw4, dy4.sum(0))


def vgg_extractor(feature, feat_len, extractor, in_channel):
    """VGGExtractor's forward on CUDA features [B, T_in, in_channel * F] -> ([B, T_in // 4, 128 * (F // 4)],
    feat_len // 4).  Fewer than 4 frames cannot be convolved (the library path fails inside ATen): refused here, before
    any launch."""
    if feature.shape[1] < 4:
        raise ValueError("VGGExtractor needs at least 4 frames per batch (time is cropped to a multiple of 4 and pooled "
                         "twice); got a batch of %d frames" % feature.shape[1])
    c1, c2, c3, c4 = extractor[0], extractor[2], extractor[5], extractor[7]
    out = VGGFn.apply(feature, in_channel, c1.weight, c1.bias, c2.weight, c2.bias, c3.weight, c3.bias, c4.weight,
                      c4.bias)
    return out, feat_len // 4


class Split:
    """fp32 matrix as (hi, lo) with hi exactly representable in TF32."""

    def __init__(self, x):
        lib = L.load()
        x = _f32c(x)
        self.hi = torch.empty_like(x)
        self.lo = torch.empty_like(x)
        with L.timed("split_tf32", 12 * x.numel()):
            L.check(lib.b200asr_split_tf32(L.ptr(x), L.ptr(self.hi), L.ptr(self.lo), x.numel(), L.stream()),
                    "split_tf32")

    def t(self):
        o = object.__new__(Split)
        o.hi, o.lo = self.hi.t(), self.lo.t()
        return o

    def view(self, *shape):
        o = object.__new__(Split)
        o.hi, o.lo = self.hi.view(*shape), self.lo.view(*shape)
        return o


def mm3(a, b, out=None, bias=None, accumulate=False):
    """out (= or +=) a @ b (+ bias) for Split operands: three error-compensated TF32 tensor-core GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        if out is None:
            out = torch.empty((a.hi.shape[0], b.hi.shape[1]), device=a.hi.device, dtype=torch.float32)
            accumulate = False
        if accumulate:
            out.addmm_(a.lo, b.hi)
        elif bias is not None:
            torch.addmm(bias, a.lo, b.hi, out=out)
        else:
            torch.mm(a.lo, b.hi, out=out)
        out.addmm_(a.hi, b.lo)
        out.addmm_(a.hi, b.hi)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def _rnn_layer_fwd(ctx, cell, x, ndir, w_ih, w_hh, bias):
    """Forward of one (bi)directional LSTM or GRU layer on the 4-slot gate layout (BiLSTMFn, BiGRUFn): per direction
    w_ih[d] [4H, I], w_hh[d] [4H, H] and bias[d] [4H], gate-major and detached -> (out [B, T, ndir*H], state stash
    [ndir, B, T, H]: c (LSTM) / h (GRU) after every step).  Saves what _rnn_layer_bwd needs on ctx."""
    lib = L.load()
    x = _f32c(x)
    B, T, I = x.shape
    H = w_hh[0].shape[1]
    dev = x.device
    ws_bytes = lib.b200asr_bilstm_workspace_bytes(B, T, H, ndir)
    if ws_bytes == 0:
        raise L.B200AsrError("bi%s: no feasible decomposition for B=%d H=%d (H must be a multiple of 16)"
                             % (cell.lower(), B, H))
    perm = gate_perm(H, dev)
    f16 = I % 4 == 0
    # one operand of x serves both directions
    xo = f16_split(x.view(B * T, I), B * T, I) if f16 else Split(x.view(B * T, I))
    gates = torch.empty((ndir, B, T, H, 4), device=dev, dtype=torch.float32)
    w_ih_p = []
    for d in range(ndir):
        wp = w_ih[d].index_select(0, perm)
        bp = bias[d].index_select(0, perm)
        if f16:
            gemm_f16x3(xo, f16_split(wp, 4 * H, I), bias=bp, out=gates[d].view(B * T, 4 * H))
        else:
            mm3(xo, Split(wp).t(), out=gates[d].view(B * T, 4 * H), bias=bp)
        w_ih_p.append(wp)
    del xo
    w_hh = torch.stack([_f32c(w) for w in w_hh]).contiguous()
    cst = torch.empty((ndir, B, T, H), device=dev, dtype=torch.float32)
    out = torch.empty((B, T, ndir * H), device=dev, dtype=torch.float32)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    fn, name = (lib.b200asr_bilstm_fwd, "bilstm_fwd") if cell == "LSTM" else (lib.b200asr_bigru_fwd, "bigru_fwd")
    # algorithmic bytes (SURVEY.md 8(d)): per step and direction read Gx[t] (16BH) + write h,c (8BH); W_hh once
    with L.timed(name, ndir * (24 * B * H * T + 16 * H * H)):
        L.check(fn(L.ptr(gates), L.ptr(w_hh), L.ptr(cst), L.ptr(out), B, T, H, ndir, L.ptr(ws), ws_bytes, L.stream()),
                name)
    ctx.cell = cell
    ctx.ndir = ndir
    ctx.dims = (B, T, I, H)
    ctx.consumed = False
    ctx.save_for_backward(x, gates, cst, out, w_hh, *w_ih_p)
    return out, cst


def _rnn_layer_bwd(ctx, dout):
    """Backward of _rnn_layer_fwd -> (dx [B, T, I] or None, per direction (dw_ih [4H, I], dw_hh [4H, H], db [4H]) in
    the gate-major 4-slot layout)."""
    lib = L.load()
    if ctx.consumed:
        raise L.B200AsrError("%s.backward ran twice: the gate stash is overwritten in place"
                             % ("BiLSTMFn" if ctx.cell == "LSTM" else "BiGRUFn"))
    ctx.consumed = True
    ndir = ctx.ndir
    B, T, I, H = ctx.dims
    x, gates, cst, out, w_hh = ctx.saved_tensors[:5]
    w_ih_p = ctx.saved_tensors[5:5 + ndir]
    dev = x.device
    dout = _f32c(dout)
    ws_bytes = lib.b200asr_bilstm_workspace_bytes(B, T, H, ndir)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    fn, name = (lib.b200asr_bilstm_bwd, "bilstm_bwd") if ctx.cell == "LSTM" else (lib.b200asr_bigru_bwd, "bigru_bwd")
    with L.timed(name, 2 * ndir * (24 * B * H * T + 16 * H * H)):
        L.check(fn(L.ptr(gates), L.ptr(w_hh), L.ptr(cst), L.ptr(dout), B, T, H, ndir, L.ptr(ws), ws_bytes,
                   L.stream()), name)
    perm = gate_perm(H, dev)
    need_dx = ctx.needs_input_grad[0]
    dx2 = torch.empty((B * T, I), device=dev, dtype=torch.float32) if need_dx else None
    f16 = I % 4 == 0
    if f16:
        xt = f16_split_t(x, I, B * T)
        # dG (d(loss)/d(pre-activation), unit-major columns) of both directions read once: its transposed images,
        # its row images and its column sums (the bias gradient)
        gts, grow, gsum = f16_split_dg(gates.view(ndir, B * T, 4 * H), row_images=need_dx)
        if need_dx:
            # dX = sum_d dG_d . W_d as one contraction over both directions
            gemm_f16x3(grow, f16_split_cat_t(w_ih_p, grow[0].shape[2] // ndir), out=dx2)
            del grow
    else:
        xs = Split(x.view(B * T, I))
    grads = []
    for d in range(ndir):
        g2 = gates[d].view(B * T, 4 * H)      # d(loss)/d(pre-activation), unit-major columns
        hd = out[:, :, d * H:(d + 1) * H]
        if f16:
            # dW_ih = dG^T . X and dW_hh = dG^T . h_prev on transposed images (h_prev's written shifted by one step
            # per utterance, zero at the sequence ends); rows written through the gate permutation by the epilogue.
            gt = gts[d]
            dw_ih = gemm_f16x3(gt, xt, permute_rows=True, name="gemm_f16_nt")
            ht = f16_split_t(hd, H, T, batches=B, ld=ndir * H, bstride=T * ndir * H, shift=(-1 if d == 0 else 1))
            dw_hh = gemm_f16x3(gt, ht, permute_rows=True, name="gemm_f16_nt")
            del gt, ht
        else:
            dG = Split(g2)
            if need_dx:
                mm3(dG, Split(w_ih_p[d]), out=dx2, accumulate=(d > 0))
            dw_ih = torch.empty((4 * H, I), device=dev, dtype=torch.float32)
            dw_ih.index_copy_(0, perm, mm3(dG.t(), xs))
            # h_{prev}: the hidden state of the previous step of this direction (zero at its first step)
            hprev = torch.zeros((B, T, H), device=dev, dtype=torch.float32)
            if T > 1:
                if d == 0:
                    hprev[:, 1:] = hd[:, :-1]
                else:
                    hprev[:, :-1] = hd[:, 1:]
            dw_hh = torch.empty((4 * H, H), device=dev, dtype=torch.float32)
            dw_hh.index_copy_(0, perm, mm3(dG.t(), Split(hprev.view(B * T, H))))
            del dG, hprev
        db = torch.empty((4 * H,), device=dev, dtype=torch.float32)
        db.index_copy_(0, perm, gsum[d] if f16 else g2.sum(0))
        grads.append((dw_ih, dw_hh, db))
    return (dx2.view(B, T, I) if need_dx else None), grads


class BiLSTMFn(Function):
    """One (bi)directional LSTM layer over zero-padded frames, zero initial state (src/module.py:129-132).

    forward(x[B,T,I], ndir, w_ih_0, w_hh_0, b_ih_0, b_hh_0 [, w_ih_1, w_hh_1, b_ih_1, b_hh_1]) -> out[B,T,ndir*H]
    The input projection and the weight-gradient contractions are tensor-core GEMMs: f16x3 when I % 4 == 0, else the
    cuBLAS 3xTF32 composition (Split + mm3); the recurrence (forward and BPTT) is the persistent kernel pair
    b200asr_bilstm_fwd / b200asr_bilstm_bwd, which needs H % 16 == 0.
    """

    @staticmethod
    def forward(ctx, x, ndir, *params):
        sink = None
        if params and isinstance(params[-1], CStateSink):
            sink, params = params[-1], params[:-1]
        assert len(params) == 4 * ndir
        out, cst = _rnn_layer_fwd(ctx, "LSTM", x, ndir, [params[4 * d].detach() for d in range(ndir)],
                                  [params[4 * d + 1].detach() for d in range(ndir)],
                                  [params[4 * d + 2].detach() + params[4 * d + 3].detach() for d in range(ndir)])
        if sink is not None:
            sink.cstate = cst
        ctx.tail = (None,) if sink is not None else ()
        return out

    @staticmethod
    def backward(ctx, dout):
        dx, per_dir = _rnn_layer_bwd(ctx, dout)
        grads = []
        for dw_ih, dw_hh, db in per_dir:
            grads += [dw_ih, dw_hh, db, db.clone()]
        return (dx, None, *grads, *ctx.tail)


class BiGRUFn(Function):
    """One (bi)directional GRU layer over zero-padded frames, zero initial state (src/module.py:129-132, the nn.GRU
    branch): the BiLSTM layer with the GRU cell.

    forward(x[B,T,I], ndir, w_ih_0, w_hh_0, b_ih_0, b_hh_0 [, ..._1]) -> out[B,T,ndir*H], parameters in nn.GRU's
    layout (gates r, z, n).  Each direction is packed into the 4-slot layout of pack_decoder_weights("GRU"), the one
    packing rule of the GRU speller and encoder: W_ih4 = [W_ir; W_iz; W_in; 0], W_hh4 = [W_hr; W_hz; 0; W_hn], bias
    (b_ir + b_hr, b_iz + b_hz, b_in, b_hn), so that the input projection and h . W_hh4^T yield (r, z, gi_n, gh_n).  The
    recurrence is b200asr_bigru_fwd / _bwd; the layer GEMMs, dX and the weight gradients are BiLSTMFn's on the 4H rows
    (the zero slots cost 4/3 of a GRU layer's contraction FLOPs), mapped back by unpack_decoder_grads("GRU").
    """

    @staticmethod
    def forward(ctx, x, ndir, *params):
        assert len(params) == 4 * ndir
        I = params[0].shape[1]
        w_ih, w_hh, bias = [], [], []
        for d in range(ndir):
            wcat, b = pack_decoder_weights("GRU", *(p.detach() for p in params[4 * d:4 * d + 4]))
            w_ih.append(wcat[:, :I])
            w_hh.append(wcat[:, I:])
            bias.append(b)
        out, _ = _rnn_layer_fwd(ctx, "GRU", x, ndir, w_ih, w_hh, bias)
        return out

    @staticmethod
    def backward(ctx, dout):
        dx, per_dir = _rnn_layer_bwd(ctx, dout)
        I = ctx.dims[2]
        grads = []
        for dw_ih, dw_hh, db in per_dir:
            grads += unpack_decoder_grads("GRU", torch.cat([dw_ih, dw_hh], 1), db, I)
        return (dx, None, *grads)


class CStateSink:
    """Passed as the last argument of BiLSTMFn.apply: receives the layer's cell-state stash [ndir, B, T, H] (c after
    every step), from which a caller reads the final cell state of each row."""
    cstate = None


def bilstm(x, lstm_params, ndir, sink=None):
    return BiLSTMFn.apply(x, ndir, *lstm_params, *((sink,) if sink is not None else ()))


def bigru(x, gru_params, ndir):
    """One (bi)directional GRU layer; gru_params = nn.GRU's (weight_ih, weight_hh, bias_ih, bias_hh) per direction."""
    return BiGRUFn.apply(x, ndir, *gru_params)


def rnn_layer_supported(B, T, H, ndir):
    """True when the persistent recurrence kernels have a plan for this layer (H a multiple of 16)."""
    return L.load().b200asr_bilstm_workspace_bytes(B, T, H, ndir) != 0


# ----------------------------------------------------------------------------------------------------------
class LogSoftmaxFn(Function):
    """log_softmax over the last dim (src/asr.py:96) + greedy argmax ids as a by-product.

    `ctc_head=True` declares that the ONLY differentiable consumer of the result is the CTC loss (ops.CTCLoss), as in
    the reference's train step (bin/train_asr.py:123-124).  ATen's CTC backward - and ours - returns
    exp(lp) - occupancy, whose class sum is zero, i.e. it already IS the logit gradient (SURVEY.md F9): the
    log-softmax backward  dx = g - exp(lp) * sum_c g  is then the identity and its 12*T*V-byte pass is skipped.
    B200ASR_CHECK_CTC_HEAD=1 runs the full backward and checks the claim."""

    @staticmethod
    def forward(ctx, logits, ctc_head=False):
        lib = L.load()
        x = _f32c(logits)
        V = x.shape[-1]
        n = x.numel() // V
        y = torch.empty_like(x)
        am = torch.empty(x.shape[:-1], device=x.device, dtype=torch.int64)
        with L.timed("log_softmax_fwd", 8 * n * V):
            L.check(lib.b200asr_log_softmax_fwd(L.ptr(x), L.ptr(y), None, L.ptr(am), n, V, L.stream()),
                    "log_softmax_fwd")
        ctx.ctc_head = bool(ctc_head)
        ctx.save_for_backward(y)
        ctx.mark_non_differentiable(am)
        return y, am

    @staticmethod
    def backward(ctx, g, _gam):
        (y,) = ctx.saved_tensors
        if ctx.ctc_head and not _CHECK_CTC_HEAD:
            return g, None
        lib = L.load()
        g = _f32c(g)
        V = y.shape[-1]
        n = y.numel() // V
        dx = torch.empty_like(y)
        with L.timed("log_softmax_bwd", 12 * n * V):
            L.check(lib.b200asr_log_softmax_bwd(L.ptr(y), L.ptr(g), L.ptr(dx), n, V, L.stream()), "log_softmax_bwd")
        if ctx.ctc_head:
            err = float((dx - g).abs().max()) / max(float(g.abs().max()), 1e-30)
            if err > 1e-4:
                raise L.B200AsrError("log_softmax(ctc_head=True): upstream gradient is not a CTC gradient "
                                     "(identity-backward error %.2e)" % err)
        return dx, None


_CHECK_CTC_HEAD = os.environ.get("B200ASR_CHECK_CTC_HEAD", "0") == "1"


def log_softmax(logits, ctc_head=False):
    return LogSoftmaxFn.apply(logits, ctc_head)


class CTCHeadOutput:
    """`ctc_output` of ASR.forward when the CTC head is fused into the loss (train step): the logits [B, T, V], their
    per-row log-sum-exp [B, T] and the arg-max ids [B, T] instead of the V-wide log-prob tensor, which the train step
    never reads except through CTCLoss (bin/train_asr.py:123-124) and arg-max (cal_er, util.py:113-127).  Quacks
    like the tensor for exactly those uses; `materialize()` gives the log-probs [B, T, V] (detached) on demand."""

    def __init__(self, logits, lse, ids, time_major=False):
        self.logits, self.lse, self.ids, self.time_major = logits, lse, ids, time_major

    @property
    def shape(self):
        s = self.logits.shape
        return torch.Size((s[1], s[0], s[2])) if self.time_major else s

    @property
    def device(self):
        return self.logits.device

    def transpose(self, a, b):
        if {a % 3, b % 3} != {0, 1}:
            raise L.B200AsrError("CTCHeadOutput only swaps batch and time")
        return CTCHeadOutput(self.logits, self.lse, self.ids, not self.time_major)

    def argmax(self, dim=-1):
        if dim not in (-1, 2):
            raise L.B200AsrError("CTCHeadOutput.argmax is over the classes")
        return self.ids.transpose(0, 1) if self.time_major else self.ids

    def detach(self):
        return CTCHeadOutput(self.logits.detach(), self.lse, self.ids, self.time_major)

    def materialize(self):
        lp = self.logits.detach() - self.lse.unsqueeze(-1)
        return lp.transpose(0, 1) if self.time_major else lp


def ctc_head(logits):
    """logits [B, T, V] -> CTCHeadOutput: one pass over the logits for the row statistics (lse + arg-max), nothing
    V-wide written."""
    lib = L.load()
    x = _f32c(logits)
    B, T, V = x.shape
    lse = torch.empty((B, T), device=x.device, dtype=torch.float32)
    am = torch.empty((B, T), device=x.device, dtype=torch.int64)
    with L.timed("log_softmax_fwd", 4 * B * T * V):
        L.check(lib.b200asr_log_softmax_fwd(L.ptr(x), None, L.ptr(lse), L.ptr(am), B * T, V, L.stream()),
                "log_softmax_fwd(stats)")
    return CTCHeadOutput(x, lse, am)


class CTCLossFn(Function):
    """sum_b weight_b * nll_b.  Forward = the alpha/beta lattice kernels (nll); backward = ONE gradient kernel that
    already multiplies by weight_b and by the upstream scalar, so no scaling pass over [T,B,V] follows.

    log_probs: [T,B,V] view of [B,T,V] memory (or any layout with unit class stride), like the reference passes
    `ctc_output.transpose(0,1)` (bin/train_asr.py:123-124).
    """

    @staticmethod
    def forward(ctx, log_probs, targets, input_lengths, target_lengths, blank, weights, row_lse=None):
        """row_lse [B, T] given: `log_probs` holds the LOGITS of the CTC head and the log-softmax is fused into the
        lattice / gradient kernels (b200asr_ctc_*_logits); the returned gradient is then the logit gradient."""
        lib = L.load()
        if log_probs.dtype != torch.float32 or log_probs.stride(2) != 1:
            if row_lse is not None:
                raise L.B200AsrError("fused CTC head: logits must be fp32 with unit class stride")
            log_probs = log_probs.float().contiguous()
        T, B, V = log_probs.shape
        dev = log_probs.device
        targets = targets.to(device=dev, dtype=torch.int64).contiguous()
        if targets.dim() != 2:
            raise L.B200AsrError("CTC targets must be a padded [B, L] tensor (cudnn-style 1-D targets unsupported)")
        Lmax = targets.shape[1]
        il = torch.as_tensor(input_lengths, dtype=torch.int64).to(dev).contiguous()
        tl = torch.as_tensor(target_lengths, dtype=torch.int64).to(dev).contiguous()
        w = _f32c(weights.to(dev))
        nll = torch.empty(B, device=dev, dtype=torch.float32)
        ws_bytes = lib.b200asr_ctc_workspace_bytes(B, T, Lmax)
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        if row_lse is not None:
            row_lse = _f32c(row_lse)
            assert tuple(row_lse.shape) == (B, T)
        with L.timed("ctc_alpha_beta", 4 * B):
            if row_lse is None:
                L.check(lib.b200asr_ctc_fwd_bwd(L.ptr(log_probs), log_probs.stride(1), log_probs.stride(0),
                                                L.ptr(targets), L.ptr(il), L.ptr(tl), B, T, V, Lmax, blank, L.ptr(nll),
                                                L.ptr(w), None, L.ptr(ws), ws_bytes, L.stream()), "ctc_fwd_bwd")
            else:
                L.check(lib.b200asr_ctc_fwd_bwd_logits(L.ptr(log_probs), L.ptr(row_lse), log_probs.stride(1),
                                                       log_probs.stride(0), L.ptr(targets), L.ptr(il), L.ptr(tl), B, T,
                                                       V, Lmax, blank, L.ptr(nll), L.ptr(w), None, L.ptr(ws), ws_bytes,
                                                       L.stream()), "ctc_fwd_bwd_logits")
        ctx.save_for_backward(log_probs, targets, il, tl, w, nll, ws)
        ctx.row_lse = row_lse
        ctx.blank = blank
        ctx.mark_non_differentiable(nll)
        loss = (nll * w).sum()
        return loss, nll

    @staticmethod
    def backward(ctx, gloss, _gnll):
        lib = L.load()
        log_probs, targets, il, tl, w, nll, ws = ctx.saved_tensors
        T, B, V = log_probs.shape
        # gradient buffer laid out like log_probs' memory
        grad = torch.empty_strided(log_probs.shape, log_probs.stride(), device=log_probs.device, dtype=torch.float32)
        up = _f32c(gloss.reshape(1))
        # algorithmic bytes (SURVEY.md 8(d)): read the log-probs and write the gradient once each
        with L.timed("ctc_grad", 8 * T * V * B):
            if ctx.row_lse is None:
                L.check(lib.b200asr_ctc_grad(L.ptr(log_probs), log_probs.stride(1), log_probs.stride(0),
                                             L.ptr(targets), L.ptr(il), L.ptr(tl), B, T, V, targets.shape[1], ctx.blank,
                                             L.ptr(nll), L.ptr(w), L.ptr(up), L.ptr(grad), L.ptr(ws), ws.numel(),
                                             L.stream()), "ctc_grad")
            else:
                L.check(lib.b200asr_ctc_grad_logits(L.ptr(log_probs), L.ptr(ctx.row_lse), log_probs.stride(1),
                                                    log_probs.stride(0), L.ptr(targets), L.ptr(il), L.ptr(tl), B, T, V,
                                                    targets.shape[1], ctx.blank, L.ptr(nll), L.ptr(w), L.ptr(up),
                                                    L.ptr(grad), L.ptr(ws), ws.numel(), L.stream()), "ctc_grad_logits")
        return grad, None, None, None, None, None, None


class CTCLoss(torch.nn.Module):
    """Drop-in for torch.nn.CTCLoss(blank, reduction, zero_infinity=False) at bin/train_asr.py:49.

    `global_batch` lets a data-parallel rank normalise by the global batch size (SURVEY.md 8(e))."""

    def __init__(self, blank=0, reduction="mean", zero_infinity=False):
        super().__init__()
        if zero_infinity:
            raise NotImplementedError("zero_infinity=True is not part of the reference path")
        self.blank = blank
        self.reduction = reduction
        self.global_batch = None

    def forward(self, log_probs, targets, input_lengths, target_lengths):
        row_lse = None
        if isinstance(log_probs, CTCHeadOutput):       # fused head: logits + row lse instead of V-wide log-probs
            if not log_probs.time_major:
                raise L.B200AsrError("CTCLoss expects [T, B, V] (pass ctc_output.transpose(0, 1))")
            row_lse = log_probs.lse
            log_probs = log_probs.logits.transpose(0, 1)
        B = log_probs.shape[1]
        dev = log_probs.device
        tl = torch.as_tensor(target_lengths, dtype=torch.int64).to(dev)
        if self.reduction == "mean":
            denom = float(self.global_batch or B)
            w = 1.0 / (tl.clamp_min(1).to(torch.float32) * denom)
        elif self.reduction == "sum":
            w = torch.ones(B, device=dev, dtype=torch.float32)
        else:
            raise NotImplementedError("reduction=%s" % self.reduction)
        loss, nll = CTCLossFn.apply(log_probs, targets, input_lengths, tl, self.blank, w, row_lse)
        self.last_nll = nll
        return loss


# ----------------------------------------------------------------------------------------------------------
class LSTMCellFn(Function):
    """Pointwise part of one LSTM step (decoder, src/asr.py:214-221): pre[B,4H] (i,f,g,o) , c_prev -> h, c."""

    @staticmethod
    def forward(ctx, pre, c_prev):
        lib = L.load()
        pre = _f32c(pre)
        c_prev = _f32c(c_prev)
        B, H4 = pre.shape
        H = H4 // 4
        gates = torch.empty_like(pre)
        c = torch.empty_like(c_prev)
        h = torch.empty_like(c_prev)
        L.check(lib.b200asr_lstm_cell_fwd(L.ptr(pre), L.ptr(c_prev), L.ptr(gates), L.ptr(c), L.ptr(h), B, H,
                                          L.stream()), "lstm_cell_fwd")
        ctx.save_for_backward(gates, c_prev, c)
        return h, c

    @staticmethod
    def backward(ctx, dh, dc):
        lib = L.load()
        gates, c_prev, c = ctx.saved_tensors
        B, H4 = gates.shape
        H = H4 // 4
        dh = _f32c(dh) if dh is not None else torch.zeros_like(c)
        dcn = _f32c(dc) if dc is not None else None
        dpre = torch.empty_like(gates)
        dcp = torch.empty_like(c)
        L.check(lib.b200asr_lstm_cell_bwd(L.ptr(gates), L.ptr(c_prev), L.ptr(c), L.ptr(dh), L.ptr(dcn), L.ptr(dpre),
                                          L.ptr(dcp), B, H, L.stream()), "lstm_cell_bwd")
        return dpre, dcp


def lstm_cell(pre, c_prev):
    return LSTMCellFn.apply(pre, c_prev)


class GRUCellFn(Function):
    """Pointwise part of one GRU step (decoder, module: 'GRU'): pre [B, 4H] (r+z sums, gi_n, gh_n), h_prev -> h.
    The backward returns dpre and only the direct part dh . z of dh_prev; the GEMM part comes back through pre."""

    @staticmethod
    def forward(ctx, pre, h_prev):
        ctx.set_materialize_grads(False)
        lib = L.load()
        pre = _f32c(pre)
        h_prev = _f32c(h_prev)
        B, H4 = pre.shape
        H = H4 // 4
        assert H4 == 4 * H and tuple(h_prev.shape) == (B, H)
        gates = torch.empty_like(pre)
        h = torch.empty_like(h_prev)
        L.check(lib.b200asr_gru_cell_fwd(L.ptr(pre), L.ptr(h_prev), L.ptr(gates), L.ptr(h), B, H, L.stream()),
                "gru_cell_fwd")
        ctx.save_for_backward(gates, h_prev)
        return h

    @staticmethod
    def backward(ctx, dh):
        lib = L.load()
        gates, h_prev = ctx.saved_tensors
        B, H = h_prev.shape
        dh = _f32c(dh) if dh is not None else None
        dpre = torch.empty_like(gates)
        dhp = torch.empty_like(h_prev)
        L.check(lib.b200asr_gru_cell_bwd(L.ptr(gates), L.ptr(h_prev), L.ptr(dh), L.ptr(dpre), L.ptr(dhp), B, H,
                                         L.stream()), "gru_cell_bwd")
        return dpre, dhp


def gru_cell(pre, h_prev):
    return GRUCellFn.apply(pre, h_prev)


def gru_preact(gi, gh):
    """The cell kernel's pre-activation layout from the two library products gi = x.W_ih^T + b_ih, gh = h.W_hh^T + b_hh
    (each [B, 3H], r|z|n): [gh_rz + gi_rz, gi_n, gh_n] (the sum in ATen's operand order)."""
    H2 = 2 * (gi.shape[1] // 3)
    return torch.cat([gh[:, :H2] + gi[:, :H2], gi[:, H2:], gh[:, H2:]], 1)


# ----------------------------------------------------------------------------------------------------------
# Decoder LSTM step (src/asr.py:214-221): the two per-step projections  x . W_ih^T + h . W_hh^T + b  are ONE skinny
# tensor-core GEMM on [x | h] . [W_ih | W_hh]^T (split-K, csrc/gemm.cu), the backward's input gradient is one more, and
# the weight gradients of all L steps are ONE  dPre^T . [x | h]  contraction over the L*B stacked rows at the end of the
# loop (same accumulator-node idea as the attention memory above) instead of 2 L library SGEMMs + 2 L accumulations.
#
# The GRU speller runs through the same step: its weights are packed so that one product yields the cell kernel's
# layout (gru_cell),  Wcat [4H, I+H] = [[W_ir W_hr]; [W_iz W_hz]; [W_in 0]; [0 W_hn]],  bias = [b_r, b_z, b_in, b_hn]
# with b_r = b_ir + b_hr, b_z = b_iz + b_hz.  The zero blocks cost 4/3 of the ideal FLOPs and weight bytes but keep
# one launch per step in each direction (DESIGN §2.3 has the measurement against two products gi / gh).
class DecMem:
    def __init__(self):
        self.dpre, self.x = [], []


def pack_decoder_weights(cell, w_ih, w_hh, b_ih, b_hh):
    """-> (wcat [4H, I+H], bias [4H]) of the step GEMM for an 'LSTM' or 'GRU' layer (PyTorch's gate order)."""
    if cell == "LSTM":
        return torch.cat([w_ih, w_hh], 1).contiguous(), (b_ih + b_hh).contiguous()
    assert cell == "GRU"
    H2, I = 2 * w_hh.shape[1], w_ih.shape[1]
    wcat = torch.zeros((2 * H2, I + H2 // 2), device=w_ih.device, dtype=w_ih.dtype)
    wcat[:H2, :I] = w_ih[:H2]
    wcat[:H2, I:] = w_hh[:H2]
    wcat[H2:H2 * 3 // 2, :I] = w_ih[H2:]
    wcat[H2 * 3 // 2:, I:] = w_hh[H2:]
    return wcat, torch.cat([b_ih[:H2] + b_hh[:H2], b_ih[H2:], b_hh[H2:]])


def unpack_decoder_grads(cell, dW, db, I):
    """Gradients of the packed (wcat, bias) -> (dW_ih, dW_hh, db_ih, db_hh) of the layer's parameters."""
    if cell == "LSTM":
        return dW[:, :I], dW[:, I:], db, db
    H2 = dW.shape[0] // 2
    H3 = H2 * 3 // 2
    return (torch.cat([dW[:H2, :I], dW[H2:H3, :I]]), torch.cat([dW[:H2, I:], dW[H3:, I:]]),
            db[:H3], torch.cat([db[:H2], db[H3:]]))


class DecWeightsFn(Function):
    @staticmethod
    def forward(ctx, mem, cell, w_ih, w_hh, b_ih, b_hh):
        ctx.set_materialize_grads(False)
        ctx.mem = mem
        ctx.cell = cell
        ctx.I = w_ih.shape[1]
        token = torch.zeros(1, device=w_ih.device, dtype=torch.float32)
        wcat, bias = pack_decoder_weights(cell, w_ih, w_hh, b_ih, b_hh)
        wlo = tf32_residual(wcat)
        ctx.mark_non_differentiable(wlo)
        return wcat, bias, token, wlo

    @staticmethod
    def backward(ctx, gW, gb, _gtoken, _gwlo=None):
        mem = ctx.mem
        dW = gW
        db = gb
        if mem.dpre:
            dpre_all = torch.cat(mem.dpre, 0)
            x_all = torch.cat(mem.x, 0)
            d = gemm_nt(dpre_all, x_all, dpre_all.shape[1], x_all.shape[1], dpre_all.shape[0])
            dW = d if gW is None else d + gW
            s = dpre_all.sum(0)
            db = s if gb is None else s + gb
            mem.dpre, mem.x = [], []
        if dW is None:
            return None, None, None, None, None, None
        return (None, None) + tuple(unpack_decoder_grads(ctx.cell, dW, db, ctx.I))


class DecStepFn(Function):
    @staticmethod
    def forward(ctx, mem, token, x, h, wcat, bias, wlo):
        ctx.set_materialize_grads(False)
        xcat = torch.cat([x, h], 1).contiguous()
        pre = gemm_tn(xcat, wcat, bias=bias, w_lo=wlo)
        ctx.save_for_backward(xcat, wcat)
        ctx.mem = mem
        ctx.I = x.shape[1]
        return pre

    @staticmethod
    def backward(ctx, dpre):
        xcat, wcat = ctx.saved_tensors
        if dpre is None:
            return None, None, None, None, None, None, None
        dpre = _f32c(dpre)
        dx = gemm_nn(dpre, wcat)
        ctx.mem.dpre.append(dpre)
        ctx.mem.x.append(xcat)
        return None, torch.zeros(1, device=dpre.device), dx[:, :ctx.I], dx[:, ctx.I:], None, None, None


def decoder_weights(w_ih, w_hh, b_ih, b_hh, cell="LSTM"):
    """-> (mem, wcat [4H, I+H], bias [4H], token) for decoder_step(); once per batch and decoder layer.
    cell: 'LSTM' (pre feeds lstm_cell) or 'GRU' (pre feeds gru_cell)."""
    mem = DecMem()
    return (mem,) + tuple(DecWeightsFn.apply(mem, cell, w_ih, w_hh, b_ih, b_hh))


def decoder_step(dw, x, h):
    """pre-activations [B, 4H] of one decoder LSTM or GRU step from decoder_weights()' handle."""
    mem, wcat, bias, token, wlo = dw
    return DecStepFn.apply(mem, token, x, h, wcat, bias, wlo)


def decoder_gemm_supported(I, H):
    return (I + H) % 4 == 0


# ----------------------------------------------------------------------------------------------------------
class CrossEntropyFn(Function):
    """CrossEntropyLoss(ignore_index) with the logit gradient produced by the same launch."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, reduction):
        lib = L.load()
        x = _f32c(logits)
        N, V = x.shape
        target = target.to(device=x.device, dtype=torch.int64).contiguous()
        if reduction == "mean":
            scale = 1.0 / (target != ignore_index).sum().to(torch.float32)
        elif reduction == "sum":
            scale = torch.ones((), device=x.device, dtype=torch.float32)
        else:
            raise NotImplementedError("reduction=%s" % reduction)
        scale = scale.reshape(1).contiguous()
        row = torch.empty(N, device=x.device, dtype=torch.float32)
        grad = torch.empty_like(x)
        with L.timed("ce_fwd_bwd", 8 * N * V):
            L.check(lib.b200asr_ce_fwd_bwd(L.ptr(x), L.ptr(target), ignore_index, N, V, L.ptr(scale), L.ptr(row),
                                           L.ptr(grad), L.stream()), "ce_fwd_bwd")
        ctx.save_for_backward(grad)
        return row.sum() * scale[0]

    @staticmethod
    def backward(ctx, gloss):
        (grad,) = ctx.saved_tensors
        return grad.mul_(gloss), None, None, None


def cross_entropy(logits, target, ignore_index=0, reduction="mean"):
    return CrossEntropyFn.apply(logits, target, ignore_index, reduction)


# ----------------------------------------------------------------------------------------------------------
class LocAttnStepFn(Function):
    """One location-aware attention step (src/module.py:234-258 + 189-195, single head) in one kernel launch;
    its backward is one launch too (+ a [B*CS, P] -> [P] reduction of the small weight-gradient partials)."""

    @staticmethod
    def forward(ctx, q, key, value, prev_att, enc_len, conv_w, proj_w, e_w, e_b, temperature):
        lib = L.load()
        q, key, value, prev_att = _f32c(q), _f32c(key), _f32c(value), _f32c(prev_att)
        B, T, D = key.shape
        E = value.shape[2]
        K, _, W = conv_w.shape
        R = (W - 1) // 2
        dev = key.device
        enc_len = enc_len.to(device=dev, dtype=torch.int64).contiguous()
        cw, pw = _f32c(conv_w.detach()), _f32c(proj_w.detach())
        ew, eb = _f32c(e_w.detach()).view(-1), _f32c(e_b.detach()).view(-1)
        attn = torch.empty((B, T), device=dev, dtype=torch.float32)
        cvec = torch.empty((B, E), device=dev, dtype=torch.float32)
        # algorithmic bytes (SURVEY.md 8(d)): key + value read once per step
        with L.timed("locattn_fwd", 4 * B * T * (D + E)):
            L.check(lib.b200asr_locattn_fwd(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev_att), L.ptr(enc_len),
                                            L.ptr(cw), L.ptr(pw), L.ptr(ew), L.ptr(eb), float(temperature), B, T, D, E,
                                            K, R, L.ptr(attn), L.ptr(cvec), L.stream()), "locattn_fwd")
        ctx.save_for_backward(q, key, value, prev_att, enc_len, cw, pw, ew, attn)
        ctx.dims = (B, T, D, E, K, R)
        ctx.temperature = float(temperature)
        ctx.w_shapes = (conv_w.shape, proj_w.shape, e_w.shape, e_b.shape)
        return cvec, attn

    @staticmethod
    def backward(ctx, dctx, dattn):
        lib = L.load()
        q, key, value, prev_att, enc_len, cw, pw, ew, attn = ctx.saved_tensors
        B, T, D, E, K, R = ctx.dims
        dev = key.device
        CS = lib.b200asr_locattn_cluster_size(T, E)
        P = lib.b200asr_locattn_wpart_floats(D, K, R)
        dctx = _f32c(dctx) if dctx is not None else torch.zeros((B, E), device=dev)
        dattn = _f32c(dattn) if dattn is not None else None
        dq_part = torch.empty((B, CS, D), device=dev, dtype=torch.float32)
        dkey = torch.empty((B, T, D), device=dev, dtype=torch.float32)
        dvalue = torch.empty((B, T, E), device=dev, dtype=torch.float32)
        dprev = torch.empty((B, T), device=dev, dtype=torch.float32)
        wpart = torch.empty((B * CS, P), device=dev, dtype=torch.float32)
        with L.timed("locattn_bwd", 4 * B * T * (2 * D + 2 * E)):
            L.check(lib.b200asr_locattn_bwd(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev_att), L.ptr(enc_len),
                                            L.ptr(cw), L.ptr(pw), L.ptr(ew), ctx.temperature, L.ptr(attn), L.ptr(dctx),
                                            L.ptr(dattn), B, T, D, E, K, R, L.ptr(dq_part), L.ptr(dkey), L.ptr(dvalue),
                                            L.ptr(dprev), L.ptr(wpart), L.stream()), "locattn_bwd")
        wsum = wpart.sum(0)
        W = 2 * R + 1
        s_conv, s_proj, s_ew, s_eb = ctx.w_shapes
        d_proj = wsum[:D * K].view(s_proj)
        d_conv = wsum[D * K:D * K + K * W].view(s_conv)
        d_ew = wsum[D * K + K * W:D * K + K * W + D].view(s_ew)
        d_eb = wsum[D * K + K * W + D:].view(s_eb)
        return dq_part.sum(1), dkey, dvalue, dprev, None, d_conv, d_proj, d_ew, d_eb, None


def loc_attention_step(q, key, value, prev_att, enc_len, conv_w, proj_w, e_w, e_b, temperature):
    """-> (context [B,E], attn [B,T])"""
    return LocAttnStepFn.apply(q, key, value, prev_att, enc_len, conv_w, proj_w, e_w, e_b, temperature)


# ----------------------------------------------------------------------------------------------------------
# The decode loop calls the attention L times on the SAME key / value / weights (src/asr.py:112-151).  Left to autograd,
# every step's backward writes a [B,T,D] and a [B,T,E] gradient that the engine then re-adds L-1 times (cfg C: 46 x
# (78 + 11) MB written and ~3x that re-read and re-written by ATen adds).  Instead the per-batch gradients live in ONE
# accumulator node:  AttnMemFn  hands key / value / the location weights (none for the dot-product attention) to the
# steps (plus a 1-element token whose only job is to make the engine run AttnMemFn.backward after the LAST step);  the
# step's backward (LocAttnMemStepFn / DotAttnMemStepFn) adds d(key) - and the location weights' partials - in place
# (b200asr_locattn_bwd_acc / b200asr_dotattn_bwd_acc) and records (attn_l, dctx_l);  AttnMemFn.backward forms
# d(value) = sum_l attn_l (x) dctx_l once (b200asr_attn_dvalue) and reduces the weight partials once.
class AttnMem:
    def __init__(self):
        self.dkey = None
        self.wpart = None
        self.attn, self.dctx = [], []
        self.meta = None


class AttnMemFn(Function):
    @staticmethod
    def forward(ctx, mem, key, value, *loc_w):
        ctx.set_materialize_grads(False)        # undefined output gradients arrive as None, not as [B,T,E] zeros
        ctx.mem = mem
        ctx.shapes = (key.shape, value.shape) + tuple(w.shape for w in loc_w)
        token = torch.zeros(1, device=key.device, dtype=torch.float32)
        return (key.view_as(key), value.view_as(value)) + tuple(w.view_as(w) for w in loc_w) + (token,)

    @staticmethod
    def backward(ctx, gkey, gvalue, *grads):
        lib = L.load()
        mem = ctx.mem
        s_key, s_value = ctx.shapes[:2]
        g_loc, _gtoken = grads[:-1], grads[-1]
        B, T, D = s_key
        E = s_value[2]
        dev = _gtoken.device
        dkey = mem.dkey if mem.dkey is not None else torch.zeros(s_key, device=dev)
        if gkey is not None:
            dkey = dkey + gkey
        if mem.attn:
            attn_all = torch.stack(mem.attn, 1).contiguous()          # [B, L, T]
            dctx_all = torch.stack(mem.dctx, 1).contiguous()          # [B, L, E]
            Lsteps = attn_all.shape[1]
            acc = gvalue is not None
            dvalue = _f32c(gvalue).clone() if acc else torch.empty(s_value, device=dev, dtype=torch.float32)
            with L.timed("attn_dvalue", 4 * B * (T * E + Lsteps * (T + E))):
                L.check(lib.b200asr_attn_dvalue(L.ptr(attn_all), L.ptr(dctx_all), B, Lsteps, T, E, L.ptr(dvalue),
                                                int(acc), L.stream()), "attn_dvalue")
        else:
            dvalue = gvalue
        d_loc = (None,) * len(g_loc)
        if mem.wpart is not None:
            s_conv, s_proj, s_ew, s_eb = ctx.shapes[2:]
            K, N, W = s_conv                                # conv weight [K, N, 2R+1]: N location channels (heads)
            C = K * N * W
            wsum = mem.wpart.sum(0)
            d_loc = (wsum[D * K:D * K + C].view(s_conv), wsum[:D * K].view(s_proj),
                     wsum[D * K + C:D * K + C + D].view(s_ew), wsum[D * K + C + D:].view(s_eb))
        add = lambda a, b: a if b is None else (b if a is None else a + b)
        mem.dkey = mem.wpart = None
        mem.attn, mem.dctx = [], []
        return (None, dkey, dvalue) + tuple(add(d, g) for d, g in zip(d_loc, g_loc))


def attention_memory(key, value, conv_w=None, proj_w=None, e_w=None, e_b=None):
    """-> (mem, key, value, conv_w, proj_w, e_w, e_b, token) for loc_attention_mem_step / loc_attention_heads_mem_step,
    or, without the location weights, (mem, key, value, token) for dot_attention_mem_step."""
    mem = AttnMem()
    loc_w = tuple(w for w in (conv_w, proj_w, e_w, e_b) if w is not None)
    if len(loc_w) not in (0, 4):
        raise ValueError("attention_memory: pass all four location weights or none")
    return (mem,) + tuple(AttnMemFn.apply(mem, _f32c(key), _f32c(value), *loc_w))


class LocAttnMemStepFn(Function):
    """One decode step on an attention memory: forward = the same single-launch kernel as LocAttnStepFn; backward =
    b200asr_locattn_bwd_acc (d(key) / weight partials added into the memory, no d(value) write)."""

    @staticmethod
    def forward(ctx, mem, token, q, key, value, prev_att, enc_len, conv_w, proj_w, e_w, e_b, temperature):
        ctx.set_materialize_grads(False)
        lib = L.load()
        q, prev_att = _f32c(q), _f32c(prev_att)
        B, T, D = key.shape
        E = value.shape[2]
        K, _, W = conv_w.shape
        R = (W - 1) // 2
        dev = key.device
        enc_len = enc_len.to(device=dev, dtype=torch.int64).contiguous()
        cw, pw = _f32c(conv_w.detach()), _f32c(proj_w.detach())
        ew, eb = _f32c(e_w.detach()).view(-1), _f32c(e_b.detach()).view(-1)
        attn = torch.empty((B, T), device=dev, dtype=torch.float32)
        cvec = torch.empty((B, E), device=dev, dtype=torch.float32)
        with L.timed("locattn_fwd", 4 * B * T * (D + E)):
            L.check(lib.b200asr_locattn_fwd(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev_att), L.ptr(enc_len),
                                            L.ptr(cw), L.ptr(pw), L.ptr(ew), L.ptr(eb), float(temperature), B, T, D, E,
                                            K, R, L.ptr(attn), L.ptr(cvec), L.stream()), "locattn_fwd")
        ctx.save_for_backward(q, key, value, prev_att, enc_len, cw, pw, ew, attn)
        ctx.mem = mem
        ctx.dims = (B, T, D, E, K, R)
        ctx.temperature = float(temperature)
        return cvec, attn

    @staticmethod
    def backward(ctx, dctx, dattn):
        lib = L.load()
        q, key, value, prev_att, enc_len, cw, pw, ew, attn = ctx.saved_tensors
        B, T, D, E, K, R = ctx.dims
        mem = ctx.mem
        dev = key.device
        CS = lib.b200asr_locattn_cluster_size(T, E)
        P = lib.b200asr_locattn_wpart_floats(D, K, R)
        if mem.dkey is None:
            mem.dkey = torch.zeros((B, T, D), device=dev, dtype=torch.float32)
            mem.wpart = torch.zeros((B * CS, P), device=dev, dtype=torch.float32)
        dctx = _f32c(dctx) if dctx is not None else torch.zeros((B, E), device=dev)
        dattn = _f32c(dattn) if dattn is not None else None
        dq_part = torch.empty((B, CS, D), device=dev, dtype=torch.float32)
        dprev = torch.empty((B, T), device=dev, dtype=torch.float32)
        with L.timed("locattn_bwd", 4 * B * T * (2 * D + E)):
            L.check(lib.b200asr_locattn_bwd_acc(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev_att), L.ptr(enc_len),
                                                L.ptr(cw), L.ptr(pw), L.ptr(ew), ctx.temperature, L.ptr(attn),
                                                L.ptr(dctx), L.ptr(dattn), B, T, D, E, K, R, L.ptr(dq_part),
                                                L.ptr(mem.dkey), L.ptr(dprev), L.ptr(mem.wpart), L.stream()),
                    "locattn_bwd_acc")
        mem.attn.append(attn)
        mem.dctx.append(dctx)
        token_grad = torch.zeros(1, device=dev, dtype=torch.float32)
        return None, token_grad, dq_part.sum(1), None, None, dprev, None, None, None, None, None, None


def loc_attention_mem_step(mem, token, q, key, value, prev_att, enc_len, conv_w, proj_w, e_w, e_b, temperature):
    """-> (context [B,E], attn [B,T]); key ... e_b and token come from attention_memory()."""
    return LocAttnMemStepFn.apply(mem, token, q, key, value, prev_att, enc_len, conv_w, proj_w, e_w, e_b, temperature)


# ----------------------------------------------------------------------------------------------------------
DOTATTN_MAX_T = 8192          # B200ASR_DOTATTN_MAX_T of include/b200asr.h


def dot_attention_supported(T, D, E):
    """The limits of b200asr_dotattn_fwd / _bwd_acc (include/b200asr.h; cluster rule of b200asr_locattn_cluster_size)."""
    cs = 4
    while cs > 1 and (E % (4 * cs) != 0 or (T < 8 * cs and E // (cs // 2) <= 1024)):
        cs >>= 1
    return 0 < T <= DOTATTN_MAX_T and 0 < D <= 512 and E > 0 and E % 4 == 0 and E // cs <= 1024


class DotAttnMemStepFn(Function):
    """One scaled dot-product attention step (src/module.py:189-212, one or more heads) on an attention memory:
    forward = b200asr_dotattn_fwd (one launch); backward = b200asr_dotattn_bwd_acc (d(key) added into the memory, no
    d(value) write; AttnMemFn forms d(value) once after the loop)."""

    @staticmethod
    def forward(ctx, mem, token, q, key, value, enc_len, num_head, temperature):
        ctx.set_materialize_grads(False)
        lib = L.load()
        q = _f32c(q)
        R, T, D = key.shape
        E = value.shape[2]
        dev = key.device
        enc_len = enc_len.to(device=dev, dtype=torch.int64).contiguous()
        attn = torch.empty((R, T), device=dev, dtype=torch.float32)
        cvec = torch.empty((R, E), device=dev, dtype=torch.float32)
        # algorithmic bytes: key + value read once, q / attn / ctx / lengths
        with L.timed("dotattn_fwd", 4 * R * T * (D + E) + 4 * R * (D + T + E) + 8 * (R // num_head)):
            L.check(lib.b200asr_dotattn_fwd(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(enc_len), int(num_head),
                                            float(temperature), R, T, D, E, L.ptr(attn), L.ptr(cvec), L.stream()),
                    "dotattn_fwd")
        ctx.save_for_backward(q, key, value, enc_len, attn)
        ctx.mem = mem
        ctx.dims = (R, T, D, E, int(num_head))
        ctx.temperature = float(temperature)
        return cvec, attn

    @staticmethod
    def backward(ctx, dctx, dattn):
        lib = L.load()
        q, key, value, enc_len, attn = ctx.saved_tensors
        R, T, D, E, N = ctx.dims
        mem = ctx.mem
        dev = key.device
        CS = lib.b200asr_locattn_cluster_size(T, E)
        if mem.dkey is None:
            mem.dkey = torch.zeros((R, T, D), device=dev, dtype=torch.float32)
        dctx = _f32c(dctx) if dctx is not None else torch.zeros((R, E), device=dev)
        dattn = _f32c(dattn) if dattn is not None else None
        dq_part = torch.empty((R, CS, D), device=dev, dtype=torch.float32)
        # value read once, key read and d(key) read + written once; q, attn, dattn, dctx, dq partials, lengths
        with L.timed("dotattn_bwd_acc", 4 * R * T * (2 * D + E) + 4 * R * (D + 2 * T + E + CS * D) + 8 * (R // N)):
            L.check(lib.b200asr_dotattn_bwd_acc(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(enc_len), N, ctx.temperature,
                                                L.ptr(attn), L.ptr(dctx), L.ptr(dattn), R, T, D, E, L.ptr(dq_part),
                                                L.ptr(mem.dkey), L.stream()), "dotattn_bwd_acc")
        mem.attn.append(attn)
        mem.dctx.append(dctx)
        token_grad = torch.zeros(1, device=dev, dtype=torch.float32)
        return None, token_grad, dq_part.sum(1), None, None, None, None, None


def dot_attention_mem_step(mem, token, q, key, value, enc_len, num_head, temperature):
    """-> (context [R,E], attn [R,T]) with R = B * num_head rows; mem, key, value and token come from
    attention_memory(key, value)."""
    return DotAttnMemStepFn.apply(mem, token, q, key, value, enc_len, num_head, temperature)


# ----------------------------------------------------------------------------------------------------------
ATTN_SMEM_OPTIN = 232448      # sm_90's opt-in shared memory per block (the library's value when no device is visible)


def loc_attention_heads_supported(N, T, D, E, K, R):
    """The limits of b200asr_locattn_heads_fwd / _bwd_acc (include/b200asr.h): N, K <= 16, D <= 512, E % 4 == 0,
    E / CS <= 1024 and both kernels' shared memory within the device's opt-in maximum."""
    if not (N > 0 and T > 0 and D > 0 and E > 0 and K > 0 and R >= 0):
        return False
    if N > 16 or K > 16 or D > 512 or E % 4 != 0:
        return False
    cs = 4
    while cs > 1 and (E % (4 * cs) != 0 or (T < 8 * cs and E // (cs // 2) <= 1024)):
        cs >>= 1
    if E // cs > 1024:
        return False
    W, TP, TS, TT = 2 * R + 1, T + 2 * R, (T + cs - 1) // cs, 16
    common = N * TP + K * N * W + D * K + D + N * D
    fwd = 4 * ((common + N * T + K * TS + 3) // 4 * 4 + 512 * 4)
    bwd = 4 * (common + D * K + N * D + 2 * N * T + N * cs * T + K * TT + 2 * TT * D + K * TP)
    optin = ATTN_SMEM_OPTIN
    if torch.cuda.is_available():
        optin = torch.cuda.get_device_properties(torch.cuda.current_device()).shared_memory_per_block_optin
    return max(fwd, bwd) + 32 * 4 <= optin      # + the kernels' static reduction scratch


class LocAttnHeadsMemStepFn(Function):
    """One multi-head location-aware attention step (src/module.py:215-258 with num_head = N > 1) on an attention
    memory: forward = b200asr_locattn_heads_fwd (one launch: one location convolution per utterance shared by its N
    heads); backward = b200asr_locattn_heads_bwd_acc (d(key) and the weight partials added into the memory, d(prev)
    for all N channels, no d(value) write; AttnMemFn forms d(value) once after the loop over the B*N rows)."""

    @staticmethod
    def forward(ctx, mem, token, q, key, value, prev_att, enc_len, num_head, conv_w, proj_w, e_w, e_b, temperature):
        ctx.set_materialize_grads(False)
        lib = L.load()
        q, prev_att = _f32c(q), _f32c(prev_att)
        rows, T, D = key.shape
        E = value.shape[2]
        N = int(num_head)
        B = rows // N
        K, _, W = conv_w.shape
        R = (W - 1) // 2
        dev = key.device
        enc_len = enc_len.to(device=dev, dtype=torch.int64).contiguous()
        cw, pw = _f32c(conv_w.detach()), _f32c(proj_w.detach())
        ew, eb = _f32c(e_w.detach()).view(-1), _f32c(e_b.detach()).view(-1)
        attn = torch.empty((rows, T), device=dev, dtype=torch.float32)
        cvec = torch.empty((rows, E), device=dev, dtype=torch.float32)
        # algorithmic bytes: key + value read once; q, prev, attn, ctx, the weights, lengths
        nbytes = 4 * rows * T * (D + E) + 4 * rows * (D + 2 * T + E) + 4 * (K * N * W + D * K + D + 1) + 8 * B
        with L.timed("locattn_heads_fwd", nbytes):
            L.check(lib.b200asr_locattn_heads_fwd(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev_att), L.ptr(enc_len),
                                                  L.ptr(cw), L.ptr(pw), L.ptr(ew), L.ptr(eb), float(temperature), B, N,
                                                  T, D, E, K, R, L.ptr(attn), L.ptr(cvec), L.stream()),
                    "locattn_heads_fwd")
        ctx.save_for_backward(q, key, value, prev_att, enc_len, cw, pw, ew, attn)
        ctx.mem = mem
        ctx.dims = (B, N, T, D, E, K, R)
        ctx.temperature = float(temperature)
        return cvec, attn

    @staticmethod
    def backward(ctx, dctx, dattn):
        lib = L.load()
        q, key, value, prev_att, enc_len, cw, pw, ew, attn = ctx.saved_tensors
        B, N, T, D, E, K, R = ctx.dims
        rows, W = B * N, 2 * R + 1
        mem = ctx.mem
        dev = key.device
        CS = lib.b200asr_locattn_cluster_size(T, E)
        P = lib.b200asr_locattn_heads_wpart_floats(N, D, K, R)
        if mem.dkey is None:
            mem.dkey = torch.zeros((rows, T, D), device=dev, dtype=torch.float32)
            mem.wpart = torch.zeros((B * CS, P), device=dev, dtype=torch.float32)
        dctx = _f32c(dctx) if dctx is not None else torch.zeros((rows, E), device=dev)
        dattn = _f32c(dattn) if dattn is not None else None
        dq_part = torch.empty((rows, CS, D), device=dev, dtype=torch.float32)
        dprev = torch.empty((B, N, T), device=dev, dtype=torch.float32)
        # value read once, key read and d(key) read + written once; q, prev, d(prev), attn, dattn, dctx, dq partials,
        # the weights, the weight partials read + written, lengths
        nbytes = (4 * rows * T * (3 * D + E) + 4 * rows * (D + 4 * T + E + CS * D) + 4 * (K * N * W + D * K + D)
                  + 8 * B * CS * P + 8 * B)
        with L.timed("locattn_heads_bwd_acc", nbytes):
            L.check(lib.b200asr_locattn_heads_bwd_acc(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev_att),
                                                      L.ptr(enc_len), L.ptr(cw), L.ptr(pw), L.ptr(ew), ctx.temperature,
                                                      L.ptr(attn), L.ptr(dctx), L.ptr(dattn), B, N, T, D, E, K, R,
                                                      L.ptr(dq_part), L.ptr(mem.dkey), L.ptr(dprev), L.ptr(mem.wpart),
                                                      L.stream()), "locattn_heads_bwd_acc")
        mem.attn.append(attn)
        mem.dctx.append(dctx)
        token_grad = torch.zeros(1, device=dev, dtype=torch.float32)
        return (None, token_grad, dq_part.sum(1), None, None, dprev, None, None, None, None, None, None, None)


def loc_attention_heads_mem_step(mem, token, q, key, value, prev_att, enc_len, num_head, conv_w, proj_w, e_w, e_b,
                                 temperature):
    """-> (context [R,E], attn [R,T]) with R = B * num_head rows, prev_att [B,N,T], conv_w [K,N,2R+1]; key ... e_b and
    token come from attention_memory()."""
    return LocAttnHeadsMemStepFn.apply(mem, token, q, key, value, prev_att, enc_len, num_head, conv_w, proj_w, e_w,
                                       e_b, temperature)


# ----------------------------------------------------------------------------------------------------------
class Linear3xFn(Function):
    """y = x W^T + b for the large dense layers of the step (CTC head, key projection, vocabulary projection) on
    the tensor cores with the error-compensated 3xTF32 scheme (fp32-class)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        shp = x.shape
        x2 = _f32c(x).reshape(-1, shp[-1])
        if x2.shape[1] % 4 == 0:
            y = gemm_tn(x2, weight.detach(), bias=bias.detach() if bias is not None else None,
                        w_lo=tf32_residual(weight.detach()))
        else:
            y = mm3(Split(x2), Split(weight.detach()).t(), bias=bias.detach() if bias is not None else None,
                    out=torch.empty((x2.shape[0], weight.shape[0]), device=x.device, dtype=torch.float32))
        ctx.save_for_backward(x2, weight)
        ctx.shp = shp
        ctx.has_bias = bias is not None
        return y.view(*shp[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, gy):
        x2, weight = ctx.saved_tensors
        gy2 = _f32c(gy).reshape(-1, weight.shape[0])
        dx = None
        own = weight.shape[0] % 4 == 0 and weight.shape[1] % 4 == 0     # else (the CTC head at V = 31) Split + mm3
        if ctx.needs_input_grad[0]:
            if own:
                dx = gemm_nn(gy2, weight.detach()).view(ctx.shp)
            else:
                dx = mm3(Split(gy2), Split(weight.detach())).view(ctx.shp)
        dw = None
        if ctx.needs_input_grad[1]:
            if own:
                dw = gemm_nt(gy2, x2, weight.shape[0], weight.shape[1], gy2.shape[0])
            else:
                dw = mm3(Split(gy2).t(), Split(x2))
        db = gy.reshape(-1, weight.shape[0]).sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return dx, dw, db


def linear3x(x, layer):
    """Apply an nn.Linear through the 3xTF32 tensor-core path when the problem is large enough to matter."""
    rows = x.numel() // x.shape[-1]
    if x.is_cuda and rows * layer.in_features * layer.out_features >= (1 << 24):
        return Linear3xFn.apply(x, layer.weight, layer.bias)
    return torch.nn.functional.linear(x, layer.weight, layer.bias)


# ----------------------------------------------------------------------------------------------------------
# RNN language model (src/lm.py): the V x E-sized gradients are added IN PLACE into the parameter's gradient - under
# optim.Optimizer the `emb.weight` view of the flat gradient buffer, zeroed by pre_step - and the backward returns None
# for the weight (the accumulator-node idea of AttnMemFn / DecWeightsFn).  Without a gradient buffer one zero [V, E]
# tensor is allocated as `.grad` once.
def _grad_view(p):
    if p.grad is None:
        p.grad = torch.zeros_like(p)
    g = p.grad
    if g.dtype != torch.float32 or not g.is_contiguous() or g.shape != p.shape:
        raise L.B200AsrError("in-place gradient needs a contiguous fp32 .grad of the parameter's shape")
    return g


def embedding_bwd_(dW, ids, dy):
    """dW[ids[n], :] += dy[n, :] in place (b200asr_embedding_bwd): deterministic, ids outside [0, V) skipped."""
    lib = L.load()
    V, E = dW.shape
    ids = ids.reshape(-1).to(device=dW.device, dtype=torch.int64).contiguous()
    dy = _f32c(dy.reshape(-1, E))
    N = ids.numel()
    if dy.shape[0] != N:
        raise L.B200AsrError("embedding_bwd: %d ids but %d gradient rows" % (N, dy.shape[0]))
    if not (dW.is_contiguous() and dW.dtype == torch.float32):
        raise L.B200AsrError("embedding_bwd: dW must be a contiguous fp32 [V, E] tensor")
    ws_bytes = lib.b200asr_embedding_bwd_workspace_bytes(N, V)
    ws = torch.empty(max(ws_bytes, 16), device=dW.device, dtype=torch.uint8)
    # algorithmic bytes: the ids and dY once, the touched rows of dW read and written (bounded by N rows)
    with L.timed("embedding_bwd", 8 * N + 4 * N * E + 8 * min(N, V) * E):
        L.check(lib.b200asr_embedding_bwd(L.ptr(ids), L.ptr(dy), N, V, E, L.ptr(dW), L.ptr(ws), ws_bytes, L.stream()),
                "embedding_bwd")
    return dW


class EmbeddingFn(Function):
    """nn.Embedding forward (ATen row gather, like the decoder's pre_embed); backward = embedding_bwd_ into
    weight.grad in place, None returned for the weight."""

    @staticmethod
    def forward(ctx, ids, weight):
        ctx.save_for_backward(ids)
        ctx.weight = weight
        return torch.nn.functional.embedding(ids, weight.detach())

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        if ctx.needs_input_grad[1]:
            embedding_bwd_(_grad_view(ctx.weight), ids, dy)
        return None, None


def embedding(ids, weight):
    return EmbeddingFn.apply(ids, weight)


class TiedLinearFn(Function):
    """y = x W^T without bias with W = emb.weight (src/lm.py:42, weight tying): the 3xTF32 GEMM of Linear3xFn; the
    weight gradient dY^T . X is accumulated by the GEMM epilogue straight into weight.grad, where the embedding kernel
    adds its part too - no second [V, E] tensor."""

    @staticmethod
    def forward(ctx, x, weight):
        shp = x.shape
        x2 = _f32c(x).reshape(-1, shp[-1])
        w = weight.detach()
        if not (x2.shape[1] % 4 == 0 and w.shape[0] % 4 == 0):
            raise L.B200AsrError("tied projection: E and V must be multiples of 4 for the tensor-core GEMM "
                                 "(E=%d V=%d)" % (x2.shape[1], w.shape[0]))
        y = gemm_tn(x2, w, w_lo=tf32_residual(w))
        ctx.save_for_backward(x2)
        ctx.weight = weight
        ctx.shp = shp
        return y.view(*shp[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy):
        (x2,) = ctx.saved_tensors
        w = ctx.weight.detach()
        V, E = w.shape
        gy2 = _f32c(gy).reshape(-1, V)
        dx = gemm_nn(gy2, w).view(ctx.shp) if ctx.needs_input_grad[0] else None
        if ctx.needs_input_grad[1]:
            gemm_nt(gy2, x2, V, E, gy2.shape[0], out=_grad_view(ctx.weight), accumulate=True)
        return dx, None


def tied_linear(x, weight):
    return TiedLinearFn.apply(x, weight)
