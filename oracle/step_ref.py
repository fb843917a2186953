"""Float64 closed forms of four kernels on the train / decode step (forward and backward as explicit expressions, not
autograd), each intermediate with an absolute-value companion, and from them a per-element bound on the fp32 rounding
of every output:
  * the decoder / LM LSTM cell, `b200asr_lstm_cell_fwd / _bwd` (csrc/lstm.cu);
  * fused log-softmax + NLL with its logit gradient, `b200asr_ce_fwd_bwd` (csrc/ce.cu);
  * the CNN prenet's Conv1d(k 4, s 2, p 1), `ops.Conv1dK4S2Fn` (three GEMMs of csrc/gemm.cu on the in-place view);
  * CTC prefix scoring, `b200asr_ctc_prefix_score` (csrc/prefix.cu).

Notation: u = 2^-24 (fp32 unit roundoff), F = 2^-126 (the smallest normal fp32: an underflowed result is off by less).
The library is built without fast math: expf and tanhf are within 2 ulp (<= 4u relative), logf and log1pf within
1 ulp; nvcc may contract a*b + c into one fma, which only removes roundings.  Each constant below is the first-order
count rounded up to the next integer, which also absorbs the second-order terms (products of two u-terms, < u^2 of the
scale).  Every bound is taken on the kernel's own fp32 inputs (given exactly in float64), so errors do not compound
between calls.  The functions return K = 2 times the bounds below for the LSTM cell, cross-entropy and the prefix
scorer: the margin for the ulp limits being maxima over the whole range, so that an fp32 emulation of the same
arithmetic (tests/test_host_step_kernels.py) stays within half of what the GPU tests allow.

LSTM cell, per element j of row b (pre = [i | f | g | o] pre-activations, exact sigmoid / tanh values i, f, g, o):
  i' = 1/(1 + expf(-a)): expf 4u, the add u, the division u          Δi = 6u i + F   (same for f, o)
  g' = tanhf(a)                                                      Δg = 4u |g| + F
  c' = fmaf(f, c_prev, i g)   P = |f c_prev| + |i g|                 Δc = 8u |f c_prev| + 13u |i g| + 2F (1 + |c_prev|)
  h' = o tanhf(c')            t = tanh(c)                            Δh = o (1 - t^2 + Δc) Δc + 12u o |t| + F
  (tanh is 1-Lipschitz and (1 - tanh^2)' is below 0.77 in magnitude, so a Δc in the argument moves it by at most
  (1 - t^2 + Δc) Δc.)
Backward, for the GIVEN stash (fp32 gates and c the forward wrote, as the autograd path passes them) and dh, dc_next:
  tc = tanhf(c) carries 4u |t|, so 1 - tc^2 is off by at most 10u ABSOLUTE: near saturation it cancels, and the
  bound is in the scale of the terms (q = |dh o|, dc~ = |dc_next| + q), not relative to the result:
  dc = dc_next + dh o (1 - tc^2)                                     Δdc = 13u dc~
  d pre_i = dc g i (1 - i)       three products, one 1 - i           Δ = 17u dc~ |g| i (1 - i) + F
  d pre_f = dc c_prev f (1 - f)                                      Δ = 17u dc~ |c_prev| f (1 - f) + F
  d pre_g = dc i (1 - g^2)       1 - g^2 off by 2u absolute          Δ = 17u dc~ i + F
  d pre_o = dh tc o (1 - o)                                          Δ = 8u |dh t| o (1 - o) + F
  dc_prev = dc f                                                     Δ = 14u dc~ f + F
  A saturated gate (|a| >= 100) is stored as exactly 0 or 1 and its d pre is exactly 0.

Cross-entropy, per valid row (target t not ignored) of V logits; one warp per row, lane l holds n <= ceil(V / 32)
logits and keeps an online (m, s); S = sum_l s_l expf(m_l - M) over a 5-level tree; lse = M + logf(S).  A term x_c
enters s with its argument x_c - m rounded (u |x_c - m|) and expf's 4u, every later rescale of s adds the rounding of
its argument (these telescope to u (m_l - x_c)), 4u and two roundings, every later add one rounding, and the lane fold
adds u (M - m_l) + 6u: the relative error of S is at most
  δS = u (M - x_min) + 6u n + 12u           (x_min: the smallest finite logit of the row)
  Δlse = δS + 2u (lse - M) + u |lse|        (logf's ulp on log S = lse - M >= 0, then the add)
  Δloss = Δlse + u |loss|
  dx_c = sc (expf(x_c - lse) - [c = t]),  p = exp(x_c - lse):
  Δdx_c = sc (p (Δlse + u |x_c - lse| + 4u) + 4u |p - [c = t]|) + F
  (the subtraction of the one-hot, the product with sc, and for ops.cross_entropy the fp32 1/n and the upstream
  scale: four roundings of |p - [c = t]|).  This replaces the earlier tensor-wide `EPS (4 (max|x| + |lse|) + V/8 + 64)`,
  whose V/8 does not follow the kernel's ceil(V/32) terms per lane at small V.
  Rows with a NaN, a +inf or only -inf logits give NaN loss and an all-NaN gradient row, as float64 ATen does; a -inf
  target gives loss +inf and a finite gradient; ignored rows are exactly 0.  One difference from ATen: an ignored row
  that holds a NaN logit gets ATen's NaN gradient (log_softmax's backward multiplies its NaN output by the row's zero
  upstream sum), while the kernel never reads an ignored row and writes 0 there.

Conv1d(C -> O, k 4, s 2, p 1) over x [B, T, C] (ops.Conv1dK4S2Fn): Tout = T // 2, half = Tout + 1, Tp = 2 half padded
rows per utterance (row 0 and rows > T zero), view row m = b half + t reads the 4C floats from padded row 2t:
  forward:  tn GEMM over M = B half - 1 view rows, K = 4C, plus bias (the rows t >= Tout are discarded);
  d w:      nt GEMM, out [O, 4C], contraction over the same M view rows (B operand pitch ldb = 2C);
  d x:      nn GEMM d cols = dy W [B half, 4C]; padded row r gets the first half of view row r // 2 and the second half
            of view row r // 2 - 1: the first add is into zeros (exact), the second one rounding, u (S0 + S1);
  d b:      the library's column sum over B Tout rows, n u sum |dy|.
Each GEMM's per-element bound is the 3xTF32 bound of tests/test_gpu_gemm_parity.py for the plan the dispatcher makes,
composed here through a callable (form, A [M, K], B [K, N], |bias|) -> bound [M, N] on the logical operands.

CTC prefix scoring (per hypothesis n and candidate c, frames t = start .. T-1, start = max(|g|, 1)):
  phi_t = r_prev[t-1, 1] (c = last token) else lae(r_prev[t-1, 0], r_prev[t-1, 1])
  r0_t = lae(r0_{t-1}, phi_t) + x[t, c];  r1_t = lae(r1_{t-1}, r0_{t-1}) + x[t, blank];  psi = lae(psi, phi_t + x[t, c])
with lae(a, b) = numpy's logaddexp (a + ln 2 when a = b, else max + log1p(exp(-|a - b|))).  One fp32 lae is within
u |lae| + 9u of the exact lae of its fp32 arguments (the argument's rounding times exp(-d) <= 1/e, expf 4u, log1pf
1 ulp of <= ln 2, the final add).  lae is 1-Lipschitz in the max norm; more precisely its gradient is the pair of softmax
weights w_a = exp(a - lae), w_b = exp(b - lae), w_a + w_b = 1, and the bound carries those weights, so that an
argument at the log-zero floor (where one fp32 ulp is 8) passes none of its rounding on to a finite score.  Per
element, with e0, e1, ep the bounds on r0, r1, psi and Δphi = u |phi| + 9u (0 for the last token):
  e0_t = w(q0) e0 + w(phi) Δphi + u |L0| + 9u + u |r0_t|           L0 = lae(r0_{t-1}, phi_t)
  e1_t = w(q1) e1 + w(q0) e0 + u |L1| + 9u + u |r1_t|              L1 = lae(r1_{t-1}, r0_{t-1})
  ep_t = w(psi) ep + w(phi + x) (Δphi + u |phi_t + x[t, c]|) + u |psi_t| + 9u
(infinite magnitudes count 0: lae(-inf, b) = b and -inf + x are exact; a -inf result is exact).  The eos candidate's
psi = lae(r_prev[T-1, 0], r_prev[T-1, 1]) is within u |psi| + 9u.  Every occurrence of the last token (and of eos)
among the candidates gets its special case; a prefix longer than T has no path: every r is log-zero and psi is
log-zero.
The reference's numpy scorer differs in three places the tests state and exclude: with duplicate candidates it treats
only the first occurrence specially; at max(|g|, 1) = T (no frame to extend over) its psi is a view of r[T-1, 0],
so its eos assignment also writes r[T-1, 0, eos]; at |g| > T it raises IndexError.
"""
import numpy as np
import torch

U = 2.0 ** -24
F = 2.0 ** -126
LOGZERO = -100000000.0
K = 2


def _sigmoid(x):
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-x))


def _fabs(x):
    """|x| with non-finite entries counted 0 (for error increments of exact operations)."""
    return np.where(np.isfinite(x), np.abs(x), 0.0)


# ------------------------------------------------------------------------------------------------ LSTM cell
def lstm_cell_fwd(pre, c_prev):
    """pre [B, 4H] (i, f, g, o), c_prev [B, H] -> (h, c, gates [B, 4H] = activated i, f, g, o) in float64."""
    pre, c_prev = np.asarray(pre, np.float64), np.asarray(c_prev, np.float64)
    H = c_prev.shape[1]
    i, f, g, o = _sigmoid(pre[:, :H]), _sigmoid(pre[:, H:2 * H]), np.tanh(pre[:, 2 * H:3 * H]), _sigmoid(pre[:, 3 * H:])
    c = f * c_prev + i * g
    return o * np.tanh(c), c, np.concatenate([i, f, g, o], 1)


def lstm_cell_fwd_bound(pre, c_prev):
    """-> (Δh, Δc, Δgates) per element (see the module docstring)."""
    _, c, gates = lstm_cell_fwd(pre, c_prev)
    H = c.shape[1]
    i, f, g, o = gates[:, :H], gates[:, H:2 * H], gates[:, 2 * H:3 * H], gates[:, 3 * H:]
    ac = np.abs(c_prev)
    dgates = np.concatenate([6 * U * i + F, 6 * U * f + F, 4 * U * np.abs(g) + F, 6 * U * o + F], 1)
    dc = 8 * U * f * ac + 13 * U * np.abs(i * g) + 2 * F * (1 + ac)
    t = np.tanh(c)
    dh = o * (1 - t * t + dc) * dc + 12 * U * o * np.abs(t) + F
    return K * dh, K * dc, K * dgates


def lstm_cell_bwd(gates, c_prev, c, dh, dc_next=None):
    """d pre [B, 4H] and dc_prev [B, H] of lstm_cell_fwd for the given stash (gates, c)."""
    gates, c_prev, c, dh = (np.asarray(a, np.float64) for a in (gates, c_prev, c, dh))
    H = c.shape[1]
    i, f, g, o = gates[:, :H], gates[:, H:2 * H], gates[:, 2 * H:3 * H], gates[:, 3 * H:]
    t = np.tanh(c)
    dc = dh * o * (1 - t * t)
    if dc_next is not None:
        dc = dc + np.asarray(dc_next, np.float64)
    dpre = np.concatenate([dc * g * i * (1 - i), dc * c_prev * f * (1 - f), dc * i * (1 - g * g),
                           dh * t * o * (1 - o)], 1)
    return dpre, dc * f


def lstm_cell_bwd_bound(gates, c_prev, c, dh, dc_next=None):
    """-> (Δd pre [B, 4H], Δdc_prev [B, H]) for the given stash."""
    gates, c_prev, c, dh = (np.asarray(a, np.float64) for a in (gates, c_prev, c, dh))
    H = c.shape[1]
    i, f, g, o = gates[:, :H], gates[:, H:2 * H], gates[:, 2 * H:3 * H], gates[:, 3 * H:]
    dct = np.abs(dh * o) + (np.abs(np.asarray(dc_next, np.float64)) if dc_next is not None else 0.0)
    t = np.tanh(c)
    dpre = np.concatenate([17 * U * dct * np.abs(g) * i * (1 - i) + F, 17 * U * dct * np.abs(c_prev) * f * (1 - f) + F,
                           17 * U * dct * i + F, 8 * U * np.abs(dh * t) * o * (1 - o) + F], 1)
    return K * dpre, K * (14 * U * dct * f + F)


# ------------------------------------------------------------------------------------------------ cross-entropy
def _row_lse(x):
    with np.errstate(invalid="ignore", over="ignore"):
        M = x.max(1, keepdims=True)
        return (M + np.log(np.exp(x - M).sum(1, keepdims=True)))[:, 0]


def ce_fwd_bwd(x, tgt, scale=1.0, ignore_index=0):
    """x [N, V] logits, tgt [N] -> (row loss [N] (0 on ignored rows), d x [N, V] = scale (softmax - onehot), 0 on
    ignored rows).  Non-finite logits follow float64 ATen: a NaN, a +inf or an all -inf row is NaN throughout."""
    x = np.asarray(x, np.float64)
    tgt = np.asarray(tgt, np.int64)
    N, V = x.shape
    keep = tgt != ignore_index
    rows = np.arange(N)
    lse = _row_lse(x)
    bad = np.isnan(x).any(1) | np.isposinf(x).any(1) | np.isneginf(x).all(1)
    lse = np.where(bad, np.nan, lse)
    with np.errstate(invalid="ignore", over="ignore"):
        loss = np.where(keep, lse - x[rows, np.where(keep, tgt, 0)], 0.0)
        p = np.exp(x - lse[:, None])
    p[rows[keep], tgt[keep]] -= 1.0
    dx = np.where(keep[:, None], scale * p, 0.0)
    return loss, dx


def ce_bounds(x, tgt, scale=1.0, ignore_index=0):
    """-> (Δ row loss [N], Δ d x [N, V]) for the rows with finite lse (other rows: NaN bounds, checked by mask)."""
    x = np.asarray(x, np.float64)
    tgt = np.asarray(tgt, np.int64)
    N, V = x.shape
    keep = tgt != ignore_index
    n = -(-V // 32)
    fin = np.where(np.isfinite(x), x, np.nan)
    with np.errstate(invalid="ignore", over="ignore"):
        M = np.nanmax(np.where(np.isnan(fin), -np.inf, fin), 1)
        xmin = np.nanmin(np.where(np.isnan(fin), np.inf, fin), 1)
        lse = _row_lse(x)
        dS = U * (M - xmin) + 6 * U * n + 12 * U
        dlse = dS + 2 * U * (lse - M) + U * np.abs(lse)
        loss = lse - x[np.arange(N), np.where(keep, tgt, 0)]
        dloss = np.where(keep, dlse + U * np.abs(loss), 0.0)
        p = np.exp(x - lse[:, None])
        arg = np.where(p > 0, U * np.abs(x - lse[:, None]), 0.0)
    onehot = np.zeros_like(x)
    onehot[np.arange(N)[keep], tgt[keep]] = 1.0
    ddx = np.abs(scale) * (p * (dlse[:, None] + arg + 4 * U) + 4 * U * np.abs(p - onehot)) + F
    return K * dloss, np.where(keep[:, None], K * ddx, 0.0)


# ------------------------------------------------------------------------------------------------ Conv1d k4 s2 p1
def conv_geometry(B, T):
    """-> (Tout, half, Tp, M): output frames, view rows per utterance, padded rows per utterance, GEMM rows."""
    Tout = T // 2
    half = Tout + 1
    return Tout, half, 2 * half, B * half - 1


def conv_view(x):
    """x [B, T, C] (float64 torch) -> the im2col view the GEMMs read: [B half, 4C], row b half + t = padded rows
    2t .. 2t+3 of utterance b (the last row of the last utterance, which would read past the buffer, is zero)."""
    B, T, C = x.shape
    _, half, Tp, _ = conv_geometry(B, T)
    xp = x.new_zeros(B * Tp + 2, C)
    xp[:B * Tp].view(B, Tp, C)[:, 1:T + 1] = x
    flat = xp.reshape(-1)
    idx = 2 * C * torch.arange(B * half, device=x.device)[:, None] + torch.arange(4 * C, device=x.device)[None, :]
    return flat[idx]


def conv_weight_matrix(w):
    """w [O, C, 4] -> [O, 4C] with K index tap * C + channel."""
    O, C, _ = w.shape
    return w.permute(0, 2, 1).reshape(O, 4 * C)


def conv_k4s2(x, w, b, dy):
    """Float64 forward and gradients as explicit view sums: x [B, T, C], w [O, C, 4], b [O] or None, dy [B, Tout, O]
    -> dict(y [B, Tout, O], dx [B, T, C], dw [O, C, 4], db [O] or None)."""
    x, w, dy = x.double(), w.double(), dy.double()
    B, T, C = x.shape
    O = w.shape[0]
    Tout, half, Tp, M = conv_geometry(B, T)
    A = conv_view(x)
    wm = conv_weight_matrix(w)
    y = (A @ wm.t()).view(B, half, O)[:, :Tout]
    if b is not None:
        y = y + b.double()
    dyf = dy.new_zeros(B, half, O)
    dyf[:, :Tout] = dy
    dy2 = dyf.view(B * half, O)
    dcols = (dy2 @ wm).view(B, half, 2, 2 * C)
    dxp = dy.new_zeros(B, half + 1, 2 * C)
    dxp[:, :half] += dcols[:, :, 0]
    dxp[:, 1:] += dcols[:, :, 1]
    dx = dxp.view(B, Tp + 2, C)[:, 1:T + 1]
    dwm = dy2[:M].t() @ A[:M]
    dw = dwm.view(O, 4, C).permute(0, 2, 1)
    db = dy.reshape(-1, O).sum(0) if b is not None else None
    return dict(y=y, dx=dx, dw=dw, db=db)


def conv_k4s2_bounds(x, w, b, dy, gemm_bound):
    """Per-element bounds of conv_k4s2's outputs.  gemm_bound(form, A [M, K], B [K, N], babs [N] or None) -> [M, N]
    is the 3xTF32 bound of one GEMM on its logical float64 operands (form 'tn', 'nn' or 'nt')."""
    x, w, dy = x.double(), w.double(), dy.double()
    B, T, C = x.shape
    O = w.shape[0]
    Tout, half, Tp, M = conv_geometry(B, T)
    A = conv_view(x)
    wm = conv_weight_matrix(w)
    babs = b.double().abs() if b is not None else None
    by = x.new_zeros(B * half, O)
    by[:M] = gemm_bound("tn", A[:M], wm.t(), babs)
    dyf = dy.new_zeros(B, half, O)
    dyf[:, :Tout] = dy
    dy2 = dyf.view(B * half, O)
    bc = gemm_bound("nn", dy2, wm, None).view(B, half, 2, 2 * C)
    sc = (dy2.abs() @ wm.abs()).view(B, half, 2, 2 * C)
    bxp = dy.new_zeros(B, half + 1, 2 * C)
    bxp[:, :half] += bc[:, :, 0] + U * sc[:, :, 0]
    bxp[:, 1:] += bc[:, :, 1] + U * sc[:, :, 1]
    bdw = gemm_bound("nt", dy2[:M].t(), A[:M], None).view(O, 4, C).permute(0, 2, 1)
    bdb = B * Tout * U * dy.abs().reshape(-1, O).sum(0) if b is not None else None
    return dict(y=by.view(B, half, O)[:, :Tout], dx=bxp.view(B, Tp + 2, C)[:, 1:T + 1], dw=bdw, db=bdb)


# ------------------------------------------------------------------------------------------------ CTC prefix scoring
def _lae_w(a, b):
    """lae(a, b) in float64 and its gradient (w_a, w_b) (0 where the result is -inf)."""
    L = np.logaddexp(a, b)
    fin = np.isfinite(L)
    Ls = np.where(fin, L, 0.0)
    return L, np.where(fin, np.exp(a - Ls), 0.0), np.where(fin, np.exp(b - Ls), 0.0)


def prefix_score(x, r_prev, prefixes, cands, blank=0, eos=1, logzero=LOGZERO):
    """x [T, V] fp32 log-probs, r_prev [N, T, 2], prefixes: N token lists, cands [N, C] ->
    (psi [N, C], r [N, C, T, 2], Δpsi [N, C], Δr [N, C, T, 2]) in float64, the kernel's semantics (module docstring)."""
    x = np.asarray(x, np.float64)
    r_prev = np.asarray(r_prev, np.float64)
    cands = np.asarray(cands, np.int64)
    N, C = cands.shape
    T = x.shape[0]
    plen = np.array([len(g) for g in prefixes])
    last = np.array([g[-1] if len(g) else -1 for g in prefixes])
    same = (plen[:, None] > 0) & (cands == last[:, None])
    start = np.maximum(plen, 1)
    r = np.full((N, C, T, 2), logzero)
    br = np.zeros((N, C, T, 2))
    q0 = np.where(plen[:, None] == 0, x[0][cands], logzero)
    r[:, :, 0, 0] = q0
    q0 = np.where((start - 1 == 0)[:, None], q0, logzero)
    q1 = np.full((N, C), logzero)
    psi = q0.copy()
    e0, e1, ep = np.zeros((N, C)), np.zeros((N, C)), np.zeros((N, C))
    lae_err = lambda L: U * _fabs(L) + 9 * U                                      # noqa: E731
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(1, T):
            live = (t >= start)[:, None]
            p0, p1 = r_prev[:, t - 1, 0][:, None], r_prev[:, t - 1, 1][:, None]
            sp = np.logaddexp(p0, p1)
            phi = np.where(same, p1, sp)
            dphi = np.where(same, 0.0, lae_err(sp))
            xc, xb = x[t][cands], x[t, blank]
            L0, w0q, w0p = _lae_w(q0, phi)
            L1, w1q, w1r = _lae_w(q1, q0)
            Lp, wps, wpx = _lae_w(psi, phi + xc)
            n0, n1 = L0 + xc, L1 + xb
            d0 = w0q * e0 + w0p * dphi + lae_err(L0) + U * _fabs(n0)
            d1 = w1q * e1 + w1r * e0 + lae_err(L1) + U * _fabs(n1)
            dp = wps * ep + wpx * (dphi + U * _fabs(phi + xc)) + lae_err(Lp)
            d0, d1, dp = (np.where(np.isfinite(v), d, 0.0) for v, d in ((n0, d0), (n1, d1), (Lp, dp)))
            q0, q1, psi = (np.where(live, a, b) for a, b in ((n0, q0), (n1, q1), (Lp, psi)))
            e0, e1, ep = (np.where(live, a, b) for a, b in ((d0, e0), (d1, e1), (dp, ep)))
            r[:, :, t, 0] = np.where(live, q0, r[:, :, t, 0])
            r[:, :, t, 1] = np.where(live, q1, r[:, :, t, 1])
            br[:, :, t, 0] = np.where(live, e0, 0.0)
            br[:, :, t, 1] = np.where(live, e1, 0.0)
        sp = np.logaddexp(r_prev[:, T - 1, 0], r_prev[:, T - 1, 1])[:, None]
    is_eos = cands == eos
    bpsi = np.where(is_eos, lae_err(sp), ep)
    psi = np.where(is_eos, sp, psi)
    return psi, r, K * bpsi, K * br
