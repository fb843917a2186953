"""Float64 closed forms of one location-aware and one scaled dot-product attention step (forward and backward, as
explicit sums, not autograd), each intermediate with an absolute-value companion, and from them a per-element bound
on the fp32 rounding of every output of the attention kernels (csrc/attention.cu).

Notation: u = 2^-24 (fp32 unit roundoff); for a sum S = sum_i x_i its companion is |S|~ = sum_i |x_i| (for nested sums
the companion of the inner sum replaces |inner|); Δx is the bound on |kernel x - exact x|.  Rows are masked at
t < len = clamp(enc_len, 0, T); key and value frames t >= len are zeroed here (the kernels never read them).

Forward (location-aware), per row:
  conv[k,t] = sum_j w_conv[k,j] prev[t+j-R]           fmaf chain of W = 2R+1 terms:       Δconv = W u conv~
  pre[t,d]  = sum_k w_proj[d,k] conv[k,t]              K more roundings, inputs off by Δconv: Δpre = (W + K) u pre~
  loc = tanh(pre)                                       tanhf is within 2 ulp (<= 4u relative): Δloc = Δpre + 4u|loc|
  x = (key + q) + loc                                   two adds:                          Δx = Δloc + 2u(|key|+|q|+|loc|)
  s = tanh(x)                                           Δs = (1 - s^2 + Δx) Δx + 4u|s|
  e = (sum_d w_e[d] s[t,d] + b_e) / temperature        per-lane fmaf chains of ceil(D/32), a 5-level warp tree, the
                                                        bias add, the division and fp32(temperature):
                                                        Δe = sum_d |w_e| Δs / temp + (ceil(D/32) + 8) u e~
  (dot-product: e = sum_d q[d] key[t,d] / temperature, Δe = (ceil(D/32) + 7) u e~.)
  attn[t] = exp(e_t - m) / sum_t' exp(e_t' - m)        a perturbation δ of the energies changes a_t by at most
                                                        a_t (|δ_t| + max |δ|) to first order; the subtraction adds
                                                        u|e_t - m| to δ_t, expf 2 ulp, the sum of T positive terms
                                                        (any order) T u, the division u:
                                                        Δa_t = a_t (δ_t + max_t' δ_t' + (T + 16) u),  δ = Δe + u|e - m|
                                                        (exactly 0 at t >= len, and the kernel must give exactly 0)
  ctx[c] = sum_{t<len} a_t value[t,c]                  Δctx = sum_t Δa_t |value| + (len + 2) u ctx~

Backward, for a GIVEN saved attention A (the kernels read the forward's fp32 output; the tests pass it here, so the
bound below does not contain the forward's Δa), d(ctx) and d(attn):
  g_t  = d(attn)_t + sum_c dctx_c value[t,c]          per CTA a lane-strided slice of E/CS, a warp tree, then the CS
                                                        partials and d(attn) added:  Δg = (ceil(E/CS/32) + CS + 8) u g~
  dot  = sum_{t<len} A_t g_t                           Δdot = sum A Δg + (T + 10) u sum A g~
  de_t = A_t (g_t - dot) / temperature  (t < len)     Δde = A (Δg + Δdot) / temp + 4u de~,  de~ = A (g~ + dot~) / temp
  location-aware (conv / pre / loc / s recomputed with the forward's bounds):
  dpre = de w_e (1 - s^2)        = d(key)              Δdpre = |w_e| (Δde + de~ (2Δs + 4u)),        dpre~ = de~ |w_e|
  dloc = dpre (1 - loc^2)                               Δdloc = Δdpre + dpre~ (2Δloc + 4u)
  d(q)      = sum_t dpre           (per-CTA partials)   Σ_t Δdpre + T u Σ_t dpre~
  d(w_proj) = sum_t dloc conv      (per-CTA partials)   Σ_t (Δdloc conv~ + dloc~ Δconv) + T u Σ_t dloc~ conv~
  d(w_e)    = sum_t de s                                Σ_t (Δde + de~ Δs) + T u Σ_t de~
  d(b_e)    = sum_t de  (exactly 0 for an exactly normalised A; here the float64 value for the given A)
                                                        Σ_t Δde + T u Σ_t de~
  dconv[k,t] = sum_d dloc w_proj[d,k]  (t < len)        Δdconv = Σ_d Δdloc |w_proj| + (ceil(D/32) + 5) u dconv~
  d(w_conv)[k,j] = sum_{t<len} dconv[k,t] prev[t+j-R]   Σ_t Δdconv |prev| + T u Σ_t dconv~ |prev|
  d(prev)[t'] = sum_{k,j} dconv[k,t'-j+R] w_conv[k,j]   Σ Δdconv |w_conv| + (ceil(K W/32) + 6) u Σ dconv~ |w_conv|
  d(value)[t,c] = A_t dctx_c  (t < len)                 one rounding, taken as 2u |A dctx|
  dot-product: d(key)[t] += de_t q, Δ = |q| Δde + 2u de~ |q| (+ u |C0|); d(q) = sum_t de_t key[t] per CTA,
  Σ_t |key| Δde + T u Σ_t de~ |key|.
Accumulators (the decode loop's _bwd_acc and attn_dvalue(accumulate = 1)): the result is C0 + step, one more rounding
(taken as 2u (|C0| + step~)) on top of the step's bound; over L steps (attn_dvalue's fmaf chain, the memory's d(key) and weight
partials) the per-step bounds add and one more level L u Σ_l step~ appears (attn_dvalue, a chain of single
roundings, is given 2 (L + 1) u of its companion).  Weight partials summed over B·CS rows in
fp32 by the caller add (B·CS) u of the companion.
A row with len = 0 follows the reference (softmax of an all -inf row): NaN attention and context; bounds are NaN there.
"""
import math

import numpy as np

U = 2.0 ** -24


def _lens(lens, T):
    return np.clip(np.asarray(lens, np.int64), 0, T)


def _valid(lens, T):
    return np.arange(T)[None, :] < lens[:, None]            # [B, T]


def _softmax(e, eb, valid, T):
    """attention and its bound from energies e and their bounds eb (masked frames excluded)."""
    en = np.where(valid, e, -np.inf)
    m = en.max(1, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        ex = np.where(valid, np.exp(en - m), 0.0)
        a = ex / ex.sum(1, keepdims=True)
        delta = np.where(valid, eb + U * np.abs(e - m), 0.0)
    ab = a * (delta + delta.max(1, keepdims=True) + (T + 16) * U)
    return a, np.where(valid, ab, 0.0)


def _context(a, ab, value, valid, lens):
    ctx = np.einsum("bt,btc->bc", a, value)
    ctx_abs = np.einsum("bt,btc->bc", np.abs(a), np.abs(value))
    ctxb = np.einsum("bt,btc->bc", ab, np.abs(value)) + (lens[:, None] + 2) * U * ctx_abs
    return ctx, ctxb


class Step:
    """One step's exact values (attribute x) and bounds (attribute x_b); gradient companions x_abs where a caller
    accumulates x over steps or rows."""


def _prep(key, value, lens, T):
    valid = _valid(lens, T)
    key = np.where(valid[:, :, None], np.asarray(key, np.float64), 0.0)
    value = np.where(valid[:, :, None], np.asarray(value, np.float64), 0.0)
    return key, value, valid


def _softmax_bwd(st, A, dctx, dattn, value, valid, temp, E, CS):
    T = A.shape[1]
    A = np.where(valid, np.asarray(A, np.float64), 0.0)
    dctx = np.asarray(dctx, np.float64)
    da = np.zeros_like(A) if dattn is None else np.asarray(dattn, np.float64)
    g = np.where(valid, da + np.einsum("bc,btc->bt", dctx, value), 0.0)
    gabs = np.where(valid, np.abs(da) + np.einsum("bc,btc->bt", np.abs(dctx), np.abs(value)), 0.0)
    gb = (math.ceil(E / CS / 32) + CS + 8) * U * gabs
    dot = (A * g).sum(1, keepdims=True)
    dot_abs = (A * gabs).sum(1, keepdims=True)
    dotb = (A * gb).sum(1, keepdims=True) + (T + 10) * U * dot_abs
    st.de = np.where(valid, A * (g - dot) / temp, 0.0)
    st.de_abs = np.where(valid, A * (gabs + dot_abs) / temp, 0.0)
    st.de_b = np.where(valid, A * (gb + dotb) / temp + 4 * U * st.de_abs, 0.0)
    st.dvalue = A[:, :, None] * dctx[:, None, :]
    st.dvalue_b = 2 * U * np.abs(st.dvalue)
    return A


def loc_step(q, key, value, prev, lens, w_conv, w_proj, w_e, b_e, temperature, dctx=None, dattn=None, attn=None):
    """q [B,D], key [B,T,D], value [B,T,E], prev [B,T], lens [B], w_conv [K,W], w_proj [D,K], w_e [D], b_e scalar.
    With dctx [B,E] (and dattn [B,T] or None) also the backward, at the given attention attn [B,T] (default: the
    exact forward attention)."""
    q = np.asarray(q, np.float64)
    B, T, D = np.shape(key)
    E = np.shape(value)[2]
    wc = np.asarray(w_conv, np.float64).reshape(-1, np.shape(w_conv)[-1])
    K, W = wc.shape
    R = (W - 1) // 2
    wp, we = np.asarray(w_proj, np.float64).reshape(D, K), np.asarray(w_e, np.float64).reshape(D)
    be = float(np.asarray(b_e, np.float64).reshape(-1)[0])
    lens = _lens(lens, T)
    key, value, valid = _prep(key, value, lens, T)
    st = Step()
    st.valid, st.lens = valid, lens
    P = np.pad(np.asarray(prev, np.float64), ((0, 0), (R, R)))                  # P[b, t + j] = prev[b, t + j - R]
    Pw = np.lib.stride_tricks.sliding_window_view(P, W, axis=1)                 # [B, T, W]
    conv = np.einsum("kj,btj->bkt", wc, Pw)
    conv_abs = np.einsum("kj,btj->bkt", np.abs(wc), np.abs(Pw))
    conv_b = W * U * conv_abs
    pre = np.einsum("dk,bkt->btd", wp, conv)
    pre_abs = np.einsum("dk,bkt->btd", np.abs(wp), conv_abs)
    loc = np.tanh(pre)
    loc_b = (W + K) * U * pre_abs + 4 * U * np.abs(loc)
    x = key + q[:, None, :] + loc
    s = np.tanh(x)
    x_b = loc_b + 2 * U * (np.abs(key) + np.abs(q)[:, None, :] + np.abs(loc))
    s_b = (1 - s * s + x_b) * x_b + 4 * U * np.abs(s)
    e = (s @ we + be) / temperature
    e_abs = (np.abs(s) @ np.abs(we) + abs(be)) / abs(temperature)
    e_b = (s_b @ np.abs(we)) / abs(temperature) + (math.ceil(D / 32) + 8) * U * e_abs
    st.conv, st.conv_abs, st.pre, st.pre_abs, st.loc, st.s, st.energy, st.energy_abs = (
        conv, conv_abs, pre, pre_abs, loc, s, e, e_abs)
    st.attn, st.attn_b = _softmax(e, e_b, valid, T)
    st.ctx, st.ctx_b = _context(st.attn, st.attn_b, value, valid, lens)
    if dctx is None:
        return st
    CS = cluster_size(T, E)
    A = _softmax_bwd(st, st.attn if attn is None else attn, dctx, dattn, value, valid, temp=temperature, E=E, CS=CS)
    de, de_abs, de_b = st.de, st.de_abs, st.de_b
    sat = 1 - s * s
    dpre = de[:, :, None] * we * sat
    dpre_abs = de_abs[:, :, None] * np.abs(we)
    dpre_b = np.abs(we) * (de_b[:, :, None] + de_abs[:, :, None] * (2 * s_b + 4 * U))
    st.dkey, st.dkey_abs, st.dkey_b = dpre, dpre_abs, dpre_b
    st.dq, st.dq_abs = dpre.sum(1), dpre_abs.sum(1)
    st.dq_b = dpre_b.sum(1) + T * U * st.dq_abs
    dloc = dpre * (1 - loc * loc)
    dloc_b = dpre_b + dpre_abs * (2 * loc_b + 4 * U)
    st.dwp = np.einsum("btd,bkt->bdk", dloc, conv)
    st.dwp_abs = np.einsum("btd,bkt->bdk", dpre_abs, conv_abs)
    st.dwp_b = (np.einsum("btd,bkt->bdk", dloc_b, conv_abs) + np.einsum("btd,bkt->bdk", dpre_abs, conv_b)
                + T * U * st.dwp_abs)
    st.dwe = np.einsum("bt,btd->bd", de, s)
    st.dwe_abs = de_abs.sum(1)[:, None] * np.ones(D)
    st.dwe_b = np.einsum("bt,btd->bd", de_b, np.ones_like(s)) + np.einsum("bt,btd->bd", de_abs, s_b) + T * U * st.dwe_abs
    st.dbe, st.dbe_abs = de.sum(1), de_abs.sum(1)
    st.dbe_b = de_b.sum(1) + T * U * st.dbe_abs
    dconv = np.where(valid[:, None, :], np.einsum("btd,dk->bkt", dloc, wp), 0.0)
    dconv_abs = np.where(valid[:, None, :], np.einsum("btd,dk->bkt", dpre_abs, np.abs(wp)), 0.0)
    dconv_b = (np.where(valid[:, None, :], np.einsum("btd,dk->bkt", dloc_b, np.abs(wp)), 0.0)
               + (math.ceil(D / 32) + 5) * U * dconv_abs)
    st.dwc = np.einsum("bkt,btj->bkj", dconv, Pw)
    st.dwc_abs = np.einsum("bkt,btj->bkj", dconv_abs, np.abs(Pw))
    st.dwc_b = np.einsum("bkt,btj->bkj", dconv_b, np.abs(Pw)) + T * U * st.dwc_abs
    flip = lambda x: np.lib.stride_tricks.sliding_window_view(np.pad(x, ((0, 0), (0, 0), (R, R))), W, axis=2)
    st.dprev = np.einsum("bktm,km->bt", flip(dconv), wc[:, ::-1])
    st.dprev_abs = np.einsum("bktm,km->bt", flip(dconv_abs), np.abs(wc[:, ::-1]))
    st.dprev_b = (np.einsum("bktm,km->bt", flip(dconv_b), np.abs(wc[:, ::-1]))
                  + (math.ceil(K * W / 32) + 6) * U * st.dprev_abs)
    return st


def dot_step(q, key, value, lens, num_head, temperature, dctx=None, dattn=None, attn=None):
    """Rows r = b·N + n: q [R,D], key [R,T,D], value [R,T,E], lens [B] (row r masked by lens[r // N])."""
    q = np.asarray(q, np.float64)
    Rr, T, D = np.shape(key)
    E = np.shape(value)[2]
    lens = np.repeat(_lens(lens, T), num_head)
    key, value, valid = _prep(key, value, lens, T)
    st = Step()
    st.valid, st.lens = valid, lens
    e = np.einsum("rd,rtd->rt", q, key) / temperature
    e_abs = np.einsum("rd,rtd->rt", np.abs(q), np.abs(key)) / abs(temperature)
    st.energy, st.energy_abs = e, e_abs
    st.attn, st.attn_b = _softmax(e, (math.ceil(D / 32) + 7) * U * e_abs, valid, T)
    st.ctx, st.ctx_b = _context(st.attn, st.attn_b, value, valid, lens)
    if dctx is None:
        return st
    CS = cluster_size(T, E)
    _softmax_bwd(st, st.attn if attn is None else attn, dctx, dattn, value, valid, temp=temperature, E=E, CS=CS)
    st.dkey = st.de[:, :, None] * q[:, None, :]
    st.dkey_abs = st.de_abs[:, :, None] * np.abs(q)[:, None, :]
    st.dkey_b = st.de_b[:, :, None] * np.abs(q)[:, None, :] + 2 * U * st.dkey_abs
    st.dq = np.einsum("rt,rtd->rd", st.de, key)
    st.dq_abs = np.einsum("rt,rtd->rd", st.de_abs, np.abs(key))
    st.dq_b = np.einsum("rt,rtd->rd", st.de_b, np.abs(key)) + T * U * st.dq_abs
    return st


def dvalue(attn_steps, dctx_steps, c0=None):
    """b200asr_attn_dvalue: C0 + sum_l attn[b,l,t] dctx[b,l,:] -> (value [B,T,E], bound)."""
    a, d = np.asarray(attn_steps, np.float64), np.asarray(dctx_steps, np.float64)
    L = a.shape[1]
    v = np.einsum("blt,blc->btc", a, d)
    vabs = np.einsum("blt,blc->btc", np.abs(a), np.abs(d))
    if c0 is not None:
        v = v + np.asarray(c0, np.float64)
        vabs = vabs + np.abs(np.asarray(c0, np.float64))
    return v, 2 * (L + 1) * U * vabs


def accumulate(c0, step_vals, step_bounds, step_abs):
    """C0 + sum over steps of a per-step quantity, with the per-step bounds and one more accumulation level."""
    c0 = np.asarray(c0, np.float64)
    L = len(step_vals)
    val = c0 + sum(step_vals)
    return val, sum(step_bounds) + (L + 1) * U * (np.abs(c0) + sum(step_abs))


def cluster_size(T, E):
    """b200asr_locattn_cluster_size: 4 CTAs where E % (4 CS) == 0 allows it; fewer for T < 8 CS unless that would
    leave more than 1024 value columns per CTA."""
    cs = 4
    while cs > 1 and (E % (4 * cs) != 0 or (T < 8 * cs and E // (cs // 2) <= 1024)):
        cs >>= 1
    return cs


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound per element; a zero bound demands equality, NaN or a mismatch in finiteness is inf."""
    got, ref, bound = (np.broadcast_to(np.asarray(x, np.float64), np.shape(ref)) for x in (got, ref, bound))
    if got.size == 0:
        return 0.0
    err = np.abs(got - ref)
    if not np.isfinite(got).all() or not np.isfinite(ref).all():
        return math.inf
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nan_to_num(r, nan=math.inf, posinf=math.inf).max())
