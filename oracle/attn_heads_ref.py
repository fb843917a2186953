"""Float64 closed form of one multi-head location-aware attention step (forward and backward, as explicit sums), each
intermediate with an absolute-value companion, and from them a per-element bound on the fp32 rounding of every output
of b200asr_locattn_heads_fwd / _bwd_acc (csrc/attention.cu).  Notation, the softmax / context / softmax-backward
bounds and the accumulator rules are those of oracle/attn_ref.py; what differs is the location term and the head sum.

Rows r = b·N + n; row r is masked at t < len[b] = clamp(enc_len[b], 0, T) (never len[r mod B]).
  conv[b,k,t] = sum_n sum_j w_conv[k,n,j] prev[b,n,t+j-R]   one fmaf chain of N·W terms (n outer, j inner):
                                                              Δconv = N W u conv~
  pre, loc                                                  as attn_ref with W -> N W: Δpre = (N W + K) u pre~
  x[r,t,d] = (key + q) + loc[b,t,d], s = tanh(x), e[r,t]    as attn_ref, per row, with loc of utterance r // N
  attn, ctx, g, dot, de, dpre = d(key), d(value)            as attn_ref, per row (the cluster partials of g: the
                                                              CS = cluster_size(T, E) CTAs of the utterance's cluster)
  d(q)[r]   = sum_t dpre[r,t]    a per-CTA chain over my frames, the tile sums added into shared memory, then the CS
                                 partials added by the caller:  Σ_t Δdpre + (T + CS) u Σ_t dpre~
  hsum[b,t,d] = sum_n dpre[bN+n,t,d]   0 + dpre_0 + ... + dpre_{N-1} in shared memory, head order:
                                 Δhsum = Σ_n Δdpre + N u Σ_n dpre~,                  hsum~ = Σ_n dpre~
  dloc = hsum (1 - loc^2)                                   Δdloc = Δhsum + hsum~ (2Δloc + 4u)
  d(w_proj)[b] = sum_t dloc conv        (per-CTA chain)     Σ_t (Δdloc conv~ + dloc~ Δconv) + T u Σ_t dloc~ conv~
  d(w_e)[b]    = sum_n sum_t de s       (per-CTA chain over the N T terms of my slice)
                                                            Σ (Δde + de~ Δs) + N T u Σ de~
  d(b_e)[b]    = sum_n sum_t de                             Σ Δde + N T u Σ de~
  dconv[b,k,t] = sum_d dloc w_proj[d,k] (t < len)           Δdconv = Σ_d Δdloc |w_proj| + (ceil(D/32) + 5) u dconv~
  d(w_conv)[b,k,n,j] = sum_{t<len} dconv[b,k,t] prev[b,n,t+j-R]   Σ_t Δdconv |prev| + T u Σ_t dconv~ |prev|
  d(prev)[b,n,t'] = sum_{k,j} dconv[b,k,t'-j+R] w_conv[k,n,j]      lane-strided over the K W terms, a warp tree:
                                                            Σ Δdconv |w_conv| + (ceil(K W/32) + 6) u Σ dconv~ |w_conv|
The weight gradients are per utterance ([B, ...]); the caller's sum over B·CS partials adds (B·CS) u as in attn_ref.
"""
import math

import numpy as np

from .attn_ref import U, Step, _context, _lens, _softmax, _softmax_bwd, cluster_size


def loc_heads_step(q, key, value, prev, lens, w_conv, w_proj, w_e, b_e, temperature, num_head, dctx=None, dattn=None,
                   attn=None):
    """q [R,D], key [R,T,D], value [R,T,E] (R = B·N rows, r = b·N + n), prev [B,N,T], lens [B], w_conv [K,N,W],
    w_proj [D,K], w_e [D], b_e scalar.  With dctx [R,E] (and dattn [R,T] or None) also the backward, at the given
    attention attn [R,T] (default: the exact forward attention)."""
    N = int(num_head)
    q = np.asarray(q, np.float64)
    Rr, T, D = np.shape(key)
    B = Rr // N
    E = np.shape(value)[2]
    wc = np.asarray(w_conv, np.float64)
    K, W = wc.shape[0], wc.shape[-1]
    wc = wc.reshape(K, N, W)
    R = (W - 1) // 2
    wp, we = np.asarray(w_proj, np.float64).reshape(D, K), np.asarray(w_e, np.float64).reshape(D)
    be = float(np.asarray(b_e, np.float64).reshape(-1)[0])
    ulens = _lens(lens, T)
    rlens = np.repeat(ulens, N)
    uvalid = np.arange(T)[None, :] < ulens[:, None]                                # [B, T]
    valid = np.repeat(uvalid, N, 0)                                                # [R, T]
    key = np.where(valid[:, :, None], np.asarray(key, np.float64), 0.0)
    value = np.where(valid[:, :, None], np.asarray(value, np.float64), 0.0)
    st = Step()
    st.valid, st.lens = valid, rlens
    P = np.pad(np.asarray(prev, np.float64).reshape(B, N, T), ((0, 0), (0, 0), (R, R)))
    Pw = np.lib.stride_tricks.sliding_window_view(P, W, axis=2)                   # [B, N, T, W]
    conv = np.einsum("knj,bntj->bkt", wc, Pw)
    conv_abs = np.einsum("knj,bntj->bkt", np.abs(wc), np.abs(Pw))
    conv_b = N * W * U * conv_abs
    pre = np.einsum("dk,bkt->btd", wp, conv)
    pre_abs = np.einsum("dk,bkt->btd", np.abs(wp), conv_abs)
    uloc = np.tanh(pre)                                                            # [B, T, D]
    uloc_b = (N * W + K) * U * pre_abs + 4 * U * np.abs(uloc)
    loc, loc_b = np.repeat(uloc, N, 0), np.repeat(uloc_b, N, 0)                    # per row
    x = key + q[:, None, :] + loc
    s = np.tanh(x)
    x_b = loc_b + 2 * U * (np.abs(key) + np.abs(q)[:, None, :] + np.abs(loc))
    s_b = (1 - s * s + x_b) * x_b + 4 * U * np.abs(s)
    e = (s @ we + be) / temperature
    e_abs = (np.abs(s) @ np.abs(we) + abs(be)) / abs(temperature)
    e_b = (s_b @ np.abs(we)) / abs(temperature) + (math.ceil(D / 32) + 8) * U * e_abs
    st.conv, st.loc, st.energy = conv, uloc, e
    st.attn, st.attn_b = _softmax(e, e_b, valid, T)
    st.ctx, st.ctx_b = _context(st.attn, st.attn_b, value, valid, rlens)
    if dctx is None:
        return st
    CS = cluster_size(T, E)
    _softmax_bwd(st, st.attn if attn is None else attn, dctx, dattn, value, valid, temp=temperature, E=E, CS=CS)
    de, de_abs, de_b = st.de, st.de_abs, st.de_b
    dpre = de[:, :, None] * we * (1 - s * s)
    dpre_abs = de_abs[:, :, None] * np.abs(we)
    dpre_b = np.abs(we) * (de_b[:, :, None] + de_abs[:, :, None] * (2 * s_b + 4 * U))
    st.dkey, st.dkey_abs, st.dkey_b = dpre, dpre_abs, dpre_b
    st.dq, st.dq_abs = dpre.sum(1), dpre_abs.sum(1)
    st.dq_b = dpre_b.sum(1) + (T + CS) * U * st.dq_abs
    heads = lambda a: a.reshape((B, N) + a.shape[1:])
    hsum, hsum_abs = heads(dpre).sum(1), heads(dpre_abs).sum(1)                    # [B, T, D]
    hsum_b = heads(dpre_b).sum(1) + N * U * hsum_abs
    dloc = hsum * (1 - uloc * uloc)
    dloc_b = hsum_b + hsum_abs * (2 * uloc_b + 4 * U)
    st.dwp = np.einsum("btd,bkt->bdk", dloc, conv)
    st.dwp_abs = np.einsum("btd,bkt->bdk", hsum_abs, conv_abs)
    st.dwp_b = (np.einsum("btd,bkt->bdk", dloc_b, conv_abs) + np.einsum("btd,bkt->bdk", hsum_abs, conv_b)
                + T * U * st.dwp_abs)
    st.dwe = heads(np.einsum("rt,rtd->rd", de, s)).sum(1)
    st.dwe_abs = heads(de_abs.sum(1)).sum(1)[:, None] * np.ones(D)
    st.dwe_b = (heads(np.einsum("rt,rtd->rd", de_b, np.ones_like(s)) + np.einsum("rt,rtd->rd", de_abs, s_b)).sum(1)
                + N * T * U * st.dwe_abs)
    st.dbe, st.dbe_abs = heads(de.sum(1)).sum(1), heads(de_abs.sum(1)).sum(1)
    st.dbe_b = heads(de_b.sum(1)).sum(1) + N * T * U * st.dbe_abs
    uv = uvalid[:, None, :]
    dconv = np.where(uv, np.einsum("btd,dk->bkt", dloc, wp), 0.0)
    dconv_abs = np.where(uv, np.einsum("btd,dk->bkt", hsum_abs, np.abs(wp)), 0.0)
    dconv_b = (np.where(uv, np.einsum("btd,dk->bkt", dloc_b, np.abs(wp)), 0.0)
               + (math.ceil(D / 32) + 5) * U * dconv_abs)
    st.dwc = np.einsum("bkt,bntj->bknj", dconv, Pw)
    st.dwc_abs = np.einsum("bkt,bntj->bknj", dconv_abs, np.abs(Pw))
    st.dwc_b = np.einsum("bkt,bntj->bknj", dconv_b, np.abs(Pw)) + T * U * st.dwc_abs
    flip = lambda a: np.lib.stride_tricks.sliding_window_view(np.pad(a, ((0, 0), (0, 0), (R, R))), W, axis=2)
    wflip = wc[:, :, ::-1]
    st.dprev = np.einsum("bktm,knm->bnt", flip(dconv), wflip)
    st.dprev_abs = np.einsum("bktm,knm->bnt", flip(dconv_abs), np.abs(wflip))
    st.dprev_b = (np.einsum("bktm,knm->bnt", flip(dconv_b), np.abs(wflip))
                  + (math.ceil(K * W / 32) + 6) * U * st.dprev_abs)
    return st
