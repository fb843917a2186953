"""CPU ORACLE (test infrastructure, NOT a product path).

numpy restatement of the reference's hot-path arithmetic.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this package; the product (end-to-end-asr-pytorch_b200/) never does
and fails loudly without its CUDA library.

The reference itself is Python glue over third-party kernels that are NOT under /root/reference:
  * torchaudio.compliance.kaldi.fbank (requirements.txt:9, unpinned; installed 2.11.0+cu128) - call site
    src/audio.py:97,104-108; algorithm restated from kaldi.py:44-83,154-217,436-511,591-646;
  * ATen LSTM / _ctc_loss / conv / softmax / cross-entropy (requirements.txt:8 torch>=1.2.0; installed
    2.11.0+cu128) - call sites src/module.py:112-113, src/asr.py:175-177, bin/train_asr.py:47-49,123-131;
    algorithms restated from the published definitions (Hochreiter&Schmidhuber LSTM with PyTorch's i,f,g,o gate
    order; Graves 2006 CTC alpha/beta with ATen's conventions, SURVEY.md F8/F9).
Pinning: tests/test_oracle.py checks every function here against golden vectors produced by RUNNING the reference
(imported from /root/reference with the shims in oracle/ref_shim.py) - see oracle/make_golden.py and tests/golden/.
The reference's own tests hold no golden values for this path (tests/test_audio.py:24,53-55,72,87,103 only pin
shapes / CMVN mean&std / delta self-consistency) - those properties are re-checked too.

All functions take / return numpy arrays; `dtype` selects float32 (mimic) or float64 (tie-break authority).
"""
import math

import numpy as np

FLT_EPS = np.float32(1.1920928955078125e-07)


# ------------------------------------------------------------------------------------------------ front end
def povey_window(n, dtype=np.float64):
    # kaldi.py:98-100  hann(periodic=False) ** 0.85
    k = np.arange(n, dtype=np.float64)
    w = (0.5 - 0.5 * np.cos(2.0 * np.pi * k / (n - 1))) ** 0.85
    return w.astype(dtype)


def mel_banks(num_bins, n_fft, sample_freq, low_freq=20.0, high_freq=0.0, dtype=np.float64):
    # kaldi.py:436-511 without VTLN; returns [num_bins, n_fft//2 + 1] (Nyquist column zero, kaldi.py:626)
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    bw = sample_freq / n_fft
    mel = lambda f: 1127.0 * np.log(1.0 + f / 700.0)
    lo, hi = mel(low_freq), mel(high_freq)
    delta = (hi - lo) / (num_bins + 1)
    b = np.arange(num_bins, dtype=np.float64)[:, None]
    left, center, right = lo + b * delta, lo + (b + 1.0) * delta, lo + (b + 2.0) * delta
    m = mel(bw * np.arange(n_fft // 2, dtype=np.float64))[None, :]
    up = (m - left) / (center - left)
    down = (right - m) / (right - center)
    bins = np.maximum(0.0, np.minimum(up, down))
    return np.pad(bins, ((0, 0), (0, 1))).astype(dtype)


def fbank(wave, sample_freq=16000.0, num_mel_bins=40, frame_length=25.0, frame_shift=10.0, preemph=0.97,
          remove_dc=True, low_freq=20.0, high_freq=0.0, dtype=np.float64):
    """wave [N] in [-1,1] -> [m, num_mel_bins] log mel energies; kaldi.py:591-646 with the reference's options
    (dither 0, snip_edges, povey window, power spectrum, log floor = float eps)."""
    x = np.asarray(wave, dtype=dtype)
    shift = int(sample_freq * frame_shift * 0.001)
    win = int(sample_freq * frame_length * 0.001)
    n_fft = 1 if win == 0 else 2 ** (win - 1).bit_length()
    n = x.shape[0]
    if n < win:
        return np.zeros((0, num_mel_bins), dtype=dtype)
    m = 1 + (n - win) // shift                                              # kaldi.py:67
    idx = np.arange(win)[None, :] + shift * np.arange(m)[:, None]
    fr = x[idx]                                                              # [m, win]
    if remove_dc:
        fr = fr - fr.mean(axis=1, keepdims=True)                             # kaldi.py:183-186
    if preemph != 0.0:
        prev = np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)               # replicate pad, kaldi.py:193-197
        fr = fr - dtype(preemph) * prev
    fr = fr * povey_window(win, dtype)[None, :]
    fr = np.pad(fr, ((0, 0), (0, n_fft - win)))
    spec = np.abs(np.fft.rfft(fr.astype(np.float64), axis=1)).astype(dtype) ** 2   # kaldi.py:616-618
    mel = spec @ mel_banks(num_mel_bins, n_fft, sample_freq, low_freq, high_freq, dtype).T
    return np.log(np.maximum(mel, dtype(FLT_EPS))).astype(dtype)             # kaldi.py:633


def fbank_tables(wave, window, mel, win, shift, remove_dc=True, preemph=0.97, use_log=True, log_floor=FLT_EPS):
    """float64 fbank on given tables: window [win] and dense mel weights [n_mel, n_fft//2 + 1], taken at the values
    passed (the kernel's fp32 tables; torchaudio builds its mel weights in fp32 even for a float64 waveform), every
    other step in float64.  wave [N] -> [m, n_mel], m = 1 + (N - win) // shift (snip_edges); log of
    max(mel, log_floor) when use_log, else the linear mel energies."""
    x = np.asarray(wave, np.float64)
    mel = np.asarray(mel, np.float64)
    n_fft = 2 * (mel.shape[1] - 1)
    if x.shape[0] < win:
        return np.zeros((0, mel.shape[0]))
    m = 1 + (x.shape[0] - win) // shift
    fr = x[np.arange(win)[None, :] + shift * np.arange(m)[:, None]]
    if remove_dc:
        fr = fr - fr.mean(axis=1, keepdims=True)
    if preemph != 0.0:
        fr = fr - float(preemph) * np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)
    fr = fr * np.asarray(window, np.float64)[None, :win]
    spec = np.abs(np.fft.rfft(fr, n=n_fft, axis=1)) ** 2
    e = spec @ mel.T
    return np.log(np.maximum(e, float(log_floor))) if use_log else e


def delta_filters(order, window):
    # src/audio.py:57-77
    scales = [[1.0]]
    for i in range(1, order + 1):
        prev_off = (len(scales[i - 1]) - 1) // 2
        cur_off = prev_off + window
        cur = [0.0] * (len(scales[i - 1]) + 2 * window)
        norm = 0.0
        for j in range(-window, window + 1):
            norm += j * j
            for k in range(-prev_off, prev_off + 1):
                cur[j + k + cur_off] += j * scales[i - 1][k + prev_off]
        scales.append([v / norm for v in cur])
    width = len(scales[-1])
    out = np.zeros((order + 1, width))
    for i, s in enumerate(scales):
        p = (width - len(s)) // 2
        out[i, p:p + len(s)] = s
    return out


def delta_cmvn(fb, order=2, window=2, apply_cmvn=True, eps=1e-10, dtype=np.float64):
    """fb [m, F] -> [m, F*(order+1)] : stacked deltas with ZERO padding in time (src/audio.py:51-54), per-utterance
    CMVN over time with the unbiased std (src/audio.py:25-27), channel-major layout (src/audio.py:85-89)."""
    fb = np.asarray(fb, dtype=dtype)
    m, F = fb.shape
    filt = delta_filters(order, window).astype(dtype)
    pad = (filt.shape[1] - 1) // 2
    xp = np.pad(fb, ((pad, pad), (0, 0)))
    chans = []
    for o in range(order + 1):
        acc = np.zeros_like(fb)
        for tap in range(filt.shape[1]):
            if filt[o, tap] != 0:
                acc = acc + filt[o, tap] * xp[tap:tap + m]
        chans.append(acc)
    x = np.stack(chans, 0)                                                   # [C, m, F]
    if apply_cmvn and m > 0:
        mean = x.mean(axis=1, keepdims=True)
        std = x.std(axis=1, ddof=1, keepdims=True) if m > 1 else np.full_like(mean, np.nan)
        x = (x - mean) / (dtype(eps) + std)
    return np.transpose(x, (1, 0, 2)).reshape(m, F * (order + 1)).astype(dtype)


# ------------------------------------------------------------------------------------------------ LSTM
def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_direction(x, w_ih, w_hh, b_ih, b_hh, reverse=False, dtype=np.float64):
    """x [B,T,I]; PyTorch parameter layout (gate rows i,f,g,o); zero initial state; returns h [B,T,H]."""
    x = np.asarray(x, dtype)
    B, T, _ = x.shape
    H = w_hh.shape[1]
    w_ih, w_hh = np.asarray(w_ih, dtype), np.asarray(w_hh, dtype)
    bias = np.asarray(b_ih, dtype) + np.asarray(b_hh, dtype)
    h = np.zeros((B, H), dtype)
    c = np.zeros((B, H), dtype)
    out = np.zeros((B, T, H), dtype)
    order = range(T - 1, -1, -1) if reverse else range(T)
    for t in order:
        g = x[:, t] @ w_ih.T + h @ w_hh.T + bias
        i, f, gg, o = _sigmoid(g[:, :H]), _sigmoid(g[:, H:2 * H]), np.tanh(g[:, 2 * H:3 * H]), _sigmoid(g[:, 3 * H:])
        c = f * c + i * gg
        h = o * np.tanh(c)
        out[:, t] = h
    return out


def bilstm(x, params, dtype=np.float64):
    """params: dict with weight_ih_l0, weight_hh_l0, bias_ih_l0, bias_hh_l0 [+ *_reverse]; runs over the padded
    frames exactly like the reference (src/module.py:129-132, no packing)."""
    fw = lstm_direction(x, params["weight_ih_l0"], params["weight_hh_l0"], params["bias_ih_l0"],
                        params["bias_hh_l0"], False, dtype)
    if "weight_ih_l0_reverse" not in params:
        return fw
    bw = lstm_direction(x, params["weight_ih_l0_reverse"], params["weight_hh_l0_reverse"],
                        params["bias_ih_l0_reverse"], params["bias_hh_l0_reverse"], True, dtype)
    return np.concatenate([fw, bw], axis=-1)


def lstm_cell(pre, c_prev):
    H = c_prev.shape[1]
    i, f, g, o = _sigmoid(pre[:, :H]), _sigmoid(pre[:, H:2 * H]), np.tanh(pre[:, 2 * H:3 * H]), _sigmoid(pre[:, 3 * H:])
    c = f * c_prev + i * g
    return o * np.tanh(c), c


# ------------------------------------------------------------------------------------------------ CTC
def log_softmax(x):
    m = x.max(axis=-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(axis=-1, keepdims=True))


def _lse(vals):
    m = max(vals)
    if m == -np.inf:
        return -np.inf
    return m + math.log(sum(math.exp(v - m) for v in vals))


def ctc_single(lp, target, blank=0):
    """lp [T,V] log-probs (T = input length), target list[int] (L = target length).
    Returns nll, alpha [T,S], beta [T,S], grad [T,V] in ATen's convention exp(lp) - exp(lcab + nll - lp)."""
    lp = np.asarray(lp, np.float64)
    T, V = lp.shape
    L = len(target)
    S = 2 * L + 1
    ext = [blank] * S
    for i, c in enumerate(target):
        ext[2 * i + 1] = int(c)
    NEG = -np.inf
    alpha = np.full((T, S), NEG)
    beta = np.full((T, S), NEG)
    if T == 0:
        return (0.0 if L == 0 else np.inf), alpha, beta, np.zeros((0, V))
    alpha[0, 0] = lp[0, blank]
    if S > 1:
        alpha[0, 1] = lp[0, ext[1]]
    for t in range(1, T):
        for s in range(S):
            v = [alpha[t - 1, s]]
            if s > 0:
                v.append(alpha[t - 1, s - 1])
            if s > 1 and ext[s] != blank and ext[s] != ext[s - 2]:
                v.append(alpha[t - 1, s - 2])
            alpha[t, s] = _lse(v) + lp[t, ext[s]]
    tail = [alpha[T - 1, S - 1]] + ([alpha[T - 1, S - 2]] if S > 1 else [])
    nll = -_lse(tail)
    beta[T - 1, S - 1] = lp[T - 1, blank]
    if S > 1:
        beta[T - 1, S - 2] = lp[T - 1, ext[S - 2]]
    for t in range(T - 2, -1, -1):
        for s in range(S):
            v = [beta[t + 1, s]]
            if s + 1 < S:
                v.append(beta[t + 1, s + 1])
            if s + 2 < S and ext[s + 2] != blank and ext[s + 2] != ext[s]:
                v.append(beta[t + 1, s + 2])
            beta[t, s] = _lse(v) + lp[t, ext[s]]
    grad = np.zeros((T, V))
    for t in range(T):
        per_class = {}
        for s in range(S):
            per_class.setdefault(ext[s], []).append(alpha[t, s] + beta[t, s])
        occ = np.full(V, NEG)
        for c, vals in per_class.items():
            occ[c] = _lse(vals)
        with np.errstate(over="ignore", invalid="ignore"):
            grad[t] = np.exp(lp[t]) - np.exp(occ + nll - lp[t])
    return nll, alpha, beta, grad


def ctc_loss(log_probs, targets, input_lengths, target_lengths, blank=0):
    """log_probs [B,T,V]; targets [B,Lmax] zero padded.  Returns (loss_mean, nll[B], grad[B,T,V]) where the loss is
    torch.nn.CTCLoss(reduction='mean') = mean_b nll_b / max(len_b,1) and grad is d(loss)/d(log_probs) in ATen's
    convention (zero beyond each input length)."""
    B, T, V = log_probs.shape
    nll = np.zeros(B)
    grad = np.zeros((B, T, V))
    for b in range(B):
        Tb, Lb = int(input_lengths[b]), int(target_lengths[b])
        n, _, _, g = ctc_single(log_probs[b, :Tb], [int(v) for v in targets[b, :Lb]], blank)
        nll[b] = n
        grad[b, :Tb] = g / (max(Lb, 1) * B)
    loss = float(np.mean(nll / np.maximum(np.asarray(target_lengths, np.float64), 1.0)))
    return loss, nll, grad


# ------------------------------------------------------------------------------------------------ attention
def loc_attention_step(q, key, value, prev_att, k_len, conv_w, proj_w, energy_w, energy_b, temperature):
    """One location-aware attention step (src/module.py:234-258 + 189-195), single head.
    q [B,D], key [B,T,D] (already tanh(proj_k)), value [B,T,E], prev_att [B,T], conv_w [K,1,2r+1], proj_w [D,K],
    energy_w [1,D], energy_b [1].  Returns (context [B,E], attn [B,T])."""
    B, T, D = key.shape
    K, _, W = conv_w.shape
    r = (W - 1) // 2
    pp = np.pad(prev_att, ((0, 0), (r, r)))
    conv = np.zeros((B, K, T))
    for j in range(W):
        conv += conv_w[None, :, 0, j, None] * pp[:, None, j:j + T]
    loc = np.tanh(np.einsum("bkt,dk->btd", conv, proj_w))
    e = np.tanh(key + q[:, None, :] + loc) @ energy_w[0] + energy_b[0]
    e = e / temperature
    mask = np.arange(T)[None, :] >= np.asarray(k_len)[:, None]
    e = np.where(mask, -np.inf, e)
    e = e - e.max(axis=1, keepdims=True)
    a = np.exp(e)
    a = a / a.sum(axis=1, keepdims=True)
    ctx = np.einsum("bt,bte->be", a, value)
    return ctx, a


# ------------------------------------------------------------------------------------------------ CE
def cross_entropy(logits, target, ignore_index=0):
    """mean over non-ignored rows of -log_softmax(logits)[target] (bin/train_asr.py:47,130-131); also the logit
    gradient."""
    lp = log_softmax(np.asarray(logits, np.float64))
    target = np.asarray(target)
    keep = target != ignore_index
    n = max(int(keep.sum()), 1)
    rows = np.arange(len(target))
    loss = float(-(lp[rows, target] * keep).sum() / n)
    grad = np.exp(lp)
    grad[rows, target] -= 1.0
    grad = grad * keep[:, None] / n
    return loss, grad


# ------------------------------------------------------------------------------------------------ CTC prefix scoring
def ctc_prefix_init(x, blank=0, logzero=-100000000.0):
    """CTCPrefixScore.init_state (src/ctc.py:27-35): x [T,V] log-probs -> r [T,2] (non-blank, blank)."""
    x = np.asarray(x, np.float32)
    r = np.full((x.shape[0], 2), logzero, dtype=np.float32)
    r[:, 1] = np.cumsum(x[:, blank].astype(np.float64)).astype(np.float32)
    return r


def ctc_prefix_cheap(x, g, r_prev, candidates, blank=0, eos=1, logzero=-100000000.0):
    """CTCPrefixScore.cheap_compute (src/ctc.py:81-116), float32 like the reference: (psi [C], r [C,T,2])."""
    x = np.asarray(x, np.float32)
    r_prev = np.asarray(r_prev, np.float32)
    T = x.shape[0]
    cand = list(candidates)
    C = len(cand)
    r = np.full((T, 2, C), logzero, dtype=np.float32)
    start = max(1, len(g))
    if len(g) == 0:
        r[0, 0, :] = x[0, cand]
    psi = r[start - 1, 0, :].copy()
    sum_prev = np.logaddexp(r_prev[:, 0], r_prev[:, 1])
    phi = np.repeat(sum_prev[:, None], C, axis=1)
    if len(g) > 0 and g[-1] in cand:
        phi[:, cand.index(g[-1])] = r_prev[:, 1]
    for t in range(start, T):
        r[t, 0, :] = np.logaddexp(r[t - 1, 0, :], phi[t - 1]) + x[t, cand]
        r[t, 1, :] = np.logaddexp(r[t - 1, 1, :], r[t - 1, 0, :]) + x[t, blank]
        psi = np.logaddexp(psi, phi[t - 1] + x[t, cand])
    if eos in cand:
        psi[cand.index(eos)] = sum_prev[-1]
    return psi, np.rollaxis(r, 2)
