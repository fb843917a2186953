"""Front end (csrc/fbank.cu: fbank_kernel, delta_stats_kernel, delta_norm_kernel) against float64, across the options
`create_transform` accepts, at the lengths and layouts where the kernels have separate code paths.

Every value is compared with a bound derived from fp32 rounding; K = 8 throughout, as in test_gpu_lstm_variants.py,
and u = 2^-24.

fbank, linear domain, per (frame, mel bin).  R_f is the float64 2-norm of the frame's RAW samples (not the
DC-removed ones: the fp32 mean subtraction errs relative to the offset, so a frame on a large DC offset legitimately
has a larger error relative to its own spectrum).  DC removal, pre-emphasis (|1 - a z^-1| <= 2) and the window (<= 1)
keep the frame's 2-norm below 2 R_f, the 512-point FFT (9 radix-2 levels' worth of rounding) then errs per bin by at
most

    |dX_k| <= E_f = K u (log2(512) + c) sqrt(512) R_f,        c = 4 (DC, pre-emphasis, window, real-FFT unpack)

so |dP_k| <= 2 |X_k| E_f + E_f^2, and the fp32 mel product over count_m bins adds (count_m + 1) u mel_m:

    |dmel_m| <= sum_k w_mk |dP_k| + K (count_m + 1) u mel_m.

Log domain: |log max(a, phi) - log max(b, phi)| <= |a - b| / max(min(a, b), phi), and min(a, b) >= b - |a - b|, so
the log-mel bound is dmel / max(mel - dmel, phi) plus K u |log mel| for logf and the fp32 result.  It stays finite at
the floor phi = FLT_EPS.

delta + CMVN, per (utterance, column), on the kernel's own fbank rows x (so the fbank error is not counted twice):
the fp32 tap chain (fp32-rounded filter taps, one fmaf per tap) errs per value by at most
e_t = (taps + 1) u sum_j |w_j| |x_{t+j}|.  The statistics are fp64 sums of those values, so they add only the
propagated tap error (mean: mean(e); std: ||e||_2 / sqrt(m - 1), plus the fp64 one-pass cancellation) and the two
fp32 roundings of mean and denominator (u |mu|, 2 u (sigma + eps)).  The output (y - mu) / (sigma + eps) is then
bounded with the denominator's lower end den_lo = max(sigma + eps - dden, eps):

    |dz_t| <= K [ (e_t + dmu + u |y_t - mu|) / den_lo + |y_t - mu| dden / ((sigma + eps) den_lo) + u |z_t| ].

tests/test_host_frontend_bounds.py emulates the pipeline in fp32 on the CPU with the same inputs and shows the bound
holds there and that eight plausible defects exceed it by at least 10x.

The contract pinned here: an utterance is its first min(frames(clamp(wave_len, 0, n_max)), t_max) frames; the CMVN
statistics cover exactly those frames, the deltas see zeros beyond them, and nothing outside them is read.
"""
import math

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from oracle.make_golden import AUDIO_CFG

pytestmark = pytest.mark.gpu
DEV = "cuda"
K = 8.0
U = 2.0 ** -24
C_FFT = 4.0
FLOOR = float(onp.FLT_EPS)
TILE_BYTES = 40 * 1024          # delta kernels' shared-memory tile limit
DC_COLS, DC_TCHUNK = 128, 64

# (name, option overrides of the shipped cfg, 16-bit PCM input, the edges the case exists for)
CASES = [
    ("shipped", {}, False, {"shipped cfg"}),
    ("80mel-hamming-pcm16", dict(feat_dim=80, window_type="hamming"), True, {"col passes=2", "hamming", "pcm16"}),
    ("128mel-rect-w4", dict(feat_dim=128, window_type="rectangular", delta_window_size=4), False,
     {"col passes=3", "empty mel filter", "tile=40KiB", "rectangular"}),
    ("4mel-order0", dict(feat_dim=4, delta_order=0, apply_cmvn=False), False, {"feat=fb"}),
    ("40mel-w8", dict(delta_window_size=8), False, {"taps=33"}),
    ("blackman-512-1ms", dict(window_type="blackman", frame_length=32, frame_shift=1), False,
     {"blackman", "win=512"}),
    ("8k-50ms", dict(sample_frequency=8000, frame_length=50, frame_shift=12.5, low_freq=0, high_freq=-200,
                     delta_order=1, delta_window_size=3), False, {"8000 Hz", "low_freq=0", "high_freq<0", "order 1"}),
    ("22k-hanning", dict(sample_frequency=22050, frame_length=20, window_type="hanning"), False,
     {"22050 Hz", "hanning"}),
    ("raw-linear-257", dict(remove_dc_offset=False, preemphasis_coefficient=0.0, use_log_fbank=False,
                            frame_length=16.0625), False,
     {"no dc removal", "no pre-emphasis", "linear mel", "win=257"}),
    ("shift40-win25", dict(frame_shift=40), False, {"shift>win"}),
]
CASE = {c[0]: c[1:] for c in CASES}

SIGNALS = ["noise 1", "tone", "silence", "dc 0.5", "noise 0.1", "tiny 1e-6", "noise 1e-3", "near floor"]


def case_seed(name, flip=False):
    return len(name) + 7 * int(flip)


def case_cfg(over):
    cfg = dict(AUDIO_CFG)
    cfg.update(over)
    return cfg


def taps_of(fe):
    return 2 * fe.delta_order * fe.delta_window + 1


def case_edges(fe, over, pcm16):
    """The code paths and options a configured front end reaches (host-side facts only)."""
    e = set()
    if not over:
        e.add("shipped cfg")
    if pcm16:
        e.add("pcm16")
    taps = taps_of(fe)
    if fe.delta_order == 0 and not fe.apply_cmvn:
        e.add("feat=fb")
    else:
        passes = -(-fe.feat_dim // DC_COLS)
        if passes > 1:
            e.add("col passes=%d" % passes)
        if taps == 33:
            e.add("taps=33")
        if (DC_TCHUNK + taps - 1) * fe.num_mel * 4 == TILE_BYTES:
            e.add("tile=40KiB")
    if fe.delta_order == 1:
        e.add("order 1")
    if int((fe.mel_count == 0).sum()):
        e.add("empty mel filter")
    wt = over.get("window_type", "povey")
    if wt != "povey":
        e.add(wt)
    if fe.sample_frequency != 16000.0:
        e.add("%d Hz" % fe.sample_frequency)
    if over.get("low_freq", 20.0) == 0:
        e.add("low_freq=0")
    if over.get("high_freq", 0.0) < 0:
        e.add("high_freq<0")
    if not fe.remove_dc:
        e.add("no dc removal")
    if fe.preemph == 0.0:
        e.add("no pre-emphasis")
    if not fe.use_log:
        e.add("linear mel")
    if fe.win_size in (257, 512):
        e.add("win=%d" % fe.win_size)
    if fe.win_shift > fe.win_size:
        e.add("shift>win")
    return e


# ------------------------------------------------------------------------------------------- inputs
def signal(kind, n, sr, rng):
    t = np.arange(n) / sr
    if kind == "silence":
        return np.zeros(n)
    if kind == "tone":                                  # on the centre of FFT bin 149: wide dynamic range
        return 0.5 * np.sin(2 * np.pi * (149 / 512) * sr * t + 0.3)
    if kind == "dc 0.5":
        return 0.5 + 1e-4 * rng.standard_normal(n)
    if kind == "tiny 1e-6":                             # every mel energy below the log floor
        return 1e-6 * rng.standard_normal(n)
    if kind == "near floor":                            # mel energies on both sides of the log floor
        return 2e-5 * rng.standard_normal(n)
    gain = float(kind.split()[1])
    return gain * rng.standard_normal(n)


def frame_counts(fe):
    """0, 1 (NaN under CMVN), 2, the tap halo, taps - 1, both sides of each 64-frame chunk edge, ~3000; unsorted."""
    taps = taps_of(fe)
    m = [0, 1, 2, (taps - 1) // 2, taps - 1, 63, 64, 65, 128, 129, 2999]
    return [m[i] for i in (6, 0, 10, 3, 1, 8, 5, 2, 9, 4, 7)]


def samples_for(fe, m, rng):
    if m == 0:
        return fe.win_size - 1
    return fe.win_size + (m - 1) * fe.win_shift + int(rng.integers(0, fe.win_shift))


def make_batch(fe, pcm16, seed):
    """Zero-padded batch (CPU): (wave fp32 or int16 [B, N], lens, frames, wave as float64 [B, N])."""
    rng = np.random.default_rng(seed)
    frames = frame_counts(fe)
    lens = [samples_for(fe, m, rng) for m in frames]
    N = max(lens)
    x = np.zeros((len(lens), N))
    for b, n in enumerate(lens):
        x[b, :n] = signal(SIGNALS[b % len(SIGNALS)], n, fe.sample_frequency, rng)
    if pcm16:
        pcm = np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.int16)
        return torch.from_numpy(pcm), lens, frames, pcm.astype(np.float64) / 32768.0
    x32 = x.astype(np.float32)
    return torch.from_numpy(x32), lens, frames, x32.astype(np.float64)


# ------------------------------------------------------------------------------------------- references and bounds
def oracle_fbank(fe, x, use_log=None):
    use_log = fe.use_log if use_log is None else use_log
    return onp.fbank_tables(x, fe.window.cpu().numpy(), fe.mel_dense.cpu().numpy(), fe.win_size, fe.win_shift,
                            fe.remove_dc, float(np.float32(fe.preemph)), use_log, FLOOR)


def fbank_bound(fe, x, use_log=None):
    """Per (frame, mel) bound on |fbank_fp32 - fbank_fp64| (module docstring)."""
    use_log = fe.use_log if use_log is None else use_log
    win, shift = fe.win_size, fe.win_shift
    if x.shape[0] < win:
        return np.zeros((0, fe.num_mel))
    m = 1 + (x.shape[0] - win) // shift
    raw = x[np.arange(win)[None, :] + shift * np.arange(m)[:, None]]
    R = np.sqrt((raw * raw).sum(1))
    fr = raw - raw.mean(1, keepdims=True) if fe.remove_dc else raw
    a = float(np.float32(fe.preemph))
    if a != 0.0:
        fr = fr - a * np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)
    fr = fr * fe.window.cpu().numpy().astype(np.float64)[None, :]
    X = np.abs(np.fft.rfft(fr, n=512, axis=1))
    mel = fe.mel_dense.cpu().numpy().astype(np.float64)
    E = (K * U * (math.log2(512) + C_FFT) * math.sqrt(512) * R)[:, None]
    lin = (X * X) @ mel.T
    cnt = fe.mel_count.cpu().numpy().astype(np.float64)[None, :]
    d = (2 * X * E + E * E) @ mel.T + K * (cnt + 1) * U * lin
    if not use_log:
        return d
    return d / np.maximum(lin - d, FLOOR) + K * U * np.abs(np.log(np.maximum(lin, FLOOR)))


def delta_cmvn_bound(fb, order, window, apply_cmvn, eps=1e-10):
    """fb [m, F] float64 (the kernel's own fbank rows) -> (float64 reference [m, D], bound [m, D])."""
    m, F = fb.shape
    ref = onp.delta_cmvn(fb, order, window, apply_cmvn, eps)
    filt = onp.delta_filters(order, window)
    taps = filt.shape[1]
    pad = (taps - 1) // 2
    xp = np.abs(np.pad(fb, ((pad, pad), (0, 0))))
    ab = np.stack([sum(abs(filt[o, j]) * xp[j:j + m] for j in range(taps)) for o in range(order + 1)], 0)
    e = np.transpose((taps + 1) * U * ab, (1, 0, 2)).reshape(m, F * (order + 1))
    if not apply_cmvn:
        return ref, K * e
    if m < 2:
        return ref, np.full_like(ref, np.nan)           # NaN like torch.std of one sample
    y = onp.delta_cmvn(fb, order, window, False)
    mu = y.mean(0)
    sd = y.std(0, ddof=1)
    s = sd + eps
    dmu = e.mean(0) + U * np.abs(mu)
    dv = 4 * (m + 2) * 2.0 ** -53 * (y * y).sum(0) / (m - 1)
    dsd = np.sqrt((e * e).sum(0) / (m - 1)) + np.minimum(np.sqrt(dv), dv / np.maximum(sd, 1e-300))
    dden = dsd + 2 * U * s
    num = np.abs(y - mu)
    den_lo = np.maximum(s - dden, eps)
    b = K * ((e + dmu + U * num) / den_lo + num * dden / (s * den_lo) + U * np.abs(ref))
    return ref, b


def worst_ratio(got, ref, bound):
    """max err / bound; NaN must sit exactly where the reference has NaN (and the bound there is NaN)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    nan = np.isnan(ref)
    if not np.array_equal(np.isnan(got), nan):
        return math.inf
    if nan.all():
        return 0.0
    err = np.abs(got - ref)[~nan]
    bnd = np.asarray(bound)[~nan]
    r = np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


# ------------------------------------------------------------------------------------------- option cases
WORST = {}


def _run_and_check(pkg, over, pcm16, seed):
    cfg = case_cfg(over)
    tr, dim = pkg.create_transform(cfg, device=DEV)
    fe = tr.frontend
    wave, lens, frames, x = make_batch(fe, pcm16, seed)
    if pcm16:
        assert int(wave.min()) == -32768 and int(wave.max()) == 32767
    t_max = max(frames) + 5
    feat, n, fb = tr.batch(wave.to(DEV), lens, t_max=t_max, return_fbank=True)
    feat2, n2, fb2 = tr.batch(wave.to(DEV), lens, t_max=t_max, return_fbank=True)
    torch.cuda.synchronize()
    assert torch.equal(bits(feat), bits(feat2)) and torch.equal(bits(fb), bits(fb2)) and torch.equal(n, n2)
    assert n.tolist() == frames and feat.shape == (len(lens), t_max, dim) == (len(lens), t_max, fe.feat_dim)
    delta_runs = fe.delta_order > 0 or fe.apply_cmvn
    if not delta_runs:
        assert feat.data_ptr() == fb.data_ptr()        # the feat = fb path: no delta / CMVN launch
    fbn, featn = fb.cpu().double().numpy(), feat.cpu().double().numpy()
    r_fb = r_ft = 0.0
    for b, m in enumerate(frames):
        xb = x[b, :lens[b]]
        r_fb = max(r_fb, worst_ratio(fbn[b, :m], oracle_fbank(fe, xb), fbank_bound(fe, xb)))
        assert not fbn[b, m:].any() and not featn[b, m:].any()        # padded rows exactly 0
        if delta_runs:
            ref, bnd = delta_cmvn_bound(fbn[b, :m], fe.delta_order, fe.delta_window, fe.apply_cmvn)
            r_ft = max(r_ft, worst_ratio(featn[b, :m], ref, bnd))
            if fe.apply_cmvn and m >= 2 and SIGNALS[b % len(SIGNALS)] in ("silence", "tiny 1e-6") and fe.use_log:
                assert not featn[b, :m, :fe.num_mel].any()   # every bin at the floor: constant static channel -> 0
    return fe, r_fb, r_ft


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_option_case_within_fp64_bound(pkg, name):
    over, pcm16, edges = CASE[name]
    fe = pkg.create_transform(case_cfg(over), device="cpu")[0].frontend
    assert edges <= case_edges(fe, over, pcm16), (edges, case_edges(fe, over, pcm16))
    ratios = {}
    for flip in (False, True):
        o = dict(over)
        if flip:
            o["use_log_fbank"] = not over.get("use_log_fbank", True)
        fe, r_fb, r_ft = _run_and_check(pkg, o, pcm16, case_seed(name, flip))
        ratios["log" if fe.use_log else "linear"] = (r_fb, r_ft)
    WORST[name] = ratios
    print("front end %s: worst err/bound (fbank, feat) %s" % (name, ratios))
    for r_fb, r_ft in ratios.values():
        assert r_fb <= 1.0 and r_ft <= 1.0, ratios


# ------------------------------------------------------------------------------------------- delta / CMVN via the C ABI
def delta_direct(pkg, fb, nfr, order, window, cmvn):
    L = pkg.lib
    lib = L.load()
    B, T, F = fb.shape
    out = torch.full((B, T, F * (order + 1)), 7.0, device=DEV)
    ws_bytes = lib.b200asr_delta_cmvn_workspace_bytes(B, T, F, order)
    ws = torch.full((max(ws_bytes, 8),), 0xFF, dtype=torch.uint8, device=DEV)      # NaN partial sums
    nf = torch.tensor(nfr, dtype=torch.int32, device=DEV)
    before = L.launch_count()
    L.check(lib.b200asr_delta_cmvn_fwd(L.ptr(fb), L.ptr(nf), B, T, F, order, window, int(cmvn), 1e-10, L.ptr(out),
                                       L.ptr(ws), ws_bytes, L.stream()), "delta_cmvn_fwd")
    torch.cuda.synchronize()
    return out, L.launch_count() - before


def crafted_fbank(nfr, T, F, seed, pad_fill=None):
    """[B, T, F]: columns 0-3 constant, 4-7 a large mean with a small spread, the rest log-mel-like noise; rows at or
    beyond the valid length zero, or NaN / 1e30 alternating (pad_fill='garbage')."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((len(nfr), T, F)) - 6.0).astype(np.float32)
    x[:, :, 0:4] = np.array([3.25, -1e3, 0.0, 1e-20], np.float32)
    x[:, :, 4:8] = (1e3 + 1e-2 * rng.standard_normal((len(nfr), T, 4))).astype(np.float32)
    for b, m in enumerate(nfr):
        m = min(max(m, 0), T)
        x[b, m:] = 0.0
        if pad_fill == "garbage":
            x[b, m::2] = np.nan
            x[b, m + 1::2] = 1e30
    return x


@pytest.mark.parametrize("order,window", [(2, 2), (1, 4), (0, 2), (2, 8)])
def test_delta_cmvn_c_abi_blind_to_padded_rows(pkg, order, window):
    T, F = 200, 40
    nfr = [150, 0, 200, 1, 2, 77]
    clean = torch.from_numpy(crafted_fbank(nfr, T, F, 3)).to(DEV)
    dirty = torch.from_numpy(crafted_fbank(nfr, T, F, 3, "garbage")).to(DEV)
    for cmvn in (1, 0):
        a, na = delta_direct(pkg, clean, nfr, order, window, cmvn)
        b, nb = delta_direct(pkg, dirty, nfr, order, window, cmvn)
        assert na == nb == (2 if cmvn else 1)          # no statistics pass without CMVN
        assert torch.equal(bits(a), bits(b))
        an = a.cpu().double().numpy()
        fb = clean.cpu().double().numpy()
        worst = 0.0
        for r, m in enumerate(nfr):
            assert not an[r, m:].any()                  # padded rows written as exact zeros
            ref, bnd = delta_cmvn_bound(fb[r, :m], order, window, bool(cmvn))
            worst = max(worst, worst_ratio(an[r, :m], ref, bnd))
            if cmvn and m >= 2:
                assert not an[r, :m, 0:4].any()          # constant static channels are exactly 0
        print("delta/CMVN C ABI order %d window %d cmvn %d: worst err/bound %.3g" % (order, window, cmvn, worst))
        assert worst <= 1.0


def test_delta_cmvn_c_abi_clamps_n_frames(pkg):
    """n_frames beyond t_max means t_max, negative means 0 (non-last rows, over-read bounded by one chunk)."""
    T, F = 192, 40
    real = [T, 0, 100, 57]
    fb = torch.from_numpy(crafted_fbank(real, T, F, 5)).to(DEV)
    for cmvn in (1, 0):
        a, _ = delta_direct(pkg, fb, real, 2, 2, cmvn)
        b, _ = delta_direct(pkg, fb, [T + 40, -7, 100, 57], 2, 2, cmvn)
        assert torch.equal(bits(a), bits(b))


def test_delta_cmvn_refuses_what_it_cannot_stage(pkg):
    L = pkg.lib
    fb = torch.zeros(2, 70, 128, device=DEV)
    for order, window in ((2, 5), (1, 9)):             # first windows whose tile exceeds 40 KB at 128 bins
        assert (DC_TCHUNK + 2 * order * window) * 128 * 4 > TILE_BYTES
        assert (DC_TCHUNK + 2 * order * (window - 1)) * 128 * 4 <= TILE_BYTES
        before = L.launch_count()
        with pytest.raises(pkg.B200AsrError):
            delta_direct(pkg, fb, [70, 3], order, window, 1)
        assert L.launch_count() == before
        delta_direct(pkg, fb, [70, 3], order, window - 1, 1)    # the largest window that fits still runs
    tr, _ = pkg.create_transform(case_cfg(dict(feat_dim=129)), device=DEV)
    before = L.launch_count()
    with pytest.raises(pkg.B200AsrError):
        tr.batch(torch.zeros(2, 4000, device=DEV), [4000, 3000])
    assert L.launch_count() == before


# ------------------------------------------------------------------------------------------- t_max / n_max contract
def test_t_max_below_longest_truncates_utterances(pkg):
    """Rows longer than t_max are their first t_max frames: n_frames == t_max, features == the fp64 oracle on the
    waveform cut to (t_max - 1) * shift + win samples, CMVN over exactly those frames."""
    tr, _ = pkg.create_transform(dict(AUDIO_CFG), device=DEV)
    fe = tr.frontend
    rng = np.random.default_rng(11)
    t_max = 200
    frames = [300, 250, 120, 180]                       # only non-last rows exceed t_max, by < 2x
    lens = [fe.win_size + (m - 1) * fe.win_shift for m in frames]
    x = np.zeros((len(lens), max(lens)), np.float32)
    for b, n in enumerate(lens):
        x[b, :n] = 0.1 * rng.standard_normal(n)
    feat, n, fb = tr.batch(torch.from_numpy(x).to(DEV), lens, t_max=t_max, return_fbank=True)
    assert n.tolist() == [min(m, t_max) for m in frames]
    fbn, featn = fb.cpu().double().numpy(), feat.cpu().double().numpy()
    for b, m in enumerate(n.tolist()):
        xb = x[b, :(m - 1) * fe.win_shift + fe.win_size].astype(np.float64)
        assert worst_ratio(fbn[b, :m], oracle_fbank(fe, xb), fbank_bound(fe, xb)) <= 1.0
        ref, bnd = delta_cmvn_bound(fbn[b, :m], 2, 2, True)
        assert worst_ratio(featn[b, :m], ref, bnd) <= 1.0
        assert not featn[b, m:].any()
    # the truncated rows equal the same utterances given exactly t_max frames of samples
    cut = [min(n_, (t_max - 1) * fe.win_shift + fe.win_size) for n_ in lens]
    feat2, n2 = tr.batch(torch.from_numpy(x).to(DEV), cut, t_max=t_max)
    assert torch.equal(n, n2) and torch.equal(bits(feat), bits(feat2))


def test_wave_len_beyond_n_max_is_clamped_on_device(pkg):
    tr, _ = pkg.create_transform(dict(AUDIO_CFG), device=DEV)
    rng = np.random.default_rng(12)
    N = 16000
    x = torch.from_numpy((0.1 * rng.standard_normal((3, N))).astype(np.float32)).to(DEV)
    over = torch.tensor([2 * N, N, 9000], dtype=torch.int32, device=DEV)   # only a non-last row, <= 2 N
    exact = torch.tensor([N, N, 9000], dtype=torch.int32, device=DEV)
    f1, n1 = tr.batch(x, over)
    f2, n2 = tr.batch(x, exact)
    assert torch.equal(n1, n2) and torch.equal(bits(f1), bits(f2))
    # with t_max above the frames of N samples, only the n_max clamp keeps row 0 from framing row 1's samples
    # (frames 98 .. 149 would end at sample 149 * 160 + 400 < 2 N, inside the buffer since row 0 is not the last)
    t_max = 150
    assert tr.frontend.num_frames(N) == 98 < t_max < tr.frontend.num_frames(2 * N)
    f1, n1, fb1 = tr.batch(x, over, t_max=t_max, return_fbank=True)
    f2, n2, fb2 = tr.batch(x, exact, t_max=t_max, return_fbank=True)
    assert n1.tolist() == n2.tolist() == [98, 98, 54]
    assert torch.equal(bits(fb1), bits(fb2)) and torch.equal(bits(f1), bits(f2))
    assert not fb1[0, 98:].any() and not f1[0, 98:].any()
    for bad in ([N + 1, N, 9000], [-1, N, 9000]):     # host-known lengths are checked before any launch
        with pytest.raises(ValueError):
            tr.batch(x, bad)
        with pytest.raises(ValueError):
            tr.batch(x, torch.tensor(bad))


def test_batch_without_a_complete_frame_is_empty_and_launches_nothing(pkg):
    """Every utterance shorter than one window (or t_max = 0): empty features, zero lengths, no kernel launched."""
    L = pkg.lib
    x = torch.ones(2, 399, device=DEV)
    for over in ({}, dict(delta_order=0, apply_cmvn=False)):
        tr, dim = pkg.create_transform(case_cfg(over), device=DEV)
        for t_max, wave in ((None, x), (0, torch.ones(2, 4000, device=DEV))):
            before = L.launch_count()
            feat, n, fb = tr.batch(wave, [wave.shape[1], 10], t_max=t_max, return_fbank=True)
            assert L.launch_count() == before
            assert feat.shape == (2, 0, dim) and fb.shape == (2, 0, tr.frontend.num_mel)
            assert n.tolist() == [0, 0] and n.dtype == torch.int64 and n.device.type == "cuda"


# ------------------------------------------------------------------------------------------- batch invariance
@pytest.mark.parametrize("name", ["shipped", "128mel-rect-w4"])
def test_utterance_bits_do_not_depend_on_the_batch(pkg, name):
    over, pcm16, _ = CASE[name]
    tr, _ = pkg.create_transform(case_cfg(over), device=DEV)
    wave, lens, frames, _ = make_batch(tr.frontend, pcm16, seed=3)
    w = wave.to(DEV)
    base, _ = tr.batch(w, lens)
    rev = list(range(len(lens)))[::-1]
    flipped, _ = tr.batch(w[rev].contiguous(), [lens[i] for i in rev], t_max=max(frames) + 200)
    for b, m in enumerate(frames):
        alone, n1 = tr.batch(w[b:b + 1, :max(lens[b], 1)].contiguous(), [lens[b]])
        assert int(n1[0]) == m
        want = bits(base[b, :m])
        assert torch.equal(bits(alone[0, :m]), want)
        assert torch.equal(bits(flipped[rev.index(b), :m]), want)
    # next to a longer and a shorter neighbour only
    for b in (frames.index(65), frames.index(2999)):
        j = frames.index(129)
        pair, _ = tr.batch(w[[j, b]].contiguous(), [lens[j], lens[b]], t_max=max(frames) + 64)
        assert torch.equal(bits(pair[1, :frames[b]]), bits(base[b, :frames[b]]))
