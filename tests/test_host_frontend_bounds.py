"""CPU checks for tests/test_gpu_frontend_variants.py: every option case reaches the edge it was written for, and the
fp32-rounding bounds used there have teeth.

The front end is emulated in float32 with numpy / scipy (fp32 framing, DC removal, pre-emphasis and window,
scipy.fft.rfft on fp32 input, the fp32 mel product and log; the delta taps as a fmaf chain on fp32-rounded taps, CMVN
statistics in fp64 rounded to fp32 mean and denominator) on the GPU cases' own inputs.  The correct emulation must
sit inside the bounds; each of eight defects a kernel could plausibly have must exceed them by at least 10x.
"""
import numpy as np
import pytest
import scipy.fft

import test_gpu_frontend_variants as V
from oracle import oracle_np as onp

F32 = np.float32
REQUIRED_EDGES = {
    "shipped cfg", "pcm16", "col passes=2", "col passes=3", "empty mel filter", "tile=40KiB", "taps=33", "feat=fb",
    "order 1", "hamming", "rectangular", "blackman", "hanning", "8000 Hz", "22050 Hz", "low_freq=0", "high_freq<0",
    "no dc removal", "no pre-emphasis", "linear mel", "win=257", "win=512", "shift>win",
}


def _fe(pkg, name):
    over, pcm16, _ = V.CASE[name]
    return pkg.create_transform(V.case_cfg(over), device="cpu")[0].frontend


# ------------------------------------------------------------------------------------------- coverage
def test_gpu_cases_cover_every_edge_once(pkg):
    """Each case reaches the edges it names; together they reach every listed edge; and each case reaches an edge
    no other case reaches, so deleting any case fails here."""
    reached = {}
    for name, (over, pcm16, edges) in V.CASE.items():
        reached[name] = V.case_edges(_fe(pkg, name), over, pcm16)
        assert edges <= reached[name], (name, edges - reached[name])
    assert set().union(*(e for _, _, _, e in V.CASES)) == REQUIRED_EDGES
    for name in V.CASE:
        others = set().union(*(r for n, r in reached.items() if n != name))
        assert V.CASE[name][2] - others, name


def test_128_bins_have_an_empty_filter(pkg):
    fe = _fe(pkg, "128mel-rect-w4")
    assert int((fe.mel_count == 0).sum()) >= 1 and fe.feat_dim == 384
    assert (V.DC_TCHUNK + V.taps_of(fe) - 1) * 128 * 4 == V.TILE_BYTES


# ------------------------------------------------------------------------------------------- fp32 emulation
def _round_bits(x, bits):
    m, e = np.frexp(x)
    return np.ldexp(np.round(m * 2.0 ** bits) / 2.0 ** bits, e).astype(F32)


def emulate_fbank(fe, x, defect=None):
    """fp32 fbank of one utterance x (float64 values that are exact in fp32)."""
    x = np.asarray(x, F32)
    win, shift = fe.win_size, fe.win_shift
    if x.shape[0] < win:
        return np.zeros((0, fe.num_mel), F32)
    m = 1 + (x.shape[0] - win) // shift
    fr = x[np.arange(win)[None, :] + shift * np.arange(m)[:, None]]
    if fe.remove_dc:
        n = 512 if defect == "DC mean over 512 samples" else win
        fr = fr - (fr.sum(1, dtype=F32) / F32(n))[:, None]
    a = F32(fe.preemph)
    if a != 0:
        first = np.zeros_like(fr[:, :1]) if defect == "zero left neighbour" else fr[:, :1]
        fr = fr - a * np.concatenate([first, fr[:, :-1]], axis=1)
    fr = fr * fe.window.numpy()[None, :]
    X = scipy.fft.rfft(fr, n=512, axis=1)
    assert X.dtype == np.complex64
    P = X.real * X.real + X.imag * X.imag
    if defect == "power in 11 bits":
        P = _round_bits(P, 11)
    mel = fe.mel_dense.numpy()
    if defect == "mel shifted one bin":
        mel = np.roll(mel, 1, axis=1)
    e = P @ mel.T
    return np.log(np.maximum(e, F32(V.FLOOR))) if fe.use_log else e


def _fmaf(w, x, acc):
    return (np.float64(w) * x.astype(np.float64) + acc.astype(np.float64)).astype(F32)


def emulate_delta_cmvn(fb, order, window, cmvn, defect=None, eps=1e-10):
    fb = np.asarray(fb, F32)
    m = fb.shape[0]
    if defect == "CMVN over one padded frame":
        fb = np.concatenate([fb, np.zeros_like(fb[:1])])
    mm = fb.shape[0]
    if mm == 0:
        return np.zeros((0, fb.shape[1] * (order + 1)), F32)
    filt = onp.delta_filters(order, window).astype(F32)
    taps = filt.shape[1]
    pad = (taps - 1) // 2
    xp = np.pad(fb, ((pad, pad), (0, 0)), mode="edge" if defect == "replicate-padded delta edges" else "constant")
    chans = []
    for o in range(order + 1):
        acc = np.zeros_like(fb)
        for j in range(taps):
            acc = _fmaf(filt[o, j], xp[j:j + mm], acc)
        chans.append(acc)
    y = np.transpose(np.stack(chans, 0), (1, 0, 2)).reshape(mm, fb.shape[1] * (order + 1))
    if not cmvn:
        return y[:m]
    if defect == "one-pass fp32 variance":
        s = np.add.accumulate(y, axis=0, dtype=F32)[-1]
        ss = np.add.accumulate(y * y, axis=0, dtype=F32)[-1]
        mean = s / F32(mm)
        var = np.maximum((ss - F32(mm) * mean * mean) / F32(mm - 1), F32(0))
        den = F32(eps) + np.sqrt(var)
    else:
        yd = y.astype(np.float64)
        ts, tss = yd.sum(0), (yd * yd).sum(0)
        mu = ts / mm
        var = (tss - ts * mu) / (mm if defect == "biased std" else mm - 1)
        mean = mu.astype(F32)
        den = F32(eps) + np.sqrt(np.maximum(var, 0.0)).astype(F32)
    return ((y - mean) / den).astype(F32)[:m]


def _fbank_ratio(fe, x, lens, frames, defect=None):
    worst = 0.0
    for b, m in enumerate(frames):
        xb = x[b, :lens[b]]
        got = emulate_fbank(fe, xb, defect)
        assert got.shape[0] == m
        worst = max(worst, V.worst_ratio(got, V.oracle_fbank(fe, xb), V.fbank_bound(fe, xb)))
    return worst


def _feat_ratio(fe, fbs, frames, defect=None, min_frames=0):
    worst = 0.0
    for fb, m in zip(fbs, frames):
        if m < min_frames:
            continue
        ref, bnd = V.delta_cmvn_bound(fb.astype(np.float64), fe.delta_order, fe.delta_window, fe.apply_cmvn)
        got = emulate_delta_cmvn(fb, fe.delta_order, fe.delta_window, fe.apply_cmvn, defect)
        worst = max(worst, V.worst_ratio(got, ref, bnd))
    return worst


def _case_inputs(pkg, name):
    fe = _fe(pkg, name)
    _, lens, frames, x = V.make_batch(fe, V.CASE[name][1], V.case_seed(name))
    return fe, lens, frames, x


@pytest.mark.parametrize("name", [c[0] for c in V.CASES])
def test_fp32_emulation_sits_inside_the_bounds(pkg, name):
    fe, lens, frames, x = _case_inputs(pkg, name)
    r_fb = _fbank_ratio(fe, x, lens, frames)
    r_ft = 0.0
    if fe.delta_order > 0 or fe.apply_cmvn:
        fbs = [emulate_fbank(fe, x[b, :lens[b]]) for b in range(len(lens))]
        r_ft = _feat_ratio(fe, fbs, frames)
    print("%s: emulation err/bound fbank %.3g feat %.3g" % (name, r_fb, r_ft))
    assert r_fb <= 0.5 and r_ft <= 0.5


@pytest.mark.parametrize("name,defect", [
    ("80mel-hamming-pcm16", "zero left neighbour"),
    ("128mel-rect-w4", "zero left neighbour"),
    ("shipped", "DC mean over 512 samples"),
    ("shipped", "mel shifted one bin"),
    ("128mel-rect-w4", "power in 11 bits"),
])
def test_fbank_bound_rejects_defects(pkg, name, defect):
    """An 11-bit power spectrum is checked where the spectrum is sharpest (rectangular window, the on-bin tone): E_f
    is a worst-case per-bin FFT bound proportional to the frame's 2-norm, so under a tapered window the tone's peak bin
    is only ~4.5x above it (povey, measured) while the fp32 pipeline itself stays below 0.06 of it."""
    fe, lens, frames, x = _case_inputs(pkg, name)
    r = _fbank_ratio(fe, x, lens, frames, defect)
    print("%s / %s: err/bound %.3g" % (name, defect, r))
    assert r >= 10.0


def test_zero_left_neighbour_is_invisible_under_the_povey_window(pkg):
    """The povey window is exactly 0 at sample 0, so the pre-emphasis edge never reaches the output: only the
    hamming / rectangular cases can catch a wrong left neighbour."""
    fe, lens, frames, x = _case_inputs(pkg, "shipped")
    assert float(fe.window[0]) == 0.0
    for b in range(len(lens)):
        xb = x[b, :lens[b]]
        assert np.array_equal(emulate_fbank(fe, xb, "zero left neighbour"), emulate_fbank(fe, xb))


@pytest.mark.parametrize("defect", ["replicate-padded delta edges", "biased std", "CMVN over one padded frame",
                                    "one-pass fp32 variance"])
def test_delta_cmvn_bound_rejects_defects(pkg, defect):
    fe, lens, frames, x = _case_inputs(pkg, "shipped")
    fbs = [emulate_fbank(fe, x[b, :lens[b]]) for b in range(len(lens))]
    r = _feat_ratio(fe, fbs, frames, defect, min_frames=2)     # rows of >= 2 frames: no NaN statistics
    print("shipped / %s: err/bound %.3g" % (defect, r))
    assert r >= 10.0
