"""Batched GPU front end: Kaldi-style fbank + delta + CMVN on waveforms resident in HBM.

Host-side mirror of the reference's `create_transform` (/root/reference/src/audio.py:115-133): same yaml keys,
same `(transform, feat_dim)` return, but the transform works on a *batch of waveforms on the GPU* (one fused
STFT+mel+log launch + one delta/CMVN launch) instead of one file path at a time inside the DataLoader workers
(src/data.py:22,31).  `transform(filepath)` is kept for drop-in use and returns the same [T, D] CPU tensor.
"""
import math

import numpy as np
import torch

from . import lib as L

_FLT_EPS = 1.1920928955078125e-07  # torch.finfo(torch.float).eps, the kaldi log floor (kaldi.py:633)


def _next_pow2(x):
    return 1 if x == 0 else 2 ** (x - 1).bit_length()


def window_function(window_type, size, blackman_coeff=0.42):
    """fp32 window table; same torch calls as kaldi.py:87-115 so the table is bit-identical."""
    if window_type == "hanning":
        return torch.hann_window(size, periodic=False)
    if window_type == "hamming":
        return torch.hamming_window(size, periodic=False, alpha=0.54, beta=0.46)
    if window_type == "povey":
        return torch.hann_window(size, periodic=False).pow(0.85)
    if window_type == "rectangular":
        return torch.ones(size)
    if window_type == "blackman":
        a = 2 * math.pi / (size - 1)
        n = torch.arange(size, dtype=torch.float32)
        return blackman_coeff - 0.5 * torch.cos(a * n) + (0.5 - blackman_coeff) * torch.cos(2 * a * n)
    raise ValueError("Invalid window type " + window_type)


def mel_filterbank(num_bins, n_fft, sample_freq, low_freq, high_freq):
    """Dense [num_bins, n_fft//2+1] triangular mel weights, fp32, arithmetic order of kaldi.py:436-511
    (no VTLN warp), last column (Nyquist) zero as at kaldi.py:626."""
    assert num_bins > 3, "Must have at least 3 mel bins"
    assert n_fft % 2 == 0
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    assert (0.0 <= low_freq < nyquist) and (0.0 < high_freq <= nyquist) and (low_freq < high_freq), \
        "Bad values in options: low-freq %s and high-freq %s vs. nyquist %s" % (low_freq, high_freq, nyquist)
    bin_width = sample_freq / n_fft
    mel_lo = 1127.0 * math.log(1.0 + low_freq / 700.0)
    mel_hi = 1127.0 * math.log(1.0 + high_freq / 700.0)
    delta = (mel_hi - mel_lo) / (num_bins + 1)
    b = torch.arange(num_bins).unsqueeze(1)
    left = mel_lo + b * delta
    center = mel_lo + (b + 1.0) * delta
    right = mel_lo + (b + 2.0) * delta
    mel = (1127.0 * (1.0 + (bin_width * torch.arange(n_fft / 2)) / 700.0).log()).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    bins = torch.max(torch.zeros(1), torch.min(up, down))
    return torch.nn.functional.pad(bins, (0, 1), mode="constant", value=0).to(torch.float32)


def sparsify_mel(dense):
    """[n_mel, n_bins] -> (start, count, offset, packed weights): each triangle as one contiguous run."""
    d = dense.numpy()
    start, count, off, w = [], [], [], []
    for row in d:
        nz = np.nonzero(row)[0]
        if len(nz) == 0:
            s, c = 0, 0
        else:
            s, c = int(nz[0]), int(nz[-1] - nz[0] + 1)
        start.append(s)
        count.append(c)
        off.append(len(w))
        w.extend(row[s:s + c].tolist())
    if not w:
        w = [0.0]
    return (np.asarray(start, np.int32), np.asarray(count, np.int32), np.asarray(off, np.int32),
            np.asarray(w, np.float32))


class FbankFrontEnd(torch.nn.Module):
    """fbank (+delta, +CMVN, channel-major interleave) for a zero-padded batch of waveforms on the GPU."""

    def __init__(self, feat_type="fbank", feat_dim=40, delta_order=0, delta_window_size=2, apply_cmvn=False,
                 sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, dither=0.0,
                 preemphasis_coefficient=0.97, remove_dc_offset=True, window_type="povey", blackman_coeff=0.42,
                 low_freq=20.0, high_freq=0.0, round_to_power_of_two=True, snip_edges=True, use_energy=False,
                 use_log_fbank=True, use_power=True, vtln_warp=1.0, energy_floor=1.0, raw_energy=True,
                 htk_compat=False, subtract_mean=False, min_duration=0.0, channel=-1, **unknown):
        super().__init__()
        if feat_type != "fbank":
            raise NotImplementedError("only feat_type 'fbank' is on the accelerated path (mfcc is unused by the "
                                      "reference's configs and skipped by its tests)")
        if unknown:
            raise TypeError("unknown fbank options: %s" % sorted(unknown))
        unsupported = []
        if dither != 0.0: unsupported.append("dither != 0")
        if not snip_edges: unsupported.append("snip_edges=False")
        if use_energy: unsupported.append("use_energy")
        if not use_power: unsupported.append("use_power=False")
        if vtln_warp != 1.0: unsupported.append("vtln_warp != 1")
        if subtract_mean: unsupported.append("subtract_mean")
        if not round_to_power_of_two: unsupported.append("round_to_power_of_two=False")
        if unsupported:
            raise NotImplementedError("fbank options outside the accelerated path: " + ", ".join(unsupported))
        self.sample_frequency = float(sample_frequency)
        self.win_shift = int(sample_frequency * frame_shift * 0.001)
        self.win_size = int(sample_frequency * frame_length * 0.001)
        self.n_fft = _next_pow2(self.win_size)
        if self.n_fft != 512:
            raise NotImplementedError("the fused kernel stages a 512-point FFT (window %d -> %d)" %
                                      (self.win_size, self.n_fft))
        self.num_mel = int(feat_dim)
        self.delta_order = int(delta_order)
        self.delta_window = int(delta_window_size)
        self.apply_cmvn = bool(apply_cmvn)
        self.preemph = float(preemphasis_coefficient)
        self.remove_dc = bool(remove_dc_offset)
        self.use_log = bool(use_log_fbank)
        self.feat_dim = self.num_mel * (self.delta_order + 1)
        win = window_function(window_type, self.win_size, blackman_coeff).to(torch.float32)
        dense = mel_filterbank(self.num_mel, self.n_fft, self.sample_frequency, low_freq, high_freq)
        start, count, off, w = sparsify_mel(dense)
        self.register_buffer("window", win, persistent=False)
        self.register_buffer("mel_dense", dense, persistent=False)
        self.register_buffer("mel_start", torch.from_numpy(start), persistent=False)
        self.register_buffer("mel_count", torch.from_numpy(count), persistent=False)
        self.register_buffer("mel_off", torch.from_numpy(off), persistent=False)
        self.register_buffer("mel_w", torch.from_numpy(w), persistent=False)

    def num_frames(self, n_samples):
        return 0 if n_samples < self.win_size else 1 + (n_samples - self.win_size) // self.win_shift

    @torch.no_grad()
    def forward(self, wave, wave_len, t_max=None, return_fbank=False):
        """wave [B, N_max] fp32 or int16 CUDA (zero padded), wave_len [B] samples (any int tensor / list).
        Returns (feat [B, t_max, D], feat_len [B] int64 on the same device) (+ the log-mel fbank [B, t_max, n_mel]
        with return_fbank).  t_max defaults to the frame count of N_max samples.

        An utterance is its first min(frames(wave_len[b]), t_max) frames: a smaller t_max truncates it (feat_len
        is then t_max, and the CMVN statistics and deltas see only the kept frames).  Lengths known on the host (a
        list or a CPU tensor) must lie in [0, N_max], else ValueError; lengths already on the device are clamped
        to [0, N_max] by the kernel, so no sample outside a row is read."""
        lib = L.load()
        if self.window.device != wave.device:
            self.to(wave.device)
        pcm16 = wave.dtype == torch.int16            # 16-bit PCM: converted on the fly by the kernel (sample / 32768)
        wave = wave.contiguous() if pcm16 else wave.to(torch.float32).contiguous()
        B, N = wave.shape
        if not (torch.is_tensor(wave_len) and wave_len.is_cuda):
            host = torch.as_tensor(wave_len)
            if host.numel() and (int(host.min()) < 0 or int(host.max()) > N):
                raise ValueError("wave_len must lie in [0, %d] (the padded length), got %s" % (N, host.tolist()))
        wl = torch.as_tensor(wave_len).to(device=wave.device, dtype=torch.int32).contiguous()
        if t_max is None:
            t_max = self.num_frames(N)
        if t_max == 0:   # no frame to compute (e.g. one utterance shorter than a window): empty, launch nothing
            fb = torch.zeros((B, 0, self.num_mel), device=wave.device)
            feat = fb if self.delta_order == 0 and not self.apply_cmvn else fb.new_zeros((B, 0, self.feat_dim))
            n = torch.zeros(B, device=wave.device, dtype=torch.int64)
            return (feat, n, fb) if return_fbank else (feat, n)
        fb = torch.empty((B, t_max, self.num_mel), device=wave.device, dtype=torch.float32)
        nfr = torch.empty(B, device=wave.device, dtype=torch.int32)
        # algorithmic bytes (SURVEY.md 8(d)): read the waveform once, write the mel features once
        with L.timed("fbank_fwd", (2 if pcm16 else 4) * int(wave.numel()) + 4 * B * t_max * self.num_mel):
            L.check((lib.b200asr_fbank_fwd_pcm16 if pcm16 else lib.b200asr_fbank_fwd)(
                L.ptr(wave), L.ptr(wl), B, N, self.win_size, self.win_shift, self.n_fft, self.preemph,
                int(self.remove_dc), L.ptr(self.window), self.num_mel, L.ptr(self.mel_start), L.ptr(self.mel_count),
                L.ptr(self.mel_off), L.ptr(self.mel_w), int(self.mel_w.numel()), int(self.use_log), _FLT_EPS,
                L.ptr(fb), t_max, L.ptr(nfr), L.stream()), "fbank_fwd")
        if self.delta_order == 0 and not self.apply_cmvn:
            feat = fb
        else:
            feat = torch.empty((B, t_max, self.feat_dim), device=wave.device, dtype=torch.float32)
            ws_bytes = lib.b200asr_delta_cmvn_workspace_bytes(B, t_max, self.num_mel, self.delta_order)
            ws = torch.empty(max(ws_bytes, 8), device=wave.device, dtype=torch.uint8)
            with L.timed("delta_cmvn_fwd", 4 * B * t_max * (self.num_mel + self.feat_dim)):
                L.check(lib.b200asr_delta_cmvn_fwd(
                    L.ptr(fb), L.ptr(nfr), B, t_max, self.num_mel, self.delta_order, self.delta_window,
                    int(self.apply_cmvn), 1e-10, L.ptr(feat), L.ptr(ws), ws_bytes, L.stream()), "delta_cmvn_fwd")
        if return_fbank:
            return feat, nfr.to(torch.int64), fb
        return feat, nfr.to(torch.int64)

    def extra_repr(self):
        return "fbank num_mel_bins=%d, delta_order=%d, cmvn=%s" % (self.num_mel, self.delta_order, self.apply_cmvn)


def load_wav(filepath):
    """[1, N] fp32 in [-1, 1] (what the historic torchaudio.load default returned, src/audio.py:102)."""
    from scipy.io import wavfile
    sr, data = wavfile.read(filepath)
    if data.dtype == np.int16:
        x = data.astype(np.float32) / 32768.0
    elif data.dtype == np.int32:
        x = data.astype(np.float32) / 2147483648.0
    else:
        x = data.astype(np.float32)
    if x.ndim == 2:
        x = x.T
    else:
        x = x[None, :]
    return torch.from_numpy(np.ascontiguousarray(x)), sr


class FileTransform(torch.nn.Module):
    """`transform(filepath) -> [T, D]` exactly like the reference's nn.Sequential (src/audio.py:115-133), and
    `transform.batch(wave, wave_len)` for the GPU-resident batched path the Solver uses."""

    def __init__(self, frontend, device="cuda"):
        super().__init__()
        self.frontend = frontend
        self.device = device

    def batch(self, wave, wave_len, t_max=None, return_fbank=False):
        return self.frontend(wave, wave_len, t_max, return_fbank)

    def forward(self, filepath):
        wave, sr = load_wav(filepath)
        if float(sr) != self.frontend.sample_frequency:
            raise ValueError("sample rate %s != configured %s" % (sr, self.frontend.sample_frequency))
        w = wave[:1].to(self.device)
        feat, flen = self.frontend(w, [w.shape[1]])
        return feat[0, :int(flen[0])].cpu()


def create_transform(audio_config, device="cuda"):
    """Same contract as /root/reference/src/audio.py:115-133: pops feat_type, feat_dim, delta_order,
    delta_window_size, apply_cmvn; forwards the remaining keys as fbank options; returns (transform, feat_dim)."""
    cfg = dict(audio_config)
    feat_type = cfg.pop("feat_type")
    feat_dim = cfg.pop("feat_dim")
    delta_order = cfg.pop("delta_order", 0)
    delta_window_size = cfg.pop("delta_window_size", 2)
    apply_cmvn = cfg.pop("apply_cmvn")
    fe = FbankFrontEnd(feat_type, feat_dim, delta_order, delta_window_size, apply_cmvn, **cfg)
    return FileTransform(fe, device), feat_dim * (delta_order + 1)
