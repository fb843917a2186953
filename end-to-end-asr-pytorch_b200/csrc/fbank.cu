// K1-K3: fused Kaldi-style filterbank front end.
//
//   fbank_kernel      : framing + DC removal + pre-emphasis + window + 512-pt real FFT (shared
//                       memory Stockham radix-4 on the packed 256-pt complex signal) + power
//                       spectrum + triangular mel filters + log  -> [B, t_max, n_mel]
//   delta_stats_kernel / delta_norm_kernel : delta / delta-delta (zero padded per utterance) + per-utterance
//                       CMVN (unbiased std, fp64 partial sums per 64-frame chunk, reduced in a fixed order) +
//                       channel-major interleave -> [B, t_max, n_mel*(order+1)]; grid (T/64, B)
//
// Reference behaviour restated (not copied):  /root/reference/src/audio.py:25-27,51-77,85-89,101-109
// and torchaudio/compliance/kaldi.py:44-83 (framing), 154-217 (window), 436-511 (mel), 591-646 (fbank).
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {

constexpr int FB_NFFT = 512;
constexpr int FB_WARPS = 4;
constexpr int FB_MAX_MEL = 128;
constexpr int FB_MAX_MELW = 2048;

struct FbankParams {
    const float* wave;
    const short* wave16;  // 16-bit PCM input (sample / 32768, like torchaudio.load's normalisation) when non-null
    const int* wave_len;
    int B, n_max;
    int win, shift;
    float preemph;
    int remove_dc;
    const float* window;
    int n_mel;
    const int* mel_start;
    const int* mel_count;
    const int* mel_off;
    const float* mel_w;
    int mel_w_total;
    float log_floor;
    int use_log;
    float* out;
    int t_max;
    int* n_frames;
};

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// One Stockham radix-4 pass of a 256-point complex FFT executed by one warp.
// x -> y (both 256 float2 in shared memory). Ns = 1, 4, 16, 64.
template <int Ns>
__device__ __forceinline__ void fft256_pass(const float2* __restrict__ x, float2* __restrict__ y,
                                            const float2* __restrict__ w512, int lane) {
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
        const int j = lane + 32 * jj;  // butterfly index 0..63
        const int k = j & (Ns - 1);
        float2 v0 = x[j], v1 = x[j + 64], v2 = x[j + 128], v3 = x[j + 192];
        if (Ns > 1) {
            const int idx = k * (128 / Ns);  // angle -2*pi*k/(4*Ns) in units of 2*pi/512
            v1 = cmul(v1, w512[idx]);
            v2 = cmul(v2, w512[2 * idx]);
            v3 = cmul(v3, w512[3 * idx]);
        }
        const float2 a0 = make_float2(v0.x + v2.x, v0.y + v2.y);
        const float2 a1 = make_float2(v0.x - v2.x, v0.y - v2.y);
        const float2 a2 = make_float2(v1.x + v3.x, v1.y + v3.y);
        const float2 a3 = make_float2(v1.x - v3.x, v1.y - v3.y);
        const int j0 = ((j - k) << 2) + k;
        y[j0] = make_float2(a0.x + a2.x, a0.y + a2.y);
        y[j0 + Ns] = make_float2(a1.x + a3.y, a1.y - a3.x);      // a1 - i*a3
        y[j0 + 2 * Ns] = make_float2(a0.x - a2.x, a0.y - a2.y);
        y[j0 + 3 * Ns] = make_float2(a1.x - a3.y, a1.y + a3.x);  // a1 + i*a3
    }
    __syncwarp();
}

__global__ void __launch_bounds__(FB_WARPS * 32) fbank_kernel(FbankParams p) {
    __shared__ float2 s_w512[FB_NFFT];
    __shared__ float s_window[FB_NFFT];
    __shared__ float s_melw[FB_MAX_MELW];
    __shared__ int s_mstart[FB_MAX_MEL], s_mcount[FB_MAX_MEL], s_moff[FB_MAX_MEL];
    __shared__ __align__(16) float s_buf[FB_WARPS][2][FB_NFFT];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int k = tid; k < FB_NFFT; k += blockDim.x) {
        float s, c;
        sincospif((float)k * (1.0f / 256.0f), &s, &c);
        s_w512[k] = make_float2(c, -s);
        s_window[k] = (k < p.win) ? p.window[k] : 0.f;
    }
    for (int k = tid; k < p.mel_w_total; k += blockDim.x) s_melw[k] = p.mel_w[k];
    for (int k = tid; k < p.n_mel; k += blockDim.x) {
        s_mstart[k] = p.mel_start[k];
        s_mcount[k] = p.mel_count[k];
        s_moff[k] = p.mel_off[k];
    }
    if (blockIdx.x == 0) {
        for (int b = tid; b < p.B; b += blockDim.x) {
            const int n = p.wave_len[b];
            p.n_frames[b] = (n >= p.win) ? 1 + (n - p.win) / p.shift : 0;
        }
    }
    __syncthreads();

    float* sA = s_buf[warp][0];
    float* sB = s_buf[warp][1];
    const long long total = (long long)p.B * p.t_max;
    const long long wstride = (long long)gridDim.x * FB_WARPS;

    for (long long item = (long long)blockIdx.x * FB_WARPS + warp; item < total; item += wstride) {
        const int b = (int)(item / p.t_max);
        const int f = (int)(item - (long long)b * p.t_max);
        const int n = p.wave_len[b];
        const int m = (n >= p.win) ? 1 + (n - p.win) / p.shift : 0;
        float* o = p.out + item * p.n_mel;
        if (f >= m) {  // padded frame
            for (int i = lane; i < p.n_mel; i += 32) o[i] = 0.f;
            continue;
        }
        const long long xoff = (long long)b * p.n_max + (long long)f * p.shift;
        const float* x = p.wave + xoff;
        const short* x16 = p.wave16 + xoff;

        // 1. load the frame, remove the DC offset (per frame mean)
        float v[FB_NFFT / 32];
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < FB_NFFT / 32; ++i) {
            const int j = lane + 32 * i;
            v[i] = (j < p.win) ? (p.wave16 ? (float)__ldg(x16 + j) * (1.0f / 32768.0f) : __ldg(x + j)) : 0.f;
            sum += v[i];
        }
        float mean = 0.f;
        if (p.remove_dc) mean = warp_sum(sum) / (float)p.win;
#pragma unroll
        for (int i = 0; i < FB_NFFT / 32; ++i) {
            const int j = lane + 32 * i;
            v[i] = (j < p.win) ? __fsub_rn(v[i], mean) : 0.f;
            sA[j] = v[i];
        }
        __syncwarp();
        // 2. pre-emphasis (replicate-padded left neighbour) and window; zero pad to 512
#pragma unroll
        for (int i = 0; i < FB_NFFT / 32; ++i) {
            const int j = lane + 32 * i;
            float y = 0.f;
            if (j < p.win) {
                const float prev = sA[j > 0 ? j - 1 : 0];
                y = __fsub_rn(v[i], __fmul_rn(p.preemph, prev));
                y = __fmul_rn(y, s_window[j]);
            }
            sB[j] = y;
        }
        __syncwarp();
        // 3. 256-pt complex FFT of z[n] = x[2n] + i x[2n+1]
        float2* cA = reinterpret_cast<float2*>(sA);
        float2* cB = reinterpret_cast<float2*>(sB);
        fft256_pass<1>(cB, cA, s_w512, lane);
        fft256_pass<4>(cA, cB, s_w512, lane);
        fft256_pass<16>(cB, cA, s_w512, lane);
        fft256_pass<64>(cA, cB, s_w512, lane);
        // 4. unpack the real FFT and take the power spectrum -> sA[0..256]
        float pw[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            const int k = lane + 32 * i;
            pw[i] = 0.f;
            if (k <= 256) {
                const float2 zk = cB[k & 255];
                float2 zc = cB[(256 - k) & 255];
                zc.y = -zc.y;
                const float er = 0.5f * (zk.x + zc.x), ei = 0.5f * (zk.y + zc.y);
                const float dr = zk.x - zc.x, di = zk.y - zc.y;
                const float orr = 0.5f * di, oi = -0.5f * dr;  // O = -i*(zk - zc)/2
                const float2 w = s_w512[k];
                const float xr = er + (w.x * orr - w.y * oi);
                const float xi = ei + (w.x * oi + w.y * orr);
                pw[i] = xr * xr + xi * xi;
            }
        }
        __syncwarp();  // everyone finished reading cB/cA before sA is overwritten
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            const int k = lane + 32 * i;
            if (k <= 256) sA[k] = pw[i];
        }
        __syncwarp();
        // 5. mel filterbank + log
        for (int i = lane; i < p.n_mel; i += 32) {
            const int s0 = s_mstart[i], cnt = s_mcount[i], off = s_moff[i];
            float acc = 0.f;
            for (int q = 0; q < cnt; ++q) acc = fmaf(s_melw[off + q], sA[s0 + q], acc);
            if (p.use_log) acc = logf(fmaxf(acc, p.log_floor));
            o[i] = acc;
        }
        __syncwarp();  // sA/sB are reused by the next frame
    }
}

// ---------------------------------------------------------------------------------------
constexpr int DC_MAX_ORDER = 2;
constexpr int DC_MAX_TAPS = 33;
constexpr int DC_COLS = 128;   // n_mel*(order+1) padded column count handled per CTA pass
constexpr int DC_ROWS = 2;     // row phases (blockDim = DC_COLS*DC_ROWS)
constexpr int DC_TCHUNK = 64;  // frames per CTA

struct DeltaParams {
    const float* fb;
    const int* n_frames;
    int B, t_max, n_mel, order, pad, taps, apply_cmvn;
    float eps;
    float* out;
    float filt[DC_MAX_ORDER + 1][DC_MAX_TAPS];
};

__device__ __forceinline__ float delta_value(const DeltaParams& p, const float* fb, int m, int t, int o, int bin) {
    // sum_tap filt[o][tap] * fb[t + tap - pad][bin], zero outside [0, m)
    float acc = 0.f;
    for (int tap = 0; tap < p.taps; ++tap) {
        const float w = p.filt[o][tap];
        const int tt = t + tap - p.pad;
        if (w != 0.f && tt >= 0 && tt < m) acc = fmaf(w, fb[(long long)tt * p.n_mel + bin], acc);
    }
    return acc;
}

// The chunk's fbank rows [t0 - pad, t0 + DC_TCHUNK + pad) are staged ONCE in shared memory (zeros outside [0, m): the
// zero padding of src/audio.py:57-77) together with the tap weights; the taps then read shared memory.  Same tap order
// and the same fmaf chain as delta_value() above (a zero tap or a zero-padded row adds exactly 0), so the values are
// bit-identical to a kernel that re-reads global memory per tap (~25 instructions per tap, branchy).
__device__ __forceinline__ void delta_stage(const DeltaParams& p, const float* fb, int m, int t0, float* s_fb,
                                            float* s_filt) {
    const int rows = DC_TCHUNK + p.taps - 1;
    for (int i = threadIdx.x; i < rows * p.n_mel; i += blockDim.x) {
        const int rl = i / p.n_mel, bin = i - rl * p.n_mel;
        const int t = t0 - p.pad + rl;
        s_fb[i] = (t >= 0 && t < m) ? fb[(long long)t * p.n_mel + bin] : 0.f;
    }
    for (int i = threadIdx.x; i < (DC_MAX_ORDER + 1) * DC_MAX_TAPS; i += blockDim.x)
        s_filt[i] = p.filt[i / DC_MAX_TAPS][i % DC_MAX_TAPS];
    __syncthreads();
}
__device__ __forceinline__ float delta_smem(const float* s_fb, const float* s_filt, int n_mel, int taps, int tl, int o,
                                            int bin) {
    float acc = 0.f;
    const float* w = s_filt + o * DC_MAX_TAPS;
    const float* x = s_fb + tl * n_mel + bin;          // row tl of the tile = frame t0 + tl - pad
    for (int tap = 0; tap < taps; ++tap) acc = fmaf(w[tap], x[tap * n_mel], acc);
    return acc;
}

// Pass 1: per (utterance, time chunk) partial sums of x and x^2 (fp64) for every output column.
// Pass 2: every CTA re-reduces the chunk partials of its utterance in a fixed order (deterministic), then
// normalises and writes its own time chunk.  Both passes recompute the (cheap) delta taps from the L2-resident fbank.

__global__ void __launch_bounds__(DC_COLS* DC_ROWS) delta_stats_kernel(DeltaParams p, double* __restrict__ partial,
                                                                      int nchunk) {
    __shared__ double s_red[2][DC_ROWS][DC_COLS];
    __shared__ float s_filt[(DC_MAX_ORDER + 1) * DC_MAX_TAPS];
    extern __shared__ float s_fb[];
    const int b = blockIdx.y, ch = blockIdx.x;
    const int D = p.n_mel * (p.order + 1);
    const int m = p.n_frames[b];
    const float* fb = p.fb + (long long)b * p.t_max * p.n_mel;
    const int r = threadIdx.x / DC_COLS, cl = threadIdx.x % DC_COLS;
    const int t0 = ch * DC_TCHUNK, t1 = min(m, t0 + DC_TCHUNK);
    if (t0 >= m) {                                      // chunk entirely in the padding: its partials are never read
        return;
    }
    delta_stage(p, fb, m, t0, s_fb, s_filt);
    for (int c0 = 0; c0 < D; c0 += DC_COLS) {
        const int col = c0 + cl;
        const bool act = col < D;
        const int o = act ? col / p.n_mel : 0;
        const int bin = act ? col - o * p.n_mel : 0;
        double s = 0.0, ss = 0.0;
        if (act)
            for (int t = t0 + r; t < t1; t += DC_ROWS) {
                const double v = (double)delta_smem(s_fb, s_filt, p.n_mel, p.taps, t - t0, o, bin);
                s += v;
                ss += v * v;
            }
        s_red[0][r][cl] = s;
        s_red[1][r][cl] = ss;
        __syncthreads();
        if (r == 0 && act) {
            double ts = 0.0, tss = 0.0;
            for (int q = 0; q < DC_ROWS; ++q) { ts += s_red[0][q][cl]; tss += s_red[1][q][cl]; }
            double* dst = partial + (((long long)b * nchunk + ch) * D + col) * 2;
            dst[0] = ts;
            dst[1] = tss;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(DC_COLS* DC_ROWS) delta_norm_kernel(DeltaParams p, const double* __restrict__ partial,
                                                                     int nchunk) {
    __shared__ float s_mean[DC_COLS], s_den[DC_COLS];
    __shared__ float s_filt[(DC_MAX_ORDER + 1) * DC_MAX_TAPS];
    extern __shared__ float s_fb[];
    const int b = blockIdx.y, ch = blockIdx.x;
    const int D = p.n_mel * (p.order + 1);
    const int m = p.n_frames[b];
    const float* fb = p.fb + (long long)b * p.t_max * p.n_mel;
    float* out = p.out + (long long)b * p.t_max * D;
    const int r = threadIdx.x / DC_COLS, cl = threadIdx.x % DC_COLS;
    const int t0 = ch * DC_TCHUNK, t1 = min(p.t_max, t0 + DC_TCHUNK);
    const int mchunks = (m + DC_TCHUNK - 1) / DC_TCHUNK;
    delta_stage(p, fb, m, t0, s_fb, s_filt);
    for (int c0 = 0; c0 < D; c0 += DC_COLS) {
        const int col = c0 + cl;
        const bool act = col < D;
        const int o = act ? col / p.n_mel : 0;
        const int bin = act ? col - o * p.n_mel : 0;
        if (p.apply_cmvn && r == 0 && act) {
            double ts = 0.0, tss = 0.0;
            for (int q = 0; q < mchunks; ++q) {
                const double* src = partial + (((long long)b * nchunk + q) * D + col) * 2;
                ts += src[0];
                tss += src[1];
            }
            const double mean = ts / (double)m;
            // unbiased variance (torch.std default); m == 1 gives 0/0 = NaN exactly like torch
            const double var = (tss - ts * mean) / (double)(m - 1);
            s_mean[cl] = (float)mean;
            s_den[cl] = p.eps + (float)sqrt(var > 0.0 || !(var == var) ? var : 0.0);
        }
        __syncthreads();
        if (act) {
            const float mean = p.apply_cmvn ? s_mean[cl] : 0.f;
            const float den = p.apply_cmvn ? s_den[cl] : 1.f;
            for (int t = t0 + r; t < t1; t += DC_ROWS) {
                float v = 0.f;
                if (t < m) {
                    v = delta_smem(s_fb, s_filt, p.n_mel, p.taps, t - t0, o, bin);
                    if (p.apply_cmvn) v = (v - mean) / den;
                }
                out[(long long)t * D + col] = v;
            }
        }
        __syncthreads();
    }
}

}  // namespace b200asr

using namespace b200asr;

static int fbank_run(const float* wave, const short* wave16, const int* wave_len, int B, int n_max, int win_size,
                     int win_shift, int n_fft, float preemph, int remove_dc, const float* window, int n_mel,
                     const int* mel_start, const int* mel_count, const int* mel_off, const float* mel_w,
                     int mel_w_total, int use_log, float log_floor, float* fbank, int t_max, int* n_frames,
                     b200asr_stream stream);

extern "C" int b200asr_fbank_fwd(const float* wave, const int* wave_len, int B, int n_max, int win_size,
                                 int win_shift, int n_fft, float preemph, int remove_dc, const float* window,
                                 int n_mel, const int* mel_start, const int* mel_count, const int* mel_off,
                                 const float* mel_w, int mel_w_total, int use_log, float log_floor, float* fbank,
                                 int t_max, int* n_frames, b200asr_stream stream) {
    B200_REQUIRE(wave, "fbank: null pointer");
    return fbank_run(wave, nullptr, wave_len, B, n_max, win_size, win_shift, n_fft, preemph, remove_dc, window, n_mel,
                     mel_start, mel_count, mel_off, mel_w, mel_w_total, use_log, log_floor, fbank, t_max, n_frames, stream);
}

extern "C" int b200asr_fbank_fwd_pcm16(const short* pcm, const int* wave_len, int B, int n_max, int win_size,
                                       int win_shift, int n_fft, float preemph, int remove_dc, const float* window,
                                       int n_mel, const int* mel_start, const int* mel_count, const int* mel_off,
                                       const float* mel_w, int mel_w_total, int use_log, float log_floor,
                                       float* fbank, int t_max, int* n_frames, b200asr_stream stream) {
    B200_REQUIRE(pcm, "fbank: null pointer");
    return fbank_run(reinterpret_cast<const float*>(pcm), pcm, wave_len, B, n_max, win_size, win_shift, n_fft, preemph,
                     remove_dc, window, n_mel, mel_start, mel_count, mel_off, mel_w, mel_w_total, use_log, log_floor,
                     fbank, t_max, n_frames, stream);
}

static int fbank_run(const float* wave, const short* wave16, const int* wave_len, int B, int n_max, int win_size,
                     int win_shift, int n_fft, float preemph, int remove_dc, const float* window, int n_mel,
                     const int* mel_start, const int* mel_count, const int* mel_off, const float* mel_w,
                     int mel_w_total, int use_log, float log_floor, float* fbank, int t_max, int* n_frames,
                     b200asr_stream stream) {
    B200_REQUIRE(n_fft == FB_NFFT, "fbank: only a 512-point padded window is supported (got %d)", n_fft);
    B200_REQUIRE(win_size >= 2 && win_size <= FB_NFFT, "fbank: window size %d not in [2,512]", win_size);
    B200_REQUIRE(win_shift > 0, "fbank: window shift must be > 0");
    B200_REQUIRE(n_mel > 0 && n_mel <= FB_MAX_MEL, "fbank: n_mel %d not in [1,%d]", n_mel, FB_MAX_MEL);
    B200_REQUIRE(mel_w_total > 0 && mel_w_total <= FB_MAX_MELW, "fbank: %d mel weights exceed %d", mel_w_total,
                 FB_MAX_MELW);
    B200_REQUIRE(B > 0 && n_max > 0 && t_max >= 0, "fbank: bad sizes B=%d n_max=%d t_max=%d", B, n_max, t_max);
    B200_REQUIRE(wave && wave_len && window && mel_start && mel_count && mel_off && mel_w && fbank && n_frames,
                 "fbank: null pointer");
    FbankParams p;
    p.wave = wave; p.wave16 = wave16; p.wave_len = wave_len; p.B = B; p.n_max = n_max; p.win = win_size; p.shift = win_shift;
    p.preemph = preemph; p.remove_dc = remove_dc; p.window = window; p.n_mel = n_mel; p.mel_start = mel_start;
    p.mel_count = mel_count; p.mel_off = mel_off; p.mel_w = mel_w; p.mel_w_total = mel_w_total;
    p.log_floor = log_floor; p.use_log = use_log; p.out = fbank; p.t_max = t_max; p.n_frames = n_frames;
    const long long items = (long long)B * (t_max > 0 ? t_max : 1);
    long long blocks = (items + FB_WARPS - 1) / FB_WARPS;
    const long long cap = (long long)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    fbank_kernel<<<(unsigned)blocks, FB_WARPS * 32, 0, (cudaStream_t)stream>>>(p);
    B200_LAUNCH_CHECK("fbank_kernel");
    return B200_OK;
}

// Delta filter taps exactly as the reference builds them (src/audio.py:57-77): order-i filter is the
// order-(i-1) filter convolved with [-w..w]/sum(j^2), all centred in a common 2*order*w+1 support.
static int build_delta_filters(int order, int window, float filt[DC_MAX_ORDER + 1][DC_MAX_TAPS], int* taps_out) {
    const int taps = 2 * order * window + 1;
    if (order < 0 || order > DC_MAX_ORDER || taps > DC_MAX_TAPS || window < 1) return -1;
    double sc[DC_MAX_ORDER + 1][DC_MAX_TAPS];
    int len[DC_MAX_ORDER + 1];
    for (int i = 0; i <= DC_MAX_ORDER; ++i)
        for (int j = 0; j < DC_MAX_TAPS; ++j) sc[i][j] = 0.0;
    sc[0][0] = 1.0;
    len[0] = 1;
    for (int i = 1; i <= order; ++i) {
        const int prev_off = (len[i - 1] - 1) / 2;
        const int cur_off = prev_off + window;
        len[i] = len[i - 1] + 2 * window;
        double norm = 0.0;
        for (int j = -window; j <= window; ++j) {
            norm += (double)j * j;
            for (int k = -prev_off; k <= prev_off; ++k) sc[i][j + k + cur_off] += (double)j * sc[i - 1][k + prev_off];
        }
        for (int j = 0; j < len[i]; ++j) sc[i][j] /= norm;
    }
    for (int i = 0; i <= DC_MAX_ORDER; ++i)
        for (int j = 0; j < DC_MAX_TAPS; ++j) filt[i][j] = 0.f;
    for (int i = 0; i <= order; ++i) {
        const int padl = (taps - len[i]) / 2;
        for (int j = 0; j < len[i]; ++j) filt[i][padl + j] = (float)sc[i][j];
    }
    *taps_out = taps;
    return 0;
}

extern "C" size_t b200asr_delta_cmvn_workspace_bytes(int B, int t_max, int n_mel, int delta_order) {
    const size_t nchunk = ((size_t)t_max + DC_TCHUNK - 1) / DC_TCHUNK;
    return (size_t)B * (nchunk ? nchunk : 1) * n_mel * (delta_order + 1) * 2 * sizeof(double);
}

extern "C" int b200asr_delta_cmvn_fwd(const float* fbank, const int* n_frames, int B, int t_max, int n_mel,
                                      int delta_order, int delta_window, int apply_cmvn, float cmvn_eps,
                                      float* feat, void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(fbank && n_frames && feat, "delta_cmvn: null pointer");
    B200_REQUIRE(B > 0 && t_max >= 0 && n_mel > 0, "delta_cmvn: bad sizes");
    DeltaParams p;
    int taps = 1;
    B200_REQUIRE(build_delta_filters(delta_order, delta_window, p.filt, &taps) == 0,
                 "delta_cmvn: unsupported delta order %d / window %d", delta_order, delta_window);
    p.fb = fbank; p.n_frames = n_frames; p.B = B; p.t_max = t_max; p.n_mel = n_mel; p.order = delta_order;
    p.taps = taps; p.pad = (taps - 1) / 2; p.apply_cmvn = apply_cmvn; p.eps = cmvn_eps; p.out = feat;
    if (t_max == 0) return B200_OK;
    const int nchunk = (t_max + DC_TCHUNK - 1) / DC_TCHUNK;
    double* partial = reinterpret_cast<double*>(workspace);
    const size_t smem = (size_t)(DC_TCHUNK + taps - 1) * n_mel * sizeof(float);
    B200_REQUIRE(smem <= 40 * 1024, "delta_cmvn: %d mel bins x %d taps do not fit the shared-memory tile", n_mel, taps);
    if (apply_cmvn) {
        B200_REQUIRE(workspace && workspace_bytes >= b200asr_delta_cmvn_workspace_bytes(B, t_max, n_mel, delta_order),
                     "delta_cmvn: workspace too small");
        delta_stats_kernel<<<dim3(nchunk, B), DC_COLS * DC_ROWS, smem, (cudaStream_t)stream>>>(p, partial, nchunk);
        B200_LAUNCH_CHECK("delta_stats_kernel");
    }
    delta_norm_kernel<<<dim3(nchunk, B), DC_COLS * DC_ROWS, smem, (cudaStream_t)stream>>>(p, partial, nchunk);
    B200_LAUNCH_CHECK("delta_norm_kernel");
    return B200_OK;
}
