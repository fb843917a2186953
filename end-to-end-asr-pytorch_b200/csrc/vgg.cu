// VGGExtractor (src/module.py:7-66) around the conv-mode 3xTF32 GEMM (b200asr_conv3x3_fwd / _wgrad, csrc/gemm.cu):
// the first layer's im2col, the 2x2 max-pool forward and backward (the backward fused with the ReLU mask of the conv
// before it) and the gradient with respect to the features.
//
// Every activation lives in a zero-haloed channels-last buffer of its (T, F): grid rows R = B (T + 2) (F + 2) plus F + 3
// trailing rows; position (b, t, f) sits at row (b (T + 2) + t + 1) (F + 2) + f + 1.  The kernels below write every row
// of the buffers they produce (zeros on the halo), so nothing needs a separate memset.
//
// Max-pool follows ATen's scan (aten/src/ATen/native/cuda/DilatedMaxPool2d.cu): the window is walked in raster order
// (time, then frequency) and an element is taken when  val > max || isnan(val),  starting from -inf; the chosen
// element's index (0..3) is kept as one byte for the backward.  Floor mode: a last odd frequency is in no window.
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {
namespace {

__host__ __device__ __forceinline__ long long grid_rows(int B, int T, int F) { return (long long)B * (T + 2) * (F + 2); }

int blocks_for(long long n) {
    const long long b = (n + 255) / 256, cap = 32LL * sm_count();
    return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

// im2col of the features for the first conv: out[m][k], m over the grid rows of (T, F), k = tap * Cin + c < 9 Cin (the
// rest of the 32 columns and every junk row: 0).  Feature element (b, t, c, f) at feat[b * ld_b + t * Cin * F + c * F + f].
__global__ void vgg_im2col_kernel(const float* __restrict__ feat, long long ld_b, int B, int T, int Cin, int F,
                                  float* __restrict__ out) {
    const long long n = grid_rows(B, T, F) * 32;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i >> 5;
        const int k = (int)(i & 31);
        const int f = (int)(m % (F + 2));
        const long long bt = m / (F + 2);
        const int t = (int)(bt % (T + 2)), b = (int)(bt / (T + 2));
        float v = 0.f;
        if (t < T && f < F && k < 9 * Cin) {
            const int tap = k / Cin, c = k - tap * Cin;
            const int tt = t + tap / 3 - 1, ff = f + tap % 3 - 1;
            if (tt >= 0 && tt < T && ff >= 0 && ff < F) v = feat[b * ld_b + ((long long)tt * Cin + c) * F + ff];
        }
        out[i] = v;
    }
}

// Pool of the padded buffer y (T, F) -> idx[b][t2][f2][c] and either the padded buffer of (T / 2, F / 2) (every row,
// halos 0) or, flat, the prenet output out[b][t2][c * F2 + f2].
__global__ void vgg_pool_fwd_kernel(const float* __restrict__ y, int B, int T, int F, int C, float* __restrict__ out,
                                    uint8_t* __restrict__ idx, int flat) {
    const int T2 = T / 2, F2 = F / 2;
    const long long n = flat ? (long long)B * T2 * F2 * C : (grid_rows(B, T2, F2) + F2 + 3) * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long row = i / C;
        int b, t2, f2;
        if (flat) {
            f2 = (int)(row % F2);
            const long long bt = row / F2;
            t2 = (int)(bt % T2);
            b = (int)(bt / T2);
        } else {
            if (row >= grid_rows(B, T2, F2)) { out[i] = 0.f; continue; }
            const int fp = (int)(row % (F2 + 2));
            const long long bt = row / (F2 + 2);
            const int tp = (int)(bt % (T2 + 2));
            b = (int)(bt / (T2 + 2));
            if (tp < 1 || tp > T2 || fp < 1 || fp > F2) { out[i] = 0.f; continue; }
            t2 = tp - 1;
            f2 = fp - 1;
        }
        const float* base = y + (((long long)b * (T + 2) + 2 * t2 + 1) * (F + 2) + 2 * f2 + 1) * C + c;
        float mx = -INFINITY;
        int k = 0;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float v = base[((long long)(w >> 1) * (F + 2) + (w & 1)) * C];
            if (v > mx || isnan(v)) { mx = v; k = w; }
        }
        idx[(((long long)b * T2 + t2) * F2 + f2) * C + c] = (uint8_t)k;
        if (flat) out[((long long)b * T2 + t2) * C * F2 + (long long)c * F2 + f2] = mx;
        else out[i] = mx;
    }
}

// Max-pool backward fused with the ReLU backward of the conv before it: every row of the padded buffer dy of (T, F) gets
// the pooled gradient where idx chose it and y > 0 (ATen's threshold_backward: y <= 0 gives 0), else 0.  The pooled
// gradient comes from the padded buffer of (T / 2, F / 2) or, flat, from the prenet output's gradient.
__global__ void vgg_pool_bwd_kernel(const float* __restrict__ dout, const uint8_t* __restrict__ idx,
                                    const float* __restrict__ y, int B, int T, int F, int C, float* __restrict__ dy,
                                    int flat) {
    const int T2 = T / 2, F2 = F / 2;
    const long long R = grid_rows(B, T, F), n = (R + F + 3) * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long row = i / C;
        float g = 0.f;
        if (row < R) {
            const int fp = (int)(row % (F + 2));
            const long long bt = row / (F + 2);
            const int tp = (int)(bt % (T + 2)), b = (int)(bt / (T + 2));
            const int t = tp - 1, f = fp - 1;
            if (t >= 0 && t < T && f >= 0 && f < 2 * F2) {
                const int t2 = t >> 1, f2 = f >> 1;
                if (idx[(((long long)b * T2 + t2) * F2 + f2) * C + c] == ((t & 1) << 1 | (f & 1)) && !(y[i] <= 0.f)) {
                    g = flat ? dout[((long long)b * T2 + t2) * C * F2 + (long long)c * F2 + f2]
                             : dout[(((long long)b * (T2 + 2) + t2 + 1) * (F2 + 2) + f2 + 1) * C + c];
                }
            }
        }
        dy[i] = g;
    }
}

// dfeat[b][t][c * F + f] = sum over (o, tap) of w1[o][c][dt][df] dy1(t + 1 - dt, f + 1 - df)[o] (dy1 padded, zero
// outside); frames t >= T (cropped by the prenet) get 0.  One thread per feature element, direct sum (not on the
// train step's path).
__global__ void vgg_feat_grad_kernel(const float* __restrict__ dy1, const float* __restrict__ w1, int B, int T, int T_in,
                                     int Cin, int F, int O, float* __restrict__ dfeat) {
    const long long n = (long long)B * T_in * Cin * F;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int f = (int)(i % F);
        const long long r = i / F;
        const int c = (int)(r % Cin);
        const long long bt = r / Cin;
        const int t = (int)(bt % T_in), b = (int)(bt / T_in);
        float s = 0.f;
        if (t < T) {
            for (int tap = 0; tap < 9; ++tap) {
                const int dt = tap / 3, df = tap % 3;
                const float* d = dy1 + (((long long)b * (T + 2) + t + 2 - dt) * (F + 2) + f + 2 - df) * O;
                const float* w = w1 + (long long)c * 9 + tap;
                for (int o = 0; o < O; ++o) s = fmaf(w[(long long)o * Cin * 9], d[o], s);
            }
        }
        dfeat[i] = s;
    }
}

}  // namespace
}  // namespace b200asr

using namespace b200asr;

static int vgg_sizes(const char* what, int B, int T, int F, int C) {
    B200_REQUIRE(B > 0 && T > 0 && F > 0 && C > 0 && grid_rows(B, T, F) * (long long)C < (1LL << 40),
                 "%s: bad sizes B=%d T=%d F=%d C=%d", what, B, T, F, C);
    return B200_OK;
}

extern "C" int b200asr_vgg_im2col(const float* feat, long long ld_b, int B, int T, int Cin, int F, float* out,
                                  b200asr_stream stream) {
    B200_REQUIRE(feat && out, "vgg_im2col: null pointer");
    B200_REQUIRE(Cin >= 1 && Cin <= 3 && ld_b >= (long long)T * Cin * F, "vgg_im2col: bad layout (Cin %d ld_b %lld)",
                 Cin, ld_b);
    const int rc = vgg_sizes("vgg_im2col", B, T, F, 32);
    if (rc != B200_OK) return rc;
    vgg_im2col_kernel<<<blocks_for(grid_rows(B, T, F) * 32), 256, 0, (cudaStream_t)stream>>>(feat, ld_b, B, T, Cin, F,
                                                                                           out);
    B200_LAUNCH_CHECK("vgg_im2col_kernel");
    return B200_OK;
}

extern "C" int b200asr_vgg_pool_fwd(const float* y, int B, int T, int F, int C, float* out, unsigned char* idx, int flat,
                                    b200asr_stream stream) {
    B200_REQUIRE(y && out && idx, "vgg_pool_fwd: null pointer");
    B200_REQUIRE(T >= 2 && (T % 2) == 0 && F >= 2, "vgg_pool_fwd: needs an even T >= 2 and F >= 2 (T %d F %d)", T, F);
    const int rc = vgg_sizes("vgg_pool_fwd", B, T, F, C);
    if (rc != B200_OK) return rc;
    const long long n = flat ? (long long)B * (T / 2) * (F / 2) * C : (grid_rows(B, T / 2, F / 2) + F / 2 + 3) * C;
    vgg_pool_fwd_kernel<<<blocks_for(n), 256, 0, (cudaStream_t)stream>>>(y, B, T, F, C, out, idx, flat);
    B200_LAUNCH_CHECK("vgg_pool_fwd_kernel");
    return B200_OK;
}

extern "C" int b200asr_vgg_pool_bwd(const float* dout, const unsigned char* idx, const float* y, int B, int T, int F,
                                    int C, float* dy, int flat, b200asr_stream stream) {
    B200_REQUIRE(dout && idx && y && dy, "vgg_pool_bwd: null pointer");
    B200_REQUIRE(T >= 2 && (T % 2) == 0 && F >= 2, "vgg_pool_bwd: needs an even T >= 2 and F >= 2 (T %d F %d)", T, F);
    const int rc = vgg_sizes("vgg_pool_bwd", B, T, F, C);
    if (rc != B200_OK) return rc;
    vgg_pool_bwd_kernel<<<blocks_for((grid_rows(B, T, F) + F + 3) * C), 256, 0, (cudaStream_t)stream>>>(
        dout, idx, y, B, T, F, C, dy, flat);
    B200_LAUNCH_CHECK("vgg_pool_bwd_kernel");
    return B200_OK;
}

extern "C" int b200asr_vgg_feat_grad(const float* dy1, const float* w1, int B, int T, int T_in, int Cin, int F, int O,
                                     float* dfeat, b200asr_stream stream) {
    B200_REQUIRE(dy1 && w1 && dfeat, "vgg_feat_grad: null pointer");
    B200_REQUIRE(Cin >= 1 && O > 0 && T_in >= T, "vgg_feat_grad: bad sizes (Cin %d O %d T %d T_in %d)", Cin, O, T, T_in);
    const int rc = vgg_sizes("vgg_feat_grad", B, T_in, F, Cin);
    if (rc != B200_OK) return rc;
    vgg_feat_grad_kernel<<<blocks_for((long long)B * T_in * Cin * F), 256, 0, (cudaStream_t)stream>>>(
        dy1, w1, B, T, T_in, Cin, F, O, dfeat);
    B200_LAUNCH_CHECK("vgg_feat_grad_kernel");
    return B200_OK;
}
