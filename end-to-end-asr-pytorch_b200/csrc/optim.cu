// K16: global gradient norm + clip + optimizer update on the flat fp32 parameter / gradient buffers.
//
// Restates /root/reference/src/solver.py:84-89 (clip_grad_norm_(params, 5.0); skip the step when the norm
// is NaN) and the torch.optim.Adadelta / Adam updates selected by src/optim.py:33-52, but decides the
// clip coefficient and the NaN skip on the device so the step needs no host synchronisation.  For the same
// reason the count of applied steps (torch's state["step"], which a skipped step does not advance) lives on
// the device, and Adam's bias corrections are formed there from it.
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {

constexpr int NORM_BLOCKS = 528;  // 4 per SM on a 132-SM part
constexpr int NORM_THREADS = 256;

__global__ void __launch_bounds__(NORM_THREADS) sumsq_partial_kernel(const float* __restrict__ g, long long n,
                                                                   double* __restrict__ partials) {
    __shared__ double s_w[NORM_THREADS / 32];
    double acc = 0.0;
    const long long n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = g4[i];
        acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const float v = g[(n4 << 2) + threadIdx.x];
        acc += (double)v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < NORM_THREADS / 32; ++w) t += s_w[w];
        partials[blockIdx.x] = t;
    }
}

__global__ void norm_final_kernel(const double* __restrict__ partials, int nparts, float* __restrict__ norm_out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < nparts; ++i) t += partials[i];
        *norm_out = (float)sqrt(t);
    }
}

// The reference skips optimizer.step() exactly when math.isnan(norm).  An Inf norm is not skipped: clip_grad_norm_
// scales by max_norm / (inf + 1e-6) = 0, so +-Inf gradient entries become NaN and every other entry 0.
__device__ __forceinline__ bool clip_coef(const float* norm_dev, float max_norm, float* coef) {
    *coef = 1.f;
    if (!norm_dev) return true;
    const float nrm = *norm_dev;
    if (isnan(nrm)) return false;
    if (max_norm > 0.f) *coef = fminf(1.f, max_norm / (nrm + 1e-6f));
    return true;
}

// One thread, launched before the update kernel: the update reads the advanced count, as torch advances
// state["step"] before it forms the bias corrections.
__global__ void advance_step_kernel(const float* __restrict__ norm_dev, long long* __restrict__ step_count) {
    if (!norm_dev || !isnan(*norm_dev)) *step_count += 1;
}

// rho / beta and their complements arrive rounded to fp32 once each, the complements formed in double on the host
// (torch's `1 - rho` is a double scalar); 1.f - rho in fp32 would be off by up to 216 u for rho = 0.999.
__global__ void __launch_bounds__(256) adadelta_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                      float* __restrict__ sq, float* __restrict__ acc, long long n,
                                                      float lr, float rho, float one_m_rho, float eps, float wd,
                                                      const float* __restrict__ norm_dev, float max_norm) {
    float coef;
    if (!clip_coef(norm_dev, max_norm, &coef)) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float gi = g[i] * coef;
        const float pi = p[i];
        if (wd != 0.f) gi = fmaf(wd, pi, gi);
        const float s = rho * sq[i] + one_m_rho * gi * gi;
        sq[i] = s;
        const float a = acc[i];
        const float delta = sqrtf(a + eps) / sqrtf(s + eps) * gi;
        acc[i] = rho * a + one_m_rho * delta * delta;
        p[i] = pi - lr * delta;
    }
}

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                  float* __restrict__ m, float* __restrict__ v, long long n, float lr,
                                                  float beta1, float one_m_beta1, double beta1_d, float beta2,
                                                  float one_m_beta2, double beta2_d, float eps, float wd,
                                                  const long long* __restrict__ step_count,
                                                  const float* __restrict__ norm_dev, float max_norm) {
    float coef;
    if (!clip_coef(norm_dev, max_norm, &coef)) return;
    // bias corrections of the applied-step count in double, as torch forms them from its Python-float betas
    const double t = (double)*step_count;
    const float step_size = (float)((double)lr / (1.0 - pow(beta1_d, t)));
    const float rsb2 = (float)(1.0 / sqrt(1.0 - pow(beta2_d, t)));
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float gi = g[i] * coef;
        const float pi = p[i];
        if (wd != 0.f) gi = fmaf(wd, pi, gi);
        const float mi = beta1 * m[i] + one_m_beta1 * gi;
        const float vi = beta2 * v[i] + one_m_beta2 * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) * rsb2 + eps;
        p[i] = pi - step_size * (mi / denom);
    }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" size_t b200asr_grad_norm_scratch_bytes(void) { return NORM_BLOCKS * sizeof(double); }

extern "C" int b200asr_grad_norm(const float* grad, long long n, float* norm_out, void* scratch,
                                 b200asr_stream stream) {
    B200_REQUIRE(grad && norm_out && scratch, "grad_norm: null pointer");
    B200_REQUIRE(n >= 0, "grad_norm: negative size");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(grad) & 15) == 0, "grad_norm: gradient buffer must be 16-byte aligned");
    sumsq_partial_kernel<<<NORM_BLOCKS, NORM_THREADS, 0, (cudaStream_t)stream>>>(grad, n,
                                                                                reinterpret_cast<double*>(scratch));
    B200_LAUNCH_CHECK("sumsq_partial_kernel");
    norm_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(reinterpret_cast<const double*>(scratch), NORM_BLOCKS,
                                                         norm_out);
    B200_LAUNCH_CHECK("norm_final_kernel");
    return B200_OK;
}

static unsigned grid_for(long long n) {
    long long b = (n + 255) / 256;
    const long long cap = (long long)sm_count() * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (unsigned)b;
}

static int advance_step(const float* grad_norm, long long* step_count, cudaStream_t stream) {
    advance_step_kernel<<<1, 1, 0, stream>>>(grad_norm, step_count);
    B200_LAUNCH_CHECK("advance_step_kernel");
    return B200_OK;
}

extern "C" int b200asr_adadelta_step(float* param, const float* grad, float* square_avg, float* acc_delta,
                                     long long n, float lr, double rho, float eps, float weight_decay,
                                     const float* grad_norm, float max_norm, long long* step_count,
                                     b200asr_stream stream) {
    B200_REQUIRE(param && grad && square_avg && acc_delta && step_count, "adadelta_step: null pointer");
    const int rc = advance_step(grad_norm, step_count, (cudaStream_t)stream);
    if (rc != B200_OK || n <= 0) return rc;
    adadelta_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(param, grad, square_avg, acc_delta, n, lr,
                                                                  (float)rho, (float)(1.0 - rho), eps, weight_decay,
                                                                  grad_norm, max_norm);
    B200_LAUNCH_CHECK("adadelta_kernel");
    return B200_OK;
}

extern "C" int b200asr_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                                 float lr, double beta1, double beta2, float eps, float weight_decay,
                                 const float* grad_norm, float max_norm, long long* step_count,
                                 b200asr_stream stream) {
    B200_REQUIRE(param && grad && exp_avg && exp_avg_sq && step_count, "adam_step: null pointer");
    const int rc = advance_step(grad_norm, step_count, (cudaStream_t)stream);
    if (rc != B200_OK || n <= 0) return rc;
    adam_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(
        param, grad, exp_avg, exp_avg_sq, n, lr, (float)beta1, (float)(1.0 - beta1), beta1, (float)beta2,
        (float)(1.0 - beta2), beta2, eps, weight_decay, step_count, grad_norm, max_norm);
    B200_LAUNCH_CHECK("adam_kernel");
    return B200_OK;
}

// ---- fp32 -> (tf32 hi, fp32 residual lo) split for error-compensated tensor-core GEMMs (3xTF32) ----------------
// hi = x rounded to TF32 (10 explicit mantissa bits, low 13 bits zero), lo = x - hi (exact in fp32).  The caller
// forms  A.B ~= A_lo.B_hi + A_hi.B_lo + A_hi.B_hi  with three TF32 tensor-core GEMMs accumulating in fp32,
// which keeps the input-projection / weight-gradient contractions within fp32-level error (~1e-6 relative).
namespace b200asr {
__global__ void __launch_bounds__(256) split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi,
                                                        float4* __restrict__ lo, long long n4, const float* xs,
                                                        float* his, float* los, int tail) {
    auto split = [](float v, float& h, float& l) {
        unsigned u = __float_as_uint(v);
        // round to nearest (ties away) on the magnitude; inf/nan pass through unchanged
        if ((u & 0x7f800000u) != 0x7f800000u) u = (u + 0x1000u) & 0xffffe000u;
        h = __uint_as_float(u);
        l = v - h;
    };
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = x[i];
        float4 h, l;
        split(v.x, h.x, l.x); split(v.y, h.y, l.y); split(v.z, h.z, l.z); split(v.w, h.w, l.w);
        hi[i] = h;
        lo[i] = l;
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < tail) {
        float h, l;
        split(xs[threadIdx.x], h, l);
        his[threadIdx.x] = h;
        los[threadIdx.x] = l;
    }
}
}  // namespace b200asr

extern "C" int b200asr_split_tf32(const float* x, float* hi, float* lo, long long n, b200asr_stream stream) {
    B200_REQUIRE(x && hi && lo, "split_tf32: null pointer");
    B200_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15) == 0,
                 "split_tf32: buffers must be 16-byte aligned");
    if (n <= 0) return B200_OK;
    const long long n4 = n >> 2;
    const int tail = (int)(n & 3);
    split_tf32_kernel<<<grid_for(n4 > 0 ? n4 : 1), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(hi), reinterpret_cast<float4*>(lo), n4,
        x + (n4 << 2), hi + (n4 << 2), lo + (n4 << 2), tail);
    B200_LAUNCH_CHECK("split_tf32_kernel");
    return B200_OK;
}
