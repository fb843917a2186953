// SURVEY.md 8(f) rank 3: CTC prefix scoring on the GPU.  Restates CTCPrefixScore.cheap_compute of the reference
// (/root/reference/src/ctc.py:81-116, Watanabe et al. TR2017-190 Algo. 2; called from src/decode.py:129-131 once per
// hypothesis and decode step, numpy, on the host): for a prefix g and a candidate token c it runs the T-long
// forward recursion  r[t,0] (prefix+c ends in c at t), r[t,1] (ends in blank)  and accumulates the prefix probability
// psi.  Candidates - and hypotheses - are independent, so ONE launch scores every (hypothesis, candidate) pair of a
// beam-search step: one thread per pair, the frame loop in registers, log-probs gathered from the [T,V] matrix.
// float32 arithmetic with the reference's finite log-zero (-1e8) and numpy's logaddexp formula.
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {

__device__ __forceinline__ float np_logaddexp(float a, float b) {
    if (a == b) return a + 0.6931471805599453f;             // numpy's branch: logaddexp(-inf, -inf) = -inf, not NaN
    const float m = fmaxf(a, b);
    const float d = -fabsf(a - b);
    return m + log1pf(expf(d));
}

__global__ void __launch_bounds__(128) ctc_prefix_kernel(const float* __restrict__ x, int T, int V,
                                                        const float* __restrict__ r_prev,
                                                        const int* __restrict__ last_char,
                                                        const int* __restrict__ prefix_len,
                                                        const int* __restrict__ cand, int N, int C, int blank, int eos,
                                                        float logzero, float* __restrict__ psi_out,
                                                        float* __restrict__ r_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * C) return;
    const int n = i / C;
    const int ci = cand[i];
    const int plen = prefix_len[n];
    const bool same = plen > 0 && ci == last_char[n];
    const float* rp = r_prev + (size_t)n * T * 2;
    float* ro = r_out + (size_t)i * T * 2;
    const int start = plen > 1 ? plen : 1;
    float r0 = logzero, r1 = logzero;
    if (plen == 0) r0 = x[ci];                              // g = <sos>: r[0,0,c] = x[0,c]
    for (int t = 0; t < start && t < T; ++t) {
        ro[2 * t] = (t == 0) ? r0 : logzero;
        ro[2 * t + 1] = logzero;
    }
    // r[start-1] as the recursion sees it (everything before `start` except r[0,0] of the empty prefix is log-zero)
    float q0 = (start - 1 == 0) ? r0 : logzero, q1 = logzero;
    float psi = q0;
    for (int t = start; t < T; ++t) {
        const float p0 = rp[2 * (t - 1)], p1 = rp[2 * (t - 1) + 1];
        const float phi = same ? p1 : np_logaddexp(p0, p1);
        const float xc = x[(size_t)t * V + ci], xb = x[(size_t)t * V + blank];
        const float n0 = np_logaddexp(q0, phi) + xc;
        const float n1 = np_logaddexp(q1, q0) + xb;
        psi = np_logaddexp(psi, phi + xc);
        q0 = n0;
        q1 = n1;
        ro[2 * t] = q0;
        ro[2 * t + 1] = q1;
    }
    if (ci == eos) psi = np_logaddexp(rp[2 * (T - 1)], rp[2 * (T - 1) + 1]);   // P(<eos> | g) = P(g)
    psi_out[i] = psi;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" int b200asr_ctc_prefix_score(const float* log_probs, int T, int V, const float* r_prev, const int* last_char,
                                        const int* prefix_len, const int* candidates, int N, int C, int blank, int eos,
                                        float* psi, float* r_out, b200asr_stream stream) {
    B200_REQUIRE(log_probs && r_prev && last_char && prefix_len && candidates && psi && r_out,
                 "ctc_prefix_score: null pointer");
    B200_REQUIRE(T > 0 && V > 0 && N > 0 && C > 0, "ctc_prefix_score: bad sizes T=%d V=%d N=%d C=%d", T, V, N, C);
    B200_REQUIRE(blank >= 0 && blank < V && eos >= -1 && eos < V, "ctc_prefix_score: blank/eos outside [0,%d)", V);
    const int total = N * C;
    ctc_prefix_kernel<<<(total + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
        log_probs, T, V, r_prev, last_char, prefix_len, candidates, N, C, blank, eos, -100000000.0f, psi, r_out);
    B200_LAUNCH_CHECK("ctc_prefix_kernel");
    return B200_OK;
}
