// K13g: one GRU cell step of the decoder (src/asr.py:214-221 with module: 'GRU'), forward and backward.
//
// The step GEMM (ops.decoder_step) delivers per row b the pre-activations in the layout
//   pre[b, 0:2H]  = gi_rz + gh_rz     (r and z, input and hidden products summed)
//   pre[b, 2H:3H] = gi_n              (x . W_in^T + b_in)
//   pre[b, 3H:4H] = gh_n              (h . W_hn^T + b_hn)
// because n needs gh_n alone: n = tanh(gi_n + r * gh_n).  The pointwise part follows ATen's GRUCell expression order
// (aten/src/ATen/native/RNN.cpp): the products and sums are rounded separately (no FMA contraction), and
// h' = (h - n) * z + n.  One thread per (b, j); the activated gates (r, z, n, gh_n) are stashed for the backward.
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {

__global__ void gru_cell_fwd_kernel(const float* __restrict__ pre, const float* __restrict__ h_prev,
                                    float* __restrict__ gates, float* __restrict__ h, int B, int H) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H) return;
    const int b = i / H, j = i - b * H;
    const float* pr = pre + (size_t)b * 4 * H;
    const float r = sigmoidf_(pr[j]), z = sigmoidf_(pr[H + j]);
    const float ghn = pr[3 * H + j];
    const float n = tanhf(__fadd_rn(pr[2 * H + j], __fmul_rn(ghn, r)));
    float* gr = gates + (size_t)b * 4 * H;
    gr[j] = r; gr[H + j] = z; gr[2 * H + j] = n; gr[3 * H + j] = ghn;
    h[i] = __fadd_rn(__fmul_rn(__fsub_rn(h_prev[i], n), z), n);
}

// dh may be NULL (h' does not reach the loss): every output is then 0 except where a gate is NaN.  A saturated gate
// (r, z in {0, 1}, n = +-1) gives exactly 0 through its derivative factor.
__global__ void gru_cell_bwd_kernel(const float* __restrict__ gates, const float* __restrict__ h_prev,
                                    const float* __restrict__ dh, float* __restrict__ dpre,
                                    float* __restrict__ dh_prev, int B, int H) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H) return;
    const int b = i / H, j = i - b * H;
    const float* gr = gates + (size_t)b * 4 * H;
    const float r = gr[j], z = gr[H + j], n = gr[2 * H + j], ghn = gr[3 * H + j];
    const float dhv = dh ? dh[i] : 0.f;
    const float dn = dhv * (1.f - z);
    const float dgin = dn * (1.f - n * n);
    float* dp = dpre + (size_t)b * 4 * H;
    dp[j] = dgin * ghn * r * (1.f - r);
    dp[H + j] = dhv * (h_prev[i] - n) * z * (1.f - z);
    dp[2 * H + j] = dgin;
    dp[3 * H + j] = dgin * r;
    dh_prev[i] = dhv * z;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" int b200asr_gru_cell_fwd(const float* preact, const float* h_prev, float* gates, float* h, int B, int H,
                                    b200asr_stream stream) {
    B200_REQUIRE(preact && h_prev && gates && h, "gru_cell_fwd: null pointer");
    B200_REQUIRE(B > 0 && H > 0 && (long long)B * H <= 0x7fffffff, "gru_cell_fwd: bad sizes");
    const int n = B * H;
    gru_cell_fwd_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(preact, h_prev, gates, h, B, H);
    B200_LAUNCH_CHECK("gru_cell_fwd_kernel");
    return B200_OK;
}

extern "C" int b200asr_gru_cell_bwd(const float* gates, const float* h_prev, const float* dh, float* dpreact,
                                    float* dh_prev, int B, int H, b200asr_stream stream) {
    B200_REQUIRE(gates && h_prev && dpreact && dh_prev, "gru_cell_bwd: null pointer");
    B200_REQUIRE(B > 0 && H > 0 && (long long)B * H <= 0x7fffffff, "gru_cell_bwd: bad sizes");
    const int n = B * H;
    gru_cell_bwd_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(gates, h_prev, dh, dpreact, dh_prev, B, H);
    B200_LAUNCH_CHECK("gru_cell_bwd_kernel");
    return B200_OK;
}
