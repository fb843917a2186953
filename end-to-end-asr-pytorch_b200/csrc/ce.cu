// K15: fused log-softmax + NLL (ignore_index) forward and logit gradient in one launch.
// Restates torch.nn.CrossEntropyLoss(ignore_index=0) at /root/reference/bin/train_asr.py:47,127-131:
// loss = mean over non-ignored rows of (lse(x) - x[target]); d loss / d x = (softmax(x) - onehot) / n_valid.
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {

__global__ void __launch_bounds__(256) ce_fwd_bwd_kernel(const float* __restrict__ x, const long long* __restrict__ tgt,
                                                        long long ignore_index, long long N, int V,
                                                        const float* __restrict__ grad_scale,
                                                        float* __restrict__ row_loss, float* __restrict__ dx) {
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= N) return;
    const float* xr = x + row * V;
    const long long t = tgt[row];
    if (t == ignore_index || t < 0 || t >= V) {
        if (lane == 0) row_loss[row] = 0.f;
        if (dx)
            for (int c = lane; c < V; c += 32) dx[row * V + c] = 0.f;
        return;
    }
    float m = NEG_INF, s = 0.f;
    for (int c = lane; c < V; c += 32) {
        const float v = xr[c];
        if (v > m) {
            s = s * expf(m - v) + 1.f;
            m = v;
        } else if (v != NEG_INF) {          // -inf adds 0; with m = -inf too, exp(-inf - -inf) would be NaN
            s += expf(v - m);
        }
    }
    const float M = warp_max(m);
    // a lane whose only finite-or-NaN values were NaN keeps m = -inf and s = NaN: s * 0 carries that NaN into S
    const float S = warp_sum(s * ((m == NEG_INF) ? 0.f : expf(m - M)));
    const float lse = M + logf(S);
    if (lane == 0) row_loss[row] = lse - xr[t];
    if (dx) {
        const float sc = grad_scale ? *grad_scale : 1.f;
        for (int c = lane; c < V; c += 32) {
            float p = expf(xr[c] - lse);
            if (c == (int)t) p -= 1.f;
            dx[row * V + c] = p * sc;
        }
    }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" int b200asr_ce_fwd_bwd(const float* logits, const long long* target, long long ignore_index,
                                  long long n_rows, int V, const float* grad_scale, float* row_loss, float* dlogits,
                                  b200asr_stream stream) {
    B200_REQUIRE(logits && target && row_loss, "ce_fwd_bwd: null pointer");
    B200_REQUIRE(n_rows >= 0 && V > 0, "ce_fwd_bwd: bad sizes");
    if (n_rows == 0) return B200_OK;
    const int wpb = 8;
    const long long blocks = (n_rows + wpb - 1) / wpb;
    ce_fwd_bwd_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(logits, target, ignore_index, n_rows, V,
                                                                              grad_scale, row_loss, dlogits);
    B200_LAUNCH_CHECK("ce_fwd_bwd_kernel");
    return B200_OK;
}
