// K9 (log-softmax half) + K10: CTC loss forward (alpha) and backward (beta, gradient) in one call.
//
//   log_softmax_fwd_kernel : one warp per row, online max/sum, writes log-probs (+ lse, argmax)
//   log_softmax_bwd_kernel : dlogits = g - exp(lp) * sum_c g
//   ctc_alpha_beta_warp_kernel : WARP-SYNCHRONOUS alpha/beta: one warp per (utterance, direction) - alpha and
//                            beta of an utterance run concurrently (they are independent) - each lane keeps R
//                            consecutive extended-label positions in registers, neighbours via warp shuffles,
//                            no barrier in the T-long chain; lattice rows stream to HBM for the gradient pass
//   ctc_alpha_beta_kernel  : block-per-(utterance, direction) variant (one thread per position, lattice row in
//                            shared memory) used for long targets (more than 63 labels), where it is faster
//   ctc_grad_kernel        : grid (T-chunks, B): per (b,t) row combines alpha+beta per class with a
//                            deterministic occurrence-chain sum and streams the V-wide gradient row
//
// Semantics restated from the reference call site bin/train_asr.py:49,123-124
// (torch.nn.CTCLoss(blank=0, zero_infinity=False) -> ATen _ctc_loss/_ctc_loss_backward; Graves 2006
// eq. 6-8, 10-11, 16) incl. the ATen convention that the returned "log_probs" gradient is
// exp(lp) - exp(log sum(alpha*beta) + nll - lp)  (SURVEY.md F9).
#include "common.cuh"
#include "../../include/b200asr.h"

namespace b200asr {

// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) log_softmax_fwd_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                             float* __restrict__ lse, long long* __restrict__ amax,
                                                             long long N, int V) {
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= N) return;
    const float* xr = x + row * V;
    float m = NEG_INF, s = 0.f;
    int mi = 0x7fffffff;
    if ((V & 3) == 0 && (reinterpret_cast<uintptr_t>(xr) & 15) == 0) {
        // 128-bit streaming, two independent loads in flight per lane, ONE rescale per 8 values (the running (max, sum)
        // pair is the only loop-carried dependency); the first index wins ties like torch.argmax
        const float4* x4 = reinterpret_cast<const float4*>(xr);
        const int n4 = V >> 2;
        for (int c = lane; c < n4; c += 64) {
            const float4 a = x4[c];
            const bool two = c + 32 < n4;
            const float4 b = two ? x4[c + 32] : make_float4(NEG_INF, NEG_INF, NEG_INF, NEG_INF);
            float bm = a.x;
            int bi = 4 * c;
            if (a.y > bm) { bm = a.y; bi = 4 * c + 1; }
            if (a.z > bm) { bm = a.z; bi = 4 * c + 2; }
            if (a.w > bm) { bm = a.w; bi = 4 * c + 3; }
            if (b.x > bm) { bm = b.x; bi = 4 * (c + 32); }
            if (b.y > bm) { bm = b.y; bi = 4 * (c + 32) + 1; }
            if (b.z > bm) { bm = b.z; bi = 4 * (c + 32) + 2; }
            if (b.w > bm) { bm = b.w; bi = 4 * (c + 32) + 3; }
            if (bm > m) {
                s *= expf(m - bm);          // m = -inf: s = 0 -> 0 * exp(-inf) = 0
                m = bm;
                mi = bi;
            }
            if (m != NEG_INF) {
                s += (expf(a.x - m) + expf(a.y - m)) + (expf(a.z - m) + expf(a.w - m));
                if (two) s += (expf(b.x - m) + expf(b.y - m)) + (expf(b.z - m) + expf(b.w - m));
            }
        }
    } else {
        for (int c = lane; c < V; c += 32) {
            const float v = xr[c];
            if (v > m) {
                s = s * expf(m - v) + 1.f;  // m=-inf: s=0 -> 0*exp(-inf)=0
                m = v;
                mi = c;
            } else {
                s += expf(v - m);
            }
        }
    }
    // warp combine (first index wins ties)
    float M = m;
    int MI = mi;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, M, o);
        const int oi = __shfl_xor_sync(0xffffffffu, MI, o);
        if (om > M || (om == M && oi < MI)) {
            M = om;
            MI = oi;
        }
    }
    const float part = (m == NEG_INF) ? 0.f : s * expf(m - M);
    const float S = warp_sum(part);
    const float L = M + logf(S);
    if (y == nullptr) {
        // statistics only (fused CTC head): the log-probs are never materialised
    } else if ((V & 3) == 0) {
        const float4* x4 = reinterpret_cast<const float4*>(xr);
        float4* y4 = reinterpret_cast<float4*>(y + row * V);
        for (int c = lane; c < (V >> 2); c += 32) {
            float4 v = x4[c];
            v.x -= L; v.y -= L; v.z -= L; v.w -= L;
            y4[c] = v;
        }
    } else {
        for (int c = lane; c < V; c += 32) y[row * V + c] = xr[c] - L;
    }
    if (lane == 0) {
        if (lse) lse[row] = L;
        if (amax) amax[row] = MI;
    }
}

__global__ void __launch_bounds__(256) log_softmax_bwd_kernel(const float* __restrict__ lp, const float* __restrict__ g,
                                                             float* __restrict__ dx, long long N, int V) {
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= N) return;
    const float* gr = g + row * V;
    const float* lr = lp + row * V;
    float s = 0.f;
    if ((V & 3) == 0) {
        const float4* g4 = reinterpret_cast<const float4*>(gr);
        const float4* l4 = reinterpret_cast<const float4*>(lr);
        float4* d4 = reinterpret_cast<float4*>(dx + row * V);
        for (int c = lane; c < (V >> 2); c += 32) {
            const float4 v = g4[c];
            s += (v.x + v.y) + (v.z + v.w);
        }
        s = warp_sum(s);
        for (int c = lane; c < (V >> 2); c += 32) {
            const float4 v = g4[c], l = l4[c];
            d4[c] = make_float4(v.x - expf(l.x) * s, v.y - expf(l.y) * s, v.z - expf(l.z) * s, v.w - expf(l.w) * s);
        }
        return;
    }
    for (int c = lane; c < V; c += 32) s += gr[c];
    s = warp_sum(s);
    for (int c = lane; c < V; c += 32) dx[row * V + c] = gr[c] - expf(lr[c]) * s;
}

// ------------------------------------------------------------------------------------------
struct CtcParams {
    const float* lp;     // log-probs, element (b,t,c) at lp[b*sb + t*st + c]
    const float* lse;    // [B,T] or null.  Non-null: `lp` holds LOGITS and log-prob(b,t,c) = lp[...] - lse[b*T + t]
                         // (the log-softmax of the CTC head fused into the loss: its V-wide output is never written)
    long long sb, st;
    const long long* targets;  // [B, L_max]
    const long long* in_len;   // [B]
    const long long* tgt_len;  // [B]
    int B, T, V, L_max, S_max, blank;
    float* nll;          // [B]
    const float* scale;  // [B] or null
    const float* upstream;  // device scalar multiplied into every gradient element (d total / d loss), or null
    float* grad;         // same strides as lp, or null
    float* alpha;        // [B,T,S_max]
    float* beta;         // [B,T,S_max]
    int* prev_same;      // [B,S_max]
    int* is_last;        // [B,S_max]
};

__device__ __forceinline__ float lse3(float a, float b, float c) {
    float m = fmaxf(a, fmaxf(b, c));
    if (m == NEG_INF) return NEG_INF;
    return logf(expf(a - m) + expf(b - m) + expf(c - m)) + m;
}

// 4-byte asynchronous global -> shared copies, tracked by commit groups (cp.async.wait_group) instead of register scoreboards
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
constexpr int CTC_PD = 8;                    // frames of emission look-ahead in the warp kernel

__global__ void __launch_bounds__(1024) ctc_alpha_beta_kernel(CtcParams p) {
    extern __shared__ float s_dyn[];
    const int S_max = p.S_max;
    float* buf0 = s_dyn;
    float* buf1 = s_dyn + S_max;
    int* lab = reinterpret_cast<int*>(s_dyn + 2 * S_max);
    int* skip = lab + S_max;

    const int b = blockIdx.x;
    const bool is_beta = blockIdx.y == 1;
    long long Tb64 = p.in_len[b];
    long long Lb64 = p.tgt_len[b];
    const int Tb = (int)(Tb64 < 0 ? 0 : (Tb64 > p.T ? p.T : Tb64));
    const int Lb = (int)(Lb64 < 0 ? 0 : (Lb64 > p.L_max ? p.L_max : Lb64));
    const int Sb = 2 * Lb + 1;
    const float* lpb = p.lp + (long long)b * p.sb;
    float* lat = (is_beta ? p.beta : p.alpha) + (long long)b * p.T * S_max;

    for (int s = threadIdx.x; s < S_max; s += blockDim.x) {
        int l = -1;
        if (s < Sb) {
            l = (s & 1) ? (int)p.targets[(long long)b * p.L_max + (s >> 1)] : p.blank;
            l = l < 0 ? 0 : (l >= p.V ? p.V - 1 : l);      // never index outside the row (torch raises on such input)
        }
        lab[s] = l;
    }
    __syncthreads();
    for (int s = threadIdx.x; s < S_max; s += blockDim.x) {
        int sk = 0;
        if (!is_beta) {
            if (s >= 2 && s < Sb && lab[s] != p.blank && lab[s] != lab[s - 2]) sk = 1;
        } else {
            if (s + 2 < Sb && lab[s + 2] != p.blank && lab[s + 2] != lab[s]) sk = 1;
        }
        skip[s] = sk;
        if (!is_beta) {
            // occurrence chains of equal labels (consumed by ctc_grad_kernel)
            int prev = -1, last = 0;
            if ((s & 1) && s < Sb) {
                const int l = lab[s];
                for (int q = s - 2; q >= 1; q -= 2)
                    if (lab[q] == l) { prev = q; break; }
                last = 1;
                for (int q = s + 2; q < Sb; q += 2)
                    if (lab[q] == l) { last = 0; break; }
            }
            p.prev_same[(long long)b * S_max + s] = prev;
            p.is_last[(long long)b * S_max + s] = last;
        }
    }
    __syncthreads();

    if (Tb == 0) {
        if (!is_beta && threadIdx.x == 0) p.nll[b] = (Lb == 0) ? 0.f : INFINITY;
        return;
    }

    float* prev = buf0;
    float* cur = buf1;
    const int t0 = is_beta ? Tb - 1 : 0;
    const int dt = is_beta ? -1 : 1;
    // boundary row
    {
        const float* lpt = lpb + (long long)t0 * p.st;
        const float ls = p.lse ? p.lse[(long long)b * p.T + t0] : 0.f;
        for (int s = threadIdx.x; s < S_max; s += blockDim.x) {
            float a = NEG_INF;
            if (!is_beta) {
                if (s == 0) a = lpt[p.blank] - ls;
                else if (s == 1 && Sb > 1) a = lpt[lab[1]] - ls;
            } else {
                if (s == Sb - 1) a = lpt[p.blank] - ls;
                else if (s == Sb - 2 && Sb > 1) a = lpt[lab[Sb - 2]] - ls;
            }
            prev[s] = a;
            lat[(long long)t0 * S_max + s] = a;
        }
    }
    if (S_max <= (int)blockDim.x) {
        // one lattice position per thread (every target shorter than 512 labels): the emission gathers run PD frames
        // ahead in a register ring, off the T-long dependency chain.  The ring holds the RAW loads (logit and row lse);
        // the subtraction happens at the consumer - an FADD next to the load makes the warp wait for the gather right
        // there.  (The cp.async ring of the warp kernel would need a block barrier per frame here.)
        constexpr int PD = 4;
        const int s = threadIdx.x;
        const bool act = s < Sb;
        const int l = act ? lab[s] : 0;
        const int sk = (s < S_max) ? skip[s] : 0;
        const float* lseb = p.lse ? p.lse + (long long)b * p.T : nullptr;
        float eq[PD], lq[PD];
#pragma unroll
        for (int d = 0; d < PD; ++d) {
            const int st = 1 + d;
            eq[d] = 0.f;
            lq[d] = 0.f;
            if (st < Tb && act) {
                eq[d] = lpb[(long long)(t0 + dt * st) * p.st + l];
                if (lseb) lq[d] = lseb[t0 + dt * st];
            }
        }
        for (int base = 1; base < Tb; base += PD) {
#pragma unroll
            for (int d = 0; d < PD; ++d) {
                const int step = base + d;
                if (step >= Tb) break;                       // block-uniform
                const int t = t0 + dt * step;
                const float e = eq[d] - lq[d];
                if (step + PD < Tb && act) {
                    eq[d] = lpb[(long long)(t + dt * PD) * p.st + l];
                    if (lseb) lq[d] = lseb[t + dt * PD];
                }
                __syncthreads();  // prev fully written
                if (s < S_max) {
                    float v = NEG_INF;
                    if (act) {
                        float a0 = prev[s], a1, a2;
                        if (!is_beta) {
                            a1 = (s > 0) ? prev[s - 1] : NEG_INF;
                            a2 = sk ? prev[s - 2] : NEG_INF;
                        } else {
                            a1 = (s + 1 < Sb) ? prev[s + 1] : NEG_INF;
                            a2 = sk ? prev[s + 2] : NEG_INF;
                        }
                        v = lse3(a0, a1, a2) + e;
                    }
                    cur[s] = v;
                    lat[(long long)t * S_max + s] = v;
                }
                float* tmp = prev; prev = cur; cur = tmp;
            }
        }
    } else
    for (int step = 1; step < Tb; ++step) {
        const int t = t0 + dt * step;
        const float* lpt = lpb + (long long)t * p.st;
        const float ls = p.lse ? p.lse[(long long)b * p.T + t] : 0.f;
        __syncthreads();  // prev fully written
        for (int s = threadIdx.x; s < S_max; s += blockDim.x) {
            float v = NEG_INF;
            if (s < Sb) {
                const float e = lpt[lab[s]] - ls;
                float a0 = prev[s], a1, a2;
                if (!is_beta) {
                    a1 = (s > 0) ? prev[s - 1] : NEG_INF;
                    a2 = skip[s] ? prev[s - 2] : NEG_INF;
                } else {
                    a1 = (s + 1 < Sb) ? prev[s + 1] : NEG_INF;
                    a2 = skip[s] ? prev[s + 2] : NEG_INF;
                }
                v = lse3(a0, a1, a2) + e;
            }
            cur[s] = v;
            lat[(long long)t * S_max + s] = v;
        }
        float* tmp = prev; prev = cur; cur = tmp;
    }
    if (!is_beta) {
        __syncthreads();
        if (threadIdx.x == 0) {
            const float l1 = prev[Sb - 1];
            const float l2 = (Sb > 1) ? prev[Sb - 2] : NEG_INF;
            const float m = fmaxf(l1, l2);
            const float ll = (m == NEG_INF) ? NEG_INF : logf(expf(l1 - m) + expf(l2 - m)) + m;
            p.nll[b] = -ll;
        }
    }
}

// ------------------------------------------------------------------------------------------
// Warp-synchronous alpha/beta: one WARP per (utterance, direction); lane l keeps the R consecutive extended-label
// positions s = l*R .. l*R+R-1 of the current lattice row in registers, the two neighbours that live in the adjacent
// lane come through one pair of warp shuffles per frame, and there is no block barrier and no shared-memory lattice
// in the T-long dependency chain.  The emission gathers of frame t+1 are issued before the update of frame t.
constexpr int CTC_WARPS = 4;

template <int R>
__global__ void __launch_bounds__(CTC_WARPS * 32) ctc_alpha_beta_warp_kernel(CtcParams p) {
    extern __shared__ float s_dyn[];                     // per warp: labels[S_max] (int) + last row [S_max]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int item = blockIdx.x * CTC_WARPS + warp;      // (b, direction)
    if (item >= 2 * p.B) return;
    const int b = item >> 1;
    const bool is_beta = item & 1;
    const int S_max = p.S_max;
    int* lab_s = reinterpret_cast<int*>(s_dyn) + (size_t)warp * 2 * S_max;
    float* row_s = reinterpret_cast<float*>(lab_s + S_max);
    constexpr int SLOT = (R + 1) * 32;                   // one frame of the look-ahead ring: [r][lane] logits + [lane] row lse
    float* ring = s_dyn + (size_t)CTC_WARPS * 2 * S_max + (size_t)warp * CTC_PD * SLOT;

    long long Tb64 = p.in_len[b];
    long long Lb64 = p.tgt_len[b];
    const int Tb = (int)(Tb64 < 0 ? 0 : (Tb64 > p.T ? p.T : Tb64));
    const int Lb = (int)(Lb64 < 0 ? 0 : (Lb64 > p.L_max ? p.L_max : Lb64));
    const int Sb = 2 * Lb + 1;
    const float* lpb = p.lp + (long long)b * p.sb;
    float* lat = (is_beta ? p.beta : p.alpha) + (long long)b * p.T * S_max;

    int lab[R];
    bool in_range[R], skip[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int s = lane * R + r;
        in_range[r] = s < Sb;
        lab[r] = (in_range[r] && (s & 1)) ? (int)p.targets[(long long)b * p.L_max + (s >> 1)] : p.blank;
        lab[r] = lab[r] < 0 ? 0 : (lab[r] >= p.V ? p.V - 1 : lab[r]);   // never index outside the row
        if (s < S_max) lab_s[s] = in_range[r] ? lab[r] : -1;
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int s = lane * R + r;
        skip[r] = false;
        if (!is_beta) {
            if (s >= 2 && s < Sb && lab[r] != p.blank && lab[r] != lab_s[s - 2]) skip[r] = true;
        } else {
            if (s + 2 < Sb && lab_s[s + 2] != p.blank && lab_s[s + 2] != lab[r]) skip[r] = true;
        }
        if (!is_beta && s < S_max) {
            // occurrence chains of equal labels (consumed by ctc_grad_kernel)
            int prev = -1, last = 0;
            if ((s & 1) && s < Sb) {
                for (int q = s - 2; q >= 1; q -= 2)
                    if (lab_s[q] == lab[r]) { prev = q; break; }
                last = 1;
                for (int q = s + 2; q < Sb; q += 2)
                    if (lab_s[q] == lab[r]) { last = 0; break; }
            }
            p.prev_same[(long long)b * S_max + s] = prev;
            p.is_last[(long long)b * S_max + s] = last;
        }
    }
    if (Tb == 0) {
        if (!is_beta && lane == 0) p.nll[b] = (Lb == 0) ? 0.f : INFINITY;
        return;
    }
    const int t0 = is_beta ? Tb - 1 : 0;
    const int dt = is_beta ? -1 : 1;
    // The emission gathers x[t, label] are independent of the recursion: they run CTC_PD frames ahead as cp.async copies
    // into a per-warp shared-memory ring, one commit group per frame; every lane reads back only what it copied itself.
    // (A register ring with the "- lse" next to the load stalls the FADD on the load it follows.)  What is left is the
    // recursion itself: ~300 dependent instructions per frame in a single warp.
    float a[R];
    const float* lseb = p.lse ? p.lse + (long long)b * p.T : nullptr;
    auto prefetch = [&](int st) {                        // frame t0 + dt * st -> ring slot st % CTC_PD
        if (st < Tb) {
            const float* lpn = lpb + (long long)(t0 + dt * st) * p.st;
            float* sl = ring + (st % CTC_PD) * SLOT;
#pragma unroll
            for (int r = 0; r < R; ++r) cp_async4(sl + r * 32 + lane, lpn + lab[r]);
            if (lseb) cp_async4(sl + R * 32 + lane, lseb + t0 + dt * st);
        }
        cp_async_commit();                               // (possibly empty) group: the group count stays one per frame
    };
    {   // boundary row
        const float* lpt = lpb + (long long)t0 * p.st;
        const float ls = lseb ? lseb[t0] : 0.f;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int s = lane * R + r;
            float v = NEG_INF;
            if (!is_beta) {
                if (s == 0) v = lpt[p.blank] - ls;
                else if (s == 1 && Sb > 1) v = lpt[lab[r]] - ls;
            } else {
                if (s == Sb - 1) v = lpt[p.blank] - ls;
                else if (s == Sb - 2 && Sb > 1) v = lpt[lab[r]] - ls;
            }
            a[r] = v;
            if (s < S_max) lat[(long long)t0 * S_max + s] = v;
        }
        for (int st = 1; st <= CTC_PD; ++st) prefetch(st);
    }
    for (int step = 1; step < Tb; ++step) {
        {
            const int t = t0 + dt * step;
            cp_async_wait<CTC_PD - 1>();                 // groups 1 .. step have landed
            float e[R];
            {
                const float* sl = ring + (step % CTC_PD) * SLOT;
                const float ls = lseb ? sl[R * 32 + lane] : 0.f;
#pragma unroll
                for (int r = 0; r < R; ++r) e[r] = sl[r * 32 + lane] - ls;
            }
            prefetch(step + CTC_PD);                     // refill the slot just read
            // neighbours across the lane boundary
            float n1, n2;
            if (!is_beta) {
                n1 = __shfl_up_sync(0xffffffffu, a[R - 1], 1);
                n2 = __shfl_up_sync(0xffffffffu, a[R >= 2 ? R - 2 : 0], 1);
                if (R == 1) n2 = __shfl_up_sync(0xffffffffu, a[0], 2);
                if (lane == 0) { n1 = NEG_INF; n2 = NEG_INF; }
                if (R == 1 && lane == 1) n2 = NEG_INF;
            } else {
                n1 = __shfl_down_sync(0xffffffffu, a[0], 1);
                n2 = __shfl_down_sync(0xffffffffu, a[R >= 2 ? 1 : 0], 1);
                if (R == 1) n2 = __shfl_down_sync(0xffffffffu, a[0], 2);
                if (lane == 31) { n1 = NEG_INF; n2 = NEG_INF; }
                if (R == 1 && lane == 30) n2 = NEG_INF;
            }
            float nw[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                float a1, a2;
                if (!is_beta) {
                    a1 = (r >= 1) ? a[r >= 1 ? r - 1 : 0] : n1;
                    a2 = (r >= 2) ? a[r >= 2 ? r - 2 : 0] : (r == 1 ? n1 : n2);
                } else {
                    a1 = (r + 1 < R) ? a[r + 1 < R ? r + 1 : 0] : n1;
                    a2 = (r + 2 < R) ? a[r + 2 < R ? r + 2 : 0] : (r + 1 < R ? n1 : n2);
                }
                if (!skip[r]) a2 = NEG_INF;
                nw[r] = in_range[r] ? lse3(a[r], a1, a2) + e[r] : NEG_INF;
            }
#pragma unroll
            for (int r = 0; r < R; ++r) {
                a[r] = nw[r];
                const int s = lane * R + r;
                if (s < S_max) lat[(long long)t * S_max + s] = nw[r];
            }
        }
    }
    if (!is_beta) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int s = lane * R + r;
            if (s < S_max) row_s[s] = a[r];
        }
        __syncwarp();
        if (lane == 0) {
            const float l1 = row_s[Sb - 1];
            const float l2 = (Sb > 1) ? row_s[Sb - 2] : NEG_INF;
            const float m = fmaxf(l1, l2);
            const float ll = (m == NEG_INF) ? NEG_INF : logf(expf(l1 - m) + expf(l2 - m)) + m;
            p.nll[b] = -ll;
        }
    }
}

template <int R>
static int launch_ctc_warp(const CtcParams& p, cudaStream_t stream) {
    const int items = 2 * p.B;
    const size_t smem = (size_t)CTC_WARPS * (2 * p.S_max + CTC_PD * (R + 1) * 32) * sizeof(float);
    ctc_alpha_beta_warp_kernel<R><<<(items + CTC_WARPS - 1) / CTC_WARPS, CTC_WARPS * 32, smem, stream>>>(p);
    return 0;
}

constexpr int CTC_GRAD_THREADS = 256;
constexpr int CTC_GRAD_TCHUNK = 8;

__global__ void __launch_bounds__(CTC_GRAD_THREADS, 8) ctc_grad_kernel(CtcParams p) {
    // grid (T chunks, B).  Phase 1 streams the dense part  g = exp(lp) * scale  of every row of the chunk (pure
    // 128-bit streaming, no barrier); phase 2 subtracts the label-occupancy term at the <= L+1 distinct classes of the
    // utterance (deterministic occurrence-chain sums, one owner thread per class, no atomics).
    extern __shared__ __align__(16) float s_dyn[];
    const int S_max = p.S_max, V = p.V;
    float* e = s_dyn;               // [warps][S_max]
    int* lab = reinterpret_cast<int*>(e + (size_t)(CTC_GRAD_THREADS / 32) * S_max);
    int* prev_same = lab + S_max;
    int* is_last = prev_same + S_max;

    const int b = blockIdx.y;
    long long Tb64 = p.in_len[b];
    long long Lb64 = p.tgt_len[b];
    const int Tb = (int)(Tb64 < 0 ? 0 : (Tb64 > p.T ? p.T : Tb64));
    const int Lb = (int)(Lb64 < 0 ? 0 : (Lb64 > p.L_max ? p.L_max : Lb64));
    const int Sb = 2 * Lb + 1;
    const float nll = p.nll[b];
    const float scale = (p.scale ? p.scale[b] : 1.f) * (p.upstream ? *p.upstream : 1.f);
    const bool vec4 = ((V & 3) == 0) && ((p.sb & 3) == 0) && ((p.st & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(p.lp) | reinterpret_cast<uintptr_t>(p.grad)) & 15) == 0;

    for (int s = threadIdx.x; s < S_max; s += blockDim.x) {
        int l = -1;
        if (s < Sb) {
            l = (s & 1) ? (int)p.targets[(long long)b * p.L_max + (s >> 1)] : p.blank;
            l = l < 0 ? 0 : (l >= V ? V - 1 : l);     // same clamp as the lattice kernels (torch raises on such input)
        }
        lab[s] = l;
        prev_same[s] = p.prev_same[(long long)b * S_max + s];
        is_last[s] = p.is_last[(long long)b * S_max + s];
    }

    const int t_begin = blockIdx.x * CTC_GRAD_TCHUNK;
    const int t_end = min(p.T, t_begin + CTC_GRAD_TCHUNK);
    // ---- phase 1: dense stream.  The chunk's rows are one flat index space, two 128-bit loads in flight per thread
    // at 8 resident blocks per SM (the register budget of __launch_bounds__(256, 8): occupancy is what hides phase 2)
    if (vec4) {
        const int n4 = V >> 2, total = (t_end - t_begin) * n4;
        const float* lp0 = p.lp + (long long)b * p.sb;
        float* g0 = p.grad + (long long)b * p.sb;
        const float* lse0 = p.lse ? p.lse + (long long)b * p.T : nullptr;
        for (int i0 = threadIdx.x; i0 < total; i0 += 2 * CTC_GRAD_THREADS) {
            const int i1 = i0 + CTC_GRAD_THREADS;
            const int r0 = i0 / n4, r1 = i1 / n4;
            const long long o0 = (long long)(t_begin + r0) * p.st + 4 * (i0 - r0 * n4);
            const long long o1 = (long long)(t_begin + r1) * p.st + 4 * (i1 - r1 * n4);
            const bool live0 = t_begin + r0 < Tb, live1 = i1 < total && t_begin + r1 < Tb;
            float4 l0 = make_float4(0.f, 0.f, 0.f, 0.f), l1 = l0;
            float ls0 = 0.f, ls1 = 0.f;
            if (live0) l0 = __ldcs(reinterpret_cast<const float4*>(lp0 + o0));
            if (live1) l1 = __ldcs(reinterpret_cast<const float4*>(lp0 + o1));
            if (lse0 && live0) ls0 = lse0[t_begin + r0];
            if (lse0 && live1) ls1 = lse0[t_begin + r1];
            const float s0 = live0 ? scale : 0.f, s1 = live1 ? scale : 0.f;
            *reinterpret_cast<float4*>(g0 + o0) =
                make_float4(expf(l0.x - ls0) * s0, expf(l0.y - ls0) * s0, expf(l0.z - ls0) * s0, expf(l0.w - ls0) * s0);
            if (i1 < total)
                *reinterpret_cast<float4*>(g0 + o1) =
                    make_float4(expf(l1.x - ls1) * s1, expf(l1.y - ls1) * s1, expf(l1.z - ls1) * s1, expf(l1.w - ls1) * s1);
        }
    } else {
        for (int t = t_begin; t < t_end; ++t) {
            float* gt = p.grad + (long long)b * p.sb + (long long)t * p.st;
            const float* lpt = p.lp + (long long)b * p.sb + (long long)t * p.st;
            const bool live = t < Tb;
            const float ls = (p.lse && live) ? p.lse[(long long)b * p.T + t] : 0.f;
            for (int c = threadIdx.x; c < V; c += blockDim.x) gt[c] = live ? expf(lpt[c] - ls) * scale : 0.f;
        }
    }
    __syncthreads();
    // ---- phase 2: occupancy of the utterance's own classes.  One WARP per frame of the chunk (warp-synchronous: the
    // block-wide version spent its time in ~10 barriers per frame, which the other resident blocks had to cover)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* ew = e + (size_t)warp * S_max;
    for (int t = t_begin + warp; t < t_end && t < Tb; t += CTC_GRAD_THREADS / 32) {
        float* gt = p.grad + (long long)b * p.sb + (long long)t * p.st;
        const float* lpt = p.lp + (long long)b * p.sb + (long long)t * p.st;
        const float* al = p.alpha + ((long long)b * p.T + t) * S_max;
        const float* be = p.beta + ((long long)b * p.T + t) * S_max;
        const float ls = p.lse ? p.lse[(long long)b * p.T + t] : 0.f;
        float mx = NEG_INF;
        for (int s = lane; s < Sb; s += 32) {
            const float v = al[s] + be[s];
            ew[s] = v;
            mx = fmaxf(mx, v);
        }
        const float m = warp_max(mx);
        for (int s = lane; s < Sb; s += 32) {
            const float v = ew[s];
            ew[s] = (v == NEG_INF) ? 0.f : expf(v - m);
        }
        __syncwarp();
        // blank (even s): fixed-order per-lane partials + fixed shuffle tree
        float part = 0.f;
        for (int s = 2 * lane; s < Sb; s += 64) part += ew[s];
        const float tot_blank = warp_sum(part);
        if (lane == 0 && tot_blank > 0.f)
            gt[p.blank] -= expf(logf(tot_blank) + m + nll - (lpt[p.blank] - ls)) * scale;
        // labels (odd s): the lane owning the last occurrence walks the chain backwards
        for (int s = 2 * lane + 1; s < Sb; s += 64) {
            if (is_last[s]) {
                float tot = 0.f;
                for (int q = s; q >= 0; q = prev_same[q]) tot += ew[q];
                const int l = lab[s];
                if (l >= 0 && l != p.blank && tot > 0.f) gt[l] -= expf(logf(tot) + m + nll - (lpt[l] - ls)) * scale;
            }
        }
        __syncwarp();
    }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" int b200asr_log_softmax_fwd(const float* logits, float* log_probs, float* lse, long long* argmax,
                                       long long n_rows, int V, b200asr_stream stream) {
    B200_REQUIRE(logits && (log_probs || lse), "log_softmax_fwd: null pointer (log_probs may be NULL when lse is given)");
    B200_REQUIRE(n_rows >= 0 && V > 0, "log_softmax_fwd: bad sizes");
    if (n_rows == 0) return B200_OK;
    const int wpb = 8;
    const long long blocks = (n_rows + wpb - 1) / wpb;
    log_softmax_fwd_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(logits, log_probs, lse, argmax,
                                                                                   n_rows, V);
    B200_LAUNCH_CHECK("log_softmax_fwd_kernel");
    return B200_OK;
}

extern "C" int b200asr_log_softmax_bwd(const float* log_probs, const float* grad_out, float* grad_in,
                                       long long n_rows, int V, b200asr_stream stream) {
    B200_REQUIRE(log_probs && grad_out && grad_in, "log_softmax_bwd: null pointer");
    B200_REQUIRE(n_rows >= 0 && V > 0, "log_softmax_bwd: bad sizes");
    if (n_rows == 0) return B200_OK;
    const int wpb = 8;
    const long long blocks = (n_rows + wpb - 1) / wpb;
    log_softmax_bwd_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(log_probs, grad_out, grad_in,
                                                                                   n_rows, V);
    B200_LAUNCH_CHECK("log_softmax_bwd_kernel");
    return B200_OK;
}

extern "C" size_t b200asr_ctc_workspace_bytes(int B, int T, int L_max) {
    const size_t S = 2 * (size_t)L_max + 1;
    return 2 * (size_t)B * T * S * sizeof(float) + 2 * (size_t)B * S * sizeof(int);
}

static int ctc_setup(CtcParams& p, const float* log_probs, const float* row_lse, long long stride_b, long long stride_t,
                     const long long* targets, const long long* input_lengths, const long long* target_lengths, int B,
                     int T, int V, int L_max, int blank, float* nll, const float* grad_scale, const float* upstream,
                     float* grad, void* workspace, size_t workspace_bytes, const char* who) {
    B200_REQUIRE(log_probs && targets && input_lengths && target_lengths && nll && workspace, "%s: null pointer", who);
    B200_REQUIRE(B > 0 && T > 0 && V > 0 && L_max >= 0, "%s: bad sizes B=%d T=%d V=%d L=%d", who, B, T, V, L_max);
    B200_REQUIRE(blank >= 0 && blank < V, "%s: blank %d outside [0,%d)", who, blank, V);
    B200_REQUIRE(workspace_bytes >= b200asr_ctc_workspace_bytes(B, T, L_max), "%s: workspace too small", who);
    p.lp = log_probs; p.lse = row_lse; p.sb = stride_b; p.st = stride_t; p.targets = targets; p.in_len = input_lengths;
    p.tgt_len = target_lengths; p.B = B; p.T = T; p.V = V; p.L_max = L_max; p.S_max = 2 * L_max + 1; p.blank = blank;
    p.nll = nll; p.scale = grad_scale; p.upstream = upstream; p.grad = grad;
    const size_t S = (size_t)p.S_max;
    float* ws = reinterpret_cast<float*>(workspace);
    p.alpha = ws;
    p.beta = ws + (size_t)B * T * S;
    p.prev_same = reinterpret_cast<int*>(ws + 2 * (size_t)B * T * S);
    p.is_last = p.prev_same + (size_t)B * S;
    return B200_OK;
}

static int ctc_launch_grad(const CtcParams& p, cudaStream_t stream) {
    const size_t S = (size_t)p.S_max;
    const size_t smem_g = S * ((CTC_GRAD_THREADS / 32) * sizeof(float) + 3 * sizeof(int));
    B200_REQUIRE(smem_g <= (size_t)max_optin_smem(), "ctc: target too long for shared memory (L=%d)", p.L_max);
    if (smem_g > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(ctc_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g));
    dim3 grid((p.T + CTC_GRAD_TCHUNK - 1) / CTC_GRAD_TCHUNK, p.B);
    ctc_grad_kernel<<<grid, CTC_GRAD_THREADS, smem_g, stream>>>(p);
    B200_LAUNCH_CHECK("ctc_grad_kernel");
    return B200_OK;
}

static int ctc_fwd_bwd_impl(const float* log_probs, const float* row_lse, long long stride_b, long long stride_t,
                            const long long* targets, const long long* input_lengths,
                            const long long* target_lengths, int B, int T, int V, int L_max, int blank,
                            float* nll, const float* grad_scale, float* grad, void* workspace,
                            size_t workspace_bytes, b200asr_stream stream) {
    CtcParams p;
    const int rc = ctc_setup(p, log_probs, row_lse, stride_b, stride_t, targets, input_lengths, target_lengths, B, T, V,
                             L_max, blank, nll, grad_scale, nullptr, grad, workspace, workspace_bytes, "ctc_fwd_bwd");
    if (rc != B200_OK) return rc;
    const int need = (p.S_max + 31) / 32;      // extended-label positions per lane
    // The warp-synchronous kernel wins while a lane holds few positions (subword targets: S <= 128); for long
    // character targets one position per thread + a block barrier is faster (V = 31, L ~ 130), so those
    // take the block kernel.
    if (need <= 4 && (size_t)CTC_WARPS * 2 * p.S_max * sizeof(float) <= 48 * 1024) {
        if (need <= 1) launch_ctc_warp<1>(p, (cudaStream_t)stream);
        else if (need <= 2) launch_ctc_warp<2>(p, (cudaStream_t)stream);
        else if (need <= 3) launch_ctc_warp<3>(p, (cudaStream_t)stream);
        else launch_ctc_warp<4>(p, (cudaStream_t)stream);
        B200_LAUNCH_CHECK("ctc_alpha_beta_warp_kernel");
    } else {
        // long targets: block-per-(utterance, direction) kernel with the lattice row in shared memory
        const size_t S = (size_t)p.S_max;
        int threads = (p.S_max + 31) / 32 * 32;
        if (threads > 1024) threads = 1024;
        const size_t smem_ab = S * (2 * sizeof(float) + 2 * sizeof(int));
        B200_REQUIRE(smem_ab <= (size_t)max_optin_smem(), "ctc_fwd_bwd: target too long for shared memory (L=%d)", L_max);
        if (smem_ab > 48 * 1024)
            B200_CUDA(cudaFuncSetAttribute(ctc_alpha_beta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem_ab));
        ctc_alpha_beta_kernel<<<dim3(B, 2), threads, smem_ab, (cudaStream_t)stream>>>(p);
        B200_LAUNCH_CHECK("ctc_alpha_beta_kernel");
    }
    if (grad) return ctc_launch_grad(p, (cudaStream_t)stream);
    return B200_OK;
}

extern "C" int b200asr_ctc_fwd_bwd(const float* log_probs, long long stride_b, long long stride_t,
                                   const long long* targets, const long long* input_lengths,
                                   const long long* target_lengths, int B, int T, int V, int L_max, int blank,
                                   float* nll, const float* grad_scale, float* grad, void* workspace,
                                   size_t workspace_bytes, b200asr_stream stream) {
    return ctc_fwd_bwd_impl(log_probs, nullptr, stride_b, stride_t, targets, input_lengths, target_lengths, B, T, V,
                            L_max, blank, nll, grad_scale, grad, workspace, workspace_bytes, stream);
}

extern "C" int b200asr_ctc_fwd_bwd_logits(const float* logits, const float* row_lse, long long stride_b,
                                          long long stride_t, const long long* targets,
                                          const long long* input_lengths, const long long* target_lengths, int B,
                                          int T, int V, int L_max, int blank, float* nll, const float* grad_scale,
                                          float* grad, void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(row_lse, "ctc_fwd_bwd_logits: null row_lse");
    return ctc_fwd_bwd_impl(logits, row_lse, stride_b, stride_t, targets, input_lengths, target_lengths, B, T, V, L_max,
                            blank, nll, grad_scale, grad, workspace, workspace_bytes, stream);
}

static int ctc_grad_impl(const float* log_probs, const float* row_lse, long long stride_b, long long stride_t,
                         const long long* targets, const long long* input_lengths, const long long* target_lengths,
                         int B, int T, int V, int L_max, int blank, const float* nll, const float* grad_scale,
                         const float* upstream, float* grad, void* workspace, size_t workspace_bytes,
                         b200asr_stream stream) {
    B200_REQUIRE(grad, "ctc_grad: null gradient pointer");
    CtcParams p;
    const int rc = ctc_setup(p, log_probs, row_lse, stride_b, stride_t, targets, input_lengths, target_lengths, B, T, V,
                             L_max, blank, const_cast<float*>(nll), grad_scale, upstream, grad, workspace,
                             workspace_bytes, "ctc_grad");
    if (rc != B200_OK) return rc;
    return ctc_launch_grad(p, (cudaStream_t)stream);
}

extern "C" int b200asr_ctc_grad(const float* log_probs, long long stride_b, long long stride_t,
                                const long long* targets, const long long* input_lengths,
                                const long long* target_lengths, int B, int T, int V, int L_max, int blank,
                                const float* nll, const float* grad_scale, const float* upstream, float* grad,
                                void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    return ctc_grad_impl(log_probs, nullptr, stride_b, stride_t, targets, input_lengths, target_lengths, B, T, V, L_max,
                         blank, nll, grad_scale, upstream, grad, workspace, workspace_bytes, stream);
}

extern "C" int b200asr_ctc_grad_logits(const float* logits, const float* row_lse, long long stride_b,
                                       long long stride_t, const long long* targets, const long long* input_lengths,
                                       const long long* target_lengths, int B, int T, int V, int L_max, int blank,
                                       const float* nll, const float* grad_scale, const float* upstream, float* grad,
                                       void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(row_lse, "ctc_grad_logits: null row_lse");
    return ctc_grad_impl(logits, row_lse, stride_b, stride_t, targets, input_lengths, target_lengths, B, T, V, L_max,
                         blank, nll, grad_scale, upstream, grad, workspace, workspace_bytes, stream);
}
