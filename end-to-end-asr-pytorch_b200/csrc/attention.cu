// K12: location-aware attention step, forward and backward, ONE launch each.
//
// Forward (per utterance b, a cluster of CS CTAs):
//   conv[k,t]  = sum_j w_conv[k,j] * prev_att[t + j - R]                (Conv1d 1->K, kernel 2R+1, pad R, no bias)
//   loc[t,d]   = tanh(sum_k w_proj[d,k] * conv[k,t])                    (Linear K->D, no bias)
//   e[t]       = (b_e + sum_d w_e[d] * tanh(key[t,d] + q[d] + loc[t,d])) / temperature
//   attn       = softmax over t < len (padded frames masked with -inf)
//   ctx[e]     = sum_t attn[t] * value[t,e]
// The CTAs of a cluster split the time axis for conv/energy, exchange the T energies through distributed
// shared memory, and split the feature axis of the context.
//
// Backward: recomputes conv/loc/tanh from the saved inputs, and produces d(q), d(key), d(value), d(prev_att)
// and per-CTA partial sums of the four small weight gradients (summed over CTAs by the caller).
//
// Restates /root/reference/src/module.py:234-258 (LocationAwareAttention.forward) + :189-195 (_attend), one head.
#include "common.cuh"
#include "../../include/b200asr.h"
#include "../../include/b200asr_debug.h"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200asr {

constexpr int ATT_TT = 32;  // time tile of the backward pass

struct AttnParams {
    const float* q;       // [B, D]
    const float* key;     // [B, T, D]
    const float* value;   // [B, T, E]
    const float* prev;    // [B, T]
    const long long* len; // [B]
    const float* w_conv;  // [K, 2R+1]
    const float* w_proj;  // [D, K]
    const float* w_e;     // [D]
    const float* b_e;     // [1]
    float temperature;
    int B, T, D, E, K, R, CS;
    // forward outputs
    float* attn;          // [B, T]
    float* ctx;           // [B, E]
    // backward inputs
    const float* attn_in; // [B, T] saved forward output
    const float* dctx;    // [B, E]
    const float* dattn;   // [B, T] or null
    // backward outputs
    float* dq_part;       // [B, CS, D]
    float* dkey;          // [B, T, D]
    float* dvalue;        // [B, T, E]
    float* dprev;         // [B, T]
    float* wpart;         // [B*CS, P], P = D*K + K*W + D + 1   (d w_proj | d w_conv | d w_e | d b_e)
    int accumulate;       // != 0: d(key) and wpart are ADDED to (the decode loop's per-batch accumulators); dvalue may
                          // then be null (d(value) = sum over steps of attn (x) dctx is formed once after the loop)
    int N;                // dot-product kernels: heads per utterance; row b is masked by len[b / N]
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ---- phases shared by the location-aware and the dot-product kernels -------------------------------------------
// frame t's energy -> s_energy[t] of every CTA of the cluster
__device__ __forceinline__ void energy_to_cluster(cg::cluster_group& cluster, float* s_energy, int rank, int CS, int t,
                                                  float e) {
    for (int rr = 0; rr < CS; ++rr) {
        float* dst = (rr == rank) ? s_energy : cluster.map_shared_rank(s_energy, rr);
        dst[t] = e;
    }
}

// masked softmax over the full time axis (redundantly in every CTA; masked frames hold -inf and get exactly 0; a row
// with len 0 gets 0/0 = NaN everywhere, as the reference's softmax of an all -inf row):
// s_energy becomes the attention; attn_row (one CTA of the cluster) receives a copy
__device__ __forceinline__ void softmax_in_place(float* s_energy, float* s_scratch, int T, float* attn_row) {
    float mx = NEG_INF;
    for (int t = threadIdx.x; t < T; t += blockDim.x) mx = fmaxf(mx, s_energy[t]);
    mx = block_max(mx, s_scratch);
    float sum = 0.f;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float x = s_energy[t];
        const float ex = (x == NEG_INF) ? 0.f : expf(x - mx);
        s_energy[t] = ex;
        sum += ex;
    }
    sum = block_sum(sum, s_scratch);
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float a = s_energy[t] / sum;
        s_energy[t] = a;
        if (attn_row) attn_row[t] = a;
    }
    __syncthreads();
}

// context slice of row b: ctx[e] for e in [rank*ES, (rank+1)*ES), frames t < len; float4 columns, time split across
// thread groups, s_ctx [blockDim.x * 4] partial sums
__device__ __forceinline__ void context_slice(const AttnParams& p, int b, int rank, int len, const float* s_attn,
                                              float* s_ctx) {
    const int T = p.T, E = p.E;
    const int ES = E / p.CS;
    const int ncol = ES >> 2;
    const int cpp = min(ncol, (int)blockDim.x);          // columns per pass
    const int ngroups = (int)blockDim.x / cpp;           // time groups
    const int grp = threadIdx.x / cpp;
    for (int cbase = 0; cbase < ncol; cbase += cpp) {
        const int col = cbase + (threadIdx.x - grp * cpp);
        const bool act = grp < ngroups && col < ncol;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (act) {
            const float* vb = p.value + (size_t)b * T * E + (size_t)rank * ES + col * 4;
#pragma unroll 4
            for (int t = grp; t < len; t += ngroups) {
                const float a = s_attn[t];
                const float4 v = *reinterpret_cast<const float4*>(vb + (size_t)t * E);
                acc.x = fmaf(a, v.x, acc.x); acc.y = fmaf(a, v.y, acc.y);
                acc.z = fmaf(a, v.z, acc.z); acc.w = fmaf(a, v.w, acc.w);
            }
        }
        *reinterpret_cast<float4*>(s_ctx + (size_t)threadIdx.x * 4) = acc;
        __syncthreads();
        if (act && grp == 0) {
            for (int g = 1; g < ngroups; ++g) {
                const float4 o = *reinterpret_cast<const float4*>(s_ctx + (size_t)(g * cpp + col - cbase) * 4);
                acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
            }
            if (len == 0) acc = make_float4(NAN, NAN, NAN, NAN);   // the reference's 0/0 attention reaches the context
            *reinterpret_cast<float4*>(p.ctx + (size_t)b * E + (size_t)rank * ES + col * 4) = acc;
        }
        __syncthreads();
    }
}

// backward, first phase: this CTA's feature slice of d(attn)[t] = dctx . value[b,t] for t < len, written into
// s_part[rank*T + t] of every CTA of the cluster (plus d(value) = attn (x) dctx when p.dvalue is set).  One warp per
// frame; the slice of d(ctx) is the same for every frame: registers; the value row of the NEXT frame of this warp is
// loaded while the current one is reduced (one row per iteration left the loop bound by the load latency).
// ES = E / CS <= 128 * MAXV.
template <int MAXV>
__device__ __forceinline__ void dattn_partials(const AttnParams& p, cg::cluster_group& cluster, int b, int rank, int len,
                                               const float* s_attn, float* s_part) {
    const int T = p.T, E = p.E, CS = p.CS;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int ES = E / CS;
    const float* dcb = p.dctx + (size_t)b * E + (size_t)rank * ES;
    const float* vb = p.value + (size_t)b * T * E + (size_t)rank * ES;
    float4 dcr[MAXV], cur[MAXV], nxt[MAXV];
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int e = lane * 4 + 128 * k;
        dcr[k] = (e < ES) ? *reinterpret_cast<const float4*>(dcb + e) : make_float4(0.f, 0.f, 0.f, 0.f);
        cur[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (warp < T && warp < len && e < ES)
            cur[k] = *reinterpret_cast<const float4*>(vb + (size_t)warp * E + e);
    }
    for (int t = warp; t < T; t += nw) {
        const float a = s_attn[t];
        float* dvr = p.dvalue + ((size_t)b * T + t) * E + (size_t)rank * ES;
        const int tn = t + nw;
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
            const int e = lane * 4 + 128 * k;
            nxt[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tn < T && tn < len && e < ES)
                nxt[k] = *reinterpret_cast<const float4*>(vb + (size_t)tn * E + e);
        }
        float part = 0.f;
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
            const int e = lane * 4 + 128 * k;
            if (e < ES) {
                const float4 dc = dcr[k], v = cur[k];
                if (t < len) part += dc.x * v.x + dc.y * v.y + dc.z * v.z + dc.w * v.w;
                if (p.dvalue) {
                    float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (t < len || len == 0) dv = make_float4(a * dc.x, a * dc.y, a * dc.z, a * dc.w);   // len 0: NaN
                    *reinterpret_cast<float4*>(dvr + e) = dv;
                }
            }
            cur[k] = nxt[k];
        }
        part = warp_sum(part);
        if (lane == 0) {
            for (int rr = 0; rr < CS; ++rr) {
                float* dst = (rr == rank) ? s_part : cluster.map_shared_rank(s_part, rr);
                dst[rank * T + t] = part;
            }
        }
    }
}

// backward, softmax phase (every CTA, full time axis, after the cluster barrier that completes dattn_partials):
// g[t] = dattn[t] + sum of the CS partials; s_de[t] = attn[t] (g[t] - sum_t' attn g) / temperature for t < len, else 0
__device__ __forceinline__ void softmax_bwd(const AttnParams& p, int b, int len, const float* s_attn, const float* s_part,
                                            float* s_de, float* s_scratch) {
    const int T = p.T, CS = p.CS;
    float dot = 0.f;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        float g = p.dattn ? p.dattn[(size_t)b * T + t] : 0.f;
        for (int rr = 0; rr < CS; ++rr) g += s_part[rr * T + t];
        s_de[t] = g;
        if (t < len) dot = fmaf(s_attn[t], g, dot);
    }
    dot = block_sum(dot, s_scratch);
    for (int t = threadIdx.x; t < T; t += blockDim.x)
        s_de[t] = (t < len) ? s_attn[t] * (s_de[t] - dot) / p.temperature : 0.f;
    __syncthreads();
}

// conv[k][tl] for the time range [t0, t0+nts) into s_conv[k*stride + tl]
__device__ __forceinline__ void conv_slice(const float* s_prev, const float* s_w, float* s_conv, int K, int W,
                                           int t0, int nts, int stride) {
    for (int idx = threadIdx.x; idx < K * nts; idx += blockDim.x) {
        const int k = idx / nts, tl = idx - k * nts;
        const float* pw = s_w + k * W;
        const float* pp = s_prev + t0 + tl;  // s_prev is shifted by R: s_prev[t + j] = prev[t + j - R]
        float acc = 0.f;
        for (int j = 0; j < W; ++j) acc = fmaf(pw[j], pp[j], acc);
        s_conv[k * stride + tl] = acc;
    }
}

__global__ void __launch_bounds__(1024) locattn_fwd_kernel(AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_scratch[32];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = p.CS;
    const int rank = (int)cluster.block_rank();
    const int b = blockIdx.x / CS;
    const int T = p.T, D = p.D, K = p.K, R = p.R, W = 2 * R + 1;
    const int TS = (T + CS - 1) / CS;
    float* s_prev = sm;                    // [T + 2R]
    float* s_w = s_prev + T + 2 * R;       // [K*W]
    float* s_pw = s_w + K * W;             // [D*K]
    float* s_ew = s_pw + D * K;            // [D]
    float* s_q = s_ew + D;                 // [D]
    float* s_energy = s_q + D;             // [T]
    float* s_conv = s_energy + T;          // [K*TS]
    float* s_ctx = sm + (((s_conv + K * TS) - sm + 3) & ~3);   // [blockDim.x * 4] partial sums, 16-B aligned

    const int len = clampi((int)p.len[b], 0, T);
    for (int i = threadIdx.x; i < T + 2 * R; i += blockDim.x) {
        const int t = i - R;
        s_prev[i] = (t >= 0 && t < T) ? p.prev[(size_t)b * T + t] : 0.f;
    }
    for (int i = threadIdx.x; i < K * W; i += blockDim.x) s_w[i] = p.w_conv[i];
    for (int i = threadIdx.x; i < D * K; i += blockDim.x) s_pw[i] = p.w_proj[i];
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
        s_ew[i] = p.w_e[i];
        s_q[i] = p.q[(size_t)b * D + i];
    }
    cluster.sync();  // all CTAs of the cluster are running (required before any remote shared-memory access)

    const int t0 = rank * TS;
    const int t1 = min(min(T, t0 + TS), len);
    const int nts = max(0, t1 - t0);
    conv_slice(s_prev, s_w, s_conv, K, W, t0, nts, TS);
    __syncthreads();

    // energies of my time slice -> every CTA of the cluster
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const float be = p.b_e[0];
    for (int tl = warp; tl < TS; tl += nw) {
        const int t = t0 + tl;
        if (t >= T) break;
        float e = NEG_INF;
        if (t < len) {
            const float* kr = p.key + ((size_t)b * T + t) * D;
            float kv[16];                                   // the frame's key row (D <= 512), all loads in flight at once
#pragma unroll
            for (int i = 0; i < 16; ++i) kv[i] = (lane + 32 * i < D) ? kr[lane + 32 * i] : 0.f;
            float part = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int d = lane + 32 * i;
                if (d < D) {
                    float pre = 0.f;
                    for (int k = 0; k < K; ++k) pre = fmaf(s_pw[d * K + k], s_conv[k * TS + tl], pre);
                    const float loc = tanhf(pre);
                    part = fmaf(s_ew[d], tanhf(kv[i] + s_q[d] + loc), part);
                }
            }
            e = (warp_sum(part) + be) / p.temperature;
        }
        if (lane == 0) energy_to_cluster(cluster, s_energy, rank, CS, t, e);
    }
    cluster.sync();

    softmax_in_place(s_energy, s_scratch, T, rank == 0 ? p.attn + (size_t)b * T : nullptr);
    context_slice(p, b, rank, len, s_energy, s_ctx);
    cluster.sync();  // keep shared memory alive until every peer has finished its remote writes/reads
}

// ------------------------------------------------------------------------------------------
// one thread per attention dim.  MINB = 2 (D <= 384, E / CS <= 512): two CTAs per SM, so that the 256 CTAs of a
// 64-utterance batch stay ONE wave; MINB = 1 (D <= 512, E / CS <= 1024):
// more registers for the value-row prefetch when all CTAs are co-resident anyway (cfg D, 32 utterances).
template <int MINB>
__global__ void __launch_bounds__(MINB == 2 ? 384 : 512, MINB) locattn_bwd_kernel(AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_scratch[32];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = p.CS;
    const int rank = (int)cluster.block_rank();
    const int b = blockIdx.x / CS;
    const int T = p.T, D = p.D, K = p.K, R = p.R, W = 2 * R + 1;
    const int TS = (T + CS - 1) / CS;
    float* s_prev = sm;                          // [T + 2R]
    float* s_w = s_prev + T + 2 * R;             // [K*W]
    float* s_pw = s_w + K * W;                   // [D*K]
    float* s_ew = s_pw + D * K;                  // [D]
    float* s_q = s_ew + D;                       // [D]
    float* s_attn = s_q + D;                     // [T]
    float* s_de = s_attn + T;                    // [T]   d(energy/temperature input) after the softmax
    float* s_part = s_de + T;                    // [CS*T] partial d(attn) of every peer
    float* s_conv = s_part + CS * T;             // [K*ATT_TT]
    float* s_dloc = s_conv + K * ATT_TT;         // [ATT_TT*D]
    float* s_dconv = s_dloc + ATT_TT * D;        // [K*(T + 2R)] full-time d(conv) with zero halo

    const int len = clampi((int)p.len[b], 0, T);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int i = threadIdx.x; i < T + 2 * R; i += blockDim.x) {
        const int t = i - R;
        s_prev[i] = (t >= 0 && t < T) ? p.prev[(size_t)b * T + t] : 0.f;
    }
    for (int i = threadIdx.x; i < K * W; i += blockDim.x) s_w[i] = p.w_conv[i];
    for (int i = threadIdx.x; i < D * K; i += blockDim.x) s_pw[i] = p.w_proj[i];
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
        s_ew[i] = p.w_e[i];
        s_q[i] = p.q[(size_t)b * D + i];
    }
    for (int i = threadIdx.x; i < T; i += blockDim.x) s_attn[i] = p.attn_in[(size_t)b * T + i];
    for (int i = threadIdx.x; i < K * (T + 2 * R); i += blockDim.x) s_dconv[i] = 0.f;
    cluster.sync();  // all CTAs running + local init visible before any remote shared-memory access

    // A. d(attn) partial over my feature slice + d(value) = attn (x) dctx
    dattn_partials<MINB == 2 ? 4 : 8>(p, cluster, b, rank, len, s_attn, s_part);   // ES <= 128 * MAXV (host-checked)
    cluster.sync();
    // B. softmax backward (every CTA, full time axis)
    softmax_bwd(p, b, len, s_attn, s_part, s_de, s_scratch);

    // C. my time slice, in tiles of ATT_TT frames: recompute conv/loc/tanh, d(key), d(q), d(w_e), d(w_proj), d(conv)
    const int t0s = rank * TS;
    const int t1s = min(T, t0s + TS);
    const int d_own = threadIdx.x;  // one thread per attention dim (blockDim >= D)
    float dq_acc = 0.f, dew_acc = 0.f, deb_acc = 0.f;
    float dpw_acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) dpw_acc[k] = 0.f;
    for (int tb = t0s; tb < t1s; tb += ATT_TT) {
        const int tv = min(min(t1s, len) - tb, ATT_TT);   // valid (unmasked) frames of this tile
        const int tn = min(t1s - tb, ATT_TT);              // frames of this tile
        // the tile's key column of this thread, issued before the location convolution so that the 32 loads overlap it
        // (a local array on purpose: fully unrolling the 32-frame body to keep it in registers measured slower)
        float kreg[ATT_TT];
#pragma unroll
        for (int tl = 0; tl < ATT_TT; ++tl)
            kreg[tl] = (d_own < D && tl < tv) ? p.key[((size_t)b * T + tb + tl) * D + d_own] : 0.f;
        if (tv > 0) conv_slice(s_prev, s_w, s_conv, K, W, tb, tv, ATT_TT);
        __syncthreads();
        if (d_own < D) {
            const float qd = s_q[d_own], ew = s_ew[d_own];
#pragma unroll 4
            for (int tl = 0; tl < ATT_TT; ++tl) {
                if (tl >= tn) break;
                const float kval = kreg[tl];
                const int t = tb + tl;
                float dpre = 0.f, dloc = 0.f;
                if (tl < tv) {
                    float pre = 0.f;
                    for (int k = 0; k < K; ++k) pre = fmaf(s_pw[d_own * K + k], s_conv[k * ATT_TT + tl], pre);
                    const float loc = tanhf(pre);
                    const float s = tanhf(kval + qd + loc);
                    const float de = s_de[t];
                    dpre = de * ew * (1.f - s * s);
                    dew_acc = fmaf(de, s, dew_acc);
                    dq_acc += dpre;
                    dloc = dpre * (1.f - loc * loc);
                    for (int k = 0; k < K; ++k) dpw_acc[k] = fmaf(dloc, s_conv[k * ATT_TT + tl], dpw_acc[k]);
                }
                if (!p.accumulate) p.dkey[((size_t)b * T + t) * D + d_own] = dpre;
                else if (tl < tv) p.dkey[((size_t)b * T + t) * D + d_own] += dpre;
                s_dloc[tl * D + d_own] = dloc;
            }
        }
        if (threadIdx.x == 0)
            for (int tl = 0; tl < tv; ++tl) deb_acc += s_de[tb + tl];
        __syncthreads();
        // d(conv)[k][t] = sum_d dloc[t,d] * w_proj[d,k]  -> every peer's full-time buffer
        for (int idx = warp; idx < tv * K; idx += nw) {
            const int tl = idx / K, k = idx - tl * K;
            float part = 0.f;
            for (int d = lane; d < D; d += 32) part = fmaf(s_dloc[tl * D + d], s_pw[d * K + k], part);
            part = warp_sum(part);
            if (lane == 0) {
                for (int rr = 0; rr < CS; ++rr) {
                    float* dst = (rr == rank) ? s_dconv : cluster.map_shared_rank(s_dconv, rr);
                    dst[k * (T + 2 * R) + R + tb + tl] = part;
                }
            }
        }
        __syncthreads();
    }
    cluster.sync();

    // D. d(w_conv) partial over my slice, d(prev) for my slice
    const int P = D * K + K * W + D + 1;
    float* wp = p.wpart + (size_t)(b * CS + rank) * P;
    const int tv_all = max(0, min(t1s, len) - t0s);
    for (int idx = threadIdx.x; idx < K * W; idx += blockDim.x) {
        const int k = idx / W, j = idx - k * W;
        const float* dc = s_dconv + k * (T + 2 * R) + R + t0s;
        const float* pp = s_prev + t0s + j;
        float acc = 0.f;
        for (int tl = 0; tl < tv_all; ++tl) acc = fmaf(dc[tl], pp[tl], acc);
        wp[D * K + idx] = p.accumulate ? wp[D * K + idx] + acc : acc;
    }
    // dprev[t'] = sum_k sum_j dconv[k][t' - j + R] * w[k][j]   (dconv zero outside [0, len))
    for (int tl = warp; tl < t1s - t0s; tl += nw) {
        const int tp = t0s + tl;
        float part = 0.f;
        for (int idx = lane; idx < K * W; idx += 32) {
            const int k = idx / W, j = idx - k * W;
            part = fmaf(s_dconv[k * (T + 2 * R) + R + tp - j + R], s_w[idx], part);
        }
        part = warp_sum(part);
        if (lane == 0) p.dprev[(size_t)b * T + tp] = part;
    }
    // E. per-CTA partial weight gradients and d(q)
    if (d_own < D) {
        if (p.accumulate) {
            for (int k = 0; k < K; ++k) wp[d_own * K + k] += dpw_acc[k];
            wp[D * K + K * W + d_own] += dew_acc;
        } else {
            for (int k = 0; k < K; ++k) wp[d_own * K + k] = dpw_acc[k];
            wp[D * K + K * W + d_own] = dew_acc;
        }
        p.dq_part[((size_t)b * CS + rank) * D + d_own] = dq_acc;
    }
    if (threadIdx.x == 0) wp[D * K + K * W + D] = p.accumulate ? wp[D * K + K * W + D] + deb_acc : deb_acc;
    cluster.sync();
}

// d(value)[b,t,:] = sum over the L decode steps of attn[b,l,t] * dctx[b,l,:]  - formed ONCE after the loop instead of
// writing (and having autograd re-add) a [B,T,E] tensor per step.  grid (ceil(T/8), B), 256 threads.
constexpr int DV_TT = 8;
__global__ void __launch_bounds__(256) attn_dvalue_kernel(const float* __restrict__ attn, const float* __restrict__ dctx,
                                                          float* __restrict__ dvalue, int B, int L, int T, int E,
                                                          int accumulate) {
    extern __shared__ float s_a[];                 // [L][DV_TT]
    const int b = blockIdx.y, t0 = blockIdx.x * DV_TT;
    for (int i = threadIdx.x; i < L * DV_TT; i += blockDim.x) {
        const int l = i / DV_TT, tt = i - l * DV_TT;
        s_a[i] = (t0 + tt < T) ? attn[((size_t)b * L + l) * T + t0 + tt] : 0.f;
    }
    __syncthreads();
    for (int e = threadIdx.x * 4; e < E; e += blockDim.x * 4) {
        float4 acc[DV_TT];
#pragma unroll
        for (int tt = 0; tt < DV_TT; ++tt) acc[tt] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int l = 0; l < L; ++l) {
            const float4 d = *reinterpret_cast<const float4*>(dctx + ((size_t)b * L + l) * E + e);
#pragma unroll
            for (int tt = 0; tt < DV_TT; ++tt) {
                const float a = s_a[l * DV_TT + tt];
                acc[tt].x = fmaf(a, d.x, acc[tt].x); acc[tt].y = fmaf(a, d.y, acc[tt].y);
                acc[tt].z = fmaf(a, d.z, acc[tt].z); acc[tt].w = fmaf(a, d.w, acc[tt].w);
            }
        }
#pragma unroll
        for (int tt = 0; tt < DV_TT; ++tt) {
            if (t0 + tt < T) {
                float4* o = reinterpret_cast<float4*>(dvalue + ((size_t)b * T + t0 + tt) * E + e);
                if (accumulate) {
                    const float4 old = *o;
                    acc[tt].x += old.x; acc[tt].y += old.y; acc[tt].z += old.z; acc[tt].w += old.w;
                }
                *o = acc[tt];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Scaled dot-product attention step (the reference's src/module.py:189-212, `_attend` + ScaleDotAttention.forward) on
// rows b of B = utterances x heads, row b masked by len[b / N]:  e[t] = (q . key[b,t]) / temperature for t < len,
// attn = softmax(e) over t < len (exactly 0 beyond), ctx = sum_t attn[t] value[b,t].  Same cluster split as the
// location-aware kernels: the CS CTAs of a row split time for the energies and the feature axis for the context.
__global__ void __launch_bounds__(512, 2) dotattn_fwd_kernel(AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_scratch[32];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = p.CS;
    const int rank = (int)cluster.block_rank();
    const int b = blockIdx.x / CS;
    const int T = p.T, D = p.D;
    const int TS = (T + CS - 1) / CS;
    float* s_energy = sm;                        // [T]
    float* s_ctx = sm + ((T + 3) & ~3);          // [blockDim.x * 4] partial sums, 16-B aligned

    const int len = clampi((int)p.len[b / p.N], 0, T);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    float qv[16];                                // the row's query (D <= 512), lane-strided like the key rows
#pragma unroll
    for (int i = 0; i < 16; ++i) qv[i] = (lane + 32 * i < D) ? p.q[(size_t)b * D + lane + 32 * i] : 0.f;
    cluster.sync();  // all CTAs of the cluster are running (required before any remote shared-memory access)

    // energies of my time slice -> every CTA of the cluster
    const int t0 = rank * TS;
    for (int tl = warp; tl < TS; tl += nw) {
        const int t = t0 + tl;
        if (t >= T) break;
        float e = NEG_INF;
        if (t < len) {
            const float* kr = p.key + ((size_t)b * T + t) * D;
            float kv[16];                        // all loads of the frame's key row in flight at once
#pragma unroll
            for (int i = 0; i < 16; ++i) kv[i] = (lane + 32 * i < D) ? kr[lane + 32 * i] : 0.f;
            float part = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) part = fmaf(qv[i], kv[i], part);
            e = warp_sum(part) / p.temperature;
        }
        if (lane == 0) energy_to_cluster(cluster, s_energy, rank, CS, t, e);
    }
    cluster.sync();  // the last remote access of this kernel: no peer touches this CTA's shared memory after it

    softmax_in_place(s_energy, s_scratch, T, rank == 0 ? p.attn + (size_t)b * T : nullptr);
    context_slice(p, b, rank, len, s_energy, s_ctx);
}

// Backward of one decode step on the per-batch accumulator (the decode loop's form, like b200asr_locattn_bwd_acc):
// g[t] = dctx . value[b,t] + dattn[t], de[t] = attn[t] (g[t] - sum attn g) / temperature;  d(key)[b,t] += de[t] q for
// t < len, dq_part[b, rank] = sum over my time slice of de[t] key[b,t].  No d(value): b200asr_attn_dvalue forms it
// once after the loop.  MINB as in the location-aware backward: 2 (E / CS <= 512) when the CTAs outnumber the SMs.
template <int MINB>
__global__ void __launch_bounds__(MINB == 2 ? 384 : 512, MINB) dotattn_bwd_kernel(AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_scratch[32];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = p.CS;
    const int rank = (int)cluster.block_rank();
    const int b = blockIdx.x / CS;
    const int T = p.T, D = p.D;
    const int TS = (T + CS - 1) / CS;
    float* s_q = sm;                             // [D]
    float* s_attn = s_q + D;                     // [T]
    float* s_de = s_attn + T;                    // [T]
    float* s_part = s_de + T;                    // [CS*T] partial d(attn) of every peer

    const int len = clampi((int)p.len[b / p.N], 0, T);
    for (int i = threadIdx.x; i < D; i += blockDim.x) s_q[i] = p.q[(size_t)b * D + i];
    for (int i = threadIdx.x; i < T; i += blockDim.x) s_attn[i] = p.attn_in[(size_t)b * T + i];
    cluster.sync();  // all CTAs running + local init visible before any remote shared-memory access

    dattn_partials<MINB == 2 ? 4 : 8>(p, cluster, b, rank, len, s_attn, s_part);
    cluster.sync();  // the last remote access of this kernel
    softmax_bwd(p, b, len, s_attn, s_part, s_de, s_scratch);

    // my time slice: one thread per attention dim; frames t >= len are neither read nor written
    const int t0s = rank * TS;
    const int t1s = min(min(T, t0s + TS), len);
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        const float qd = s_q[d];
        float acc = 0.f;
#pragma unroll 4
        for (int t = t0s; t < t1s; ++t) {
            const float de = s_de[t];
            const size_t off = ((size_t)b * T + t) * D + d;
            acc = fmaf(de, p.key[off], acc);
            p.dkey[off] += de * qd;
        }
        p.dq_part[((size_t)b * CS + rank) * D + d] = acc;
    }
}

// CTAs per row: 4 where the feature split allows it (E % (4 CS) == 0); fewer for short memories (T < 8 CS: a speed
// preference only), but never so few that E / CS exceeds the backward's 1024-column limit.
static int pick_cluster(int T, int E) {
    int cs = 4;
    while (cs > 1 && (E % (4 * cs) != 0 || (T < 8 * cs && E / (cs / 2) <= 1024))) cs >>= 1;
    return cs;
}

constexpr size_t ATT_STATIC_SMEM = 32 * sizeof(float);   // s_scratch of every attention kernel

static int launch_attn(const char* what, const void* fn, AttnParams& p, int threads, size_t smem,
                       cudaStream_t stream) {
    B200_REQUIRE(smem + ATT_STATIC_SMEM <= (size_t)max_optin_smem(),
                 "%s: %zu bytes of shared memory needed (T=%d D=%d too large)", what, smem + ATT_STATIC_SMEM, p.T, p.D);
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.B * p.CS);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = p.CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    void* args[] = {&p};
    B200_CUDA(cudaLaunchKernelExC(&cfg, fn, args));
    count_launch();
    return B200_OK;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" int b200asr_locattn_cluster_size(int T, int E) { return pick_cluster(T, E); }

extern "C" size_t b200asr_locattn_wpart_floats(int D, int K, int R) { return (size_t)D * K + (size_t)K * (2 * R + 1) + D + 1; }

extern "C" int b200asr_locattn_fwd(const float* q, const float* key, const float* value, const float* prev_att,
                                   const long long* enc_len, const float* w_conv, const float* w_proj,
                                   const float* w_energy, const float* b_energy, float temperature, int B, int T, int D,
                                   int E, int K, int R, float* attn, float* ctx, b200asr_stream stream) {
    B200_REQUIRE(q && key && value && prev_att && enc_len && w_conv && w_proj && w_energy && b_energy && attn && ctx,
                 "locattn_fwd: null pointer");
    B200_REQUIRE(B > 0 && T > 0 && D > 0 && E > 0 && K > 0 && R >= 0, "locattn_fwd: bad sizes");
    B200_REQUIRE(E % 4 == 0, "locattn_fwd: value dim %d must be a multiple of 4", E);
    B200_REQUIRE(K <= 16, "locattn_fwd: at most 16 location kernels (got %d)", K);
    AttnParams p = {};
    p.q = q; p.key = key; p.value = value; p.prev = prev_att; p.len = enc_len; p.w_conv = w_conv; p.w_proj = w_proj;
    p.w_e = w_energy; p.b_e = b_energy; p.temperature = temperature; p.B = B; p.T = T; p.D = D; p.E = E; p.K = K;
    p.R = R; p.CS = pick_cluster(T, E); p.attn = attn; p.ctx = ctx;
    B200_REQUIRE(D <= 512, "locattn_fwd: attention dim %d > 512", D);
    const int threads = 512;
    const int W = 2 * R + 1, TS = (T + p.CS - 1) / p.CS;
    const size_t smem = sizeof(float) * ((size_t)T + 2 * R + (size_t)K * W + (size_t)D * K + 2 * D + T + (size_t)K * TS +
                                         (size_t)threads * 4 + 4);
    return launch_attn("loc_attention", (const void*)locattn_fwd_kernel, p, threads, smem, (cudaStream_t)stream);
}

// MINB of the backward kernel: 2 when the CTAs outnumber the SMs and the smaller register budget fits the shape
static int locattn_bwd_minb(int B, int T, int D, int E) {
    const int cs = pick_cluster(T, E);
    return ((long long)B * cs > sm_count() && D <= 384 && E / cs <= 512) ? 2 : 1;
}

extern "C" int b200asr_debug_locattn_bwd_minb(int B, int T, int D, int E) {
    return (B > 0 && T > 0 && E > 0) ? locattn_bwd_minb(B, T, D, E) : 0;
}

static int locattn_bwd_impl(const float* q, const float* key, const float* value, const float* prev_att,
                            const long long* enc_len, const float* w_conv, const float* w_proj,
                            const float* w_energy, float temperature, const float* attn, const float* dctx,
                            const float* dattn, int B, int T, int D, int E, int K, int R, float* dq_part,
                            float* dkey, float* dvalue, float* dprev, float* wpart, int accumulate,
                            b200asr_stream stream) {
    B200_REQUIRE(q && key && value && prev_att && enc_len && w_conv && w_proj && w_energy && attn && dctx && dq_part &&
                     dkey && (dvalue || accumulate) && dprev && wpart,
                 "locattn_bwd: null pointer");
    B200_REQUIRE(B > 0 && T > 0 && D > 0 && E > 0 && K > 0 && R >= 0, "locattn_bwd: bad sizes");
    B200_REQUIRE(E % 4 == 0, "locattn_bwd: value dim %d must be a multiple of 4", E);
    B200_REQUIRE(K <= 16, "locattn_bwd: at most 16 location kernels (got %d)", K);
    B200_REQUIRE(D <= 512, "locattn_bwd: attention dim %d > 512", D);
    B200_REQUIRE(E / pick_cluster(T, E) <= 1024, "locattn_bwd: value dim %d too large for %d-CTA clusters", E, pick_cluster(T, E));
    AttnParams p = {};
    p.q = q; p.key = key; p.value = value; p.prev = prev_att; p.len = enc_len; p.w_conv = w_conv; p.w_proj = w_proj;
    p.w_e = w_energy; p.temperature = temperature; p.B = B; p.T = T; p.D = D; p.E = E; p.K = K; p.R = R;
    p.CS = pick_cluster(T, E); p.attn_in = attn; p.dctx = dctx; p.dattn = dattn; p.dq_part = dq_part; p.dkey = dkey;
    p.dvalue = dvalue; p.dprev = dprev; p.wpart = wpart; p.accumulate = accumulate;
    int threads = (D + 31) / 32 * 32;
    if (threads < 128) threads = 128;
    const int W = 2 * R + 1;
    const size_t smem = sizeof(float) * ((size_t)T + 2 * R + (size_t)K * W + (size_t)D * K + 2 * D + 2 * (size_t)T +
                                         (size_t)p.CS * T + (size_t)K * ATT_TT + (size_t)ATT_TT * D +
                                         (size_t)K * (T + 2 * R));
    const bool two_per_sm = locattn_bwd_minb(B, T, D, E) == 2;
    return launch_attn("loc_attention", two_per_sm ? (const void*)locattn_bwd_kernel<2> : (const void*)locattn_bwd_kernel<1>,
                       p, threads, smem, (cudaStream_t)stream);
}

extern "C" int b200asr_locattn_bwd(const float* q, const float* key, const float* value, const float* prev_att,
                                   const long long* enc_len, const float* w_conv, const float* w_proj,
                                   const float* w_energy, float temperature, const float* attn, const float* dctx,
                                   const float* dattn, int B, int T, int D, int E, int K, int R, float* dq_part,
                                   float* dkey, float* dvalue, float* dprev, float* wpart, b200asr_stream stream) {
    return locattn_bwd_impl(q, key, value, prev_att, enc_len, w_conv, w_proj, w_energy, temperature, attn, dctx, dattn, B,
                            T, D, E, K, R, dq_part, dkey, dvalue, dprev, wpart, 0, stream);
}

extern "C" int b200asr_locattn_bwd_acc(const float* q, const float* key, const float* value, const float* prev_att,
                                       const long long* enc_len, const float* w_conv, const float* w_proj,
                                       const float* w_energy, float temperature, const float* attn, const float* dctx,
                                       const float* dattn, int B, int T, int D, int E, int K, int R, float* dq_part,
                                       float* dkey_acc, float* dprev, float* wpart_acc, b200asr_stream stream) {
    return locattn_bwd_impl(q, key, value, prev_att, enc_len, w_conv, w_proj, w_energy, temperature, attn, dctx, dattn, B,
                            T, D, E, K, R, dq_part, dkey_acc, nullptr, dprev, wpart_acc, 1, stream);
}

extern "C" int b200asr_attn_dvalue(const float* attn_steps, const float* dctx_steps, int B, int L, int T, int E,
                                   float* dvalue, int accumulate, b200asr_stream stream) {
    B200_REQUIRE(attn_steps && dctx_steps && dvalue, "attn_dvalue: null pointer");
    B200_REQUIRE(B > 0 && L > 0 && T > 0 && E > 0 && E % 4 == 0, "attn_dvalue: bad sizes B=%d L=%d T=%d E=%d", B, L, T, E);
    const size_t smem = (size_t)L * DV_TT * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "attn_dvalue: %d decode steps do not fit", L);
    dim3 grid((T + DV_TT - 1) / DV_TT, B);
    attn_dvalue_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(attn_steps, dctx_steps, dvalue, B, L, T, E, accumulate);
    B200_LAUNCH_CHECK("attn_dvalue_kernel");
    return B200_OK;
}

// ---- scaled dot-product attention ----------------------------------------------------------------------------------
// The limits of include/b200asr.h, checked before any CUDA call (ops.dot_attention_supported restates them).
static int dotattn_check(const char* what, int R, int N, int T, int D, int E) {
    B200_REQUIRE(R > 0 && N > 0 && T > 0 && D > 0 && E > 0 && R % N == 0,
                 "%s: bad sizes R=%d N=%d T=%d D=%d E=%d (R must be a multiple of N)", what, R, N, T, D, E);
    B200_REQUIRE(T <= B200ASR_DOTATTN_MAX_T, "%s: %d frames > %d", what, T, B200ASR_DOTATTN_MAX_T);
    B200_REQUIRE(D <= 512, "%s: attention dim %d > 512", what, D);
    B200_REQUIRE(E % 4 == 0, "%s: value dim %d must be a multiple of 4", what, E);
    B200_REQUIRE(E / pick_cluster(T, E) <= 1024, "%s: value dim %d too large for %d-CTA clusters", what, E,
                 pick_cluster(T, E));
    return B200_OK;
}

static AttnParams dotattn_params(const float* q, const float* key, const float* value, const long long* enc_len,
                                 int num_head, float temperature, int R, int T, int D, int E) {
    AttnParams p = {};
    p.q = q; p.key = key; p.value = value; p.len = enc_len; p.N = num_head; p.temperature = temperature;
    p.B = R; p.T = T; p.D = D; p.E = E; p.CS = pick_cluster(T, E);
    return p;
}

static int dotattn_bwd_minb(int R, int T, int E) {
    const int cs = pick_cluster(T, E);
    return ((long long)R * cs > sm_count() && E / cs <= 512) ? 2 : 1;
}

extern "C" int b200asr_dotattn_supported(int T, int D, int E) {
    return T > 0 && T <= B200ASR_DOTATTN_MAX_T && D > 0 && D <= 512 && E > 0 && E % 4 == 0 &&
           E / pick_cluster(T, E) <= 1024;
}

extern "C" int b200asr_debug_dotattn_bwd_minb(int R, int T, int E) {
    return (R > 0 && T > 0 && E > 0) ? dotattn_bwd_minb(R, T, E) : 0;
}

extern "C" int b200asr_dotattn_fwd(const float* q, const float* key, const float* value, const long long* enc_len,
                                   int num_head, float temperature, int R, int T, int D, int E, float* attn, float* ctx,
                                   b200asr_stream stream) {
    B200_REQUIRE(q && key && value && enc_len && attn && ctx, "dotattn_fwd: null pointer");
    const int rc = dotattn_check("dotattn_fwd", R, num_head, T, D, E);
    if (rc != B200_OK) return rc;
    AttnParams p = dotattn_params(q, key, value, enc_len, num_head, temperature, R, T, D, E);
    p.attn = attn; p.ctx = ctx;
    const int threads = 512;
    const size_t smem = sizeof(float) * (((size_t)T + 3) / 4 * 4 + (size_t)threads * 4);
    return launch_attn("dotattn_fwd", (const void*)dotattn_fwd_kernel, p, threads, smem, (cudaStream_t)stream);
}

extern "C" int b200asr_dotattn_bwd_acc(const float* q, const float* key, const float* value, const long long* enc_len,
                                       int num_head, float temperature, const float* attn, const float* dctx,
                                       const float* dattn, int R, int T, int D, int E, float* dq_part, float* dkey_acc,
                                       b200asr_stream stream) {
    B200_REQUIRE(q && key && value && enc_len && attn && dctx && dq_part && dkey_acc, "dotattn_bwd_acc: null pointer");
    const int rc = dotattn_check("dotattn_bwd_acc", R, num_head, T, D, E);
    if (rc != B200_OK) return rc;
    AttnParams p = dotattn_params(q, key, value, enc_len, num_head, temperature, R, T, D, E);
    p.attn_in = attn; p.dctx = dctx; p.dattn = dattn; p.dq_part = dq_part; p.dkey = dkey_acc;
    const bool two_per_sm = dotattn_bwd_minb(R, T, E) == 2;
    const int threads = two_per_sm ? 384 : 512;
    const size_t smem = sizeof(float) * ((size_t)D + 2 * (size_t)T + (size_t)p.CS * T);
    return launch_attn("dotattn_bwd_acc", two_per_sm ? (const void*)dotattn_bwd_kernel<2> : (const void*)dotattn_bwd_kernel<1>,
                       p, threads, smem, (cudaStream_t)stream);
}

// ---- multi-head location-aware attention ---------------------------------------------------------------------------
// The reference's LocationAwareAttention with N > 1 heads (src/module.py:234-258): ONE location convolution per
// utterance over the N channels of prev_att [B,N,T], its projection shared by the N heads (loc.repeat(1,N,1,1)); row
// r = b*N + n of q / key / value / attn / ctx is head n of utterance b, masked by len[b]:
//   conv[k,t]  = sum_n sum_j w_conv[k,n,j] * prev[b,n,t+j-R]         (one fmaf chain, n outer, j inner)
//   loc[t,d]   = tanh(sum_k w_proj[d,k] * conv[k,t])
//   e[r,t]     = (b_e + sum_d w_e[d] * tanh(key[r,t,d] + q[r,d] + loc[t,d])) / temperature
// One cluster of CS CTAs per UTTERANCE covers all N heads: the CTAs split time for conv / loc / the N heads' energies
// (conv and loc computed once per frame, not once per head), exchange the N energy rows through distributed shared
// memory, and each runs the N masked softmaxes and an E/CS slice of the N contexts.  The backward sums d(loc) over the
// heads in shared memory in head order (no atomics) and writes d(prev) for all N channels.
namespace b200asr {

constexpr int LH_TT = 16;  // frame tile of the multi-head backward

// conv[k][tl] over the N channels for frames [t0, t0+nts) into s_conv[k*stride + tl]; s_prev holds N rows of T + 2R
__device__ __forceinline__ void conv_heads_slice(const float* s_prev, const float* s_w, float* s_conv, int K, int N,
                                                 int W, int TP, int t0, int nts, int stride) {
    for (int idx = threadIdx.x; idx < K * nts; idx += blockDim.x) {
        const int k = idx / nts, tl = idx - k * nts;
        float acc = 0.f;
        for (int n = 0; n < N; ++n) {
            const float* pw = s_w + (k * N + n) * W;
            const float* pp = s_prev + n * TP + t0 + tl;
            for (int j = 0; j < W; ++j) acc = fmaf(pw[j], pp[j], acc);
        }
        s_conv[k * stride + tl] = acc;
    }
}

// prev rows of utterance b (zero halo of R frames each side), the weights and the N query rows into shared memory
__device__ __forceinline__ void heads_load_common(const AttnParams& p, int b, float* s_prev, float* s_w, float* s_pw,
                                                  float* s_ew, float* s_q) {
    const int N = p.N, T = p.T, D = p.D, K = p.K, R = p.R, W = 2 * R + 1, TP = T + 2 * R;
    for (int i = threadIdx.x; i < N * TP; i += blockDim.x) {
        const int n = i / TP, t = i - n * TP - R;
        s_prev[i] = (t >= 0 && t < T) ? p.prev[((size_t)b * N + n) * T + t] : 0.f;
    }
    for (int i = threadIdx.x; i < K * N * W; i += blockDim.x) s_w[i] = p.w_conv[i];
    for (int i = threadIdx.x; i < D * K; i += blockDim.x) s_pw[i] = p.w_proj[i];
    for (int i = threadIdx.x; i < D; i += blockDim.x) s_ew[i] = p.w_e[i];
    for (int i = threadIdx.x; i < N * D; i += blockDim.x) s_q[i] = p.q[(size_t)b * N * D + i];
}

__global__ void __launch_bounds__(512, 1) locattn_heads_fwd_kernel(AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_scratch[32];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = p.CS;
    const int rank = (int)cluster.block_rank();
    const int b = blockIdx.x / CS;                  // utterance
    const int N = p.N, T = p.T, D = p.D, K = p.K, R = p.R, W = 2 * R + 1, TP = T + 2 * R;
    const int TS = (T + CS - 1) / CS;
    float* s_prev = sm;                             // [N*(T + 2R)]
    float* s_w = s_prev + N * TP;                   // [K*N*W]
    float* s_pw = s_w + K * N * W;                  // [D*K]
    float* s_ew = s_pw + D * K;                     // [D]
    float* s_q = s_ew + D;                          // [N*D]
    float* s_energy = s_q + N * D;                  // [N*T]
    float* s_conv = s_energy + N * T;               // [K*TS]
    float* s_ctx = sm + (((s_conv + K * TS) - sm + 3) & ~3);   // [blockDim.x * 4] partial sums, 16-B aligned

    const int len = clampi((int)p.len[b], 0, T);
    heads_load_common(p, b, s_prev, s_w, s_pw, s_ew, s_q);
    cluster.sync();  // all CTAs of the cluster are running (required before any remote shared-memory access)

    const int t0 = rank * TS;
    const int nts = max(0, min(min(T, t0 + TS), len) - t0);
    conv_heads_slice(s_prev, s_w, s_conv, K, N, W, TP, t0, nts, TS);
    __syncthreads();

    // one warp per frame of my slice: loc once, then the N heads' energies -> every CTA of the cluster
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const float be = p.b_e[0];
    for (int tl = warp; tl < TS; tl += nw) {
        const int t = t0 + tl;
        if (t >= T) break;
        if (t >= len) {
            if (lane == 0)
                for (int n = 0; n < N; ++n) energy_to_cluster(cluster, s_energy + n * T, rank, CS, t, NEG_INF);
            continue;
        }
        float lc[16];                                   // loc[t, lane + 32 i] (D <= 512)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int d = lane + 32 * i;
            lc[i] = 0.f;
            if (d < D) {
                float pre = 0.f;
                for (int k = 0; k < K; ++k) pre = fmaf(s_pw[d * K + k], s_conv[k * TS + tl], pre);
                lc[i] = tanhf(pre);
            }
        }
        for (int n = 0; n < N; ++n) {
            const float* kr = p.key + (((size_t)b * N + n) * T + t) * D;
            float kv[16];                               // the frame's key row of head n, all loads in flight at once
#pragma unroll
            for (int i = 0; i < 16; ++i) kv[i] = (lane + 32 * i < D) ? kr[lane + 32 * i] : 0.f;
            float part = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int d = lane + 32 * i;
                if (d < D) part = fmaf(s_ew[d], tanhf(kv[i] + s_q[n * D + d] + lc[i]), part);
            }
            const float e = warp_sum(part) + be;        // divided by the temperature below
            if (lane == 0) energy_to_cluster(cluster, s_energy + n * T, rank, CS, t, e);
        }
    }
    cluster.sync();  // the last remote access of this kernel: no peer touches this CTA's shared memory after it
    // the division outside the energy loop: its slow path is a subroutine call, which there would need a stack frame
    for (int i = threadIdx.x; i < N * T; i += blockDim.x) s_energy[i] = s_energy[i] / p.temperature;
    __syncthreads();

#pragma unroll 1
    for (int n = 0; n < N; ++n) {
        const int r = b * N + n;
        softmax_in_place(s_energy + n * T, s_scratch, T, rank == 0 ? p.attn + (size_t)r * T : nullptr);
        context_slice(p, r, rank, len, s_energy + n * T, s_ctx);
    }
}

// Backward of one decode step on the per-batch accumulators (the decode loop's form): per head the d(attn) partials
// and the softmax backward of the shared helpers; then, in tiles of LH_TT frames of my time slice, one thread per
// attention dim recomputes conv / loc once per frame and, per head, s = tanh(key + q + loc): d(key) += dpre,
// d(q) and d(w_e) partials, and the head sum dpre_0 + ... + dpre_{N-1} in s_dloc (head order) before d(loc) =
// sum * (1 - loc^2) feeds d(w_proj) and d(conv).  d(conv) goes to every peer's full-time buffer; each CTA then forms
// its slice of d(w_conv) [K,N,W] and d(prev) [N, slice].  MINB as in the single-head backward.
template <int MINB>
__global__ void __launch_bounds__(MINB == 2 ? 384 : 512, MINB) locattn_heads_bwd_kernel(AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_scratch[32];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = p.CS;
    const int rank = (int)cluster.block_rank();
    const int b = blockIdx.x / CS;
    const int N = p.N, T = p.T, D = p.D, K = p.K, R = p.R, W = 2 * R + 1, TP = T + 2 * R;
    const int TS = (T + CS - 1) / CS;
    float* s_prev = sm;                             // [N*(T + 2R)]
    float* s_w = s_prev + N * TP;                   // [K*N*W]
    float* s_pw = s_w + K * N * W;                  // [D*K]
    float* s_ew = s_pw + D * K;                     // [D]
    float* s_q = s_ew + D;                          // [N*D]
    float* s_attn = s_q + N * D;                    // [N*T]
    float* s_de = s_attn + N * T;                   // [N*T]
    float* s_part = s_de + N * T;                   // [N*CS*T] partial d(attn) of every peer, per head
    float* s_conv = s_part + N * CS * T;            // [K*LH_TT]
    float* s_loc = s_conv + K * LH_TT;              // [LH_TT*D]
    float* s_dloc = s_loc + LH_TT * D;              // [LH_TT*D]
    float* s_dq = s_dloc + LH_TT * D;               // [N*D]    d(q) of my slice, thread d owns column d
    float* s_dpw = s_dq + N * D;                    // [D*K]    d(w_proj) of my slice, thread d owns row d
    float* s_dconv = s_dpw + D * K;                 // [K*(T + 2R)] full-time d(conv) with zero halo

    const int len = clampi((int)p.len[b], 0, T);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    heads_load_common(p, b, s_prev, s_w, s_pw, s_ew, s_q);
    for (int i = threadIdx.x; i < N * T; i += blockDim.x) s_attn[i] = p.attn_in[(size_t)b * N * T + i];
    for (int i = threadIdx.x; i < N * D; i += blockDim.x) s_dq[i] = 0.f;
    for (int i = threadIdx.x; i < D * K; i += blockDim.x) s_dpw[i] = 0.f;
    for (int i = threadIdx.x; i < K * TP; i += blockDim.x) s_dconv[i] = 0.f;
    cluster.sync();  // all CTAs running + local init visible before any remote shared-memory access

    // A. d(attn) partials of the N rows over my feature slice
#pragma unroll 1
    for (int n = 0; n < N; ++n)
        dattn_partials<MINB == 2 ? 4 : 8>(p, cluster, b * N + n, rank, len, s_attn + n * T, s_part + n * CS * T);
    cluster.sync();
    // B. softmax backward of the N rows (every CTA, full time axis)
#pragma unroll 1
    for (int n = 0; n < N; ++n)
        softmax_bwd(p, b * N + n, len, s_attn + n * T, s_part + n * CS * T, s_de + n * T, s_scratch);

    // C. my time slice, frames t < len only
    const int t0s = rank * TS;
    const int t1s = min(T, t0s + TS);
    const int tend = min(t1s, len);
    const int d_own = threadIdx.x;  // one thread per attention dim (blockDim >= D)
    float dew_acc = 0.f, deb_acc = 0.f;
    for (int tb = t0s; tb < tend; tb += LH_TT) {
        const int tv = min(tend - tb, LH_TT);
        conv_heads_slice(s_prev, s_w, s_conv, K, N, W, TP, tb, tv, LH_TT);
        __syncthreads();
        if (d_own < D) {
            for (int tl = 0; tl < tv; ++tl) {
                float pre = 0.f;
                for (int k = 0; k < K; ++k) pre = fmaf(s_pw[d_own * K + k], s_conv[k * LH_TT + tl], pre);
                s_loc[tl * D + d_own] = tanhf(pre);
                s_dloc[tl * D + d_own] = 0.f;
            }
            const float ew = s_ew[d_own];
            for (int n = 0; n < N; ++n) {
                const size_t off = (((size_t)b * N + n) * T + tb) * D + d_own;
                const float qd = s_q[n * D + d_own];
                const float* de_n = s_de + n * T + tb;
                float dq = 0.f;
#pragma unroll 2                                    // 4 spills in the two-CTAs-per-SM instance
                for (int tl = 0; tl < tv; ++tl) {
                    const float s = tanhf(p.key[off + (size_t)tl * D] + qd + s_loc[tl * D + d_own]);
                    const float de = de_n[tl];
                    const float dpre = de * ew * (1.f - s * s);
                    dew_acc = fmaf(de, s, dew_acc);
                    dq += dpre;
                    p.dkey[off + (size_t)tl * D] += dpre;
                    s_dloc[tl * D + d_own] += dpre;
                }
                s_dq[n * D + d_own] += dq;
            }
            for (int tl = 0; tl < tv; ++tl) {
                const float loc = s_loc[tl * D + d_own];
                const float dloc = s_dloc[tl * D + d_own] * (1.f - loc * loc);
                s_dloc[tl * D + d_own] = dloc;
                for (int k = 0; k < K; ++k)
                    s_dpw[d_own * K + k] = fmaf(dloc, s_conv[k * LH_TT + tl], s_dpw[d_own * K + k]);
            }
        }
        if (threadIdx.x == 0)
            for (int n = 0; n < N; ++n)
                for (int tl = 0; tl < tv; ++tl) deb_acc += s_de[n * T + tb + tl];
        __syncthreads();
        // d(conv)[k][t] = sum_d dloc[t,d] * w_proj[d,k]  -> every peer's full-time buffer
        for (int idx = warp; idx < tv * K; idx += nw) {
            const int tl = idx / K, k = idx - tl * K;
            float part = 0.f;
            for (int d = lane; d < D; d += 32) part = fmaf(s_dloc[tl * D + d], s_pw[d * K + k], part);
            part = warp_sum(part);
            if (lane == 0) {
                for (int rr = 0; rr < CS; ++rr) {
                    float* dst = (rr == rank) ? s_dconv : cluster.map_shared_rank(s_dconv, rr);
                    dst[k * TP + R + tb + tl] = part;
                }
            }
        }
        __syncthreads();
    }
    cluster.sync();  // the last remote access of this kernel: every peer's d(conv) is in place

    // D. d(w_conv)[k,n,j] partial over my slice, d(prev)[n, t'] for my slice
    const int P = D * K + K * N * W + D + 1;
    float* wp = p.wpart + (size_t)(b * CS + rank) * P;
    const int tv_all = max(0, tend - t0s);
    for (int idx = threadIdx.x; idx < K * N * W; idx += blockDim.x) {
        const int k = idx / (N * W), nj = idx - k * N * W, n = nj / W, j = nj - n * W;
        const float* dc = s_dconv + k * TP + R + t0s;
        const float* pp = s_prev + n * TP + t0s + j;
        float acc = 0.f;
        for (int tl = 0; tl < tv_all; ++tl) acc = fmaf(dc[tl], pp[tl], acc);
        wp[D * K + idx] += acc;
    }
    // dprev[n, t'] = sum_k sum_j dconv[k][t' - j + R] * w[k,n,j]   (dconv zero outside [0, len))
    const int ns = t1s - t0s;
    for (int o = warp; o < N * ns; o += nw) {
        const int n = o / ns, tp = t0s + (o - n * ns);
        float part = 0.f;
        for (int idx = lane; idx < K * W; idx += 32) {
            const int k = idx / W, j = idx - k * W;
            part = fmaf(s_dconv[k * TP + R + tp - j + R], s_w[(k * N + n) * W + j], part);
        }
        part = warp_sum(part);
        if (lane == 0) p.dprev[((size_t)b * N + n) * T + tp] = part;
    }
    // E. per-CTA partial weight gradients and d(q)
    if (d_own < D) {
        for (int k = 0; k < K; ++k) wp[d_own * K + k] += s_dpw[d_own * K + k];
        wp[D * K + K * N * W + d_own] += dew_acc;
        for (int n = 0; n < N; ++n) p.dq_part[(((size_t)b * N + n) * CS + rank) * D + d_own] = s_dq[n * D + d_own];
    }
    if (threadIdx.x == 0) wp[D * K + K * N * W + D] += deb_acc;
}

static size_t locattn_heads_fwd_smem(int N, int T, int D, int K, int R, int CS) {
    const size_t W = 2 * (size_t)R + 1, TP = (size_t)T + 2 * R, TS = ((size_t)T + CS - 1) / CS;
    const size_t head = N * TP + K * N * W + (size_t)D * K + D + (size_t)N * D + (size_t)N * T + K * TS;
    return sizeof(float) * ((head + 3) / 4 * 4 + 512 * 4);
}

static size_t locattn_heads_bwd_smem(int N, int T, int D, int K, int R, int CS) {
    const size_t W = 2 * (size_t)R + 1, TP = (size_t)T + 2 * R;
    return sizeof(float) * (N * TP + K * N * W + 2 * (size_t)D * K + D + 2 * (size_t)N * D + 2 * (size_t)N * T +
                            (size_t)N * CS * T + (size_t)K * LH_TT + 2 * (size_t)LH_TT * D + K * TP);
}

// The limits of include/b200asr.h, checked before any CUDA call (b200asr_locattn_heads_supported reports the same set;
// ops.loc_attention_heads_supported restates it).
static int locattn_heads_check(const char* what, int B, int N, int T, int D, int E, int K, int R) {
    B200_REQUIRE(B > 0 && N > 0 && T > 0 && D > 0 && E > 0 && K > 0 && R >= 0,
                 "%s: bad sizes B=%d N=%d T=%d D=%d E=%d K=%d R=%d", what, B, N, T, D, E, K, R);
    B200_REQUIRE(N <= 16, "%s: at most 16 heads (got %d)", what, N);
    B200_REQUIRE(K <= 16, "%s: at most 16 location kernels (got %d)", what, K);
    B200_REQUIRE(D <= 512, "%s: attention dim %d > 512", what, D);
    B200_REQUIRE(E % 4 == 0, "%s: value dim %d must be a multiple of 4", what, E);
    const int cs = pick_cluster(T, E);
    B200_REQUIRE(E / cs <= 1024, "%s: value dim %d too large for %d-CTA clusters", what, E, cs);
    const size_t fwd = locattn_heads_fwd_smem(N, T, D, K, R, cs), bwd = locattn_heads_bwd_smem(N, T, D, K, R, cs);
    const size_t need = fwd > bwd ? fwd : bwd;
    B200_REQUIRE(need + ATT_STATIC_SMEM <= (size_t)max_optin_smem(),
                 "%s: %zu bytes of shared memory needed (N=%d T=%d D=%d K=%d R=%d too large)", what,
                 need + ATT_STATIC_SMEM, N, T, D, K, R);
    return B200_OK;
}

static AttnParams locattn_heads_params(const float* q, const float* key, const float* value, const float* prev_att,
                                       const long long* enc_len, const float* w_conv, const float* w_proj,
                                       const float* w_energy, float temperature, int B, int N, int T, int D, int E,
                                       int K, int R) {
    AttnParams p = {};
    p.q = q; p.key = key; p.value = value; p.prev = prev_att; p.len = enc_len; p.w_conv = w_conv; p.w_proj = w_proj;
    p.w_e = w_energy; p.temperature = temperature; p.B = B; p.N = N; p.T = T; p.D = D; p.E = E; p.K = K; p.R = R;
    p.CS = pick_cluster(T, E);
    return p;
}

}  // namespace b200asr

extern "C" int b200asr_locattn_heads_supported(int N, int T, int D, int E, int K, int R) {
    return locattn_heads_check("locattn_heads_supported", 1, N, T, D, E, K, R) == B200_OK;
}

extern "C" size_t b200asr_locattn_heads_wpart_floats(int N, int D, int K, int R) {
    return (size_t)D * K + (size_t)K * N * (2 * R + 1) + D + 1;
}

extern "C" int b200asr_debug_locattn_heads_bwd_minb(int B, int N, int T, int D, int E) {
    return (B > 0 && N > 0 && T > 0 && E > 0) ? locattn_bwd_minb(B, T, D, E) : 0;   // the single-head rule
}

extern "C" int b200asr_locattn_heads_fwd(const float* q, const float* key, const float* value, const float* prev_att,
                                         const long long* enc_len, const float* w_conv, const float* w_proj,
                                         const float* w_energy, const float* b_energy, float temperature, int B,
                                         int N, int T, int D, int E, int K, int R, float* attn, float* ctx,
                                         b200asr_stream stream) {
    B200_REQUIRE(q && key && value && prev_att && enc_len && w_conv && w_proj && w_energy && b_energy && attn && ctx,
                 "locattn_heads_fwd: null pointer");
    const int rc = locattn_heads_check("locattn_heads_fwd", B, N, T, D, E, K, R);
    if (rc != B200_OK) return rc;
    AttnParams p = locattn_heads_params(q, key, value, prev_att, enc_len, w_conv, w_proj, w_energy, temperature, B, N,
                                        T, D, E, K, R);
    p.b_e = b_energy; p.attn = attn; p.ctx = ctx;
    return launch_attn("locattn_heads_fwd", (const void*)locattn_heads_fwd_kernel, p, 512,
                       locattn_heads_fwd_smem(N, T, D, K, R, p.CS), (cudaStream_t)stream);
}

extern "C" int b200asr_locattn_heads_bwd_acc(const float* q, const float* key, const float* value,
                                             const float* prev_att, const long long* enc_len, const float* w_conv,
                                             const float* w_proj, const float* w_energy, float temperature,
                                             const float* attn, const float* dctx, const float* dattn, int B, int N,
                                             int T, int D, int E, int K, int R, float* dq_part, float* dkey_acc,
                                             float* dprev, float* wpart_acc, b200asr_stream stream) {
    B200_REQUIRE(q && key && value && prev_att && enc_len && w_conv && w_proj && w_energy && attn && dctx && dq_part &&
                     dkey_acc && dprev && wpart_acc,
                 "locattn_heads_bwd_acc: null pointer");
    const int rc = locattn_heads_check("locattn_heads_bwd_acc", B, N, T, D, E, K, R);
    if (rc != B200_OK) return rc;
    AttnParams p = locattn_heads_params(q, key, value, prev_att, enc_len, w_conv, w_proj, w_energy, temperature, B, N,
                                        T, D, E, K, R);
    p.attn_in = attn; p.dctx = dctx; p.dattn = dattn; p.dq_part = dq_part; p.dkey = dkey_acc; p.dprev = dprev;
    p.wpart = wpart_acc; p.accumulate = 1;
    int threads = (D + 31) / 32 * 32;
    if (threads < 128) threads = 128;
    const bool two_per_sm = locattn_bwd_minb(B, T, D, E) == 2;
    return launch_attn("locattn_heads_bwd_acc",
                       two_per_sm ? (const void*)locattn_heads_bwd_kernel<2> : (const void*)locattn_heads_bwd_kernel<1>,
                       p, threads, locattn_heads_bwd_smem(N, T, D, K, R, p.CS), (cudaStream_t)stream);
}
