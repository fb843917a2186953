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
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

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
    const int T = p.T, D = p.D, E = p.E, K = p.K, R = p.R, W = 2 * R + 1;
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
        if (lane == 0) {
            for (int rr = 0; rr < CS; ++rr) {
                float* dst = (rr == rank) ? s_energy : cluster.map_shared_rank(s_energy, rr);
                dst[t] = e;
            }
        }
    }
    cluster.sync();

    // masked softmax over the full time axis (redundantly in every CTA)
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
        if (rank == 0) p.attn[(size_t)b * T + t] = a;
    }
    __syncthreads();

    // context slice: e in [rank*ES, (rank+1)*ES); float4 columns, time split across thread groups
    const int ES = E / CS;
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
                const float a = s_energy[t];
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
            *reinterpret_cast<float4*>(p.ctx + (size_t)b * E + (size_t)rank * ES + col * 4) = acc;
        }
        __syncthreads();
    }
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
    const int T = p.T, D = p.D, E = p.E, K = p.K, R = p.R, W = 2 * R + 1;
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
    const int ES = E / CS;
    {
        // the slice of d(ctx) is the same for every frame: registers; the value row of the NEXT frame of this warp is
        // loaded while the current one is reduced (one row per iteration left the loop bound by the load latency)
        constexpr int MAXV = MINB == 2 ? 4 : 8;              // ES <= 128 * MAXV (checked by the host wrapper)
        const float* dcb = p.dctx + (size_t)b * E + (size_t)rank * ES;
        float4 dcr[MAXV], cur[MAXV], nxt[MAXV];
#pragma unroll
        for (int k = 0; k < MAXV; ++k) {
            const int e = lane * 4 + 128 * k;
            dcr[k] = (e < ES) ? *reinterpret_cast<const float4*>(dcb + e) : make_float4(0.f, 0.f, 0.f, 0.f);
            cur[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (warp < T && warp < len && e < ES)
                cur[k] = *reinterpret_cast<const float4*>(p.value + ((size_t)b * T + warp) * E + (size_t)rank * ES + e);
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
                    nxt[k] = *reinterpret_cast<const float4*>(p.value + ((size_t)b * T + tn) * E + (size_t)rank * ES + e);
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
                        if (t < len) dv = make_float4(a * dc.x, a * dc.y, a * dc.z, a * dc.w);
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
    cluster.sync();
    // B. softmax backward (every CTA, full time axis)
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

static int pick_cluster(int T, int E) {
    int cs = 4;
    while (cs > 1 && (E % (4 * cs) != 0 || T < 8 * cs)) cs >>= 1;
    return cs;
}

static int launch_attn(const void* fn, AttnParams& p, int threads, size_t smem, cudaStream_t stream) {
    B200_REQUIRE(smem <= (size_t)max_optin_smem(), "loc_attention: %zu bytes of shared memory needed (T=%d D=%d too large)",
                 smem, p.T, p.D);
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
    return launch_attn((const void*)locattn_fwd_kernel, p, threads, smem, (cudaStream_t)stream);
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
    const bool two_per_sm = (long long)B * p.CS > sm_count() && D <= 384 && E / p.CS <= 512;
    return launch_attn(two_per_sm ? (const void*)locattn_bwd_kernel<2> : (const void*)locattn_bwd_kernel<1>, p, threads,
                       smem, (cudaStream_t)stream);
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
