// K7/K8: persistent (Bi)LSTM recurrence, forward and BPTT backward, fp32.
//
// Decomposition (same for fwd and bwd): one CTA per (direction, batch-group, unit-block). A CTA owns UB hidden units
// (= 4*UB gate columns) for Bc batch rows and keeps its slice of W_hh resident in shared memory for all T steps.
// The Bc rows are processed as NH = 2 independent halves by two thread GROUPS of 128 threads that run their own
// step loops and drift out of phase: while one group waits for its state exchange, the FMA pipes work for the other,
// so the cross-SM latency is hidden behind compute.
//
//   group g (4 warps), step GEMM in one of two forms (the planner decides per shape, make_plan):
//     tensor cores (default whenever a half is exactly 16 rows, H % 32 == 0, UB even <= 16: every BASELINE shape):
//              error-compensated 3xTF32 mma.sync.m16n8k8 with fragment-major operands, see "Tensor-core variant" below;
//     fp32 FMA (every other shape): 32 register tiles of 4 gates x 8 rows (one W float4 feeds 32 FMAs), K split over
//              4 lanes (one per bulk-copy chunk, chunks padded apart in shared memory), packed FFMA2 inner loops with
//              explicit A/B register double buffering, two warp shuffles reduce the K-chunks, then each of the 4 lanes
//              finishes the pointwise cell update of two rows.
//     In both forms the two groups take turns on the math pipes (mbarrier hand-off), so that one group's exchange is
//     hidden behind the other group's loop.
//   control warp g (1 lane): waits on the group's "done" mbarrier, issues ONE fence + release for the whole group
//              (off the compute warps' critical path), spins on the peers' counter, then pulls the next [H,Bh] state
//              block (fwd) / [nub,Bh,UB] inbox of partial products (bwd) from L2 with 1-D bulk async copies (TMA)
//              that complete on per-chunk "full" mbarriers.
// There is no CTA-wide or grid-wide barrier in the step loops; the backward has one 128-thread named barrier per step
// (the dG tile of a group feeds all of its GEMM tiles).  Batches whose CTAs cannot all be co-resident are processed as
// consecutive launches over row blocks (Plan::nsplit).
//
//   fwd step : gates[b, 4UB] = Gx[b,t] + h_{t-1}[b,:] . Wslice^T ; pointwise ; publish h_t slice
//   bwd step : dh = dOut[b,t] + sum_src partial_src[b, my units] ; pointwise -> dG[b,4UB] ;
//              partial_me[b, :] = dG . Wslice  (scattered to every destination's inbox, deterministic, no atomics)
//
// The input projection (x . W_ih^T + b_ih + b_hh, K6) and the weight-gradient contractions are tensor-core GEMMs
// done by the caller; this file is the sequential part.
//
// Reference behaviour restated: torch.nn.LSTM as called from /root/reference/src/module.py:112-113,129-132 (single
// layer, batch_first, zero initial state, run over the zero-padded frames - no packing, SURVEY.md F5), gates i,f,g,o.
#include "common.cuh"
#include "lstm_umma.h"
#include "../../include/b200asr.h"
#include "../../include/b200asr_debug.h"

namespace b200asr {

constexpr int LSTM_GTHREADS = 128;                  // compute threads per group (one group per batch half)
constexpr int LSTM_THREADS = 2 * LSTM_GTHREADS + 64;  // two groups + two control warps
constexpr int LSTM_NCHUNK = 4;
constexpr int LSTM_MAX_TILES = 32;                  // register tiles (4 gates x R rows) per group
constexpr int LSTM_CHUNK_PAD = 4;                   // floats between the K-chunks of the state block in smem
constexpr int LSTM_COUNTER_BYTES = 4096;

struct LstmParams {
    float* gates;        // [ndir][B][T][H][4]
    const float* whh;    // packed, see lstm_pack_kernel
    float* cst;          // [ndir][B][T][H]
    float* out;          // fwd: layer output [B][T][ndir*H]; bwd: dOut (read only)
    float* xbuf;         // exchange buffers
    unsigned* counters;  // [ndir][nbg][NH]
    int* err_flag;
    long long* trace;    // optional [T][16] clock64 stamps of CTA 0 / group 0 (debug; NULL in production)
    int B, T, H, ndir, UB, Bc, nub, nbg, NH, R;
    int b0, Bend;        // this launch covers batch rows [b0, Bend) of the B rows the tensors hold
    int flags;           // debug switches: bit 2 = first-generation MMA loops (every warp polls, compiler-pipelined),
                         // bit 3 = clock64 trace of the backward instead of the forward kernel
    int mma;             // 1: tensor-core (3xTF32 mma.sync) step GEMMs, see the *_mma kernels
};

#define LSTM_TRACE(slot) \
    do { if (p.trace && blockIdx.x == 0) p.trace[(size_t)step * 16 + (slot)] = clock64(); } while (0)

__device__ __forceinline__ void spin_until(const unsigned* ctr, unsigned target, int* err_flag) {
    const long long t0 = clock64();
    while (ld_acquire_u32(ctr) < target) {
        if (clock64() - t0 > (1LL << 33)) {  // ~4 s: a peer died; abort instead of hanging the GPU
            *err_flag = 1;
            __threadfence_system();
            __trap();
        }
    }
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------------------------------
// Weight packing. Source: PyTorch layout w[dir][g*H + j][k] (gate-major rows).
//   fwd pack: dst[dir][ub][k][u][g]           (per-CTA slice contiguous, k-major)
//   bwd pack: dst[dir][ub][u][g][k]           (per-CTA slice contiguous, row-major over k)
__global__ void lstm_pack_kernel(const float* __restrict__ w, float* __restrict__ dst, int H, int UB, int ndir,
                                 int for_bwd) {
    const long long n = (long long)ndir * 4 * H * H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        long long r = i;
        const int dir = (int)(r / (4LL * H * H));
        r -= (long long)dir * 4 * H * H;
        const int ub = (int)(r / (4LL * UB * H));
        r -= (long long)ub * 4 * UB * H;
        int k, u, g;
        if (!for_bwd) {
            k = (int)(r / (4 * UB));
            const int q = (int)(r - (long long)k * 4 * UB);
            u = q >> 2;
            g = q & 3;
        } else {
            const int q = (int)(r / H);
            k = (int)(r - (long long)q * H);
            u = q >> 2;
            g = q & 3;
        }
        const int j = ub * UB + u;
        dst[i] = w[((long long)dir * 4 * H + (long long)g * H + j) * H + k];
    }
}

// Control lane of one group: publishes the group's step (one fence + one release per CTA-group and step, off the
// compute warps' critical path), waits for the peers, then pulls the next step's block into shared memory.
// (Measured and dropped: issuing the four chunk copies from four lanes, and relying on the release alone without
// the fence - neither moved the step time.)
__device__ __forceinline__ void control_loop(const LstmParams& p, int T, unsigned nub, uint64_t* done, uint64_t* full,
                                             unsigned* ctr, const float* src_even, const float* src_odd, float* dst,
                                             const uint32_t* src_off, const uint32_t* dst_off,
                                             const uint32_t* chunk_bytes, bool trace_me) {
    for (int step = 0; step + 1 < T; ++step) {
        mbar_wait(done, (uint32_t)(step & 1));          // every compute warp of the group finished `step`
        if (trace_me) LSTM_TRACE(8);
        __threadfence();                                // their global stores (made visible to me through the
        if (trace_me) LSTM_TRACE(9);                    // mbarrier) are ordered before the release
        red_release_add_u32(ctr, 1u);
        spin_until(ctr, (unsigned)(step + 1) * nub, p.err_flag);
        if (trace_me) LSTM_TRACE(10);
        fence_proxy_async();
        const float* src = (step & 1) ? src_odd : src_even;
        for (int c = 0; c < LSTM_NCHUNK; ++c) {
            mbar_expect_tx(&full[c], chunk_bytes[c]);
            if (chunk_bytes[c]) bulk_g2s(dst + dst_off[c], src + src_off[c], chunk_bytes[c], &full[c]);
        }
        if (trace_me) LSTM_TRACE(11);
    }
}

// Pairs of fp32 FMAs on a packed register pair: d.{lo,hi} = a.{lo,hi} * b + c.{lo,hi} with a scalar multiplier.  Hopper
// has no packed fp32 FMA instruction: the pair is two FFMAs (same rounding as the packed form).
__device__ __forceinline__ unsigned long long ffma2_vs(unsigned long long a, float b, unsigned long long c) {
    float alo, ahi, clo, chi;
    unsigned long long d;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(alo), "=f"(ahi) : "l"(a));
    asm("mov.b64 {%0, %1}, %2;" : "=f"(clo), "=f"(chi) : "l"(c));
    asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(fmaf(alo, b, clo)), "f"(fmaf(ahi, b, chi)));
    return d;
}
__device__ __forceinline__ unsigned long long pack2(float lo, float hi) {
    unsigned long long d;
    asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(lo), "f"(hi));
    return d;
}
__device__ __forceinline__ void unpack2(unsigned long long v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}

// pick the RL consecutive rows [kq*RL, kq*RL + RL) of an R-row accumulator tile (RL = R/4) without dynamic indexing
template <int R>
__device__ __forceinline__ float pick_row(const float (&acc)[R][4], int kq, int i, int q) {
    constexpr int RL = R / 4;
    float v = acc[i][q];
    if (kq == 1) v = acc[RL + i][q];
    if (kq == 2) v = acc[2 * RL + i][q];
    if (kq == 3) v = acc[3 * RL + i][q];
    return v;
}

// ------------------------------------------------------------------------------------------
// Forward compute group: 128 threads = 32 register tiles (4 gates x R rows) x 4 K-chunks.  lane = kq*8 + tile%8.
template <int R>
__device__ __forceinline__ void fwd_group(const LstmParams& p, int g, int gt, int dir, int bg, int ub, const float4* Ws,
                                          const float* hsg, uint64_t* full, uint64_t* done, float* xbg,
                                          uint64_t* turn) {
    constexpr int RL = R / 4;                 // rows each lane finishes
    const int H = p.H, UB = p.UB, T = p.T;
    const int Bh = p.Bc / p.NH;
    const int NBO = Bh / R;                   // row blocks per half
    const int KC = H / LSTM_NCHUNK;
    const int lane = gt & 31;
    const int kq = lane >> 3;
    const int tile = (gt >> 5) * 8 + (lane & 7);
    const int NT = UB * NBO;
    const bool has_tile = tile < NT;
    const int u = has_tile ? tile % UB : 0;
    const int bo = has_tile ? tile / UB : 0;
    const int ug = ub * UB + u;
    const int bl0 = bo * R + kq * RL;         // my RL rows within the half
    const int bglob0 = p.b0 + bg * p.Bc + g * Bh + bl0;
    const size_t half_elems = (size_t)H * Bh;
    const int chunk_stride = KC * Bh + LSTM_CHUNK_PAD;   // padded so the 4 chunks start in different banks
    const bool trc = (g == 0 && gt == 0);
    float c_reg[RL];
#pragma unroll
    for (int i = 0; i < RL; ++i) c_reg[i] = 0.f;

    for (int step = 0; step < T; ++step) {
        const int tt = dir ? (T - 1 - step) : step;
        if (trc) LSTM_TRACE(0);
        float4 gx[RL];
#pragma unroll
        for (int i = 0; i < RL; ++i) {
            gx[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int b = bglob0 + i;
            if (has_tile && b < p.Bend)
                gx[i] = *reinterpret_cast<const float4*>(p.gates + ((((size_t)dir * p.B + b) * T + tt) * H + ug) * 4);
        }
        float acc[R][4];
#pragma unroll
        for (int i = 0; i < R; ++i)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][q] = 0.f;

        if (step > 0) {
            // Turn taking: the two groups of a CTA alternate on the FMA pipes (A, B, A, B, ...).  A group's loop runs
            // faster alone than next to the other group's loop, and in strict alternation each group's state
            // exchange is hidden behind the other group's loop instead of both groups waiting at once.
            if (p.NH == 2) {
                if (g == 1) mbar_wait(&turn[1], (uint32_t)((step - 1) & 1));
                else if (step >= 2) mbar_wait(&turn[0], (uint32_t)(step & 1));
            }
            // warp-uniform wait: the 4 K-chunk lanes of a warp need all 4 chunks (a per-lane wait would diverge the
            // warp and serialise the four K-chunk loops)
#pragma unroll
            for (int c = 0; c < LSTM_NCHUNK; ++c) mbar_wait(&full[c], (uint32_t)((step - 1) & 1));
            __syncwarp();
            if (trc) LSTM_TRACE(1);
            if (has_tile) {
                const float4* hp = reinterpret_cast<const float4*>(hsg + (size_t)kq * chunk_stride + bo * R);
                const float4* wp = Ws + (size_t)kq * KC * UB + u;
                const int hstride = Bh >> 2;  // float4 per k row
                // accumulators as row pairs: accp[rp][q] = (acc[2rp][q], acc[2rp+1][q])
                unsigned long long accp[R / 2][4];
#pragma unroll
                for (int rp = 0; rp < R / 2; ++rp)
#pragma unroll
                    for (int q = 0; q < 4; ++q) accp[rp][q] = 0ull;
                // explicit register double buffering (A/B) over pairs of k, last pair peeled: every load is
                // unconditional and is issued one full FMA block (16 packed FMAs) ahead of its first use
#define LSTM_FWD_LOAD(hreg, wreg, k_)                                              \
    {                                                                              \
        wreg = wp[(size_t)(k_) * UB];                                              \
        _Pragma("unroll") for (int j = 0; j < RL; ++j) hreg[j] = hp[(size_t)(k_) * hstride + j]; \
    }
#define LSTM_FWD_FMA(hreg, wreg)                                                   \
    _Pragma("unroll") for (int j = 0; j < RL; ++j) {                               \
        const unsigned long long h01 = pack2(hreg[j].x, hreg[j].y), h23 = pack2(hreg[j].z, hreg[j].w); \
        accp[2 * j][0] = ffma2_vs(h01, wreg.x, accp[2 * j][0]);                    \
        accp[2 * j][1] = ffma2_vs(h01, wreg.y, accp[2 * j][1]);                    \
        accp[2 * j][2] = ffma2_vs(h01, wreg.z, accp[2 * j][2]);                    \
        accp[2 * j][3] = ffma2_vs(h01, wreg.w, accp[2 * j][3]);                    \
        accp[2 * j + 1][0] = ffma2_vs(h23, wreg.x, accp[2 * j + 1][0]);            \
        accp[2 * j + 1][1] = ffma2_vs(h23, wreg.y, accp[2 * j + 1][1]);            \
        accp[2 * j + 1][2] = ffma2_vs(h23, wreg.z, accp[2 * j + 1][2]);            \
        accp[2 * j + 1][3] = ffma2_vs(h23, wreg.w, accp[2 * j + 1][3]);            \
    }
                float4 hA[RL], hB[RL], wA, wB;
                LSTM_FWD_LOAD(hA, wA, 0)
#pragma unroll 2
                for (int kk = 0; kk < KC - 2; kk += 2) {
                    LSTM_FWD_LOAD(hB, wB, kk + 1)
                    LSTM_FWD_FMA(hA, wA)
                    LSTM_FWD_LOAD(hA, wA, kk + 2)
                    LSTM_FWD_FMA(hB, wB)
                }
                LSTM_FWD_LOAD(hB, wB, KC - 1)
                LSTM_FWD_FMA(hA, wA)
                LSTM_FWD_FMA(hB, wB)
#undef LSTM_FWD_LOAD
#undef LSTM_FWD_FMA
#pragma unroll
                for (int rp = 0; rp < R / 2; ++rp)
#pragma unroll
                    for (int q = 0; q < 4; ++q) unpack2(accp[rp][q], acc[2 * rp][q], acc[2 * rp + 1][q]);
            }
            if (trc) LSTM_TRACE(3);
            if (p.NH == 2) {             // hand the FMA pipes to the other group
                __syncwarp();
                if (lane == 0) mbar_arrive(&turn[1 - g]);
            }
            // reduce the 4 K-chunks held by lanes l, l^8, l^16, l^24
#pragma unroll
            for (int i = 0; i < R; ++i)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float v = acc[i][q];
                    v += __shfl_xor_sync(0xffffffffu, v, 8);
                    v += __shfl_xor_sync(0xffffffffu, v, 16);
                    acc[i][q] = v;
                }
            if (trc) LSTM_TRACE(4);
        }
        float hq[RL], cq[RL];
        float4 gq[RL];
#pragma unroll
        for (int i = 0; i < RL; ++i) {
            hq[i] = 0.f;
            const int b = bglob0 + i;
            if (has_tile && b < p.Bend) {
                const float ig = sigmoidf_(gx[i].x + pick_row<R>(acc, kq, i, 0));
                const float fg = sigmoidf_(gx[i].y + pick_row<R>(acc, kq, i, 1));
                const float gg = tanhf(gx[i].z + pick_row<R>(acc, kq, i, 2));
                const float og = sigmoidf_(gx[i].w + pick_row<R>(acc, kq, i, 3));
                const float c = fmaf(fg, c_reg[i], ig * gg);
                c_reg[i] = c;
                hq[i] = og * tanhf(c);
                cq[i] = c;
                gq[i] = make_float4(ig, fg, gg, og);
            }
        }
        // publish the new state FIRST (it is on the critical path of every peer CTA), then write the stash
        if (step + 1 < T) {
            if (has_tile) {
                float* dstp = xbg + (size_t)(step & 1) * half_elems + (size_t)ug * Bh + bl0;
#pragma unroll
                for (int i = 0; i < RL; ++i) dstp[i] = hq[i];
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(done);
            if (trc) LSTM_TRACE(5);
        }
#pragma unroll
        for (int i = 0; i < RL; ++i) {
            const int b = bglob0 + i;
            if (has_tile && b < p.Bend) {
                const size_t row = ((size_t)dir * p.B + b) * T + tt;
                *reinterpret_cast<float4*>(p.gates + (row * H + ug) * 4) = gq[i];
                p.cst[row * H + ug] = cq[i];
                p.out[((size_t)b * T + tt) * (p.ndir * H) + (size_t)dir * H + ug] = hq[i];
            }
        }
    }
}

__global__ void __launch_bounds__(LSTM_THREADS, 1) bilstm_fwd_kernel(LstmParams p) {
    extern __shared__ __align__(128) unsigned char s_raw[];
    const int H = p.H, UB = p.UB, Bc = p.Bc, T = p.T, NH = p.NH;
    const int Bh = Bc / NH;
    const int KC = H / LSTM_NCHUNK;
    const int chunk_stride = KC * Bh + LSTM_CHUNK_PAD;
    const size_t hs_half = (size_t)LSTM_NCHUNK * chunk_stride;                   // padded floats per half
    float4* Ws = reinterpret_cast<float4*>(s_raw);                               // [H][UB] float4 (4 gates)
    float* hs = reinterpret_cast<float*>(Ws + (size_t)H * UB);                   // [NH][4 chunks, padded]
    uint64_t* full = reinterpret_cast<uint64_t*>(hs + 2 * ((size_t)LSTM_NCHUNK * (KC * (Bc / NH) + LSTM_CHUNK_PAD)));
    uint64_t* done = full + 2 * LSTM_NCHUNK;                                     // [2]
    uint64_t* turn = done + 2;                                                   // [2] FMA-loop turn taking

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    int blk = blockIdx.x;
    const int ub = blk % p.nub; blk /= p.nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;

    {   // resident W_hh slice
        const float4* src = reinterpret_cast<const float4*>(p.whh) + ((size_t)dir * p.nub + ub) * (size_t)H * UB;
        for (int i = tid; i < H * UB; i += LSTM_THREADS) Ws[i] = src[i];
    }
    if (tid == 0) {
        for (int i = 0; i < 2 * LSTM_NCHUNK; ++i) mbar_init(&full[i], 1);
        for (int i = 0; i < 2; ++i) mbar_init(&done[i], LSTM_GTHREADS / 32);
        for (int i = 0; i < 2; ++i) mbar_init(&turn[i], LSTM_GTHREADS / 32);
        mbar_fence_init();
    }
    __syncthreads();

    const size_t half_elems = (size_t)H * Bh;                                    // floats per state block
    float* xb = p.xbuf + ((size_t)dir * p.nbg + bg) * NH * 2 * half_elems;       // [NH][2][H*Bh]
    unsigned* ctr0 = p.counters + ((size_t)dir * p.nbg + bg) * NH;

    if (warp >= 2 * (LSTM_GTHREADS / 32)) {
        // ===== control warps: warp 8 -> group 0, warp 9 -> group 1 =====
        const int g = warp - 2 * (LSTM_GTHREADS / 32);
        if (lane == 0 && g < NH) {
            uint32_t soff[LSTM_NCHUNK], doff[LSTM_NCHUNK], bytes[LSTM_NCHUNK];
            for (int c = 0; c < LSTM_NCHUNK; ++c) {
                soff[c] = (uint32_t)((size_t)c * KC * Bh);
                doff[c] = (uint32_t)((size_t)c * chunk_stride);
                bytes[c] = (uint32_t)((size_t)KC * Bh * sizeof(float));
            }
            control_loop(p, T, (unsigned)p.nub, &done[g], &full[g * LSTM_NCHUNK], ctr0 + g,
                         xb + ((size_t)g * 2 + 0) * half_elems, xb + ((size_t)g * 2 + 1) * half_elems,
                         hs + (size_t)g * hs_half, soff, doff, bytes, g == 0);
        }
        return;
    }
    const int g = tid / LSTM_GTHREADS;
    if (g >= NH) return;
    const int gt = tid - g * LSTM_GTHREADS;
    if (p.R == 8)
        fwd_group<8>(p, g, gt, dir, bg, ub, Ws, hs + (size_t)g * hs_half, &full[g * LSTM_NCHUNK], &done[g],
                     xb + (size_t)g * 2 * half_elems, turn);
    else
        fwd_group<4>(p, g, gt, dir, bg, ub, Ws, hs + (size_t)g * hs_half, &full[g * LSTM_NCHUNK], &done[g],
                     xb + (size_t)g * 2 * half_elems, turn);
}

// ------------------------------------------------------------------------------------------
// Backward compute group.
template <int R>
__device__ __forceinline__ void bwd_group(const LstmParams& p, int g, int gt, int dir, int bg, int ub, const float* Wr,
                                          const float* inb, float* dgs, uint64_t* full, uint64_t* done, float* xbg,
                                          uint64_t* turn) {
    constexpr int RL = R / 4;
    const int H = p.H, UB = p.UB, T = p.T, nub = p.nub;
    const int Bh = p.Bc / p.NH;
    const int NBO = Bh / R;
    const int lane = gt & 31;
    const int kq = lane >> 3;
    const int tile = (gt >> 5) * 8 + (lane & 7);
    const int NT = UB * NBO;
    const bool has_tile = tile < NT;
    const int u = has_tile ? tile % UB : 0;
    const int bo = has_tile ? tile / UB : 0;
    const int ug = ub * UB + u;
    const int bl0 = bo * R + kq * RL;
    const int bglob0 = p.b0 + bg * p.Bc + g * Bh + bl0;
    const size_t inbox_elems = (size_t)Bh * H;
    const int SC = (nub + LSTM_NCHUNK - 1) / LSTM_NCHUNK;        // sources per chunk
    const bool vec_ok = (UB % 4) == 0;
    float dc_reg[RL];
#pragma unroll
    for (int i = 0; i < RL; ++i) dc_reg[i] = 0.f;

    for (int step = 0; step < T; ++step) {
        const int fstep = T - 1 - step;                    // forward step index being differentiated
        const int tt = dir ? (T - 1 - fstep) : fstep;      // its time index
        const int tt_prev = dir ? tt + 1 : tt - 1;         // time index of the previous forward step
        float4 gtv[RL];
        float ct[RL], cp[RL], dh[RL];
#pragma unroll
        for (int i = 0; i < RL; ++i) {
            gtv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            ct[i] = cp[i] = dh[i] = 0.f;
            const int b = bglob0 + i;
            if (has_tile && b < p.Bend) {
                const size_t row = ((size_t)dir * p.B + b) * T + tt;
                gtv[i] = *reinterpret_cast<const float4*>(p.gates + (row * H + ug) * 4);
                ct[i] = p.cst[row * H + ug];
                if (fstep > 0) cp[i] = p.cst[(((size_t)dir * p.B + b) * T + tt_prev) * H + ug];
                dh[i] = p.out[((size_t)b * T + tt) * (p.ndir * H) + (size_t)dir * H + ug];
            }
        }
        if (step > 0) {
            // my K-chunk of the sources for all R rows of the tile, then reduce over the 4 chunk lanes
            float part[R];
#pragma unroll
            for (int i = 0; i < R; ++i) part[i] = 0.f;
#pragma unroll
            for (int c = 0; c < LSTM_NCHUNK; ++c) mbar_wait(&full[c], (uint32_t)((step - 1) & 1));
            __syncwarp();
            const int s0 = min(nub, kq * SC), s1 = min(nub, s0 + SC);
            if (has_tile) {
                for (int s = s0; s < s1; ++s) {
                    const float* ib = inb + ((size_t)s * Bh + bo * R) * UB + u;
#pragma unroll
                    for (int i = 0; i < R; ++i) part[i] += ib[i * UB];
                }
            }
#pragma unroll
            for (int i = 0; i < R; ++i) {
                float v = part[i];
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                part[i] = v;
            }
#pragma unroll
            for (int i = 0; i < RL; ++i) {
                float v = part[i];
                if (kq == 1) v = part[RL + i];
                if (kq == 2) v = part[2 * RL + i];
                if (kq == 3) v = part[3 * RL + i];
                dh[i] += v;
            }
        }
        // pointwise backward of the cell for my rows
#pragma unroll
        for (int i = 0; i < RL; ++i) {
            const int b = bglob0 + i;
            float4 dg = make_float4(0.f, 0.f, 0.f, 0.f);
            if (has_tile && b < p.Bend) {
                const float ig = gtv[i].x, fg = gtv[i].y, gg = gtv[i].z, og = gtv[i].w;
                const float tc = tanhf(ct[i]);
                const float dc = dc_reg[i] + dh[i] * og * (1.f - tc * tc);
                dg.x = dc * gg * ig * (1.f - ig);
                dg.y = dc * cp[i] * fg * (1.f - fg);
                dg.z = dc * ig * (1.f - gg * gg);
                dg.w = dh[i] * tc * og * (1.f - og);
                dc_reg[i] = dc * fg;
                const size_t row = ((size_t)dir * p.B + b) * T + tt;
                *reinterpret_cast<float4*>(p.gates + (row * H + ug) * 4) = dg;
            }
            if (has_tile) {
                float* d = dgs + (size_t)(u * 4) * Bh + bl0 + i;
                d[0] = dg.x; d[Bh] = dg.y; d[2 * Bh] = dg.z; d[3 * Bh] = dg.w;
            }
        }
        named_bar_sync(1 + g, LSTM_GTHREADS);              // the dG tile of this step is complete
        if (step + 1 < T) {
            // turn taking on the FMA pipes (see the forward kernel): the groups alternate on this GEMM
            if (p.NH == 2) {
                if (g == 1) mbar_wait(&turn[1], (uint32_t)(step & 1));
                else if (step >= 1) mbar_wait(&turn[0], (uint32_t)((step - 1) & 1));
            }
            // partial[b][k] = sum_c dGs[c][b] * Wr[c][k]; thread tiles of R rows x (2 strided float4 of k)
            const int NKQ = H / 8;
            const int ntiles = NKQ * NBO;
            float* outbase = xbg + (size_t)(step & 1) * nub * inbox_elems;
            for (int t2 = gt; t2 < ntiles; t2 += LSTM_GTHREADS) {
                const int kq2 = t2 % NKQ;
                const int bo2 = t2 / NKQ;
                // packed accumulators: a2[i][j] = (partial[row i][k0 + 2j], partial[row i][k0 + 2j + 1])
                unsigned long long a2[R][4];
#pragma unroll
                for (int i = 0; i < R; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) a2[i][j] = 0ull;
                const int C = 4 * UB;
                const float* wptr = Wr + kq2 * 4;
                const float* dptr = dgs + bo2 * R;
#define LSTM_BWD_LOAD(dreg, wareg, wbreg, c_)                                       \
    {                                                                              \
        wareg = *reinterpret_cast<const float4*>(wptr + (size_t)(c_) * H);         \
        wbreg = *reinterpret_cast<const float4*>(wptr + (size_t)(c_) * H + (H >> 1)); \
        _Pragma("unroll") for (int j = 0; j < RL; ++j)                             \
            dreg[j] = *reinterpret_cast<const float4*>(dptr + (size_t)(c_) * Bh + j * 4); \
    }
#define LSTM_BWD_FMA(dreg, wareg, wbreg)                                           \
    {                                                                              \
        const unsigned long long w01 = pack2(wareg.x, wareg.y), w23 = pack2(wareg.z, wareg.w); \
        const unsigned long long w45 = pack2(wbreg.x, wbreg.y), w67 = pack2(wbreg.z, wbreg.w); \
        _Pragma("unroll") for (int j = 0; j < RL; ++j) {                           \
            const float dv[4] = {dreg[j].x, dreg[j].y, dreg[j].z, dreg[j].w};      \
            _Pragma("unroll") for (int r = 0; r < 4; ++r) {                        \
                a2[j * 4 + r][0] = ffma2_vs(w01, dv[r], a2[j * 4 + r][0]);         \
                a2[j * 4 + r][1] = ffma2_vs(w23, dv[r], a2[j * 4 + r][1]);         \
                a2[j * 4 + r][2] = ffma2_vs(w45, dv[r], a2[j * 4 + r][2]);         \
                a2[j * 4 + r][3] = ffma2_vs(w67, dv[r], a2[j * 4 + r][3]);         \
            }                                                                      \
        }                                                                          \
    }
                float4 dA[RL], dB[RL], waA, wbA, waB, wbB;
                LSTM_BWD_LOAD(dA, waA, wbA, 0)
#pragma unroll 1
                for (int c = 0; c < C - 2; c += 2) {
                    LSTM_BWD_LOAD(dB, waB, wbB, c + 1)
                    LSTM_BWD_FMA(dA, waA, wbA)
                    LSTM_BWD_LOAD(dA, waA, wbA, c + 2)
                    LSTM_BWD_FMA(dB, waB, wbB)
                }
                LSTM_BWD_LOAD(dB, waB, wbB, C - 1)
                LSTM_BWD_FMA(dA, waA, wbA)
                LSTM_BWD_FMA(dB, waB, wbB)
#undef LSTM_BWD_LOAD
#undef LSTM_BWD_FMA
                float a[R][8];
#pragma unroll
                for (int i = 0; i < R; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) unpack2(a2[i][j], a[i][2 * j], a[i][2 * j + 1]);
                // scatter to the destination inboxes: element (dst, src=ub, row, u')
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int k0 = r * (H >> 1) + kq2 * 4;
                    if (vec_ok) {
                        const int dst = k0 / UB, uu = k0 - dst * UB;
                        float* o = outbase + (((size_t)dst * nub + ub) * Bh + bo2 * R) * UB + uu;
#pragma unroll
                        for (int i = 0; i < R; ++i)
                            *reinterpret_cast<float4*>(o + (size_t)i * UB) =
                                make_float4(a[i][r * 4], a[i][r * 4 + 1], a[i][r * 4 + 2], a[i][r * 4 + 3]);
                    } else {
                        // unit blocks that are not a multiple of 4 (e.g. UB = 10 at H = 640): resolve the destination
                        // of each of the 4 k columns once (the runtime division is expensive), then store row by row
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int k = k0 + j;
                            const int dst = k / UB, uu = k - dst * UB;
                            float* o = outbase + (((size_t)dst * nub + ub) * Bh + bo2 * R) * UB + uu;
#pragma unroll
                            for (int i = 0; i < R; ++i) o[(size_t)i * UB] = a[i][r * 4 + j];
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                if (p.NH == 2) mbar_arrive(&turn[1 - g]);
                mbar_arrive(done);
            }
        }
    }
}

// Shared memory: Wr[4UB][H] | inbox[NH][nub*Bh*UB] | dGs[NH][4UB*Bh] | barriers
__global__ void __launch_bounds__(LSTM_THREADS, 1) bilstm_bwd_kernel(LstmParams p) {
    extern __shared__ __align__(128) unsigned char s_raw[];
    const int H = p.H, UB = p.UB, Bc = p.Bc, T = p.T, nub = p.nub, NH = p.NH;
    const int Bh = Bc / NH;
    float* Wr = reinterpret_cast<float*>(s_raw);                 // [4UB][H]
    float* inbox = Wr + (size_t)4 * UB * H;                      // [NH][nub*Bh*UB]  (= Bc*H floats)
    float* dGs = inbox + (size_t)Bc * H;                         // [NH][4UB*Bh]
    uint64_t* full = reinterpret_cast<uint64_t*>(dGs + (size_t)4 * UB * Bc);
    uint64_t* done = full + 2 * LSTM_NCHUNK;
    uint64_t* turn = done + 2;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    int blk = blockIdx.x;
    const int ub = blk % nub; blk /= nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;

    {
        const float4* src = reinterpret_cast<const float4*>(p.whh) + ((size_t)dir * nub + ub) * (size_t)H * UB;
        float4* dst = reinterpret_cast<float4*>(Wr);
        for (int i = tid; i < H * UB; i += LSTM_THREADS) dst[i] = src[i];
    }
    if (tid == 0) {
        for (int i = 0; i < 2 * LSTM_NCHUNK; ++i) mbar_init(&full[i], 1);
        for (int i = 0; i < 2; ++i) mbar_init(&done[i], LSTM_GTHREADS / 32);
        for (int i = 0; i < 2; ++i) mbar_init(&turn[i], LSTM_GTHREADS / 32);
        mbar_fence_init();
    }
    __syncthreads();

    // global inbox layout per (dir, bg, half, parity): [dst nub][src nub][Bh][UB]
    const size_t inbox_elems = (size_t)Bh * H;                   // floats one destination receives per step
    float* xb = p.xbuf + ((size_t)dir * p.nbg + bg) * NH * 2 * (size_t)nub * inbox_elems;
    unsigned* ctr0 = p.counters + ((size_t)dir * p.nbg + bg) * NH;
    const int SC = (nub + LSTM_NCHUNK - 1) / LSTM_NCHUNK;

    if (warp >= 2 * (LSTM_GTHREADS / 32)) {
        const int g = warp - 2 * (LSTM_GTHREADS / 32);
        if (lane == 0 && g < NH) {
            uint32_t off[LSTM_NCHUNK], bytes[LSTM_NCHUNK];
            for (int c = 0; c < LSTM_NCHUNK; ++c) {
                const int s0 = min(nub, c * SC), s1 = min(nub, s0 + SC);
                off[c] = (uint32_t)((size_t)s0 * Bh * UB);
                bytes[c] = (uint32_t)((size_t)(s1 - s0) * Bh * UB * sizeof(float));
            }
            control_loop(p, T, (unsigned)nub, &done[g], &full[g * LSTM_NCHUNK], ctr0 + g,
                         xb + (((size_t)g * 2 + 0) * nub + ub) * inbox_elems,
                         xb + (((size_t)g * 2 + 1) * nub + ub) * inbox_elems, inbox + (size_t)g * inbox_elems, off, off,
                         bytes, false);
        }
        return;
    }
    const int g = tid / LSTM_GTHREADS;
    if (g >= NH) return;
    const int gt = tid - g * LSTM_GTHREADS;
    if (p.R == 8)
        bwd_group<8>(p, g, gt, dir, bg, ub, Wr, inbox + (size_t)g * inbox_elems, dGs + (size_t)g * 4 * UB * Bh,
                     &full[g * LSTM_NCHUNK], &done[g], xb + (size_t)g * 2 * nub * inbox_elems, turn);
    else
        bwd_group<4>(p, g, gt, dir, bg, ub, Wr, inbox + (size_t)g * inbox_elems, dGs + (size_t)g * 4 * UB * Bh,
                     &full[g * LSTM_NCHUNK], &done[g], xb + (size_t)g * 2 * nub * inbox_elems, turn);
}


// ==========================================================================================
// Tensor-core variant of the two step kernels (used when a group's batch half is exactly 16 rows = the M of one
// warp-level MMA, H % 32 == 0 and UB is even and <= 16: every BASELINE shape).  Same CTA decomposition, same
// exchange protocol and control warps as above; only the per-step GEMM of a group changes from packed fp32 FMAs to
// error-compensated TF32 tensor-core MMAs (3xTF32: hi*hi + lo*hi + hi*lo with fp32 accumulation, the same scheme the
// input-projection GEMMs use), issued as warp-level mma.sync.m16n8k8 from the group's four warps.  The operands live
// in shared memory in FRAGMENT-MAJOR order, so that every operand fetch is one conflict-free 128-bit load per lane:
//   fwd  A = h_{t-1} [16 rows x H]   : exchanged between CTAs directly in fragment order [H/8][lane][a0..a3]
//        B = W slice [H x 4UB]       : [H/8][pair][lane][b0,b1 of tile0 | b0,b1 of tile1]; a "pair" = 4 units,
//                                      tile0 = gates (i,f), tile1 = gates (g,o), column 2*tig+{0,1} <-> unit tig,
//                                      so lane (gid,tig) ends up with all 4 gates of unit tig for rows gid, gid+8
//                                      and finishes the pointwise cell update without any shuffle
//   bwd  A = dG [16 rows x 4UB]      : written by the pointwise pass in fragment order [4UB/8][lane][a0..a3]
//        B = W slice [4UB x H]       : [H/32][4UB/8][lane][4 tiles x (b0,b1)]
// MMA fragment coordinates (PTX ISA, m16n8k8 .tf32; gid = lane>>2, tig = lane&3):
//   A: a0=(gid,tig) a1=(gid+8,tig) a2=(gid,tig+4) a3=(gid+8,tig+4);  B: b0=(k=tig,n=gid) b1=(k=tig+4,n=gid)
//   D: d0=(gid,2tig) d1=(gid,2tig+1) d2=(gid+8,2tig) d3=(gid+8,2tig+1)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x) & 0xffffe000u;                   // the 10 mantissa bits TF32 keeps
    lo = __float_as_uint(x - __uint_as_float(hi));           // exact residual
}
__device__ __forceinline__ void split4(const float4& v, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    split_tf32(v.x, hi[0], lo[0]);
    split_tf32(v.y, hi[1], lo[1]);
    split_tf32(v.z, hi[2], lo[2]);
    split_tf32(v.w, hi[3], lo[3]);
}

// fwd pack: dst[dir][ub][ks = H/8][pair][lane][4];  bwd pack: dst[dir][ub][nb = H/32][ks = 4UB/8][lane][8]
__global__ void lstm_pack_mma_kernel(const float* __restrict__ w, float* __restrict__ dst, int H, int UB, int ndir,
                                     int for_bwd) {
    const int npairs = (UB + 3) / 4;
    const int nub = H / UB;
    const long long per_cta = for_bwd ? (long long)H * 4 * UB : (long long)H * npairs * 16;
    const long long n = (long long)ndir * nub * per_cta;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        long long r = i;
        const int cta = (int)(r / per_cta);
        r -= (long long)cta * per_cta;
        const int dir = cta / nub, ub = cta - dir * nub;
        int k, unit, gate;
        if (!for_bwd) {
            const int reg = (int)(r & 3);
            const int lane = (int)((r >> 2) & 31);
            const int q = (int)(r >> 7);                  // ks * npairs + pair
            const int ks = q / npairs, pair = q - ks * npairs;
            const int gid = lane >> 2, tig = lane & 3;
            const int tile = reg >> 1;                    // 0: gates i,f   1: gates g,o
            k = ks * 8 + tig + 4 * (reg & 1);
            unit = pair * 4 + (gid >> 1);
            gate = 2 * tile + (gid & 1);
        } else {
            const int f = (int)(r & 7);
            const int lane = (int)((r >> 3) & 31);
            const int q = (int)(r >> 8);                  // nb * KS2 + ks
            const int KS2 = (4 * UB) / 8;
            const int nb = q / KS2, ks = q - nb * KS2;
            const int gid = lane >> 2, tig = lane & 3;
            const int j = f >> 1;
            k = (nb * 4 + j) * 8 + gid;
            const int c = ks * 8 + tig + 4 * (f & 1);
            unit = c >> 2;
            gate = c & 3;
        }
        float v = 0.f;
        if (unit < UB) v = w[((long long)dir * 4 * H + (long long)gate * H + (ub * UB + unit)) * H + k];
        dst[i] = v;
    }
}

// ---- forward group, tensor cores: warp w of the group owns units [4w, 4w+4) of the CTA's unit block.
// NS = number of k-step parities accumulated separately: a warp carries 6*NS independent MMA accumulator chains
// (2 tiles x 3 products x NS); the dependent-issue latency of mma.sync is long enough that 6 chains leave the
// tensor pipe idle.
template <int NS>
__device__ __forceinline__ void fwd_group_mma(const LstmParams& p, int g, int gt, int dir, int bg, int ub,
                                              const float4* Wm, const float* hsg, uint64_t* full, uint64_t* done,
                                              float* xbg, uint64_t* turn) {
    const int H = p.H, UB = p.UB, T = p.T;
    const int KC = H / LSTM_NCHUNK;
    const int KSC = KC / 8;                               // k-steps per bulk-copy chunk
    const int npairs = (UB + 3) / 4;
    const int warp = gt >> 5, lane = gt & 31, gid = lane >> 2, tig = lane & 3;
    const bool has_pair = warp < npairs;
    const int u = warp * 4 + tig;
    const bool has_unit = has_pair && u < UB;
    const int ug = ub * UB + (has_unit ? u : 0);
    const int brow[2] = {p.b0 + bg * p.Bc + g * 16 + gid, p.b0 + bg * p.Bc + g * 16 + gid + 8};
    const size_t half_elems = (size_t)H * 16;
    const int chunk_stride = KC * 16 + LSTM_CHUNK_PAD;
    // where my two h values go in the NEXT step's A operand: k = ug -> k-step ug/8, column ug%8
    const size_t pub_off = ((size_t)(ug >> 3) * 32 + gid * 4 + (ug & 3)) * 4 + 2 * ((ug >> 2) & 1);
    const bool trc = (g == 0 && gt == 0);
    float c_reg[2] = {0.f, 0.f};

    for (int step = 0; step < T; ++step) {
        const int tt = dir ? (T - 1 - step) : step;
        if (trc) LSTM_TRACE(0);
        float4 gx[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            gx[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (has_unit && brow[i] < p.Bend)
                gx[i] = *reinterpret_cast<const float4*>(p.gates + ((((size_t)dir * p.B + brow[i]) * T + tt) * H + ug) * 4);
        }
        float t0[4] = {0.f, 0.f, 0.f, 0.f}, t1[4] = {0.f, 0.f, 0.f, 0.f};   // gates (i,f) / (g,o) x rows (gid, gid+8)
        if (step > 0) {
            // three independent accumulator chains per tile (hi*hi, lo*hi, hi*lo) keep the tensor pipe busy
            float d0[3 * NS][4], d1[3 * NS][4];
#pragma unroll
            for (int q = 0; q < 3 * NS; ++q)
#pragma unroll
                for (int i = 0; i < 4; ++i) d0[q][i] = d1[q][i] = 0.f;
            // the two groups alternate on the tensor pipe (see the FMA kernel): in phase they would share it AND wait
            // for their exchanges at the same time; in alternation one group's exchange hides behind the other's MMAs
            if (g == 1) mbar_wait(&turn[1], (uint32_t)((step - 1) & 1));
            else if (step >= 2) mbar_wait(&turn[0], (uint32_t)(step & 1));
            if (trc) LSTM_TRACE(2);
#pragma unroll 1
            for (int c = 0; c < LSTM_NCHUNK; ++c) {
                // every warp waits (also one without units): the wait is what keeps a warp from running a step
                // ahead and arriving twice in one phase of the group's `done` barrier
                mbar_wait(&full[c], (uint32_t)((step - 1) & 1));
                if (trc && c == 0) LSTM_TRACE(1);
                if (!has_pair) continue;
                const float4* ap = reinterpret_cast<const float4*>(hsg + (size_t)c * chunk_stride) + lane;
                const float4* wp = Wm + ((size_t)c * KSC * npairs + warp) * 32 + lane;
#pragma unroll 2
                for (int ks = 0; ks < KSC; ks += NS) {
#pragma unroll
                    for (int s = 0; s < NS; ++s) {
                        const float4 av = ap[(size_t)(ks + s) * 32];
                        const float4 wv = wp[(size_t)(ks + s) * npairs * 32];
                        uint32_t ah[4], al[4], bh[4], bl[4];
                        split4(av, ah, al);
                        split4(wv, bh, bl);
                        mma_tf32(d0[3 * s + 0], ah, bh[0], bh[1]);
                        mma_tf32(d1[3 * s + 0], ah, bh[2], bh[3]);
                        mma_tf32(d0[3 * s + 1], al, bh[0], bh[1]);
                        mma_tf32(d1[3 * s + 1], al, bh[2], bh[3]);
                        mma_tf32(d0[3 * s + 2], ah, bl[0], bl[1]);
                        mma_tf32(d1[3 * s + 2], ah, bl[2], bl[3]);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int s = NS - 1; s >= 0; --s) {        // residual products first, then the hi*hi sums
                    s0 += d0[3 * s + 1][i] + d0[3 * s + 2][i];
                    s1 += d1[3 * s + 1][i] + d1[3 * s + 2][i];
                }
#pragma unroll
                for (int s = 0; s < NS; ++s) {
                    s0 += d0[3 * s][i];
                    s1 += d1[3 * s][i];
                }
                t0[i] = s0;
                t1[i] = s1;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&turn[1 - g]);
            if (trc) LSTM_TRACE(3);
        }
        float hq[2] = {0.f, 0.f}, cq[2] = {0.f, 0.f};
        float4 gq[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            gq[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (has_unit && brow[i] < p.Bend) {
                const float ig = sigmoidf_(gx[i].x + t0[2 * i]);
                const float fg = sigmoidf_(gx[i].y + t0[2 * i + 1]);
                const float gg = tanhf(gx[i].z + t1[2 * i]);
                const float og = sigmoidf_(gx[i].w + t1[2 * i + 1]);
                const float c = fmaf(fg, c_reg[i], ig * gg);
                c_reg[i] = c;
                hq[i] = og * tanhf(c);
                cq[i] = c;
                gq[i] = make_float4(ig, fg, gg, og);
            }
        }
        if (step + 1 < T) {
            if (has_unit)
                *reinterpret_cast<float2*>(xbg + (size_t)(step & 1) * half_elems + pub_off) = make_float2(hq[0], hq[1]);
            __syncwarp();
            if (lane == 0) mbar_arrive(done);
            if (trc) LSTM_TRACE(5);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (has_unit && brow[i] < p.Bend) {
                const size_t row = ((size_t)dir * p.B + brow[i]) * T + tt;
                *reinterpret_cast<float4*>(p.gates + (row * H + ug) * 4) = gq[i];
                p.cst[row * H + ug] = cq[i];
                p.out[((size_t)brow[i] * T + tt) * (p.ndir * H) + (size_t)dir * H + ug] = hq[i];
            }
        }
    }
}

// ---- forward group, tensor cores, v2: (a) only warp 0 of the group polls the turn / chunk mbarriers, the other three
// warps are parked in a hardware named barrier - a polling warp steals issue slots from the one compute warp its
// scheduler has during the other group's turn; (b) the flat K loop is software-pipelined by hand over blocks of
// four k-steps (two register stages), so that every shared-memory load is issued a whole block (24 MMAs) before
// its first use.  Needs H % 128 == 0 (blocks of four k-steps never straddle a bulk-copy chunk).
__device__ __forceinline__ void fwd_group_mma_v2(const LstmParams& p, int g, int gt, int dir, int bg, int ub,
                                                 const float4* Wm, const float* hsg, uint64_t* full, uint64_t* done,
                                                 float* xbg, uint64_t* turn) {
    const int H = p.H, UB = p.UB, T = p.T;
    const int KS = H / 8;
    const int KSC = KS / LSTM_NCHUNK;
    const int npairs = (UB + 3) / 4;
    const int warp = gt >> 5, lane = gt & 31, gid = lane >> 2, tig = lane & 3;
    const bool has_pair = warp < npairs;
    const int u = warp * 4 + tig;
    const bool has_unit = has_pair && u < UB;
    const int ug = ub * UB + (has_unit ? u : 0);
    const int brow[2] = {p.b0 + bg * p.Bc + g * 16 + gid, p.b0 + bg * p.Bc + g * 16 + gid + 8};
    const size_t half_elems = (size_t)H * 16;
    const size_t pub_off = ((size_t)(ug >> 3) * 32 + gid * 4 + (ug & 3)) * 4 + 2 * ((ug >> 2) & 1);
    const bool trc = (g == 0 && gt == 0);
    float c_reg[2] = {0.f, 0.f};

    for (int step = 0; step < T; ++step) {
        const int tt = dir ? (T - 1 - step) : step;
        if (trc) LSTM_TRACE(0);
        float4 gx[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            gx[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (has_unit && brow[i] < p.Bend)
                gx[i] = *reinterpret_cast<const float4*>(p.gates + ((((size_t)dir * p.B + brow[i]) * T + tt) * H + ug) * 4);
        }
        float t0[4] = {0.f, 0.f, 0.f, 0.f}, t1[4] = {0.f, 0.f, 0.f, 0.f};
        if (step > 0) {
            if (warp == 0) {
                if (g == 1) mbar_wait(&turn[1], (uint32_t)((step - 1) & 1));
                else if (step >= 2) mbar_wait(&turn[0], (uint32_t)(step & 1));
                if (trc) LSTM_TRACE(2);
#pragma unroll
                for (int c = 0; c < LSTM_NCHUNK; ++c) mbar_wait(&full[c], (uint32_t)((step - 1) & 1));
                if (trc) LSTM_TRACE(1);
            }
            named_bar_sync(3 + g, LSTM_GTHREADS);
            if (has_pair) {
                float d0[3][4], d1[3][4];
#pragma unroll
                for (int q = 0; q < 3; ++q)
#pragma unroll
                    for (int i = 0; i < 4; ++i) d0[q][i] = d1[q][i] = 0.f;
                const float4* ap = reinterpret_cast<const float4*>(hsg) + lane;     // + ks*32 + chunk (1 float4 pad)
                const float4* wp = Wm + (size_t)warp * 32 + lane;                   // + ks*npairs*32
                const size_t wstride = (size_t)npairs * 32;
                int ldk = 0, ldrem = KSC, ldpad = 0;
#define LSTM_MMA_LOAD(areg, wreg)                                                   \
    {                                                                               \
        _Pragma("unroll") for (int j = 0; j < 4; ++j) {                             \
            areg[j] = ap[(size_t)(ldk + j) * 32 + ldpad];                           \
            wreg[j] = wp[(size_t)(ldk + j) * wstride];                              \
        }                                                                           \
        ldk += 4; ldrem -= 4;                                                       \
        if (ldrem == 0) { ldrem = KSC; ++ldpad; }                                   \
    }
#define LSTM_MMA_BLOCK(areg, wreg)                                                  \
    _Pragma("unroll") for (int j = 0; j < 4; ++j) {                                 \
        uint32_t ah[4], al[4], bh[4], bl[4];                                        \
        split4(areg[j], ah, al);                                                    \
        split4(wreg[j], bh, bl);                                                    \
        mma_tf32(d0[0], ah, bh[0], bh[1]);                                          \
        mma_tf32(d1[0], ah, bh[2], bh[3]);                                          \
        mma_tf32(d0[1], al, bh[0], bh[1]);                                          \
        mma_tf32(d1[1], al, bh[2], bh[3]);                                          \
        mma_tf32(d0[2], ah, bl[0], bl[1]);                                          \
        mma_tf32(d1[2], ah, bl[2], bl[3]);                                          \
    }
                float4 aA[4], wA[4], aB[4], wB[4];
                LSTM_MMA_LOAD(aA, wA)
                int ks0 = 0;
#pragma unroll 1
                for (; ks0 + 8 < KS; ks0 += 8) {
                    LSTM_MMA_LOAD(aB, wB)
                    LSTM_MMA_BLOCK(aA, wA)
                    LSTM_MMA_LOAD(aA, wA)
                    LSTM_MMA_BLOCK(aB, wB)
                }
                LSTM_MMA_LOAD(aB, wB)
                LSTM_MMA_BLOCK(aA, wA)
                LSTM_MMA_BLOCK(aB, wB)
#undef LSTM_MMA_LOAD
#undef LSTM_MMA_BLOCK
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    t0[i] = d0[0][i] + (d0[1][i] + d0[2][i]);
                    t1[i] = d1[0][i] + (d1[1][i] + d1[2][i]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&turn[1 - g]);
            if (trc) LSTM_TRACE(3);
        }
        float hq[2] = {0.f, 0.f}, cq[2] = {0.f, 0.f};
        float4 gq[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            gq[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (has_unit && brow[i] < p.Bend) {
                const float ig = sigmoidf_(gx[i].x + t0[2 * i]);
                const float fg = sigmoidf_(gx[i].y + t0[2 * i + 1]);
                const float gg = tanhf(gx[i].z + t1[2 * i]);
                const float og = sigmoidf_(gx[i].w + t1[2 * i + 1]);
                const float c = fmaf(fg, c_reg[i], ig * gg);
                c_reg[i] = c;
                hq[i] = og * tanhf(c);
                cq[i] = c;
                gq[i] = make_float4(ig, fg, gg, og);
            }
        }
        if (step + 1 < T) {
            if (has_unit)
                *reinterpret_cast<float2*>(xbg + (size_t)(step & 1) * half_elems + pub_off) = make_float2(hq[0], hq[1]);
            __syncwarp();
            if (lane == 0) mbar_arrive(done);
            if (trc) LSTM_TRACE(5);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (has_unit && brow[i] < p.Bend) {
                const size_t row = ((size_t)dir * p.B + brow[i]) * T + tt;
                *reinterpret_cast<float4*>(p.gates + (row * H + ug) * 4) = gq[i];
                p.cst[row * H + ug] = cq[i];
                p.out[((size_t)brow[i] * T + tt) * (p.ndir * H) + (size_t)dir * H + ug] = hq[i];
            }
        }
    }
}

__global__ void __launch_bounds__(LSTM_THREADS, 1) bilstm_fwd_mma_kernel(LstmParams p) {
    extern __shared__ __align__(128) unsigned char s_raw[];
    const int H = p.H, UB = p.UB, T = p.T, NH = p.NH;
    const int KC = H / LSTM_NCHUNK;
    const int npairs = (UB + 3) / 4;
    const int chunk_stride = KC * 16 + LSTM_CHUNK_PAD;
    const size_t hs_half = (size_t)LSTM_NCHUNK * chunk_stride;
    const size_t wm_vec = (size_t)H * npairs * 4;                                // float4 elements
    float4* Wm = reinterpret_cast<float4*>(s_raw);
    float* hs = reinterpret_cast<float*>(Wm + wm_vec);
    uint64_t* full = reinterpret_cast<uint64_t*>(hs + 2 * hs_half);
    uint64_t* done = full + 2 * LSTM_NCHUNK;
    uint64_t* turn = done + 2;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    int blk = blockIdx.x;
    const int ub = blk % p.nub; blk /= p.nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;
    {
        const float4* src = reinterpret_cast<const float4*>(p.whh) + ((size_t)dir * p.nub + ub) * wm_vec;
        for (size_t i = tid; i < wm_vec; i += LSTM_THREADS) Wm[i] = src[i];
    }
    if (tid == 0) {
        for (int i = 0; i < 2 * LSTM_NCHUNK; ++i) mbar_init(&full[i], 1);
        for (int i = 0; i < 2; ++i) mbar_init(&done[i], LSTM_GTHREADS / 32);
        for (int i = 0; i < 2; ++i) mbar_init(&turn[i], LSTM_GTHREADS / 32);
        mbar_fence_init();
    }
    __syncthreads();
    const size_t half_elems = (size_t)H * 16;
    float* xb = p.xbuf + ((size_t)dir * p.nbg + bg) * NH * 2 * half_elems;
    unsigned* ctr0 = p.counters + ((size_t)dir * p.nbg + bg) * NH;
    if (warp >= 2 * (LSTM_GTHREADS / 32)) {
        const int g = warp - 2 * (LSTM_GTHREADS / 32);
        if (lane == 0 && g < NH) {
            uint32_t soff[LSTM_NCHUNK], doff[LSTM_NCHUNK], bytes[LSTM_NCHUNK];
            for (int c = 0; c < LSTM_NCHUNK; ++c) {
                soff[c] = (uint32_t)((size_t)c * KC * 16);
                doff[c] = (uint32_t)((size_t)c * chunk_stride);
                bytes[c] = (uint32_t)((size_t)KC * 16 * sizeof(float));
            }
            control_loop(p, T, (unsigned)p.nub, &done[g], &full[g * LSTM_NCHUNK], ctr0 + g,
                         xb + ((size_t)g * 2 + 0) * half_elems, xb + ((size_t)g * 2 + 1) * half_elems,
                         hs + (size_t)g * hs_half, soff, doff, bytes, g == 0);
        }
        return;
    }
    const int g = tid / LSTM_GTHREADS;
    if (g >= NH) return;
    if (!(p.flags & 4) && H % 128 == 0)
        fwd_group_mma_v2(p, g, tid - g * LSTM_GTHREADS, dir, bg, ub, Wm, hs + (size_t)g * hs_half,
                         &full[g * LSTM_NCHUNK], &done[g], xb + (size_t)g * 2 * half_elems, turn);
    else if (p.mma == 2)
        fwd_group_mma<2>(p, g, tid - g * LSTM_GTHREADS, dir, bg, ub, Wm, hs + (size_t)g * hs_half,
                         &full[g * LSTM_NCHUNK], &done[g], xb + (size_t)g * 2 * half_elems, turn);
    else
        fwd_group_mma<1>(p, g, tid - g * LSTM_GTHREADS, dir, bg, ub, Wm, hs + (size_t)g * hs_half,
                         &full[g * LSTM_NCHUNK], &done[g], xb + (size_t)g * 2 * half_elems, turn);
}

// ---- backward group, tensor cores
__device__ __forceinline__ void bwd_group_mma(const LstmParams& p, int g, int gt, int dir, int bg, int ub,
                                              const float4* Wm, const float* inb, float* dgs, uint64_t* full,
                                              uint64_t* done, float* xbg, uint64_t* turn) {
    const int H = p.H, UB = p.UB, T = p.T, nub = p.nub;
    const int warp = gt >> 5, lane = gt & 31, gid = lane >> 2, tig = lane & 3;
    const int KS2 = (4 * UB) / 8;                              // k-steps of the dG . W product (UB even)
    const int NB = H / 32;                                     // batches of 4 n-tiles (32 columns of dh)
    const size_t inbox_elems = (size_t)16 * H;
    const unsigned inv_ub = (65536u + UB - 1) / UB;            // k / UB = (k * inv_ub) >> 16 for k < 65536 / UB
    // pointwise items: (row, unit) pairs of the 16 x UB tile, consecutive lanes -> consecutive units
    int it_u[2], it_b[2], it_row[2];
    bool it_ok[2], it_in[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int i = gt + j * LSTM_GTHREADS;
        it_in[j] = i < 16 * UB;
        it_b[j] = it_in[j] ? i / UB : 0;
        it_u[j] = it_in[j] ? i - it_b[j] * UB : 0;
        it_row[j] = p.b0 + bg * p.Bc + g * 16 + it_b[j];
        it_ok[j] = it_in[j] && it_row[j] < p.Bend;
    }
    float dc_reg[2] = {0.f, 0.f};
    const bool lead = (p.flags & 4) == 0;
    const bool trc = (g == 0 && gt == 0);

    for (int step = 0; step < T; ++step) {
        const int fstep = T - 1 - step;
        const int tt = dir ? (T - 1 - fstep) : fstep;
        const int tt_prev = dir ? tt + 1 : tt - 1;
        if (trc) LSTM_TRACE(0);
        float4 gtv[2];
        float ct[2], cp[2], dh[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            gtv[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            ct[j] = cp[j] = dh[j] = 0.f;
            if (it_ok[j]) {
                const int ug = ub * UB + it_u[j];
                const size_t row = ((size_t)dir * p.B + it_row[j]) * T + tt;
                gtv[j] = *reinterpret_cast<const float4*>(p.gates + (row * H + ug) * 4);
                ct[j] = p.cst[row * H + ug];
                if (fstep > 0) cp[j] = p.cst[(((size_t)dir * p.B + it_row[j]) * T + tt_prev) * H + ug];
                dh[j] = p.out[((size_t)it_row[j] * T + tt) * (p.ndir * H) + (size_t)dir * H + ug];
            }
        }
        if (step > 0) {
            if (lead) {
                // only warp 0 polls; the other warps park in a hardware barrier and leave their schedulers' issue
                // slots to the other group's MMA loop
                if (warp == 0) {
#pragma unroll
                    for (int c = 0; c < LSTM_NCHUNK; ++c) mbar_wait(&full[c], (uint32_t)((step - 1) & 1));
                }
                named_bar_sync(3 + g, LSTM_GTHREADS);
            } else {
#pragma unroll
                for (int c = 0; c < LSTM_NCHUNK; ++c) mbar_wait(&full[c], (uint32_t)((step - 1) & 1));
                __syncwarp();
            }
            if (trc) LSTM_TRACE(1);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (it_in[j]) {
                    const float* ib = inb + (size_t)it_b[j] * UB + it_u[j];
                    float s0 = 0.f, s1 = 0.f;
                    int s = 0;
                    for (; s + 1 < nub; s += 2) {
                        s0 += ib[(size_t)s * 16 * UB];
                        s1 += ib[(size_t)(s + 1) * 16 * UB];
                    }
                    if (s < nub) s0 += ib[(size_t)s * 16 * UB];
                    dh[j] += s0 + s1;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            float4 dg = make_float4(0.f, 0.f, 0.f, 0.f);
            if (it_ok[j]) {
                const float ig = gtv[j].x, fg = gtv[j].y, gg = gtv[j].z, og = gtv[j].w;
                const float tc = tanhf(ct[j]);
                const float dc = dc_reg[j] + dh[j] * og * (1.f - tc * tc);
                dg.x = dc * gg * ig * (1.f - ig);
                dg.y = dc * cp[j] * fg * (1.f - fg);
                dg.z = dc * ig * (1.f - gg * gg);
                dg.w = dh[j] * tc * og * (1.f - og);
                dc_reg[j] = dc * fg;
                const size_t row = ((size_t)dir * p.B + it_row[j]) * T + tt;
                *reinterpret_cast<float4*>(p.gates + (row * H + ub * UB + it_u[j]) * 4) = dg;
            }
            if (it_in[j]) {
                // A operand of the step GEMM, fragment order: element (row b, c = 4u + gate)
                const int b = it_b[j], u = it_u[j];
                float* d = dgs + ((size_t)(u >> 1) * 32 + (b & 7) * 4) * 4 + (b >> 3) + 2 * (u & 1);
                d[0] = dg.x; d[4] = dg.y; d[8] = dg.z; d[12] = dg.w;
            }
        }
        if (lead && warp == 0 && step + 1 < T) {                            // groups alternate on the tensor pipe
            if (g == 1) mbar_wait(&turn[1], (uint32_t)(step & 1));
            else if (step >= 1) mbar_wait(&turn[0], (uint32_t)((step - 1) & 1));
        }
        named_bar_sync(1 + g, LSTM_GTHREADS);                              // dG tile complete (and turn acquired)
        if (step + 1 < T) {
            if (!lead) {
                if (g == 1) mbar_wait(&turn[1], (uint32_t)(step & 1));
                else if (step >= 1) mbar_wait(&turn[0], (uint32_t)((step - 1) & 1));
            }
            float* outbase = xbg + (size_t)(step & 1) * nub * inbox_elems;
            if (trc) LSTM_TRACE(2);
            const float4* ap = reinterpret_cast<const float4*>(dgs) + lane;
            for (int nb = warp; nb < NB; nb += LSTM_GTHREADS / 32) {
                float d[4][3][4];
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int q = 0; q < 3; ++q)
#pragma unroll
                        for (int i = 0; i < 4; ++i) d[j][q][i] = 0.f;
                const float4* wp = Wm + ((size_t)nb * KS2 * 32 + lane) * 2;
#pragma unroll 2
                for (int ks = 0; ks < KS2; ++ks) {
                    const float4 av = ap[(size_t)ks * 32];
                    const float4 w01 = wp[(size_t)ks * 64], w23 = wp[(size_t)ks * 64 + 1];
                    uint32_t ah[4], al[4], bh[4], bl[4];
                    split4(av, ah, al);
                    split4(w01, bh, bl);
                    mma_tf32(d[0][0], ah, bh[0], bh[1]);
                    mma_tf32(d[1][0], ah, bh[2], bh[3]);
                    mma_tf32(d[0][1], al, bh[0], bh[1]);
                    mma_tf32(d[1][1], al, bh[2], bh[3]);
                    mma_tf32(d[0][2], ah, bl[0], bl[1]);
                    mma_tf32(d[1][2], ah, bl[2], bl[3]);
                    split4(w23, bh, bl);
                    mma_tf32(d[2][0], ah, bh[0], bh[1]);
                    mma_tf32(d[3][0], ah, bh[2], bh[3]);
                    mma_tf32(d[2][1], al, bh[0], bh[1]);
                    mma_tf32(d[3][1], al, bh[2], bh[3]);
                    mma_tf32(d[2][2], ah, bl[0], bl[1]);
                    mma_tf32(d[3][2], ah, bl[2], bl[3]);
                }
                // scatter to the destination inboxes: element (dst, src = ub, row, unit'); UB even -> float2
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int k = (nb * 4 + j) * 8 + 2 * tig;
                    const int dst = (int)(((unsigned)k * inv_ub) >> 16);
                    const int uu = k - dst * UB;
                    float* o = outbase + (((size_t)dst * nub + ub) * 16 + gid) * UB + uu;
                    const float v0 = d[j][0][0] + (d[j][1][0] + d[j][2][0]);
                    const float v1 = d[j][0][1] + (d[j][1][1] + d[j][2][1]);
                    const float v2 = d[j][0][2] + (d[j][1][2] + d[j][2][2]);
                    const float v3 = d[j][0][3] + (d[j][1][3] + d[j][2][3]);
                    *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
                    *reinterpret_cast<float2*>(o + (size_t)8 * UB) = make_float2(v2, v3);
                }
            }
            if (trc) LSTM_TRACE(3);
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&turn[1 - g]);
                mbar_arrive(done);
            }
            if (trc) LSTM_TRACE(5);
        }
    }
}

__global__ void __launch_bounds__(LSTM_THREADS, 1) bilstm_bwd_mma_kernel(LstmParams p) {
    extern __shared__ __align__(128) unsigned char s_raw[];
    const int H = p.H, UB = p.UB, Bc = p.Bc, T = p.T, nub = p.nub, NH = p.NH;
    float* Wr = reinterpret_cast<float*>(s_raw);
    float* inbox = Wr + (size_t)4 * UB * H;
    float* dGs = inbox + (size_t)Bc * H;
    uint64_t* full = reinterpret_cast<uint64_t*>(dGs + (size_t)4 * UB * Bc);
    uint64_t* done = full + 2 * LSTM_NCHUNK;
    uint64_t* turn = done + 2;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    int blk = blockIdx.x;
    const int ub = blk % nub; blk /= nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;
    {
        const float4* src = reinterpret_cast<const float4*>(p.whh) + ((size_t)dir * nub + ub) * (size_t)H * UB;
        float4* dst = reinterpret_cast<float4*>(Wr);
        for (int i = tid; i < H * UB; i += LSTM_THREADS) dst[i] = src[i];
    }
    if (tid == 0) {
        for (int i = 0; i < 2 * LSTM_NCHUNK; ++i) mbar_init(&full[i], 1);
        for (int i = 0; i < 2; ++i) mbar_init(&done[i], LSTM_GTHREADS / 32);
        for (int i = 0; i < 2; ++i) mbar_init(&turn[i], LSTM_GTHREADS / 32);
        mbar_fence_init();
    }
    __syncthreads();
    const size_t inbox_elems = (size_t)16 * H;
    float* xb = p.xbuf + ((size_t)dir * p.nbg + bg) * NH * 2 * (size_t)nub * inbox_elems;
    unsigned* ctr0 = p.counters + ((size_t)dir * p.nbg + bg) * NH;
    const int SC = (nub + LSTM_NCHUNK - 1) / LSTM_NCHUNK;
    if (warp >= 2 * (LSTM_GTHREADS / 32)) {
        const int g = warp - 2 * (LSTM_GTHREADS / 32);
        if (lane == 0 && g < NH) {
            uint32_t off[LSTM_NCHUNK], bytes[LSTM_NCHUNK];
            for (int c = 0; c < LSTM_NCHUNK; ++c) {
                const int s0 = min(nub, c * SC), s1 = min(nub, s0 + SC);
                off[c] = (uint32_t)((size_t)s0 * 16 * UB);
                bytes[c] = (uint32_t)((size_t)(s1 - s0) * 16 * UB * sizeof(float));
            }
            control_loop(p, T, (unsigned)nub, &done[g], &full[g * LSTM_NCHUNK], ctr0 + g,
                         xb + (((size_t)g * 2 + 0) * nub + ub) * inbox_elems,
                         xb + (((size_t)g * 2 + 1) * nub + ub) * inbox_elems, inbox + (size_t)g * inbox_elems, off, off,
                         bytes, g == 0);
        }
        return;
    }
    const int g = tid / LSTM_GTHREADS;
    if (g >= NH) return;
    bwd_group_mma(p, g, tid - g * LSTM_GTHREADS, dir, bg, ub, reinterpret_cast<const float4*>(Wr),
                  inbox + (size_t)g * inbox_elems, dGs + (size_t)g * 4 * UB * 16, &full[g * LSTM_NCHUNK], &done[g],
                  xb + (size_t)g * 2 * nub * inbox_elems, turn);
}

// ------------------------------------------------------------------------------------------
__global__ void lstm_cell_fwd_kernel(const float* __restrict__ pre, const float* __restrict__ c_prev,
                                     float* __restrict__ gates, float* __restrict__ c, float* __restrict__ h, int B,
                                     int H) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H) return;
    const int b = i / H, j = i - b * H;
    const float* pr = pre + (size_t)b * 4 * H;
    const float ig = sigmoidf_(pr[j]), fg = sigmoidf_(pr[H + j]), gg = tanhf(pr[2 * H + j]),
                og = sigmoidf_(pr[3 * H + j]);
    const float cn = fmaf(fg, c_prev[i], ig * gg);
    float* gr = gates + (size_t)b * 4 * H;
    gr[j] = ig; gr[H + j] = fg; gr[2 * H + j] = gg; gr[3 * H + j] = og;
    c[i] = cn;
    h[i] = og * tanhf(cn);
}

__global__ void lstm_cell_bwd_kernel(const float* __restrict__ gates, const float* __restrict__ c_prev,
                                     const float* __restrict__ c, const float* __restrict__ dh,
                                     const float* __restrict__ dc_next, float* __restrict__ dpre,
                                     float* __restrict__ dc_prev, int B, int H) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H) return;
    const int b = i / H, j = i - b * H;
    const float* gr = gates + (size_t)b * 4 * H;
    const float ig = gr[j], fg = gr[H + j], gg = gr[2 * H + j], og = gr[3 * H + j];
    const float tc = tanhf(c[i]);
    const float dhv = dh[i];
    const float dc = (dc_next ? dc_next[i] : 0.f) + dhv * og * (1.f - tc * tc);
    float* dp = dpre + (size_t)b * 4 * H;
    dp[j] = dc * gg * ig * (1.f - ig);
    dp[H + j] = dc * c_prev[i] * fg * (1.f - fg);
    dp[2 * H + j] = dc * ig * (1.f - gg * gg);
    dp[3 * H + j] = dhv * tc * og * (1.f - og);
    dc_prev[i] = dc * fg;
}

// ------------------------------------------------------------------------------------------
struct Plan {
    int UB, Bc, nub, nbg, ctas, NH, R, mma;
    int Bsub, nsplit;    // the batch is processed as nsplit consecutive launches of <= Bsub rows
    size_t smem_fwd, smem_bwd, pack_bytes, xbuf_fwd_bytes, xbuf_bwd_bytes;
};

#ifndef LSTM_UMMA_BWD_DEFAULT
#define LSTM_UMMA_BWD_DEFAULT 1
#endif
static int g_lstm_flags = 0;  // experiment switches, see LstmParams::flags (set through the upper bits of the mode)
static int g_lstm_mode = 0;   // 0: wgmma (lstm_umma.cu) when the shape allows, else mma.sync, else fp32 FMA;
                              // 1: always the fp32-FMA kernels, 2: mma.sync with 6 instead of 12 accumulator chains
                              // (measurement only), 3: never wgmma (the mma.sync generation, for A/B comparisons)

static int halves_for(int Bc) { return (Bc % 8 == 0) ? 2 : 1; }
static int rows_for(int Bc) { return ((Bc / halves_for(Bc)) % 8 == 0) ? 8 : 4; }
static size_t smem_fwd_bytes(int H, int UB, int Bc) {
    const int Bh = Bc / halves_for(Bc);
    return (size_t)H * UB * 16 + 2 * ((size_t)H * Bh + LSTM_NCHUNK * LSTM_CHUNK_PAD) * 4 + (2 * LSTM_NCHUNK + 4) * 8 + 128;
}
static size_t smem_bwd_bytes(int H, int UB, int Bc) {
    return (size_t)4 * UB * H * 4 + (size_t)Bc * H * 4 + (size_t)4 * UB * Bc * 4 + (2 * LSTM_NCHUNK + 4) * 8 + 128;
}
static size_t smem_fwd_mma_bytes(int H, int UB) {
    const int npairs = (UB + 3) / 4;
    return (size_t)H * npairs * 64 + 2 * ((size_t)H * 16 + LSTM_NCHUNK * LSTM_CHUNK_PAD) * 4 + (2 * LSTM_NCHUNK + 4) * 8 + 128;
}

// One launch over B rows: every (direction, batch-group, unit-block) CTA must be co-resident.
static int plan_one(int B, int H, int ndir, Plan* out) {
    const int sms = sm_count();
    const size_t smem_cap = (size_t)max_optin_smem();
    long long best_cost = -1;
    Plan best{};
    for (int UB = 1; UB <= H; ++UB) {
        if (H % UB) continue;
        for (int Bc = 4; Bc <= 64; Bc += 4) {
            const int NH = halves_for(Bc);
            const int R = rows_for(Bc);
            if (UB * (Bc / NH / R) > LSTM_MAX_TILES) continue;   // register tiles per group
            const int nbg = (B + Bc - 1) / Bc;
            const int nub = H / UB;
            const int ctas = ndir * nbg * nub;
            if (ctas > sms) continue;
            const size_t sf = smem_fwd_bytes(H, UB, Bc), sb = smem_bwd_bytes(H, UB, Bc);
            if (sf > smem_cap || sb > smem_cap) continue;
            // bulk copies need 16-B multiples
            if (((size_t)(H / LSTM_NCHUNK) * (Bc / NH) * 4) % 16) continue;
            if (((size_t)(Bc / NH) * UB * 4) % 16) continue;
            if ((long long)ndir * nbg * NH * 4 > LSTM_COUNTER_BYTES - 64) continue;
            // cost: per-CTA FMA work per step; tie-break on the state tile pulled per step
            const long long cost = (long long)UB * Bc * 1000 + Bc;
            if (best_cost < 0 || cost < best_cost) {
                best_cost = cost;
                best.UB = UB; best.Bc = Bc; best.nub = nub; best.nbg = nbg; best.ctas = ctas; best.NH = NH; best.R = R;
                best.smem_fwd = sf; best.smem_bwd = sb; best.mma = 0;
            }
        }
    }
    // Tensor-core step GEMMs: a group's batch half is exactly one 16-row MMA tile (Bc = 32, two groups), the unit
    // block is even and <= 16 (4 warps x 4 units).  The MMA path sustains > 2x the MACs of the FMA loops, so it is
    // taken whenever its per-CTA work is not more than 1.5x that of the best FMA decomposition.
    if (g_lstm_mode != 1 && H % 32 == 0 && H <= 2048) {
        long long best_mma = -1;
        Plan bm{};
        for (int UB = 2; UB <= 16 && UB <= H; UB += 2) {
            if (H % UB) continue;
            const int Bc = 32, NH = 2;
            const int nbg = (B + Bc - 1) / Bc;
            const int nub = H / UB;
            const int ctas = ndir * nbg * nub;
            if (ctas > sms) continue;
            const size_t sf = smem_fwd_mma_bytes(H, UB), sb = smem_bwd_bytes(H, UB, Bc);
            if (sf > smem_cap || sb > smem_cap) continue;
            if ((long long)ndir * nbg * NH * 4 > LSTM_COUNTER_BYTES - 64) continue;
            const long long cost = (long long)UB * Bc * 1000 + Bc;
            if (best_mma < 0 || cost < best_mma) {
                best_mma = cost;
                bm.UB = UB; bm.Bc = Bc; bm.nub = nub; bm.nbg = nbg; bm.ctas = ctas; bm.NH = NH; bm.R = 8;
                bm.smem_fwd = sf; bm.smem_bwd = sb;
                bm.mma = (g_lstm_mode != 2 && (H / 32) % 2 == 0) ? 2 : 1;   // 2: twelve accumulator chains per warp
            }
        }
        if (best_mma >= 0 && (best_cost < 0 || 2 * best_mma <= 3 * best_cost)) {
            best = bm;
            best_cost = best_mma;
        }
    }
    if (best_cost < 0) return -2;
    *out = best;
    return 0;
}

static int make_plan(int B, int H, int ndir, Plan* out) {
    if (H % 16 != 0) return -1;  // K chunks (H/4) and the 16-wide k tiles of the backward pass
    // batches whose CTAs cannot all be co-resident run as consecutive launches over row blocks
    Plan best{};
    int rc = -2;
    for (int n = 1; n <= B; ++n) {
        const int Bs = (B + n - 1) / n;
        rc = plan_one(Bs, H, ndir, &best);
        if (rc == 0) {
            best.Bsub = Bs;
            best.nsplit = (B + Bs - 1) / Bs;
            break;
        }
        if (Bs <= 4) break;
    }
    if (rc != 0) return rc;
    const int npairs = (best.UB + 3) / 4;
    best.pack_bytes = (size_t)ndir * 4 * H * H * sizeof(float);
    if (best.mma) {
        const size_t pf = (size_t)ndir * best.nub * H * npairs * 16 * sizeof(float);
        if (pf > best.pack_bytes) best.pack_bytes = pf;
    }
    best.xbuf_fwd_bytes = (size_t)ndir * best.nbg * 2 * (size_t)H * best.Bc * sizeof(float);
    best.xbuf_bwd_bytes = (size_t)ndir * best.nbg * 2 * (size_t)best.nub * best.Bc * H * sizeof(float);
    *out = best;
    return 0;
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static long long* g_trace = nullptr;   // debug only: set through b200asr_debug_set_lstm_trace

}  // namespace b200asr

using namespace b200asr;

extern "C" size_t b200asr_bilstm_workspace_bytes(int B, int T, int H, int ndir) {
    (void)T;
    Plan pl;
    if (make_plan(B, H, ndir, &pl) != 0) return 0;
    const size_t x = pl.xbuf_fwd_bytes > pl.xbuf_bwd_bytes ? pl.xbuf_fwd_bytes : pl.xbuf_bwd_bytes;
    const size_t legacy = align_up(pl.pack_bytes, 256) + align_up(x, 256) + LSTM_COUNTER_BYTES /*counters + err flag*/;
    const size_t um = lstm_umma_workspace_bytes(B, H, ndir);
    return legacy > um ? legacy : um;
}

extern "C" int b200asr_bilstm_uses_tcgen05(int B, int H, int ndir) {
    return (g_lstm_mode == 0 && lstm_umma_fwd_supported(B, H, ndir)) ? 1 : 0;
}

extern "C" int b200asr_bilstm_plan(int B, int H, int ndir, int* unit_block, int* batch_block, int* n_ctas) {
    Plan pl;
    const int rc = make_plan(B, H, ndir, &pl);
    B200_REQUIRE(rc == 0, "bilstm_plan: no feasible decomposition for B=%d H=%d ndir=%d (H must be a multiple of 16)",
                 B, H, ndir);
    if (unit_block) *unit_block = pl.UB;
    if (batch_block) *batch_block = pl.Bc;
    if (n_ctas) *n_ctas = pl.ctas;
    return B200_OK;
}

extern "C" int b200asr_bilstm_uses_tensor_cores(int B, int H, int ndir) {
    Plan pl;
    if (make_plan(B, H, ndir, &pl) != 0) return -1;
    return pl.mma ? 1 : 0;
}

static int bilstm_run(bool bwd, float* gates, const float* w_hh, float* cstate, float* out_or_dout, int B, int T,
                      int H, int ndir, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    B200_REQUIRE(gates && w_hh && cstate && out_or_dout && workspace, "bilstm: null pointer");
    B200_REQUIRE(B > 0 && T > 0 && H > 0 && (ndir == 1 || ndir == 2), "bilstm: bad sizes B=%d T=%d H=%d ndir=%d", B, T,
                 H, ndir);
    Plan pl;
    B200_REQUIRE(make_plan(B, H, ndir, &pl) == 0,
                 "bilstm: no feasible decomposition for B=%d H=%d ndir=%d (H must be a multiple of 16)", B, H, ndir);
    B200_REQUIRE(workspace_bytes >= b200asr_bilstm_workspace_bytes(B, T, H, ndir), "bilstm: workspace too small");
    if (!bwd && g_lstm_mode == 0 && lstm_umma_fwd_supported(B, H, ndir))
        return lstm_umma_fwd(gates, w_hh, cstate, out_or_dout, B, T, H, ndir, workspace, workspace_bytes,
                             (g_lstm_flags & 8) ? nullptr : g_trace, g_lstm_flags >> 4, stream);
    // flag bit 5 (mode 512) toggles the backward between the wgmma kernel and the mma.sync generation
    if (bwd && g_lstm_mode == 0 && (((g_lstm_flags & 32) != 0) != (LSTM_UMMA_BWD_DEFAULT != 0)) &&
        lstm_umma_bwd_supported(B, H, ndir, g_lstm_flags >> 4))
        return lstm_umma_bwd(gates, w_hh, cstate, out_or_dout, B, T, H, ndir, workspace, workspace_bytes,
                             (g_lstm_flags & 8) ? g_trace : nullptr, g_lstm_flags >> 4, stream);
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    float* packed = reinterpret_cast<float*>(ws);
    const size_t xoff = align_up(pl.pack_bytes, 256);
    const size_t xbytes = pl.xbuf_fwd_bytes > pl.xbuf_bwd_bytes ? pl.xbuf_fwd_bytes : pl.xbuf_bwd_bytes;
    float* xbuf = reinterpret_cast<float*>(ws + xoff);
    unsigned* counters = reinterpret_cast<unsigned*>(ws + xoff + align_up(xbytes, 256));
    int* err_flag = reinterpret_cast<int*>(counters + (LSTM_COUNTER_BYTES / 4 - 4));

    {
        const long long n = (long long)(pl.pack_bytes / sizeof(float));
        int blocks = (int)((n + 255) / 256);
        if (blocks > 4096) blocks = 4096;
        if (pl.mma) lstm_pack_mma_kernel<<<blocks, 256, 0, stream>>>(w_hh, packed, H, pl.UB, ndir, bwd ? 1 : 0);
        else lstm_pack_kernel<<<blocks, 256, 0, stream>>>(w_hh, packed, H, pl.UB, ndir, bwd ? 1 : 0);
        B200_LAUNCH_CHECK("lstm_pack_kernel");
    }
    LstmParams p;
    p.gates = gates; p.whh = packed; p.cst = cstate; p.out = out_or_dout; p.xbuf = xbuf; p.counters = counters;
    p.err_flag = err_flag; p.B = B; p.T = T; p.H = H; p.ndir = ndir; p.UB = pl.UB; p.Bc = pl.Bc; p.nub = pl.nub;
    p.nbg = pl.nbg; p.NH = pl.NH; p.R = pl.R; p.mma = pl.mma; p.flags = g_lstm_flags;
    p.trace = (bwd == ((g_lstm_flags & 8) != 0)) ? g_trace : nullptr;   // flag bit 3: trace the backward kernel
    const void* fn = !pl.mma ? (bwd ? (const void*)bilstm_bwd_kernel : (const void*)bilstm_fwd_kernel)
                             : (bwd ? (const void*)bilstm_bwd_mma_kernel : (const void*)bilstm_fwd_mma_kernel);
    const size_t smem = bwd ? pl.smem_bwd : pl.smem_fwd;
    B200_REQUIRE(smem <= (size_t)max_optin_smem(), "bilstm: %zu B of shared memory exceed the device limit", smem);
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, LSTM_THREADS, smem));
    B200_REQUIRE((long long)per_sm * sm_count() >= pl.ctas, "bilstm: %d CTAs cannot be co-resident (%d/SM x %d SMs)",
                 pl.ctas, per_sm, sm_count());
    for (int sp = 0; sp < pl.nsplit; ++sp) {
        p.b0 = sp * pl.Bsub;
        p.Bend = p.b0 + pl.Bsub < B ? p.b0 + pl.Bsub : B;
        B200_CUDA(cudaMemsetAsync(counters, 0, LSTM_COUNTER_BYTES, stream));
        void* args[] = {&p};
        B200_CUDA(cudaLaunchCooperativeKernel(fn, dim3(pl.ctas), dim3(LSTM_THREADS), args, smem, stream));
        count_launch();
    }
    return B200_OK;
}

extern "C" void b200asr_debug_set_lstm_trace(long long* device_buffer) { g_trace = device_buffer; }
extern "C" void b200asr_debug_set_lstm_mode(int mode) {
    g_lstm_mode = mode & 3;
    g_lstm_flags = mode >> 4;
}

extern "C" int b200asr_bilstm_fwd(float* gates, const float* w_hh, float* cstate, float* out, int B, int T, int H,
                                  int ndir, void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    return bilstm_run(false, gates, w_hh, cstate, out, B, T, H, ndir, workspace, workspace_bytes,
                      (cudaStream_t)stream);
}

extern "C" int b200asr_bilstm_bwd(float* gates, const float* w_hh, const float* cstate, const float* dout, int B,
                                  int T, int H, int ndir, void* workspace, size_t workspace_bytes,
                                  b200asr_stream stream) {
    return bilstm_run(true, gates, w_hh, const_cast<float*>(cstate), const_cast<float*>(dout), B, T, H, ndir,
                      workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_lstm_cell_fwd(const float* preact, const float* c_prev, float* gates, float* c, float* h,
                                     int B, int H, b200asr_stream stream) {
    B200_REQUIRE(preact && c_prev && gates && c && h, "lstm_cell_fwd: null pointer");
    B200_REQUIRE(B > 0 && H > 0, "lstm_cell_fwd: bad sizes");
    const int n = B * H;
    lstm_cell_fwd_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(preact, c_prev, gates, c, h, B, H);
    B200_LAUNCH_CHECK("lstm_cell_fwd_kernel");
    return B200_OK;
}

extern "C" int b200asr_lstm_cell_bwd(const float* gates, const float* c_prev, const float* c, const float* dh,
                                     const float* dc_next, float* dpreact, float* dc_prev, int B, int H,
                                     b200asr_stream stream) {
    B200_REQUIRE(gates && c_prev && c && dh && dpreact && dc_prev, "lstm_cell_bwd: null pointer");
    B200_REQUIRE(B > 0 && H > 0, "lstm_cell_bwd: bad sizes");
    const int n = B * H;
    lstm_cell_bwd_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(gates, c_prev, c, dh, dc_next, dpreact,
                                                                          dc_prev, B, H);
    B200_LAUNCH_CHECK("lstm_cell_bwd_kernel");
    return B200_OK;
}
