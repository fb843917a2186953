// K7 on the Hopper tensor cores: the persistent BiLSTM recurrence with the step GEMM issued as warpgroup MMAs (wgmma,
// f16 operands in shared memory, fp32 accumulators in registers) instead of warp-level mma.sync.  Same CTA
// decomposition and the same cross-SM exchange protocol as csrc/lstm.cu (one CTA per (direction, batch group of 32
// rows, unit block), W_hh slice resident in shared memory for all T steps, per-step release/acquire counter + 1-D bulk
// copies of the next state).
//
// fp32 parity on a 16-bit tensor-core path - the "2 x 2 block" split product.  Every fp32 operand x is held as two
// fp16 numbers  x = hi + lo / 2048,  hi = fp16(x),  lo = fp16((x - hi) * 2048)  (22+ significant bits; h in (-1,1) and
// recurrent weights are far inside the fp16 range).  The step product h . W^T then needs hi.hi + (hi.lo + lo.hi)/2048.
// Because a single CTA only has 32 batch rows, the M = 64 of a warpgroup MMA has room to spare, so the hi and lo parts
// are STACKED along M and N:
//        A = [ h_hi ; h_lo ]  (M = 64 rows)        B = [ W_hi ; W_lo ]  (N = 8*UB rows),   both K-major over k = 0..H-1
// and one MMA per 16 values of k produces all four blocks hi.hi | hi.lo / lo.hi | lo.lo of D.  The epilogue adds
// D[hi,hi] + (D[hi,lo] + D[lo,hi]) / 2048  (lo.lo is below fp32 resolution and dropped).
// Row / column orders are chosen so that no shuffle or shared-memory round trip is needed after the MMA:
//   A rows  : warp q of a warpgroup (rows 16q..16q+15) = [hi of batch rows 8q..8q+7 ; lo of the same 8 rows]
//   B rows  : warpgroup j owns rows 32j..32j+31 = [hi | lo] x column groups (gates i,f | g,o) x (unit 4j + tq, gate e)
//   so thread (r = lane/4, tq = lane%4) of warp q in warpgroup j receives, in its 16 accumulator registers, the hi row
//   AND the lo row of batch row 8q+r for all four gates of unit 4j + tq, against W_hi and W_lo: one LSTM cell per thread.
// The state exchange moves the next A operand between CTAs already in its shared-memory image (fp16 hi/lo, K-major,
// 128-byte swizzle) and is pipelined per K ATOM (64 values of k = the hidden units of 64/UB producer CTAs): every
// epilogue warp releases its stores with one red.release on the counter of the atom(s) its units belong to; lane a of
// the consumer's control warp polls counter a and pulls atom a with one 8 KB bulk copy as soon as ITS producers are
// done, and the warpgroups issue the four MMAs of an atom when it lands - the slowest producer, the copies and the MMAs
// of one step overlap instead of running back to back.  No CTA-wide barrier, fence or grid-wide counter in the loop.
//
// Reference behaviour restated: torch.nn.LSTM as called from the reference's src/module.py:112-113,129-132 (single
// layer, batch_first, zero initial state, run over the zero-padded frames, gates i,f,g,o).
#include <cuda_fp16.h>
#include "common.cuh"
#include "wgmma.cuh"
#include "lstm_umma.h"

namespace b200asr {
namespace {

constexpr int UL_BC = 32;                 // batch rows per CTA (A operand: 32 hi rows + 32 lo rows = M 64)
constexpr int UL_MAX_CTRL = 8;            // control warps (each owns every UL_MAX_CTRL-th K atom)
constexpr int UL_ATOM_A = 64 * 128;       // bytes of one K atom (64 values of k) of the A operand
constexpr int UL_MAX_ATOMS = 16;
constexpr int UL_COUNTER_BYTES = 4096;

struct UlParams {
    float* gates;          // [ndir][B][T][H][4]  in: x.W_ih^T + b (gate-interleaved), out: activated gates (stash)
    const uint8_t* wpack;  // [ndir][nub] shared-memory images of the B operand
    float* cst;            // [ndir][B][T][H]
    float* out;            // [B][T][ndir*H]
    uint8_t* xbuf;         // [ndir][nbg][2] images of the A operand
    unsigned* counters;    // [ndir][nbg]
    int* err_flag;
    long long* trace;
    int B, T, H, ndir, UB, nub, nbg, NA, NC, flags;
    int b0, Bend;
};

__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void red_relaxed_add_u32(unsigned* p, unsigned v) {
    asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Consumer side of the exchange.  The producer orders its data stores before the flag with a gpu-scope fence; the
// consumer polls the flag with RELAXED gpu-scope loads (served at the L2 coherence point) and then only ISSUES A BULK
// COPY, whose reads are performed by the TMA unit at L2 - this thread never reads the data through its own L1, and the
// copy is control-dependent on the polled value.  `strict` adds the formal acquire (one more L2 round trip) and the
// generic->async proxy fence of the PTX memory model; both variants are tested.
__device__ __forceinline__ void ul_spin_until(const unsigned* ctr, unsigned target, int* err_flag, bool strict = false) {
    const long long t0 = clock64();
    while (ld_relaxed_u32(ctr) < target) {
        if (clock64() - t0 > (1LL << 33)) {  // ~4 s: a peer died; abort instead of hanging the GPU
            *err_flag = 1;
            __threadfence_system();
            __trap();
        }
    }
    if (strict) {
        (void)ld_acquire_u32(ctr);
        fence_proxy_async();
    }
}
// ---- "data is the flag" exchange (UL_POLL kernels) ----------------------------------------------------------------
// The exchange buffers start out filled with a bit pattern that a real value never takes (fp16 0xFFFF / fp32
// 0xFFFFFFFF: NaNs that arithmetic does not produce).  A producer just STORES its slice; a consumer polls the data with
// relaxed gpu-scope loads (served at L2) until no poison is left, so a step's hand-over costs one store -> L2 -> load
// round trip instead of  fence -> flag -> poll -> bulk copy.  Buffers rotate over UL_NBUF steps; the producer re-poisons
// its slice of the buffer that will be written again UL_NBUF-2 steps later - at that point every consumer is provably
// done with it (they all published the step after reading it).
constexpr int UL_NBUF = 8;
#ifndef UL_POLL_FWD_DEFAULT
#define UL_POLL_FWD_DEFAULT 0     // 1 once the polling exchange of the forward kernel is the validated default
#endif
#ifndef UL_POLL_BWD_DEFAULT
#define UL_POLL_BWD_DEFAULT 1
#endif
__device__ __forceinline__ uint4 ld_relaxed_v4(const void* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float ld_relaxed_f32(const float* p) {
    float v;
    asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_v2(void* p, uint32_t a, uint32_t b) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void st_relaxed_b16(void* p, unsigned short a) {
    asm volatile("st.relaxed.gpu.global.u16 [%0], %1;" ::"l"(p), "h"(a) : "memory");
}
// any 16-bit half of the chunk still 0xFFFF?
__device__ __forceinline__ bool has_poison16(const uint4& v) {
    return (__vcmpeq2(v.x, 0xFFFFFFFFu) | __vcmpeq2(v.y, 0xFFFFFFFFu) | __vcmpeq2(v.z, 0xFFFFFFFFu) |
            __vcmpeq2(v.w, 0xFFFFFFFFu)) != 0u;
}
__device__ __forceinline__ void ul_watchdog(long long t0, int* err_flag) {
    if (clock64() - t0 > (1LL << 33)) {  // ~4 s: a peer died; abort instead of hanging the GPU
        *err_flag = 1;
        __threadfence_system();
        __trap();
    }
}

__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void ul_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn((x - __half2float(hi)) * 2048.f);
}

// W_hh [ndir][4H][H] (PyTorch gate-major rows) -> per-CTA shared-memory images of B = [W_hi ; W_lo]
template <int UBP>
__global__ void ul_pack_fwd_kernel(const float* __restrict__ w, uint8_t* __restrict__ dst, int H, int UB, int ndir) {
    constexpr int N = 8 * UBP, NH = 4 * UBP;
    const int nub = H / UB, NA = H / 64;
    const long long per_cta = (long long)N * H;
    const long long n_el = (long long)ndir * nub * per_cta;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_el; i += (long long)gridDim.x * blockDim.x) {
        const int cta = (int)(i / per_cta);
        const int r = (int)(i - (long long)cta * per_cta);
        const int n = r / H, k = r - n * H;
        const int dir = cta / nub, ub = cta - dir * nub;
        const int nn = n % NH;
        const int g = nn >> 3, tq = (nn >> 1) & 3, e = nn & 1;
        const int unit = (g >> 1) * 4 + tq, gate = 2 * (g & 1) + e;
        float v = 0.f;
        if (unit < UB) v = w[((long long)dir * 4 * H + (long long)gate * H + (ub * UB + unit)) * H + k];
        __half hi, lo;
        split_f16(v, hi, lo);
        uint8_t* img = dst + (size_t)cta * ((size_t)NA * N * 128);
        const int row = 32 * (g >> 1) + (n < NH ? 0 : 16) + 8 * (g & 1) + (nn & 7);   // warpgroup g/2: [hi | lo] x (if | go)
        const uint32_t off = (uint32_t)(k >> 6) * (N * 128) + wgmma::sw128_offset(row, (k & 63) * 2);
        *reinterpret_cast<__half*>(img + off) = (n < NH) ? hi : lo;
    }
}

#define UL_TRACE(slot) \
    do { if (p.trace && blockIdx.x == 0) p.trace[(size_t)step * 16 + (slot)] = clock64(); } while (0)

// Warp roles: warps [0, UBP) MMA + epilogue / pointwise - UBP/4 warpgroups; warp w is warp q = w % 4 of warpgroup
// j = w / 4 (the unit quad), i.e. ONE cell (batch row 8q + lane/4, unit 4j + lane%4) per thread; warp UBP = publisher
// (one lane: ONE gpu-scope fence + release per CTA and step, after the epilogue warps arrived on `pub`); warps
// UBP+1 .. UBP+NC = control, one lane each, control warp c owns K atoms c, c+NC, ...
template <int UBP, bool POLL>
__global__ void __launch_bounds__(32 * (UBP + 1 + UL_MAX_CTRL), 1) bilstm_fwd_umma_kernel(UlParams p) {
    constexpr int N = 8 * UBP;            // B operand rows (gate columns, hi + lo copies)
    extern __shared__ __align__(1024) uint8_t smem[];
    const int H = p.H, T = p.T, NA = p.NA, UB = p.UB;
    uint8_t* sA = smem;
    uint8_t* sB = smem + (size_t)NA * UL_ATOM_A;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + (size_t)NA * N * 128);    // [UL_MAX_ATOMS]
    uint64_t* mma_done = full + UL_MAX_ATOMS;    // the MMAs of a step have read every atom of A (one arrival per warp)
    uint64_t* wload = mma_done + 1;
    uint64_t* pub = mma_done + 2;                // the epilogue warps have stored h_step
    uint64_t* landed = mma_done + 3;             // [UL_MAX_ATOMS] polling exchange: a bulk copy of the atom has landed

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NC = p.NC;
    int blk = blockIdx.x;
    const int ub = blk % p.nub; blk /= p.nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;

    if (tid == 0) {
        for (int a = 0; a < UL_MAX_ATOMS; ++a) {
            mbar_init(&full[a], 1);
            mbar_init(&landed[a], 1);
        }
        mbar_init(pub, UBP);
        mbar_init(mma_done, UBP);
        mbar_init(wload, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const size_t img_bytes = (size_t)NA * UL_ATOM_A;             // one image of the A operand
    uint8_t* xb = p.xbuf + ((size_t)dir * p.nbg + bg) * (POLL ? UL_NBUF : 2) * img_bytes;
    unsigned* ctr0 = p.counters + ((size_t)dir * p.nbg + bg) * UL_MAX_ATOMS;

    if (POLL && warp >= UBP) {
        // ------------------------------------------------------------------ loader warps (warp UBP only loads W)
        const int c = warp - UBP;                     // 0 .. UL_MAX_CTRL
        if (c == 0) {
            if (lane == 0) {
                const uint8_t* wsrc = p.wpack + ((size_t)dir * p.nub + ub) * ((size_t)NA * N * 128);
                mbar_expect_tx(wload, (uint32_t)(NA * N * 128));
                for (int a = 0; a < NA; ++a)
                    bulk_g2s(sB + (size_t)a * N * 128, wsrc + (size_t)a * N * 128, N * 128, wload);
            }
        } else {
            // loader warp c-1 owns K atoms c-1, c-1+NC, ...  Per atom and step: (1) lanes 0..7 spin on the LAST row of the
            // atom in the exchange buffer (8 chunks = a slice of every producer) until no poison is left - the data
            // itself is the flag, nobody fences; (2) lane 0 pulls the atom with ONE bulk copy; (3) the warp checks the
            // landed image for poison (a slower producer warp's rows may lag the sentinel row) and re-pulls if needed;
            // (4) the atom is released to the MMA lane.
            uint32_t nland[2] = {0u, 0u};                 // bulk copies completed per owned atom (barrier phase)
            for (int step = 0; step + 1 < T; ++step) {
                // my own MMAs of `step` (which read the atoms about to be overwritten) are done
                if (step > 0) mbar_wait(mma_done, (uint32_t)((step - 1) & 1));
                const uint8_t* img = xb + (size_t)(step % UL_NBUF) * img_bytes;
                int own = 0;
                for (int a = c - 1; a < NA; a += NC, ++own) {
                    const uint8_t* src = img + (size_t)a * UL_ATOM_A;
                    uint8_t* dst = sA + (size_t)a * UL_ATOM_A;
                    const long long t0 = clock64();
                    bool bad = true;
                    while (bad) {
                        if (lane < 8) {
                            uint4 v = ld_relaxed_v4(src + 63 * 128 + lane * 16);
                            while (has_poison16(v)) {
                                ul_watchdog(t0, p.err_flag);
                                v = ld_relaxed_v4(src + 63 * 128 + lane * 16);
                            }
                        }
                        __syncwarp();
                        if (a == 0 && lane == 0) UL_TRACE(10);
                        if (lane == 0) {
                            mbar_expect_tx(&landed[a], UL_ATOM_A);
                            bulk_g2s(dst, src, UL_ATOM_A, &landed[a]);
                        }
                        mbar_wait(&landed[a], nland[own & 1] & 1u);
                        ++nland[own & 1];
                        bool p16 = false;
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            p16 |= has_poison16(*reinterpret_cast<const uint4*>(dst + (size_t)(j * 32 + lane) * 16));
                        bad = __any_sync(0xffffffffu, p16);
                        if (bad) ul_watchdog(t0, p.err_flag);
                    }
                    __syncwarp();
                    if (lane == 0) ul_arrive(&full[a]);
                    if (a == 0 && lane == 0) UL_TRACE(11);
                    if (a == NA - 1 && lane == 0) UL_TRACE(15);
                }
            }
        }
    } else if (warp == UBP) {
        // ------------------------------------------------------------------ publisher lane
        if (lane == 0) {
            const int a0 = (ub * UB) >> 6, a1 = (ub * UB + UB - 1) >> 6;
            for (int step = 0; step + 1 < T; ++step) {
                mbar_wait(pub, (uint32_t)(step & 1));       // every epilogue warp stored its part of h_step
                UL_TRACE(8);
                fence_acq_rel_gpu();                        // their stores (observed through the mbarrier) first ...
                red_relaxed_add_u32(ctr0 + a0, 1u);         // ... then the flag(s) of the K atom(s) of my unit block
                if (a1 != a0) red_relaxed_add_u32(ctr0 + a1, 1u);
                UL_TRACE(9);
            }
        }
    } else if (warp > UBP) {
        // ------------------------------------------------------------------ control warps (one lane each)
        const int c = warp - UBP - 1;
        if (lane == 0 && c < NC) {
            if (c == 0) {
                const uint8_t* wsrc = p.wpack + ((size_t)dir * p.nub + ub) * ((size_t)NA * N * 128);
                mbar_expect_tx(wload, (uint32_t)(NA * N * 128));
                for (int a = 0; a < NA; ++a)
                    bulk_g2s(sB + (size_t)a * N * 128, wsrc + (size_t)a * N * 128, N * 128, wload);
            }
            unsigned per_step[(UL_MAX_ATOMS + 1) / 2];
            for (int i = 0, a = c; a < NA; a += NC, ++i) {
                unsigned nprod = 0;                       // producer CTAs whose units fall into atom a
                for (int u = 0; u < p.nub; ++u)
                    if ((u * UB) / 64 <= a && (u * UB + UB - 1) / 64 >= a) ++nprod;
                per_step[i] = nprod;
            }
            for (int step = 0; step + 1 < T; ++step) {
                // my own MMAs of `step` must have read the atoms before they are overwritten (they finished long
                // ago: every producer ran the same MMAs before it could publish)
                if (step > 0) mbar_wait(mma_done, (uint32_t)((step - 1) & 1));
                for (int i = 0, a = c; a < NA; a += NC, ++i) {
                    ul_spin_until(ctr0 + a, (unsigned)(step + 1) * per_step[i], p.err_flag, (p.flags & 1) != 0);
                    if (a == 0) UL_TRACE(10);
                    if (a == NA - 1) UL_TRACE(15);
                    const uint8_t* src = xb + (size_t)(step & 1) * ((size_t)NA * UL_ATOM_A) + (size_t)a * UL_ATOM_A;
                    mbar_expect_tx(&full[a], UL_ATOM_A);
                    bulk_g2s(sA + (size_t)a * UL_ATOM_A, src, UL_ATOM_A, &full[a]);
                    if (a == 0) UL_TRACE(11);
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ MMA + epilogue / pointwise warps
        const int q = warp & 3, jq = warp >> 2, r = lane >> 2, tq = lane & 3;
        const int brow = p.b0 + bg * UL_BC + 8 * q + r;
        const int unit = 4 * jq + tq;                     // my unit of the CTA's block
        const bool ok = (brow < p.Bend) && (unit < UB);
        const int ug = ub * UB + (unit < UB ? unit : 0);  // = my k in the next A operand
        const uint32_t a_base = smem_u32(sA), b_base = smem_u32(sB) + jq * (32 * 128);
        float d[16];
        const int a_row_hi = 16 * q + r, a_row_lo = 16 * q + 8 + r;
        const uint32_t pub_hi = (uint32_t)(ug >> 6) * UL_ATOM_A + wgmma::sw128_offset(a_row_hi, (ug & 63) * 2);
        const uint32_t pub_lo = (uint32_t)(ug >> 6) * UL_ATOM_A + wgmma::sw128_offset(a_row_lo, (ug & 63) * 2);
        float c_reg = 0.f;
        const bool trc = (warp == 0 && lane == 0);
        float4 st_g = make_float4(0.f, 0.f, 0.f, 0.f);
        float st_c = 0.f, st_h = 0.f;
        size_t st_row = 0, st_out = 0;
        bool st_pending = false;

        for (int step = 0; step < T; ++step) {
            const int tt = dir ? (T - 1 - step) : step;
            if (trc) UL_TRACE(0);
            const size_t rowbase = ((size_t)dir * p.B + (ok ? brow : 0)) * T + tt;
            float4 pre = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok) pre = *reinterpret_cast<const float4*>(p.gates + (rowbase * H + ug) * 4);
            if (step > 0) {
                if (step == 1) mbar_wait(wload, 0);
                wgmma::fence_operand(d);
                wgmma::fence();
                for (int a = 0; a < NA; ++a) {
                    mbar_wait(&full[a], (uint32_t)((step - 1) & 1));
                    if (trc && a == 0) UL_TRACE(1);
                    if (trc && a == NA - 1) UL_TRACE(6);
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        wgmma::mma_f16_n32(d, wgmma::desc_k_sw128(a_base + a * UL_ATOM_A + j * 32),
                                           wgmma::desc_k_sw128(b_base + a * (N * 128) + j * 32), (a | j) != 0);
                }
                wgmma::commit_group();
                if (trc) UL_TRACE(2);
                wgmma::wait_all();
                wgmma::fence_operand(d);
                __syncwarp();
                if (lane == 0) ul_arrive(mma_done);     // the control warps may overwrite the atoms of A
                if (trc) UL_TRACE(3);
                // d[0..7]: hi and lo row against W_hi, gates (i,f) then (g,o); d[8..15]: the same against W_lo
                const float *dif = d, *dgo = d + 4, *eif = d + 8, *ego = d + 12;
                if (trc) UL_TRACE(4);
                if (st_pending) {
                    *reinterpret_cast<float4*>(p.gates + (st_row * H + ug) * 4) = st_g;
                    p.cst[st_row * H + ug] = st_c;
                    p.out[st_out] = st_h;
                    st_pending = false;
                }
                const float k = 1.f / 2048.f;
                pre.x += dif[0] + (dif[2] + eif[0]) * k;
                pre.y += dif[1] + (dif[3] + eif[1]) * k;
                pre.z += dgo[0] + (dgo[2] + ego[0]) * k;
                pre.w += dgo[1] + (dgo[3] + ego[1]) * k;
            }
            const float ig = sigmoidf_(pre.x);
            const float fg = sigmoidf_(pre.y);
            const float gg = tanhf(pre.z);
            const float og = sigmoidf_(pre.w);
            const float c = fmaf(fg, c_reg, ig * gg);
            c_reg = ok ? c : 0.f;
            const float hq = ok ? og * tanhf(c) : 0.f;
            if (trc) UL_TRACE(7);
            if (step + 1 < T) {
                // publish h_step as element (A row, k = ug) of the next A operand, fp16 hi / lo
                uint8_t* dstimg = xb + (size_t)(POLL ? (step % UL_NBUF) : (step & 1)) * img_bytes;
                if (POLL) {
                    // data is the flag: plain gpu-scope stores; re-poison my slice of the buffer used UL_NBUF-2 steps on
                    uint8_t* poison = xb + (size_t)((step + UL_NBUF - 2) % UL_NBUF) * img_bytes;
                    __half hi, lo;
                    split_f16(hq, hi, lo);
                    if ((UB & 3) == 0) {
                        uint32_t wh = __half_as_ushort(hi), wl = __half_as_ushort(lo);
                        wh |= __shfl_down_sync(0xffffffffu, wh, 1) << 16;
                        wl |= __shfl_down_sync(0xffffffffu, wl, 1) << 16;
                        const uint32_t wh2 = __shfl_down_sync(0xffffffffu, wh, 2);
                        const uint32_t wl2 = __shfl_down_sync(0xffffffffu, wl, 2);
                        if (tq == 0 && unit < UB) {
                            st_relaxed_v2(poison + pub_hi, 0xFFFFFFFFu, 0xFFFFFFFFu);
                            st_relaxed_v2(poison + pub_lo, 0xFFFFFFFFu, 0xFFFFFFFFu);
                            st_relaxed_v2(dstimg + pub_hi, wh, wh2);
                            st_relaxed_v2(dstimg + pub_lo, wl, wl2);
                        }
                    } else if (unit < UB) {
                        st_relaxed_b16(poison + pub_hi, 0xFFFFu);
                        st_relaxed_b16(poison + pub_lo, 0xFFFFu);
                        st_relaxed_b16(dstimg + pub_hi, __half_as_ushort(hi));
                        st_relaxed_b16(dstimg + pub_lo, __half_as_ushort(lo));
                    }
                } else {
                    __half hi, lo;
                    split_f16(hq, hi, lo);
                    if ((UB & 3) == 0) {
                        // the four lanes of a unit quad hold k = ug .. ug+3 of the same A row: one 8-byte store each
                        // for the hi and the lo row instead of four 2-byte ones
                        uint32_t wh = __half_as_ushort(hi), wl = __half_as_ushort(lo);
                        wh |= __shfl_down_sync(0xffffffffu, wh, 1) << 16;
                        wl |= __shfl_down_sync(0xffffffffu, wl, 1) << 16;
                        const uint32_t wh2 = __shfl_down_sync(0xffffffffu, wh, 2);
                        const uint32_t wl2 = __shfl_down_sync(0xffffffffu, wl, 2);
                        if (tq == 0 && unit < UB) {
                            *reinterpret_cast<uint2*>(dstimg + pub_hi) = make_uint2(wh, wh2);
                            *reinterpret_cast<uint2*>(dstimg + pub_lo) = make_uint2(wl, wl2);
                        }
                    } else if (unit < UB) {
                        *reinterpret_cast<__half*>(dstimg + pub_hi) = hi;
                        *reinterpret_cast<__half*>(dstimg + pub_lo) = lo;
                    }
                }
                if (!POLL) {
                    __syncwarp();
                    if (lane == 0) ul_arrive(pub);
                }
                if (trc) UL_TRACE(5);
            }
            // the stash / output stores of this step are issued during the NEXT step (after its MMAs): stores
            // in flight while the publisher runs its gpu-scope fence lengthen that fence by their L2 round trip
            st_g = make_float4(ig, fg, gg, og);
            st_c = c;
            st_h = hq;
            st_row = rowbase;
            st_out = ((size_t)brow * T + tt) * (p.ndir * H) + (size_t)dir * H + ug;
            st_pending = ok;
        }
        if (st_pending) {
            *reinterpret_cast<float4*>(p.gates + (st_row * H + ug) * 4) = st_g;
            p.cst[st_row * H + ug] = st_c;
            p.out[st_out] = st_h;
        }
    }
}

// =====================================================================================================================
// Backward (BPTT) step on wgmma.  Per CTA (direction, batch group of 32 rows, unit block of UB units) and step:
//   dh = dOut[b,t] + sum_src partial_src[b, my units]          (inbox: one [32 x UB] fp32 block per source CTA)
//   pointwise -> dG[b, 4*UB] (written to the gate stash in place), dc carried in a register
//   partial_me[b, 0..H) = dG[32 x 4UB] . W_slice[4UB x H]      -> scattered to every destination CTA's inbox
// The step GEMM has K = 4*UB <= 64 (ONE 128-byte K atom) and N = H, so the tensor core is fed with
//   A1 = [ dG_hi ; dG_lo ]  and  A2 = [ 0 ; dG_hi ]   (M = 64: per warp 8 "hi" rows then 8 "lo" rows)
//   D[:, n-block] = A1 . W_hi^T + A2 . W_lo^T
// i.e. the hi rows of D hold dG_hi.W_hi and the lo rows hold dG_lo.W_hi + dG_hi.W_lo (both scaled by 2048); of every
// 256 columns, warpgroup jq accumulates columns 64jq .. 64jq+63 (2*(4UB/16) MMAs of N = 64), and the accumulator
// fragment hands every thread the (hi, lo) pair of the same (row, column).  dG has no bounded range, so every batch
// row is scaled by a power of two that brings its largest |dG| to [2^13, 2^14) before the fp16 hi/lo split; the drain
// undoes it.
template <int UB>
__global__ void ul_pack_bwd_kernel(const float* __restrict__ w, uint8_t* __restrict__ dst, int H, int ndir) {
    const int nub = H / UB;
    const long long per_cta = (long long)2 * H * 64;           // (part, n, k) elements; k < 4*UB used
    const long long n_el = (long long)ndir * nub * per_cta;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_el; i += (long long)gridDim.x * blockDim.x) {
        const int cta = (int)(i / per_cta);
        int r = (int)(i - (long long)cta * per_cta);
        const int part = r / (H * 64);
        r -= part * H * 64;
        const int n = r >> 6, k = r & 63;
        const int dir = cta / nub, ub = cta - dir * nub;
        const int u = k >> 2, g = k & 3;
        float v = 0.f;
        if (u < UB) v = w[((long long)dir * 4 * H + (long long)g * H + (ub * UB + u)) * H + n];
        __half hi, lo;
        split_f16(v, hi, lo);
        uint8_t* img = dst + (size_t)cta * ((size_t)2 * H * 128) + (size_t)part * H * 128;
        *reinterpret_cast<__half*>(img + wgmma::sw128_offset(n, k * 2)) = part ? lo : hi;
    }
}


constexpr int ULB_EPI_WARPS = 16;
constexpr int ULB_CTRL = 4;

// POLL = the "data is the flag" exchange for the backward: every fp32 partial carries the parity of its buffer
// generation in its least significant mantissa bit (2^-24 relative - below the resolution of the hi/lo product), the
// destination polls its inbox IN GLOBAL MEMORY (L2) with relaxed loads until every word shows the expected tag and sums
// straight from registers: no fence, no counter, no bulk copy, no shared-memory inbox.
template <int UB, bool POLL>
__global__ void __launch_bounds__(32 * (ULB_EPI_WARPS + 1 + ULB_CTRL), 1) bilstm_bwd_umma_kernel(UlParams p) {
    constexpr int KS = (4 * UB) / 16;               // MMAs (k-steps of 16) per product and n-block
    extern __shared__ __align__(1024) uint8_t smem[];
    const int H = p.H, T = p.T, nub = p.nub;
    const int NB = (H + 255) / 256;                 // n-blocks of (up to) 256 columns, 64 per warpgroup
    uint8_t* sWhi = smem;
    uint8_t* sWlo = smem + (size_t)H * 128;
    uint8_t* sA1 = sWlo + (size_t)H * 128;
    uint8_t* sA2 = sA1 + 8192;
    float* inbox = reinterpret_cast<float*>(sA2 + 8192);                       // [nub][32][UB]
    const size_t inbox_bytes = POLL ? 0 : (size_t)nub * UL_BC * UB * sizeof(float);   // POLL sums straight from L2
    float* rscale = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(inbox) + inbox_bytes);   // [32]
    uint64_t* in_full = reinterpret_cast<uint64_t*>(rscale + 32);
    uint64_t* a_ready = in_full + 1;
    uint64_t* mma_done = in_full + 2;               // the MMAs of a step have read the A tiles (one arrival per warp)
    uint64_t* pub = in_full + 3;
    uint64_t* wload = in_full + 4;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    int blk = blockIdx.x;
    const int ub = blk % p.nub; blk /= p.nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;

    for (int i = tid; i < 16384 / 16; i += blockDim.x) reinterpret_cast<uint4*>(sA1)[i] = make_uint4(0, 0, 0, 0);
    if (tid == 0) {
        mbar_init(in_full, ULB_CTRL);
        mbar_init(a_ready, ULB_EPI_WARPS);
        mbar_init(mma_done, ULB_EPI_WARPS);
        mbar_init(pub, ULB_EPI_WARPS);
        mbar_init(wload, 1);
        mbar_fence_init();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const size_t xelems = (size_t)nub * nub * UL_BC * UB;                       // one parity buffer of one (dir, bg)
    float* xb = reinterpret_cast<float*>(p.xbuf) + ((size_t)dir * p.nbg + bg) * 2 * xelems;
    unsigned* ctr = p.counters + ((size_t)dir * p.nbg + bg);

    if (POLL && warp >= ULB_EPI_WARPS) {
        if (warp == ULB_EPI_WARPS + 1 && lane == 0) {            // only the W load is left for the control warps
            const uint8_t* wsrc = p.wpack + ((size_t)dir * p.nub + ub) * ((size_t)2 * H * 128);
            mbar_expect_tx(wload, (uint32_t)(2 * H * 128));
            for (int off = 0; off < 2 * H * 128; off += 32768)
                bulk_g2s(sWhi + off, wsrc + off, 32768, wload);
        }
    } else if (warp == ULB_EPI_WARPS) {
        // ------------------------------------------------------------------ publisher lane
        if (lane == 0) {
            for (int step = 0; step + 1 < T; ++step) {
                mbar_wait(pub, (uint32_t)(step & 1));
                UL_TRACE(8);
                fence_acq_rel_gpu();
                red_relaxed_add_u32(ctr, 1u);
                UL_TRACE(9);
            }
        }
    } else if (warp > ULB_EPI_WARPS) {
        // ------------------------------------------------------------------ control lanes: W load, inbox pulls
        const int c = warp - ULB_EPI_WARPS - 1;
        if (lane == 0) {
            if (c == 0) {
                const uint8_t* wsrc = p.wpack + ((size_t)dir * p.nub + ub) * ((size_t)2 * H * 128);
                mbar_expect_tx(wload, (uint32_t)(2 * H * 128));
                for (int off = 0; off < 2 * H * 128; off += 32768)
                    bulk_g2s(sWhi + off, wsrc + off, 32768, wload);
            }
            const uint32_t chunk = (uint32_t)(inbox_bytes / ULB_CTRL);
            for (int step = 0; step + 1 < T; ++step) {
                // my epilogue warps summed the inbox of `step` before they released the A tile of `step`
                mbar_wait(mma_done, (uint32_t)(step & 1));
                ul_spin_until(ctr, (unsigned)(step + 1) * (unsigned)nub, p.err_flag, (p.flags & 1) != 0);
                if (c == 0) UL_TRACE(10);
                const uint8_t* src = reinterpret_cast<const uint8_t*>(xb + (size_t)(step & 1) * xelems +
                                                                      (size_t)ub * nub * UL_BC * UB) + (size_t)c * chunk;
                mbar_expect_tx(in_full, chunk);
                bulk_g2s(reinterpret_cast<uint8_t*>(inbox) + (size_t)c * chunk, src, chunk, in_full);
                if (c == 0) UL_TRACE(11);
            }
        }
    } else {
        // ------------------------------------------------------------------ pointwise + MMA + drain warps
        // pointwise mapping: cell i = warp*32 + lane -> (batch row b = i / UB, unit u = i % UB)
        const int ci = warp * 32 + lane;
        const bool cell = ci < UL_BC * UB;
        const int b = cell ? ci / UB : 0, u = cell ? ci % UB : 0;
        const int brow = p.b0 + bg * UL_BC + b;
        const bool ok = cell && brow < p.Bend;
        const int ug = ub * UB + u;
        const int row_hi = 16 * (b >> 3) + (b & 7), row_lo = row_hi + 8;
        const uint32_t off_hi = wgmma::sw128_offset(row_hi, 8 * u), off_lo = wgmma::sw128_offset(row_lo, 8 * u);
        // MMA / drain mapping: warp q of warpgroup jq = column quarter jq of every n-block
        const int q = warp & 3, jq = warp >> 2, r = lane >> 2, tq = lane & 3;
        const int drow = 8 * q + r;
        const uint32_t a1 = smem_u32(sA1), a2 = smem_u32(sA2), whi = smem_u32(sWhi), wlo = smem_u32(sWlo);
        float d[32];
        float dc_reg = 0.f;
        const bool trc = (warp == 0 && lane == 0);

        for (int step = 0; step < T; ++step) {
            const int fstep = T - 1 - step;
            const int tt = dir ? (T - 1 - fstep) : fstep;
            const int tt_prev = dir ? tt + 1 : tt - 1;
            if (trc) UL_TRACE(0);
            float4 gtv = make_float4(0.f, 0.f, 0.f, 0.f);
            float ct = 0.f, cp = 0.f, dh = 0.f;
            const size_t row = ((size_t)dir * p.B + (ok ? brow : 0)) * T + tt;
            if (ok) {
                gtv = *reinterpret_cast<const float4*>(p.gates + (row * H + ug) * 4);
                ct = p.cst[row * H + ug];
                if (fstep > 0) cp = p.cst[(((size_t)dir * p.B + brow) * T + tt_prev) * H + ug];
                dh = p.out[((size_t)brow * T + tt) * (p.ndir * H) + (size_t)dir * H + ug];
            }
            if (POLL && step > 0) {
                if (cell) {
                    const float* ib = xb + (size_t)((step - 1) & 1) * xelems + (size_t)ub * nub * UL_BC * UB +
                                      (size_t)b * UB + u;                       // [src] stride UL_BC * UB
                    const uint32_t tag = (uint32_t)(((step - 1) >> 1) & 1) ^ 1u;
                    const long long t0 = clock64();
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
                    for (int sb = 0; sb < nub; sb += 32) {
                        // cheap spin on one word, then the block of 32 sources (they finish within a few hundred cycles)
                        float v[32];
                        const int nhere = min(32, nub - sb);          // nub = 40 at H = 640: a tail block of 8 sources
                        v[0] = ld_relaxed_f32(ib + (size_t)sb * UL_BC * UB);
                        while ((__float_as_uint(v[0]) & 1u) != tag) {
                            ul_watchdog(t0, p.err_flag);
                            v[0] = ld_relaxed_f32(ib + (size_t)sb * UL_BC * UB);
                        }
#pragma unroll
                        for (int j = 1; j < 32; ++j)
                            v[j] = (j < nhere) ? ld_relaxed_f32(ib + (size_t)(sb + j) * UL_BC * UB) : __uint_as_float(tag);
                        uint32_t pending = 0;
#pragma unroll
                        for (int j = 1; j < 32; ++j) pending |= ((__float_as_uint(v[j]) & 1u) != tag) ? (1u << j) : 0u;
                        while (pending) {
                            ul_watchdog(t0, p.err_flag);
#pragma unroll
                            for (int j = 1; j < 32; ++j)
                                if (pending & (1u << j)) {
                                    v[j] = ld_relaxed_f32(ib + (size_t)(sb + j) * UL_BC * UB);
                                    if ((__float_as_uint(v[j]) & 1u) == tag) pending &= ~(1u << j);
                                }
                        }
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            if (j < nhere) {                          // nub is a multiple of 4 (ulb_plan)
                                s0 += v[j]; s1 += v[j + 1]; s2 += v[j + 2]; s3 += v[j + 3];
                            }
                        }
                    }
                    dh += (s0 + s1) + (s2 + s3);
                }
                if (trc) UL_TRACE(3);
            }
            if (!POLL && step > 0) {
                mbar_wait(in_full, (uint32_t)((step - 1) & 1));
                if (trc) UL_TRACE(3);
                if (cell) {
                    const float* ib = inbox + (size_t)b * UB + u;
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
                    int s = 0;
                    for (; s + 3 < nub; s += 4) {
                        s0 += ib[(size_t)s * UL_BC * UB];
                        s1 += ib[(size_t)(s + 1) * UL_BC * UB];
                        s2 += ib[(size_t)(s + 2) * UL_BC * UB];
                        s3 += ib[(size_t)(s + 3) * UL_BC * UB];
                    }
                    for (; s < nub; ++s) s0 += ib[(size_t)s * UL_BC * UB];
                    dh += (s0 + s1) + (s2 + s3);
                }
            }
            float4 dg = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok) {
                const float ig = gtv.x, fg = gtv.y, gg = gtv.z, og = gtv.w;
                const float tc = tanhf(ct);
                const float dc = dc_reg + dh * og * (1.f - tc * tc);
                dg.x = dc * gg * ig * (1.f - ig);
                dg.y = dc * cp * fg * (1.f - fg);
                dg.z = dc * ig * (1.f - gg * gg);
                dg.w = dh * tc * og * (1.f - og);
                dc_reg = dc * fg;
                *reinterpret_cast<float4*>(p.gates + (row * H + ug) * 4) = dg;
            }
            if (trc) UL_TRACE(4);
            if (step + 1 < T) {
                // per-row power-of-two scale: the row's largest |dG| goes to [2^13, 2^14)
                float m = fmaxf(fmaxf(fabsf(dg.x), fabsf(dg.y)), fmaxf(fabsf(dg.z), fabsf(dg.w)));
#pragma unroll
                for (int o = 1; o < UB; o <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                int e = (int)((__float_as_uint(m) >> 23) & 0xffu) - 127;
                e = e < -100 ? -100 : (e > 100 ? 100 : e);
                const float sc = __uint_as_float((uint32_t)(127 + 13 - e) << 23);
                // every warpgroup's MMAs of the previous step have read the A tiles (and the drains the row scales)
                if (step > 0) mbar_wait(mma_done, (uint32_t)((step - 1) & 1));
                if (cell) {
                    if (u == 0) rscale[b] = __uint_as_float((uint32_t)(127 + e - 13) << 23);
                    __half hi[4], lo[4];
                    split_f16(dg.x * sc, hi[0], lo[0]);
                    split_f16(dg.y * sc, hi[1], lo[1]);
                    split_f16(dg.z * sc, hi[2], lo[2]);
                    split_f16(dg.w * sc, hi[3], lo[3]);
                    const uint2 vh = make_uint2((uint32_t)__half_as_ushort(hi[0]) | ((uint32_t)__half_as_ushort(hi[1]) << 16),
                                                (uint32_t)__half_as_ushort(hi[2]) | ((uint32_t)__half_as_ushort(hi[3]) << 16));
                    const uint2 vl = make_uint2((uint32_t)__half_as_ushort(lo[0]) | ((uint32_t)__half_as_ushort(lo[1]) << 16),
                                                (uint32_t)__half_as_ushort(lo[2]) | ((uint32_t)__half_as_ushort(lo[3]) << 16));
                    *reinterpret_cast<uint2*>(sA1 + off_hi) = vh;
                    *reinterpret_cast<uint2*>(sA1 + off_lo) = vl;
                    *reinterpret_cast<uint2*>(sA2 + off_lo) = vh;
                }
                fence_proxy_async_smem();       // my generic-proxy writes of the A tiles -> visible to the tensor core
                __syncwarp();
                if (lane == 0) ul_arrive(a_ready);
                if (trc) UL_TRACE(5);
                if (step == 0) mbar_wait(wload, 0);
                mbar_wait(a_ready, (uint32_t)(step & 1));           // all 16 warps wrote (and fenced) their part of A
                if (trc) UL_TRACE(1);
                // ---- MMA + drain of the accumulator into the destinations' inboxes, n-block by n-block
                float* outbase = xb + (size_t)(step & 1) * xelems;
                for (int j = 0; j < NB; ++j) {
                    if (256 * j + 64 * jq >= H) continue;             // the last block of H = 640 is only 128 wide
                    const uint32_t boff = (uint32_t)(256 * j + 64 * jq) * 128u;
                    wgmma::fence_operand(d);
                    wgmma::fence();
#pragma unroll
                    for (int kk = 0; kk < KS; ++kk) {
                        wgmma::mma_f16_n64(d, wgmma::desc_k_sw128(a1 + kk * 32), wgmma::desc_k_sw128(whi + boff + kk * 32), kk > 0);
                        wgmma::mma_f16_n64(d, wgmma::desc_k_sw128(a2 + kk * 32), wgmma::desc_k_sw128(wlo + boff + kk * 32), 1);
                    }
                    wgmma::commit_group();
                    wgmma::wait_all();
                    wgmma::fence_operand(d);
                    if (trc && j == 0) UL_TRACE(6);
                    const float* v0 = d;
                    const float* v1 = d + 16;
                    const float rs = rscale[drow];
                    const float k = 1.f / 2048.f;
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            const float* v = hh ? &v1[4 * g] : &v0[4 * g];
                            const int n = 256 * j + 64 * jq + 32 * hh + 8 * g + 2 * tq;
                            const int dst = n / UB, uu = n - dst * UB;
                            const float o0 = (v[0] + v[2] * k) * rs;
                            const float o1 = (v[1] + v[3] * k) * rs;
                            float* optr = outbase + (((size_t)dst * nub + ub) * UL_BC + drow) * UB + uu;
                            if (POLL) {
                                const uint32_t tagw = (uint32_t)((step >> 1) & 1) ^ 1u;
                                st_relaxed_v2(optr, (__float_as_uint(o0) & ~1u) | tagw, (__float_as_uint(o1) & ~1u) | tagw);
                            } else {
                                *reinterpret_cast<float2*>(optr) = make_float2(o0, o1);
                            }
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) {
                    ul_arrive(mma_done);
                    if (!POLL) ul_arrive(pub);
                }
                if (trc) UL_TRACE(7);
            }
        }
    }
}

struct UlPlan {
    int UB, UBp, nub, nbg, ctas, NA, Bsub, nsplit;
    size_t smem, pack_bytes, xbuf_bytes;
};

int ul_plan(int B, int H, int ndir, UlPlan* out) {
    if (H % 64 != 0 || H / 64 > UL_MAX_ATOMS) return -1;
    const int sms = sm_count();
    const size_t cap = (size_t)max_optin_smem();
    const int NA = H / 64;
    for (int n = 1; n <= B; ++n) {
        const int Bs = (B + n - 1) / n;
        const int nbg = (Bs + UL_BC - 1) / UL_BC;
        for (int UB = 2; UB <= 16; ++UB) {           // smallest unit block whose CTAs are all co-resident
            if (H % UB) continue;
            const int UBp = (UB + 3) / 4 * 4;
            if (UBp != 8 && UBp != 12 && UBp != 16) continue;
            const int nub = H / UB;
            const int ctas = ndir * nbg * nub;
            if (ctas > sms) continue;
            const size_t smem = (size_t)NA * UL_ATOM_A + (size_t)NA * 8 * UBp * 128 + 512;
            if (smem > cap) continue;
            if ((size_t)ndir * nbg * UL_MAX_ATOMS * 4 > UL_COUNTER_BYTES - 64) continue;
            out->UB = UB; out->UBp = UBp; out->nub = nub; out->nbg = nbg; out->ctas = ctas; out->NA = NA;
            out->Bsub = Bs; out->nsplit = (B + Bs - 1) / Bs; out->smem = smem;
            out->pack_bytes = (size_t)ndir * nub * NA * 8 * UBp * 128;
            out->xbuf_bytes = (size_t)ndir * nbg * UL_NBUF * NA * UL_ATOM_A;   // (2 images suffice for the flag protocol)
            return 0;
        }
        if (Bs <= UL_BC) break;
    }
    return -2;
}

size_t ul_align(size_t x) { return (x + 255) / 256 * 256; }

template <int UBP, bool POLL>
int ul_launch_fwd(const UlPlan& pl, UlParams p, const float* w_hh, cudaStream_t stream) {
    {
        const long long n = (long long)p.ndir * pl.nub * 8 * UBP * p.H;
        int blocks = (int)((n + 255) / 256);
        if (blocks > 8192) blocks = 8192;
        ul_pack_fwd_kernel<UBP><<<blocks, 256, 0, stream>>>(w_hh, const_cast<uint8_t*>(p.wpack), p.H, pl.UB, p.ndir);
        B200_LAUNCH_CHECK("ul_pack_fwd_kernel");
    }
    const void* fn = (const void*)bilstm_fwd_umma_kernel<UBP, POLL>;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
    int per_sm = 0;
    const int threads = 32 * (UBP + 1 + p.NC);
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, pl.smem));
    B200_REQUIRE((long long)per_sm * sm_count() >= pl.ctas, "bilstm(umma): %d CTAs cannot be co-resident (%d/SM x %d SMs)",
                 pl.ctas, per_sm, sm_count());
    for (int sp = 0; sp < pl.nsplit; ++sp) {
        p.b0 = sp * pl.Bsub;
        p.Bend = p.b0 + pl.Bsub < p.B ? p.b0 + pl.Bsub : p.B;
        B200_CUDA(cudaMemsetAsync(p.counters, 0, UL_COUNTER_BYTES, stream));
        if (POLL) B200_CUDA(cudaMemsetAsync(p.xbuf, 0xFF, pl.xbuf_bytes, stream));      // poison every exchange image
        void* args[] = {&p};
        B200_CUDA(cudaLaunchCooperativeKernel(fn, dim3(pl.ctas), dim3(threads), args, pl.smem, stream));
        count_launch();
    }
    return B200_OK;
}

struct UlbPlan {
    int UB, nub, nbg, ctas, Bsub, nsplit;
    size_t smem, pack_bytes, xbuf_bytes;
};

int ulb_plan(int B, int H, int ndir, bool poll, UlbPlan* out) {
    // accumulator = H columns in n-blocks of 256, 64 per warpgroup: 256 | 512 | 640 | 768 (a last block of 128 or 256)
    if (H % 128 != 0 || H < 256 || H > 768) return -1;
    const int sms = sm_count();
    const size_t cap = (size_t)max_optin_smem();
    for (int n = 1; n <= B; ++n) {
        const int Bs = (B + n - 1) / n;
        const int nbg = (Bs + UL_BC - 1) / UL_BC;
        for (int UB = 8; UB <= 16; UB += 8) {
            if (H % UB) continue;
            const int nub = H / UB;
            const int ctas = ndir * nbg * nub;
            if (ctas > sms) continue;
            if (nub % 4) continue;
            const size_t inbox = (size_t)nub * UL_BC * UB * 4;
            // the polling exchange keeps no inbox in shared memory (which is what lets H = 640 fit)
            const size_t smem = (size_t)2 * H * 128 + 16384 + (poll ? 0 : inbox) + 128 + 128;
            if (smem > cap || (inbox / ULB_CTRL) % 16 || (2 * H * 128) % 32768) continue;
            out->UB = UB; out->nub = nub; out->nbg = nbg; out->ctas = ctas; out->Bsub = Bs;
            out->nsplit = (B + Bs - 1) / Bs; out->smem = smem;
            out->pack_bytes = (size_t)ndir * nub * 2 * H * 128;
            out->xbuf_bytes = (size_t)ndir * nbg * 2 * nub * inbox;
            return 0;
        }
        if (Bs <= UL_BC) break;
    }
    return -2;
}

template <int UB, bool POLL>
int ul_launch_bwd(const UlbPlan& pl, UlParams p, const float* w_hh, cudaStream_t stream) {
    {
        const long long n = (long long)p.ndir * pl.nub * 2 * p.H * 64;
        int blocks = (int)((n + 255) / 256);
        if (blocks > 8192) blocks = 8192;
        ul_pack_bwd_kernel<UB><<<blocks, 256, 0, stream>>>(w_hh, const_cast<uint8_t*>(p.wpack), p.H, p.ndir);
        B200_LAUNCH_CHECK("ul_pack_bwd_kernel");
    }
    const void* fn = (const void*)bilstm_bwd_umma_kernel<UB, POLL>;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
    int per_sm = 0;
    const int threads = 32 * (ULB_EPI_WARPS + 1 + ULB_CTRL);
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, pl.smem));
    B200_REQUIRE((long long)per_sm * sm_count() >= pl.ctas, "bilstm(umma bwd): %d CTAs cannot be co-resident (%d/SM x %d SMs)",
                 pl.ctas, per_sm, sm_count());
    for (int sp = 0; sp < pl.nsplit; ++sp) {
        p.b0 = sp * pl.Bsub;
        p.Bend = p.b0 + pl.Bsub < p.B ? p.b0 + pl.Bsub : p.B;
        B200_CUDA(cudaMemsetAsync(p.counters, 0, UL_COUNTER_BYTES, stream));
        if (POLL) B200_CUDA(cudaMemsetAsync(p.xbuf, 0, pl.xbuf_bytes, stream));     // generation tags start at 0
        void* args[] = {&p};
        B200_CUDA(cudaLaunchCooperativeKernel(fn, dim3(pl.ctas), dim3(threads), args, pl.smem, stream));
        count_launch();
    }
    return B200_OK;
}

}  // namespace

static bool ulb_poll(int flags) { return ((flags & 8) != 0) != (UL_POLL_BWD_DEFAULT != 0); }

bool lstm_umma_bwd_supported(int B, int H, int ndir, int flags) {
    UlbPlan pl;
    return ulb_plan(B, H, ndir, ulb_poll(flags), &pl) == 0;
}

int lstm_umma_bwd(float* gates, const float* w_hh, const float* cstate, const float* dout, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, long long* trace, int flags, cudaStream_t stream) {
    UlbPlan pl;
    // flag bit 3 (debug mode 2048) selects the OTHER exchange protocol than the default one
    const bool poll = ulb_poll(flags);
    B200_REQUIRE(ulb_plan(B, H, ndir, poll, &pl) == 0, "bilstm(umma bwd): unsupported shape B=%d H=%d ndir=%d", B, H, ndir);
    B200_REQUIRE(workspace_bytes >= lstm_umma_workspace_bytes(B, H, ndir), "bilstm(umma bwd): workspace too small");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    UlParams p;
    p.gates = gates; p.cst = const_cast<float*>(cstate); p.out = const_cast<float*>(dout);
    p.wpack = ws;
    p.xbuf = ws + ul_align(pl.pack_bytes);
    p.counters = reinterpret_cast<unsigned*>(ws + ul_align(pl.pack_bytes) + ul_align(pl.xbuf_bytes));
    p.err_flag = reinterpret_cast<int*>(p.counters + (UL_COUNTER_BYTES / 4 - 4));
    p.trace = trace;
    p.flags = flags;
    p.B = B; p.T = T; p.H = H; p.ndir = ndir; p.UB = pl.UB; p.nub = pl.nub; p.nbg = pl.nbg; p.NA = 0; p.NC = ULB_CTRL;
    p.b0 = 0; p.Bend = B;
    if (pl.UB == 16) return poll ? ul_launch_bwd<16, true>(pl, p, w_hh, stream) : ul_launch_bwd<16, false>(pl, p, w_hh, stream);
    return poll ? ul_launch_bwd<8, true>(pl, p, w_hh, stream) : ul_launch_bwd<8, false>(pl, p, w_hh, stream);
}

bool lstm_umma_fwd_supported(int B, int H, int ndir) {
    UlPlan pl;
    return ul_plan(B, H, ndir, &pl) == 0;
}

size_t lstm_umma_workspace_bytes(int B, int H, int ndir) {
    UlPlan pl;
    UlbPlan pb;
    size_t f = 0, b = 0;
    if (ul_plan(B, H, ndir, &pl) == 0) f = ul_align(pl.pack_bytes) + ul_align(pl.xbuf_bytes) + UL_COUNTER_BYTES;
    for (int poll = 0; poll < 2; ++poll)
        if (ulb_plan(B, H, ndir, poll != 0, &pb) == 0) {
            const size_t bb = ul_align(pb.pack_bytes) + ul_align(pb.xbuf_bytes) + UL_COUNTER_BYTES;
            b = bb > b ? bb : b;
        }
    return f > b ? f : b;
}

int lstm_umma_plan(int B, int H, int ndir, int* unit_block, int* batch_block, int* n_ctas) {
    UlPlan pl;
    if (ul_plan(B, H, ndir, &pl) != 0) return -1;
    if (unit_block) *unit_block = pl.UB;
    if (batch_block) *batch_block = UL_BC;
    if (n_ctas) *n_ctas = pl.ctas;
    return 0;
}

int lstm_umma_fwd(float* gates, const float* w_hh, float* cstate, float* out, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, long long* trace, int flags, cudaStream_t stream) {
    UlPlan pl;
    B200_REQUIRE(ul_plan(B, H, ndir, &pl) == 0, "bilstm(umma): unsupported shape B=%d H=%d ndir=%d", B, H, ndir);
    B200_REQUIRE(workspace_bytes >= lstm_umma_workspace_bytes(B, H, ndir), "bilstm(umma): workspace too small");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    UlParams p;
    p.gates = gates; p.cst = cstate; p.out = out;
    p.wpack = ws;
    p.xbuf = ws + ul_align(pl.pack_bytes);
    p.counters = reinterpret_cast<unsigned*>(ws + ul_align(pl.pack_bytes) + ul_align(pl.xbuf_bytes));
    p.err_flag = reinterpret_cast<int*>(p.counters + (UL_COUNTER_BYTES / 4 - 4));
    p.trace = trace;
    p.flags = flags;
    p.B = B; p.T = T; p.H = H; p.ndir = ndir; p.UB = pl.UB; p.nub = pl.nub; p.nbg = pl.nbg; p.NA = pl.NA;
    p.NC = pl.NA < UL_MAX_CTRL ? pl.NA : UL_MAX_CTRL;
    p.b0 = 0; p.Bend = B;
    // flag bit 2 (debug mode 1024) selects the OTHER exchange protocol than the default one
    const bool poll = ((flags & 4) != 0) != (UL_POLL_FWD_DEFAULT != 0);
    switch (pl.UBp) {
        case 8: return poll ? ul_launch_fwd<8, true>(pl, p, w_hh, stream) : ul_launch_fwd<8, false>(pl, p, w_hh, stream);
        case 12: return poll ? ul_launch_fwd<12, true>(pl, p, w_hh, stream) : ul_launch_fwd<12, false>(pl, p, w_hh, stream);
        default: return poll ? ul_launch_fwd<16, true>(pl, p, w_hh, stream) : ul_launch_fwd<16, false>(pl, p, w_hh, stream);
    }
}

}  // namespace b200asr
