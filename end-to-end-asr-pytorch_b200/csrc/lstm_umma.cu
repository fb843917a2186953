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
#include "rnn_cell.cuh"

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
    int B, T, H, ndir, UB, nub, nbg, NA, NC;
    int strict;            // forward: formal acquire after the flag poll (debug mode 256)
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
// generic->async proxy fence of the PTX memory model (debug mode 256); tests/test_gpu_lstm_variants.py runs both.
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
// ---- the backward's "data is the flag" exchange: relaxed gpu-scope loads and stores of tagged partials -------------
__device__ __forceinline__ float ld_relaxed_f32(const float* p) {
    float v;
    asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_v2(void* p, uint32_t a, uint32_t b) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
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

// Warp roles: warps [0, UBP) MMA + epilogue / pointwise - UBP/4 warpgroups; warp w is warp q = w % 4 of warpgroup
// j = w / 4 (the unit quad), i.e. ONE cell (batch row 8q + lane/4, unit 4j + lane%4) per thread; warp UBP = publisher
// (one lane: ONE gpu-scope fence + release per CTA and step, after the epilogue warps arrived on `pub`); warps
// UBP+1 .. UBP+NC = control, one lane each, control warp c owns K atoms c, c+NC, ...
template <int CELL, int UBP>
__device__ __forceinline__ void fwd_umma_body(const UlParams& p) {
    constexpr int N = 8 * UBP;            // B operand rows (gate columns, hi + lo copies)
    extern __shared__ __align__(1024) uint8_t smem[];
    const int H = p.H, T = p.T, NA = p.NA, UB = p.UB;
    uint8_t* sA = smem;
    uint8_t* sB = smem + (size_t)NA * UL_ATOM_A;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + (size_t)NA * N * 128);    // [UL_MAX_ATOMS]
    uint64_t* mma_done = full + UL_MAX_ATOMS;    // the MMAs of a step have read every atom of A (one arrival per warp)
    uint64_t* wload = mma_done + 1;
    uint64_t* pub = mma_done + 2;                // the epilogue warps have stored h_step

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NC = p.NC;
    int blk = blockIdx.x;
    const int ub = blk % p.nub; blk /= p.nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;

    if (tid == 0) {
        for (int a = 0; a < UL_MAX_ATOMS; ++a) mbar_init(&full[a], 1);
        mbar_init(pub, UBP);
        mbar_init(mma_done, UBP);
        mbar_init(wload, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const size_t img_bytes = (size_t)NA * UL_ATOM_A;             // one image of the A operand
    uint8_t* xb = p.xbuf + ((size_t)dir * p.nbg + bg) * 2 * img_bytes;
    unsigned* ctr0 = p.counters + ((size_t)dir * p.nbg + bg) * UL_MAX_ATOMS;

    if (warp == UBP) {
        // ------------------------------------------------------------------ publisher lane
        if (lane == 0) {
            const int a0 = (ub * UB) >> 6, a1 = (ub * UB + UB - 1) >> 6;
            for (int step = 0; step + 1 < T; ++step) {
                mbar_wait(pub, (uint32_t)(step & 1));       // every epilogue warp stored its part of h_step
                fence_acq_rel_gpu();                        // their stores (observed through the mbarrier) first ...
                red_relaxed_add_u32(ctr0 + a0, 1u);         // ... then the flag(s) of the K atom(s) of my unit block
                if (a1 != a0) red_relaxed_add_u32(ctr0 + a1, 1u);
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
                    ul_spin_until(ctr0 + a, (unsigned)(step + 1) * per_step[i], p.err_flag, p.strict != 0);
                    const uint8_t* src = xb + (size_t)(step & 1) * ((size_t)NA * UL_ATOM_A) + (size_t)a * UL_ATOM_A;
                    mbar_expect_tx(&full[a], UL_ATOM_A);
                    bulk_g2s(sA + (size_t)a * UL_ATOM_A, src, UL_ATOM_A, &full[a]);
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
        float4 st_g = make_float4(0.f, 0.f, 0.f, 0.f);
        float st_c = 0.f, st_h = 0.f;
        size_t st_row = 0, st_out = 0;
        bool st_pending = false;

        for (int step = 0; step < T; ++step) {
            const int tt = dir ? (T - 1 - step) : step;
            const size_t rowbase = ((size_t)dir * p.B + (ok ? brow : 0)) * T + tt;
            float4 pre = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok) pre = *reinterpret_cast<const float4*>(p.gates + (rowbase * H + ug) * 4);
            if (step > 0) {
                if (step == 1) mbar_wait(wload, 0);
                wgmma::fence_operand(d);
                wgmma::fence();
                for (int a = 0; a < NA; ++a) {
                    mbar_wait(&full[a], (uint32_t)((step - 1) & 1));
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        wgmma::mma_f16_n32(d, wgmma::desc_k_sw128(a_base + a * UL_ATOM_A + j * 32),
                                           wgmma::desc_k_sw128(b_base + a * (N * 128) + j * 32), (a | j) != 0);
                }
                wgmma::commit_group();
                wgmma::wait_all();
                wgmma::fence_operand(d);
                __syncwarp();
                if (lane == 0) ul_arrive(mma_done);     // the control warps may overwrite the atoms of A
                // d[0..7]: hi and lo row against W_hi, gates (i,f) then (g,o); d[8..15]: the same against W_lo
                const float *dif = d, *dgo = d + 4, *eif = d + 8, *ego = d + 12;
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
            float c = c_reg;                              // c_t (LSTM) / h_t (GRU) after the cell
            float4 gq;
            cell_fwd<CELL>([&](int q) { return f4_at(pre, q); }, c, gq);
            c_reg = ok ? c : 0.f;
            const float hq = ok ? cell_h<CELL>(gq, c) : 0.f;
            if (step + 1 < T) {
                // publish h_step as element (A row, k = ug) of the next A operand, fp16 hi / lo
                uint8_t* dstimg = xb + (size_t)(step & 1) * img_bytes;
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
                __syncwarp();
                if (lane == 0) ul_arrive(pub);
            }
            // the stash / output stores of this step are issued during the NEXT step (after its MMAs): stores
            // in flight while the publisher runs its gpu-scope fence lengthen that fence by their L2 round trip
            st_g = gq;
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
// the step kernels of the two cells (csrc/rnn_cell.cuh) on one body
template <int UBP>
__global__ void __launch_bounds__(32 * (UBP + 1 + UL_MAX_CTRL), 1) bilstm_fwd_umma_kernel(UlParams p) {
    fwd_umma_body<CELL_LSTM, UBP>(p);
}
template <int UBP>
__global__ void __launch_bounds__(32 * (UBP + 1 + UL_MAX_CTRL), 1) bigru_fwd_umma_kernel(UlParams p) {
    fwd_umma_body<CELL_GRU, UBP>(p);
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


__device__ __forceinline__ float add_ftz(float a, float b) {
    float r;
    asm("add.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
// ---- distributed shared memory of a thread-block cluster ------------------------------------------------------------
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, int rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_v2(uint32_t addr, uint32_t a, uint32_t b) {
    asm volatile("st.relaxed.cluster.shared::cluster.v2.u32 [%0], {%1,%2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint2 ld_cluster_v2(uint32_t addr) {
    uint2 v;
    asm volatile("ld.relaxed.cluster.shared::cta.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

constexpr int ULB_EPI_WARPS = 16;
constexpr int ULB_CTRL = 4;
constexpr size_t ULB_SMEM_FIXED = 16384 + 128 + 128;   // A tiles, row scales, barriers (+ 2 H 128 B of W_hh)

// Bytes of the cluster staging buffers: two parity buffers of the partials that the CS - 1 other ranks send to the
// destinations this rank aggregates (nub / CS of them, 32 x UB fp32 each).
__host__ __device__ inline size_t ulb_staging_bytes(int nub, int UB, int CS) {
    return CS > 1 ? (size_t)2 * (CS - 1) * (nub / CS) * UL_BC * UB * 4 : 0;
}

// The state exchange is "data is the flag": every fp32 partial carries the parity of its buffer generation in its
// least significant mantissa bit (2^-24 relative - below the resolution of the hi/lo product), the destination polls
// its inbox IN GLOBAL MEMORY (L2) with relaxed loads until every word shows the expected tag and sums straight from
// registers (flushing subnormals, so that a tagged zero adds nothing): no fence, no counter, no bulk copy, no
// shared-memory inbox.
// Two-level exchange (CS > 1): the CTAs of one (direction, batch group) run as clusters of CS consecutive unit blocks.
// Cluster rank d % CS aggregates the cluster's partials for destination d: the other ranks store theirs into its
// staging buffer in distributed shared memory (tagged the same way, two parity buffers), it polls its own shared
// memory, sums the CS contributions in rank order with flushing adds, re-tags the sum and stores it to d's L2 inbox.
// A destination then polls nub / CS sources (one per cluster) instead of nub, and the L2 traffic per step drops CS x.
// Warp roles: warps [0, 16) pointwise + MMA + drain; lane 0 of warp 17 loads W_hh.  Warps 16 and 18 .. 20 have no work
// but stay in the block: __launch_bounds__ and ul_launch_bwd's occupancy check count them.
template <int CELL, int UB, int CS>
__device__ __forceinline__ void bwd_umma_body(const UlParams& p) {
    constexpr int KS = (4 * UB) / 16;               // MMAs (k-steps of 16) per product and n-block
    // the 64 columns of a warpgroup's n-block start on a multiple of UB * CS units, so the aggregating rank of each
    // accumulator column group depends only on its offset inside the block
    static_assert(64 % (UB * CS) == 0, "cluster size");
    extern __shared__ __align__(1024) uint8_t smem[];
    const int H = p.H, T = p.T, nub = p.nub;
    const int NB = (H + 255) / 256;                 // n-blocks of (up to) 256 columns, 64 per warpgroup
    uint8_t* sWhi = smem;
    uint8_t* sWlo = smem + (size_t)H * 128;
    uint8_t* sA1 = sWlo + (size_t)H * 128;
    uint8_t* sA2 = sA1 + 8192;
    float* rscale = reinterpret_cast<float*>(sA2 + 8192);                      // [32]
    uint64_t* a_ready = reinterpret_cast<uint64_t*>(rscale + 32);
    uint64_t* mma_done = a_ready + 1;               // the MMAs of a step have read the A tiles (one arrival per warp)
    uint64_t* wload = a_ready + 2;
    // [parity][CS - 1 sender slots][nub / CS destinations][UL_BC][UB] fp32 (CS > 1)
    float* stg = reinterpret_cast<float*>(sA1 + ULB_SMEM_FIXED);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    int blk = blockIdx.x;
    const int ub = blk % p.nub; blk /= p.nub;
    const int bg = blk % p.nbg; blk /= p.nbg;
    const int dir = blk;
    const int crank = ub % CS;                      // = the block's rank in its cluster (clusters along unit blocks)
    const int nsrc = nub / CS;                      // sources per L2 inbox: one per cluster
    constexpr int PB = 32 / CS;                     // sources polled as one block (registers)

    for (int i = tid; i < 16384 / 16; i += blockDim.x) reinterpret_cast<uint4*>(sA1)[i] = make_uint4(0, 0, 0, 0);
    if (CS > 1) {                                   // generation tags start at 0
        for (int i = tid; i < (int)(ulb_staging_bytes(nub, UB, CS) / 16); i += blockDim.x)
            reinterpret_cast<uint4*>(stg)[i] = make_uint4(0, 0, 0, 0);
    }
    if (tid == 0) {
        mbar_init(a_ready, ULB_EPI_WARPS);
        mbar_init(mma_done, ULB_EPI_WARPS);
        mbar_init(wload, 1);
        mbar_fence_init();
    }
    fence_proxy_async_smem();
    if (CS > 1) cluster_sync_all();                 // every peer runs and has zeroed its staging before a remote store
    else __syncthreads();
    const size_t xelems = (size_t)nub * nsrc * UL_BC * UB;                      // one parity buffer of one (dir, bg)
    float* xb = reinterpret_cast<float*>(p.xbuf) + ((size_t)dir * p.nbg + bg) * 2 * xelems;
    const uint32_t stg_base = smem_u32(stg), stg_slot = (uint32_t)nsrc * (UL_BC * UB * 4);   // bytes per sender slot

    if (warp >= ULB_EPI_WARPS) {
        if (warp == ULB_EPI_WARPS + 1 && lane == 0) {
            const uint8_t* wsrc = p.wpack + ((size_t)dir * p.nub + ub) * ((size_t)2 * H * 128);
            mbar_expect_tx(wload, (uint32_t)(2 * H * 128));
            for (int off = 0; off < 2 * H * 128; off += 32768)
                bulk_g2s(sWhi + off, wsrc + off, 32768, wload);
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

        for (int step = 0; step < T; ++step) {
            const int fstep = T - 1 - step;
            const int tt = dir ? (T - 1 - fstep) : fstep;
            const int tt_prev = dir ? tt + 1 : tt - 1;
            float4 gtv = make_float4(0.f, 0.f, 0.f, 0.f);
            float ct = 0.f, cp = 0.f, dh = 0.f;
            const size_t row = ((size_t)dir * p.B + (ok ? brow : 0)) * T + tt;
            if (ok) {
                gtv = *reinterpret_cast<const float4*>(p.gates + (row * H + ug) * 4);
                ct = p.cst[row * H + ug];
                if (fstep > 0) cp = p.cst[(((size_t)dir * p.B + brow) * T + tt_prev) * H + ug];
                dh = p.out[((size_t)brow * T + tt) * (p.ndir * H) + (size_t)dir * H + ug];
            }
            if (step > 0) {
                if (cell) {
                    const float* ib = xb + (size_t)((step - 1) & 1) * xelems + (size_t)ub * nsrc * UL_BC * UB +
                                      (size_t)b * UB + u;                       // [src] stride UL_BC * UB
                    const uint32_t tag = (uint32_t)(((step - 1) >> 1) & 1) ^ 1u;
                    const long long t0 = clock64();
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
                    for (int sb = 0; sb < nsrc; sb += PB) {
                        // cheap spin on one word, then the block of PB sources (they finish within a few hundred cycles)
                        float v[PB];
                        const int nhere = min(PB, nsrc - sb);         // nub = 40 at H = 640: a tail block of 8 sources
                        v[0] = ld_relaxed_f32(ib + (size_t)sb * UL_BC * UB);
                        while ((__float_as_uint(v[0]) & 1u) != tag) {
                            ul_watchdog(t0, p.err_flag);
                            v[0] = ld_relaxed_f32(ib + (size_t)sb * UL_BC * UB);
                        }
#pragma unroll
                        for (int j = 1; j < PB; ++j)
                            v[j] = (j < nhere) ? ld_relaxed_f32(ib + (size_t)(sb + j) * UL_BC * UB) : __uint_as_float(tag);
                        uint32_t pending = 0;
#pragma unroll
                        for (int j = 1; j < PB; ++j) pending |= ((__float_as_uint(v[j]) & 1u) != tag) ? (1u << j) : 0u;
                        while (pending) {
                            ul_watchdog(t0, p.err_flag);
#pragma unroll
                            for (int j = 1; j < PB; ++j)
                                if (pending & (1u << j)) {
                                    v[j] = ld_relaxed_f32(ib + (size_t)(sb + j) * UL_BC * UB);
                                    if ((__float_as_uint(v[j]) & 1u) == tag) pending &= ~(1u << j);
                                }
                        }
                        // flush-to-zero adds: a zero partial arrives with its tag as the smallest subnormal, and a
                        // zero dout row must still get dG = 0 exactly (same FADD instruction, no extra work)
#pragma unroll
                        for (int j = 0; j < PB; j += 4) {
                            if (j < nhere) {                          // nub / CS is a multiple of 4 (ulb_plan)
                                s0 = add_ftz(s0, v[j]); s1 = add_ftz(s1, v[j + 1]);
                                s2 = add_ftz(s2, v[j + 2]); s3 = add_ftz(s3, v[j + 3]);
                            }
                        }
                    }
                    dh += (s0 + s1) + (s2 + s3);
                }
            }
            float4 dg = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok) {
                cell_bwd<CELL>(gtv, ct, cp, dh, dc_reg, dg);
                *reinterpret_cast<float4*>(p.gates + (row * H + ug) * 4) = dg;
            }
            if (step + 1 < T) {
                // per-row power-of-two scale: the row's largest |dG| goes to [2^13, 2^14)
                float m = fmaxf(fmaxf(fabsf(dg.x), fabsf(dg.y)), fmaxf(fabsf(dg.z), fabsf(dg.w)));
#pragma unroll
                for (int o = 1; o < UB; o <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                // e in [-113, 127] keeps sc = 2^(13-e) and its inverse 2^(e-13) normal: a tighter upper clamp would
                // leave a row whose largest |dG| is >= 2^(clamp+3) above 65504 after scaling (hi = inf, lo = -inf)
                int e = (int)((__float_as_uint(m) >> 23) & 0xffu) - 127;
                e = e < -113 ? -113 : (e > 127 ? 127 : e);
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
                if (step == 0) mbar_wait(wload, 0);
                mbar_wait(a_ready, (uint32_t)(step & 1));           // all 16 warps wrote (and fenced) their part of A
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
                    const float* v0 = d;
                    const float* v1 = d + 16;
                    const float rs = rscale[drow];
                    const float k = 1.f / 2048.f;
                    const uint32_t tagw = (uint32_t)((step >> 1) & 1) ^ 1u;
                    // CS = 1: every partial to its destination's L2 inbox.  CS > 1: the partials another rank
                    // aggregates go to that rank's staging buffer first; this rank's own share (column group
                    // m = 4 hh + g with aggregator (8 m / UB) % CS == crank, the idx-th such group) waits in own[] for
                    // the second pass, after these stores are on their way.
                    constexpr int G = UB / 8;                  // column groups of 8 per destination
                    float own[16 / CS];
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            const float* v = hh ? &v1[4 * g] : &v0[4 * g];
                            const int m = 4 * hh + g;
                            const int n = 256 * j + 64 * jq + 8 * m + 2 * tq;
                            const int dst = n / UB, uu = n - dst * UB;
                            const int agg = (8 * m / UB) % CS;         // = dst % CS
                            const float o0 = (v[0] + v[2] * k) * rs;
                            const float o1 = (v[1] + v[3] * k) * rs;
                            if (CS > 1 && agg == crank) {
                                const int idx = (m / G) / CS * G + m % G;
                                own[2 * idx] = o0;
                                own[2 * idx + 1] = o1;
                                continue;
                            }
                            const uint32_t w0 = (__float_as_uint(o0) & ~1u) | tagw, w1 = (__float_as_uint(o1) & ~1u) | tagw;
                            if (CS == 1) {
                                st_relaxed_v2(outbase + (((size_t)dst * nsrc + ub) * UL_BC + drow) * UB + uu, w0, w1);
                            } else {
                                const int slot = (crank - agg - 1 + CS) % CS;
                                const uint32_t sa = stg_base + (uint32_t)((step & 1) * (CS - 1) + slot) * stg_slot +
                                                    (uint32_t)(((dst / CS) * UL_BC + drow) * UB + uu) * 4u;
                                st_cluster_v2(mapa_shared(sa, agg), w0, w1);
                            }
                        }
                    }
                    if (CS > 1) {
                        const long long t0 = clock64();
#pragma unroll
                        for (int idx = 0; idx < 8 / CS; ++idx) {
                            const int m = G * (crank + CS * (idx / G)) + idx % G;
                            const int n = 256 * j + 64 * jq + 8 * m + 2 * tq;
                            const int dst = n / UB, uu = n - dst * UB;
                            const uint32_t soff = (uint32_t)(((dst / CS) * UL_BC + drow) * UB + uu) * 4u;
                            // the CS contributions in rank order; flushing adds drop the tagged zeros
                            float s0 = 0.f, s1 = 0.f;
#pragma unroll
                            for (int rr = 0; rr < CS; ++rr) {
                                float x0 = own[2 * idx], x1 = own[2 * idx + 1];
                                if (rr != crank) {
                                    const int slot = (rr - crank - 1 + CS) % CS;
                                    const uint32_t sa = stg_base + (uint32_t)((step & 1) * (CS - 1) + slot) * stg_slot + soff;
                                    uint2 w = ld_cluster_v2(sa);
                                    while (((w.x & 1u) != tagw) || ((w.y & 1u) != tagw)) {
                                        ul_watchdog(t0, p.err_flag);
                                        w = ld_cluster_v2(sa);
                                    }
                                    x0 = __uint_as_float(w.x);
                                    x1 = __uint_as_float(w.y);
                                }
                                s0 = add_ftz(s0, x0);
                                s1 = add_ftz(s1, x1);
                            }
                            st_relaxed_v2(outbase + (((size_t)dst * nsrc + ub / CS) * UL_BC + drow) * UB + uu,
                                          (__float_as_uint(s0) & ~1u) | tagw, (__float_as_uint(s1) & ~1u) | tagw);
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) ul_arrive(mma_done);
            }
        }
    }
    if (CS > 1) cluster_sync_all();                 // no peer accesses this block's shared memory after it exits
}
template <int UB, int CS>
__global__ void __launch_bounds__(32 * (ULB_EPI_WARPS + 1 + ULB_CTRL), 1) bilstm_bwd_umma_kernel(UlParams p) {
    bwd_umma_body<CELL_LSTM, UB, CS>(p);
}
template <int UB, int CS>
__global__ void __launch_bounds__(32 * (ULB_EPI_WARPS + 1 + ULB_CTRL), 1) bigru_bwd_umma_kernel(UlParams p) {
    bwd_umma_body<CELL_GRU, UB, CS>(p);
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
            out->xbuf_bytes = (size_t)ndir * nbg * 2 * NA * UL_ATOM_A;
            return 0;
        }
        if (Bs <= UL_BC) break;
    }
    return -2;
}

size_t ul_align(size_t x) { return (x + 255) / 256 * 256; }

template <int CELL, int UBP>
int ul_launch_fwd(const UlPlan& pl, UlParams p, const float* w_hh, cudaStream_t stream) {
    {
        const long long n = (long long)p.ndir * pl.nub * 8 * UBP * p.H;
        int blocks = (int)((n + 255) / 256);
        if (blocks > 8192) blocks = 8192;
        ul_pack_fwd_kernel<UBP><<<blocks, 256, 0, stream>>>(w_hh, const_cast<uint8_t*>(p.wpack), p.H, pl.UB, p.ndir);
        B200_LAUNCH_CHECK("ul_pack_fwd_kernel");
    }
    const void* fn = CELL == CELL_GRU ? (const void*)bigru_fwd_umma_kernel<UBP> : (const void*)bilstm_fwd_umma_kernel<UBP>;
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
        void* args[] = {&p};
        B200_CUDA(cudaLaunchCooperativeKernel(fn, dim3(pl.ctas), dim3(threads), args, pl.smem, stream));
        count_launch();
    }
    return B200_OK;
}

struct UlbPlan {
    int UB, nub, nbg, ctas, Bsub, nsplit;
    int CS;                // cluster size of the two-level exchange (1: every partial straight to L2)
    size_t smem, pack_bytes, xbuf_bytes;
};

int g_ulb_cs_cap = 0;              // test cap on CS (debug lstm mode bits 4..6; 0: none)
bool g_ulb_coop_refused = false;   // the runtime refused a cooperative cluster launch: CS = 1 from then on

const void* ulb_kernel(int cell, int UB, int CS) {
    if (cell == CELL_GRU) {
        if (UB == 16)
            return CS == 4 ? (const void*)bigru_bwd_umma_kernel<16, 4>
                           : CS == 2 ? (const void*)bigru_bwd_umma_kernel<16, 2> : (const void*)bigru_bwd_umma_kernel<16, 1>;
        return CS == 4 ? (const void*)bigru_bwd_umma_kernel<8, 4>
                       : CS == 2 ? (const void*)bigru_bwd_umma_kernel<8, 2> : (const void*)bigru_bwd_umma_kernel<8, 1>;
    }
    if (UB == 16)
        return CS == 4 ? (const void*)bilstm_bwd_umma_kernel<16, 4>
                       : CS == 2 ? (const void*)bilstm_bwd_umma_kernel<16, 2> : (const void*)bilstm_bwd_umma_kernel<16, 1>;
    return CS == 4 ? (const void*)bilstm_bwd_umma_kernel<8, 4>
                   : CS == 2 ? (const void*)bilstm_bwd_umma_kernel<8, 2> : (const void*)bilstm_bwd_umma_kernel<8, 1>;
}

void ulb_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int ctas, int CS, size_t smem,
                       cudaStream_t stream) {
    *cfg = cudaLaunchConfig_t{};
    cfg->gridDim = dim3(ctas);
    cfg->blockDim = dim3(32 * (ULB_EPI_WARPS + 1 + ULB_CTRL));
    cfg->dynamicSmemBytes = smem;
    cfg->stream = stream;
    attr[0].id = cudaLaunchAttributeCooperative;    // every CTA of the launch co-resident, as the exchange needs
    attr[0].val.cooperative = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = CS;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg->attrs = attr;
    cfg->numAttrs = 2;
}

// Clusters of CS blocks of this instance that the device holds at once (0 when it cannot be asked: no device, or a
// runtime without the query).  The planner asks the LSTM instance for both cells: the GRU instances use no more
// registers and the same shared memory (tests/test_host_gru_encoder.py checks it on the compiler's report), so the
// plan and the variant queries are one for both cells.
int ulb_max_clusters(int UB, int CS, int ctas, size_t smem) {
    const void* fn = ulb_kernel(CELL_LSTM, UB, CS);
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[2];
    ulb_launch_config(&cfg, attr, ctas, CS, smem, 0);
    cfg.attrs = attr + 1;                           // the occupancy query takes the cluster shape only
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, fn, &cfg) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return n;
}

// The largest CS in {4, 2} whose staging buffers fit in shared memory, that divides nub into a multiple of 4 sources
// per inbox, and whose clusters the device holds all at once; else 1.
int ulb_cluster(const UlbPlan& pl, size_t cap) {
    for (int cs = 4; cs >= 2; cs >>= 1) {
        if (g_ulb_coop_refused || (g_ulb_cs_cap != 0 && cs > g_ulb_cs_cap)) continue;
        if (pl.nub % cs || (pl.nub / cs) % 4) continue;
        const size_t smem = pl.smem + ulb_staging_bytes(pl.nub, pl.UB, cs);
        if (smem > cap) continue;
        if ((long long)ulb_max_clusters(pl.UB, cs, pl.ctas, smem) * cs < pl.ctas) continue;
        return cs;
    }
    return 1;
}

int ulb_plan(int B, int H, int ndir, UlbPlan* out, bool cluster = true) {
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
            const size_t inbox = (size_t)nub * UL_BC * UB * 4;      // partials one destination receives per step (CS = 1)
            const size_t smem = (size_t)2 * H * 128 + ULB_SMEM_FIXED;
            if (smem > cap || (inbox / ULB_CTRL) % 16 || (2 * H * 128) % 32768) continue;
            out->UB = UB; out->nub = nub; out->nbg = nbg; out->ctas = ctas; out->Bsub = Bs;
            out->nsplit = (B + Bs - 1) / Bs; out->smem = smem;
            out->pack_bytes = (size_t)ndir * nub * 2 * H * 128;
            out->xbuf_bytes = (size_t)ndir * nbg * 2 * nub * inbox;
            out->CS = cluster ? ulb_cluster(*out, cap) : 1;
            out->smem += ulb_staging_bytes(nub, UB, out->CS);
            return 0;
        }
        if (Bs <= UL_BC) break;
    }
    return -2;
}

// One launch per row block.  A cooperative cluster launch that the runtime refuses runs nothing: the launches then
// fall back to CS = 1 (and the planner never picks CS > 1 again in this process).
template <int CELL, int UB>
int ul_launch_bwd(UlbPlan pl, UlParams p, const float* w_hh, cudaStream_t stream) {
    {
        const long long n = (long long)p.ndir * pl.nub * 2 * p.H * 64;
        int blocks = (int)((n + 255) / 256);
        if (blocks > 8192) blocks = 8192;
        ul_pack_bwd_kernel<UB><<<blocks, 256, 0, stream>>>(w_hh, const_cast<uint8_t*>(p.wpack), p.H, p.ndir);
        B200_LAUNCH_CHECK("ul_pack_bwd_kernel");
    }
    for (;;) {
        const void* fn = ulb_kernel(CELL, UB, pl.CS);
        B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
        if (pl.CS == 1) {
            int per_sm = 0;
            B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 32 * (ULB_EPI_WARPS + 1 + ULB_CTRL),
                                                                    pl.smem));
            B200_REQUIRE((long long)per_sm * sm_count() >= pl.ctas,
                         "bilstm(umma bwd): %d CTAs cannot be co-resident (%d/SM x %d SMs)", pl.ctas, per_sm, sm_count());
        }
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute attr[2];
        ulb_launch_config(&cfg, attr, pl.ctas, pl.CS, pl.smem, stream);
        bool refused = false;
        for (int sp = 0; sp < pl.nsplit; ++sp) {
            p.b0 = sp * pl.Bsub;
            p.Bend = p.b0 + pl.Bsub < p.B ? p.b0 + pl.Bsub : p.B;
            B200_CUDA(cudaMemsetAsync(p.counters, 0, UL_COUNTER_BYTES, stream));
            B200_CUDA(cudaMemsetAsync(p.xbuf, 0, pl.xbuf_bytes, stream));     // generation tags start at 0
            void* args[] = {&p};
            const cudaError_t e = cudaLaunchKernelExC(&cfg, fn, args);
            if (e != cudaSuccess && pl.CS > 1 && sp == 0) {
                (void)cudaGetLastError();
                refused = true;
                break;
            }
            B200_CUDA(e);
            count_launch();
        }
        if (!refused) return B200_OK;
        g_ulb_coop_refused = true;
        pl.smem -= ulb_staging_bytes(pl.nub, UB, pl.CS);
        pl.CS = 1;
    }
}

}  // namespace

bool lstm_umma_bwd_variant(int B, int H, int ndir, int* ub, int* nsplit) {
    UlbPlan pl;
    if (ulb_plan(B, H, ndir, &pl, false) != 0) return false;
    *ub = pl.UB;
    *nsplit = pl.nsplit;
    return true;
}

int lstm_umma_bwd_cluster(int B, int H, int ndir) {
    UlbPlan pl;
    return ulb_plan(B, H, ndir, &pl) == 0 ? pl.CS : -1;
}

void lstm_umma_set_cluster_cap(int cap) { g_ulb_cs_cap = cap; }

bool lstm_umma_fwd_variant(int B, int H, int ndir, int* ub, int* ubp, int* nsplit) {
    UlPlan pl;
    if (ul_plan(B, H, ndir, &pl) != 0) return false;
    *ub = pl.UB;
    *ubp = pl.UBp;
    *nsplit = pl.nsplit;
    return true;
}

int lstm_umma_bwd(int cell, float* gates, const float* w_hh, const float* cstate, const float* dout, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    UlbPlan pl;
    B200_REQUIRE(ulb_plan(B, H, ndir, &pl) == 0, "bilstm(umma bwd): unsupported shape B=%d H=%d ndir=%d", B, H, ndir);
    B200_REQUIRE(workspace_bytes >= lstm_umma_workspace_bytes(B, H, ndir), "bilstm(umma bwd): workspace too small");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    UlParams p;
    p.gates = gates; p.cst = const_cast<float*>(cstate); p.out = const_cast<float*>(dout);
    p.wpack = ws;
    p.xbuf = ws + ul_align(pl.pack_bytes);
    p.counters = reinterpret_cast<unsigned*>(ws + ul_align(pl.pack_bytes) + ul_align(pl.xbuf_bytes));
    p.err_flag = reinterpret_cast<int*>(p.counters + (UL_COUNTER_BYTES / 4 - 4));
    p.B = B; p.T = T; p.H = H; p.ndir = ndir; p.UB = pl.UB; p.nub = pl.nub; p.nbg = pl.nbg; p.NA = 0; p.NC = ULB_CTRL;
    p.strict = 0;
    p.b0 = 0; p.Bend = B;
    if (cell == CELL_GRU) {
        if (pl.UB == 16) return ul_launch_bwd<CELL_GRU, 16>(pl, p, w_hh, stream);
        return ul_launch_bwd<CELL_GRU, 8>(pl, p, w_hh, stream);
    }
    if (pl.UB == 16) return ul_launch_bwd<CELL_LSTM, 16>(pl, p, w_hh, stream);
    return ul_launch_bwd<CELL_LSTM, 8>(pl, p, w_hh, stream);
}

size_t lstm_umma_workspace_bytes(int B, int H, int ndir) {
    UlPlan pl;
    UlbPlan pb;
    size_t f = 0, b = 0;
    if (ul_plan(B, H, ndir, &pl) == 0) f = ul_align(pl.pack_bytes) + ul_align(pl.xbuf_bytes) + UL_COUNTER_BYTES;
    if (ulb_plan(B, H, ndir, &pb, false) == 0) b = ul_align(pb.pack_bytes) + ul_align(pb.xbuf_bytes) + UL_COUNTER_BYTES;
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

int lstm_umma_fwd(int cell, float* gates, const float* w_hh, float* cstate, float* out, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, bool strict, cudaStream_t stream) {
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
    p.B = B; p.T = T; p.H = H; p.ndir = ndir; p.UB = pl.UB; p.nub = pl.nub; p.nbg = pl.nbg; p.NA = pl.NA;
    p.NC = pl.NA < UL_MAX_CTRL ? pl.NA : UL_MAX_CTRL;
    p.strict = strict ? 1 : 0;
    p.b0 = 0; p.Bend = B;
    if (cell == CELL_GRU) {
        switch (pl.UBp) {
            case 8: return ul_launch_fwd<CELL_GRU, 8>(pl, p, w_hh, stream);
            case 12: return ul_launch_fwd<CELL_GRU, 12>(pl, p, w_hh, stream);
            default: return ul_launch_fwd<CELL_GRU, 16>(pl, p, w_hh, stream);
        }
    }
    switch (pl.UBp) {
        case 8: return ul_launch_fwd<CELL_LSTM, 8>(pl, p, w_hh, stream);
        case 12: return ul_launch_fwd<CELL_LSTM, 12>(pl, p, w_hh, stream);
        default: return ul_launch_fwd<CELL_LSTM, 16>(pl, p, w_hh, stream);
    }
}

}  // namespace b200asr
