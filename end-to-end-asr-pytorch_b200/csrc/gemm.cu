// K6 / K9 / K11: the dense contractions of the step on the Hopper tensor cores (wgmma), fp32 in and out, fp32-class
// accuracy ("3xTF32").  ONE kernel template serves the three operand arrangements of a layer y = x . W^T + b:
//   tn :  C[M,N] (+)= A[M,K] . B[N,K]^T + bias      forward  (x . W^T): both operands K-major (K contiguous)
//   nn :  C[M,N] (+)= A[M,K] . B[K,N]               input gradient (dY . W): B is MN-major (N contiguous)
//   nt :  C[M,N] (+)= sum_r A[r,M]^T . B[r,N]       weight gradient (dY^T . X): the contraction runs over the B*T rows,
//                                                    both operands MN-major; rows are addressed as (batch, time) so
//                                                    that B can be read SHIFTED by one time step (dW_hh = dG^T . h_prev
//                                                    without materialising h_prev: the row before the first / after the
//                                                    last step of an utterance is out of bounds = zero-filled by TMA)
//   conv mode (conv3x3_gemm_kernel, the same body): a 3x3 convolution over a zero-haloed channels-last buffer as an implicit GEMM - tn with the A
//                     box of each 32-wide K block (one tap) loaded at that tap's row shift, nt (weight gradient) with
//                     each B box at its tap's shift; see GemmArgs and b200asr_conv3x3_fwd / _wgrad (VGGExtractor)
//   reference call sites: the input projection inside nn.LSTM (src/module.py:112-113,131), the CTC head (src/asr.py:29,
//   96), proj_k / char_trans / pj (src/asr.py:242-243,177,220; src/module.py:123,155) and their autograd backward.
//
// wgmma .tf32 reads fp32 bit patterns from shared memory and ignores the low 13 mantissa bits (the tn form on W^T, which
// reads B raw, and the nn form, which truncates B explicitly, give bit-equal results: tests/test_gpu_gemm_mainloop.py),
// so a raw K-major fp32 B tile IS the TF32 "hi" operand; the residual  lo = x - trunc(x)  is a second tile of the same
// layout.  A is split into hi and lo in registers.  Per 32-wide K block the two consumer warpgroups accumulate
// A_hi.B + A_lo.B + A_hi.B_lo  in one fp32 register accumulator.
// wgmma has no MN-major form for 32-bit types: an MN-major B is loaded as plain [32 k][32 column] boxes and transposed
// into the K-major swizzled image (hi and lo at once); an MN-major A is gathered into the register fragments with
// transposed addressing.
//
// One 128 x 128 tile per CTA (x split-K slices when the tile grid alone cannot fill the SMs: partial tiles go to a
// workspace and a second small kernel sums them in a fixed order - deterministic).
//
// Warp roles.  Warpgroup 0 (setmaxnreg 40): lane 0 of warp 0 issues the TMA loads (out-of-bounds rows / K tail
// zero-filled by the hardware); warps 1..3 make the B operand's TF32 images when the stage does not bring them
// (MN-major B: transpose into the K-major swizzled hi / lo images; K-major B without a pre-computed residual: the lo
// tile) and signal them on their own barrier.  Warpgroups 1 and 2 (setmaxnreg 232) are the consumers, 64 tile rows
// each: per K block every thread loads its A fragment from the stage, splits it into hi = trunc_tf32(x) and
// lo = x - hi in registers and issues  A_hi.B, A_lo.B, A_hi.B_lo  per 8 k with A from registers (wgmma RS form), so
// only B is read by the tensor core from shared memory.  Block i+1 is issued before block i is waited for
// (wait_group 1); the wait that retires a block releases its stage (one arrive per warp), and the A fragments are
// double-buffered because a register operand may not change before its MMAs retire.  The accumulation chain is cut
// every G_CH K blocks and summed with IEEE fp32 adds in a second register tile (the tensor core's fp32 accumulate is
// not IEEE-rounded); each chunk is one straight-line body (mma_chunk) that ends in the only drain of the loop.  The
// epilogue (+ bias [+ C]) runs from those registers.
//
// Shared memory per K block of a tn stage: wgmma B reads 96 KB + A fragment loads 16 KB + TMA writes 48 KB (B lo
// pre-computed) = 160 KB for 1536 tensor-core cycles, ~104 B/clk against the ~128 B/clk an SM moves.  An nt stage adds
// the B transpose (16 KB read, 32 KB written): 208 KB, ~135 B/clk.
//
// Shared-memory images.  K-major operand, R rows: R consecutive 128-byte rows (32 k each), 128-byte swizzle; one MMA
// (8 k) advances the descriptor start by 32 bytes.  MN-major operand as loaded: R/32 boxes of [32 k][32 columns] =
// 4096 bytes each (a TMA box {32 columns, 32 rows}); A's boxes with the 128-byte swizzle (see AFragAddr), B's
// without (the transposing pass reads one k row of 32 columns per warp load).
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/b200asr.h"
#include "../../include/b200asr_debug.h"

namespace b200asr {
namespace {

constexpr int G_BM = 128, G_BN = 128, G_BK = 32;
constexpr int G_TILE = G_BM * G_BK * 4;         // 16 KB: one operand tile (G_BM == G_BN)
constexpr int G_CONSUMERS = 256;                // two warpgroups
constexpr int G_THREADS = 128 + G_CONSUMERS;    // warpgroup 0: TMA producer + B image makers
constexpr int G_PREP_WARPS = 3;                 // warps 1..3
constexpr int G_PRODUCER_REGS = 40, G_CONSUMER_REGS = 232;   // 128 * 40 + 256 * 232 <= 65536
constexpr int G_BOX = 32 * G_BK * 4;            // one MN-major box: 32 columns x 32 k
constexpr int G_MAX_SPLIT = 32;
constexpr int G_CH_DEFAULT = 4;                 // K blocks per accumulation chunk; 1, 2 or 4

// stage: [A as loaded | B as loaded | B lo | B hi (K-major image, MN-major B only)]
template <bool B_MN>
struct GemmSmem {
    static constexpr int STAGE = (B_MN ? 4 : 3) * G_TILE;
    static constexpr int STAGES = B_MN ? 3 : 4;                 // 192 KB either way
    static constexpr int B_LO = 2 * G_TILE;
    static constexpr int B_HI = B_MN ? 3 * G_TILE : G_TILE;     // K-major B: the raw tile is the hi operand
};

struct GemmArgs {
    const float* bias;
    float* C;
    float* partial;        // [nsplit][M][N] when nsplit > 1
    int M, N, ldc, accumulate, perm;
    int KB;                // K blocks (of 32) in total
    int kb_per_split;
    int kbt;               // K blocks per batch entry (MN-major operands walk (batch, time)); KB = batches * kbt
    int a_shift, b_shift;  // time shift of the rows read from A / B (nt form)
    int ch;                // K blocks per accumulation chunk
    // Conv mode (CONV kernels): 3x3 convolution over a zero-haloed channels-last buffer [batches][T + 2][F + 2][C] as
    // an implicit GEMM.  K = taps * C in (tap, channel) order; the K block at k reads tap k / cv_c, whose rows sit
    // (tap / 3) (F + 2) + tap % 3 rows after the output row (tn: A rows; nt: B rows).  Output row m is the padded
    // position m of the grid (t = (m / (F + 2)) % (T + 2), f = m % (F + 2)); rows with t >= T or f >= F are junk.
    int cv_c, cv_fp, cv_t, cv_f;
    int cv_relu;           // tn epilogue: + bias, then ReLU
    const float* cv_mask;  // tn epilogue: zero where mask <= 0 (ReLU backward on the saved activation), pitch ldc
};

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::
            "r"(smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void g_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ float tf32_residual(float x) { return x - tf32_trunc(x); }

// Residual of a K-major tile (elementwise: the image keeps its layout); pt = thread index among the image makers.
__device__ __forceinline__ void split_k_tile(const uint8_t* raw, uint8_t* lo, int pt) {
    const float4* src = reinterpret_cast<const float4*>(raw);
    float4* dst = reinterpret_cast<float4*>(lo);
#pragma unroll 4
    for (int j = pt; j < G_TILE / 16; j += G_PREP_WARPS * 32) {
        const float4 v = src[j];
        dst[j] = make_float4(tf32_residual(v.x), tf32_residual(v.y), tf32_residual(v.z), tf32_residual(v.w));
    }
}
// [32 k][32 column] boxes -> K-major swizzled hi and lo images.  Work item = (box, 4 consecutive k); warp pw moves
// items pw, pw + G_PREP_WARPS, ..., lane = column.  Loads: one k row of 32 columns per warp instruction (conflict-free);
// stores: 16 bytes per lane, 8 consecutive rows hit 8 different swizzled chunks (conflict-free).
__device__ __forceinline__ void split_mn_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int boxes, int pw,
                                              int lane) {
    for (int it = pw; it < boxes * 8; it += G_PREP_WARPS) {
        const int j = it >> 3, k0 = (it & 7) * 4;
        const float* b = reinterpret_cast<const float*>(raw + j * G_BOX) + k0 * 32 + lane;
        const float x0 = b[0], x1 = b[32], x2 = b[64], x3 = b[96];
        const uint32_t off = wgmma::sw128_offset(32 * j + lane, k0 * 4);
        *reinterpret_cast<float4*>(hi + off) = make_float4(tf32_trunc(x0), tf32_trunc(x1), tf32_trunc(x2), tf32_trunc(x3));
        *reinterpret_cast<float4*>(lo + off) =
            make_float4(tf32_residual(x0), tf32_residual(x1), tf32_residual(x2), tf32_residual(x3));
    }
}

// MN-major A: MMA row r of the tile reads (and the epilogue writes) tile row mn_row(r), which rotates bits 2..4 of the
// row index: bit 2 moves to bit 4, bits 3..4 move to bits 2..3.  See AFragAddr for why.
__host__ __device__ __forceinline__ int mn_row(int r) { return (r & 0x63) | ((r & 0x04) << 2) | ((r & 0x18) >> 1); }

// A fragment of one thread per K block: [hi | lo][k8 step][register of the RS operand].
struct AFrag {
    uint32_t v[2][G_BK / 8][4];
};

// Byte offsets (inside the stage's A tile) of the thread's fragment elements for q = 0 (k = 8 k4 + l%4) and q = 1
// (k = 8 k4 + l%4 + 4), h = 0 (MMA row r) and h = 1 (row r + 8); k4 adds k4 * K4_STEP.  r = 64 wg + 16 w + l/4.
//   K-major A: element (row m, k) at sw128_offset(m, 4 k); for one load instruction the 8 rows m = r0 + l/4 have
//     m & 7 = l/4, so the chunks (2 k4 + q) ^ (l/4) are 8 different ones and l%4 picks the word: 32 banks.
//   MN-major A (swizzled [32 k][32 m] boxes): element (k, m) at 4096 (m >> 5) + 128 k + 16 (((m >> 2) & 7) ^ (k & 7))
//     + 4 (m & 3).  With m = mn_row(r): bits 0..1 of m are l%4's partner l/4 & 3, bit 4 is l/4 >> 2, bits 2..3 are
//     fixed per (warp, h).  k & 7 = l%4 + 4q, so the chunk's bits 0..1 are (fixed) ^ l%4 and bit 2 is (l/4 >> 2) ^ q:
//     bank = 4 chunk + (m & 3) takes each of the 32 values once.  Without the row permutation bit 2 of the chunk
//     would come from both l/4 and l%4 (two-way conflict); without the swizzle every lane of a column would share
//     a bank (four-way).
template <bool A_MN>
struct AFragAddr {
    static constexpr uint32_t K4_STEP = A_MN ? 8 * 128 : 32;
    uint32_t off[2][2];   // [q][h]
    __device__ __forceinline__ AFragAddr(int r) {
        const int tq = threadIdx.x & 3;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int rr = r + 8 * h;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                if (A_MN) {
                    const int m = mn_row(rr), k = tq + 4 * q;
                    off[q][h] = (uint32_t)((m >> 5) * G_BOX + k * 128 + ((((m >> 2) & 7) ^ k) << 4) + (m & 3) * 4);
                } else {
                    off[q][h] = wgmma::sw128_offset((uint32_t)rr, (uint32_t)(16 * q + 4 * tq));
                }
            }
        }
    }
    // K-major: the k4 step moves 32 bytes inside the row, i.e. chunk c -> c + 2 before the swizzle: XOR form
    __device__ __forceinline__ uint32_t at(int k4, int q, int h) const {
        if (A_MN) return off[q][h] + k4 * K4_STEP;
        return off[q][h] ^ (uint32_t)(k4 * 32);
    }
};

template <bool A_MN>
__device__ __forceinline__ void load_a_frag(AFrag& f, const uint8_t* a_tile, const AFragAddr<A_MN>& ad) {
#pragma unroll
    for (int k4 = 0; k4 < G_BK / 8; ++k4)
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t x = *reinterpret_cast<const uint32_t*>(a_tile + ad.at(k4, q, h));
                const uint32_t hi = x & 0xffffe000u;
                f.v[0][k4][2 * q + h] = hi;
                f.v[1][k4][2 * q + h] = __float_as_uint(__uint_as_float(x) - __uint_as_float(hi));
            }
}
__device__ __forceinline__ void keep(AFrag& f) {
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int k4 = 0; k4 < G_BK / 8; ++k4) wgmma::fence_operand(f.v[p][k4]);
}

// One accumulation chunk of LEN K blocks, starting at block i0 of the slice, into d (overwritten): block j + 1 is
// issued before block j is waited for (wait_group 1), the wait that retires a block releases its stage (one arrive per
// warp), the chunk ends in a drain.  Straight-line code with the fragments local to the chunk, so that the compiler sees
// which wait retires which register operand and adds no wait of its own (it would at a loop back-edge that carries
// MMAs in flight).  The consumers wait for the TMA bytes (full: A is read with generic loads) and, when warps 1..3
// make B's images, for those as well (ready).
template <int LEN, bool A_MN, bool B_PREP, class L>
__device__ __forceinline__ void mma_chunk(float (&d)[64], int i0, const uint8_t* smem, uint64_t* full, uint64_t* ready,
                                          uint64_t* empty, const AFragAddr<A_MN>& ad, int lane) {
    AFrag f[2];
#pragma unroll
    for (int j = 0; j < LEN; ++j) {
        const int i = i0 + j, s = i % L::STAGES;
        const uint32_t phase = (uint32_t)((i / L::STAGES) & 1);
        mbar_wait(&full[s], phase);
        if (B_PREP) mbar_wait(&ready[s], phase);
        const uint8_t* st = smem + s * L::STAGE;
        load_a_frag<A_MN>(f[j & 1], st, ad);
        const uint32_t b = smem_u32(st) + L::B_HI, blo = smem_u32(st) + L::B_LO;
        wgmma::fence_operand(d);
        wgmma::fence();
#pragma unroll
        for (int k4 = 0; k4 < G_BK / 8; ++k4) {
            const uint64_t db = wgmma::desc_k_sw128(b + k4 * 32);
            wgmma::mma_tf32_n128_rs(d, f[j & 1].v[0][k4], db, (j | k4) != 0);
            wgmma::mma_tf32_n128_rs(d, f[j & 1].v[1][k4], db, 1);
            wgmma::mma_tf32_n128_rs(d, f[j & 1].v[0][k4], wgmma::desc_k_sw128(blo + k4 * 32), 1);
        }
        wgmma::commit_group();
        if (j + 1 < LEN) wgmma::wait_group<1>();       // block j - 1 retired, block j stays in flight
        else wgmma::wait_all();
        if (j > 0) keep(f[(j - 1) & 1]);
        if (lane == 0 && j > 0) g_arrive(&empty[(i - 1) % L::STAGES]);
    }
    wgmma::fence_operand(d);
    keep(f[(LEN - 1) & 1]);
    if (lane == 0) g_arrive(&empty[(i0 + LEN - 1) % L::STAGES]);
}

// Epilogue of a consumer thread: its accumulator fragment (tile rows row0 / row1, columns n0 + 8 gq + 2 (lane % 4) + {0,1})
// -> C (+ bias, + C when accumulating, rows through the gate permutation when perm), or -> its split-K partial tile.
__device__ __forceinline__ void store_acc(const float (&acc)[64], const float* bias_in, float* C, float* partial, int M,
                                          int N, int ldc_in, int accumulate_in, int perm, int row0, int row1, int n0,
                                          int lane) {
    const bool to_partial = gridDim.z > 1;
    float* Cb = to_partial ? partial + (size_t)blockIdx.z * M * N : C;
    const int ldc = to_partial ? N : ldc_in;
    const float* bias = to_partial ? nullptr : bias_in;
    const int accumulate = to_partial ? 0 : accumulate_in;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = h ? row1 : row0;
        if (row >= M) continue;
        const int orow = (!to_partial && perm) ? (row & 3) * (M >> 2) + (row >> 2) : row;
        float* crow = Cb + (size_t)orow * ldc;
        const bool vec = ((ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(Cb) & 7) == 0);
#pragma unroll
        for (int gq = 0; gq < 16; ++gq) {
            const int n = n0 + 8 * gq + 2 * (lane & 3);
            float o0 = acc[4 * gq + 2 * h], o1 = acc[4 * gq + 2 * h + 1];
            if (bias && n < N) o0 += bias[n];
            if (bias && n + 1 < N) o1 += bias[n + 1];
            if (vec && n + 1 < N) {
                float2* p2 = reinterpret_cast<float2*>(crow + n);
                if (accumulate) { const float2 old = *p2; o0 += old.x; o1 += old.y; }
                *p2 = make_float2(o0, o1);
            } else {
                if (n < N) crow[n] = accumulate ? crow[n] + o0 : o0;
                if (n + 1 < N) crow[n + 1] = accumulate ? crow[n + 1] + o1 : o1;
            }
        }
    }
}

// Epilogue of the conv-mode tn form (never split): per output row of the grid, + bias, ReLU or the ReLU-backward mask,
// and exact zeros on junk rows.  C (and the mask) are addressed at the row's zero-haloed position, so junk rows land on
// the halo of the next buffer and keep it zero.  N % 4 == 0 (checked by the host).
__device__ __forceinline__ void conv_store(const float (&acc)[64], const GemmArgs& g, int row0, int row1, int n0,
                                           int lane) {
    const int per = (g.cv_t + 2) * g.cv_fp;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = h ? row1 : row0;
        if (row >= g.M) continue;
        const int r = row % per, t = r / g.cv_fp, f = r - t * g.cv_fp;
        const bool junk = t >= g.cv_t || f >= g.cv_f;
        float* crow = g.C + (size_t)row * g.ldc;
        const float* mrow = g.cv_mask ? g.cv_mask + (size_t)row * g.ldc : nullptr;
#pragma unroll
        for (int gq = 0; gq < 16; ++gq) {
            const int n = n0 + 8 * gq + 2 * (lane & 3);
            if (n >= g.N) continue;
            float o0 = acc[4 * gq + 2 * h], o1 = acc[4 * gq + 2 * h + 1];
            if (g.bias) { o0 += g.bias[n]; o1 += g.bias[n + 1]; }
            if (g.cv_relu) { o0 = o0 < 0.f ? 0.f : o0; o1 = o1 < 0.f ? 0.f : o1; }    // NaN stays NaN, as clamp_min
            if (mrow) {                                                               // as ATen's threshold_backward
                const float2 mk = *reinterpret_cast<const float2*>(mrow + n);
                o0 = mk.x <= 0.f ? 0.f : o0;
                o1 = mk.y <= 0.f ? 0.f : o1;
            }
            if (junk) o0 = o1 = 0.f;
            *reinterpret_cast<float2*>(crow + n) = make_float2(o0, o1);
        }
    }
}

// B_PRE: the residual of a K-major B comes from a pre-computed residual matrix (same shape / layout: the weights, split
// once per step by b200asr_tf32_residual) through its own tensor map.  An MN-major B goes through the transposing
// pass, which makes its residual in the same sweep.
// The kernel body, shared by gemm3x_kernel (the dense forms) and conv3x3_gemm_kernel (CONV: the conv mode).
template <bool A_MN, bool B_MN, bool B_PRE, bool CONV>
__device__ __forceinline__ void gemm3x_body(const CUtensorMap& map_a, const CUtensorMap& map_b,
                                            const CUtensorMap& map_blo, const GemmArgs& g) {
    using L = GemmSmem<B_MN>;
    static_assert(!(B_PRE && B_MN), "only a K-major B brings a pre-computed residual");
    constexpr bool B_PREP = B_MN || !B_PRE;                        // warps 1..3 make B images
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::STAGES * L::STAGE);      // TMA landed
    uint64_t* ready = full + L::STAGES;                                              // B images made (B_PREP)
    uint64_t* empty = ready + L::STAGES;                                             // MMAs of the stage retired

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * G_BM, n0 = blockIdx.x * G_BN;
    const int M = g.M, N = g.N;
    const int kb0 = blockIdx.z * g.kb_per_split;
    // K blocks of this slice (>= 1 by construction of the grid).  Evaluated by each role after its setmaxnreg: a value
    // live across the register reallocation is kept in local memory.
    auto slice_blocks = [&]() { return min(g.KB, kb0 + g.kb_per_split) - kb0; };
    const int a_boxes = min(G_BM / 32, (M - m0 + 31) / 32);      // MN-major: 32-column boxes that hold real data
    const int b_boxes = min(G_BN / 32, (N - n0 + 31) / 32);
    const uint32_t a_bytes = A_MN ? (uint32_t)a_boxes * G_BOX : (uint32_t)G_TILE;
    const uint32_t b_bytes = B_MN ? (uint32_t)b_boxes * G_BOX : (uint32_t)G_TILE;

    if (tid == 0) {
        for (int s = 0; s < L::STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&ready[s], G_PREP_WARPS * 32);
            mbar_init(&empty[s], G_CONSUMERS / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(G_PRODUCER_REGS) : "memory");
        const int nkb = slice_blocks();
        if (warp == 0) {
            if (lane == 0) {
                for (int i = 0; i < nkb; ++i) {
                    const int kb = kb0 + i;
                    const int s = i % L::STAGES;
                    if (i >= L::STAGES) mbar_wait(&empty[s], (uint32_t)(((i / L::STAGES) - 1) & 1));
                    uint8_t* st = smem + s * L::STAGE;
                    mbar_expect_tx(&full[s], a_bytes + (B_PRE ? 2 * b_bytes : b_bytes));
                    const int bt = kb / g.kbt, t0 = (kb - bt * g.kbt) * G_BK;
                    if (CONV && !A_MN) {
                        const int k = kb * G_BK, tap = k / g.cv_c;
                        tma_load_2d(st, &map_a, k - tap * g.cv_c, m0 + (tap / 3) * g.cv_fp + tap % 3, &full[s]);
                    } else if (A_MN) {
                        for (int j = 0; j < a_boxes; ++j)
                            tma_load_3d(st + j * G_BOX, &map_a, m0 + 32 * j, t0 + g.a_shift, bt, &full[s]);
                    } else {
                        tma_load_2d(st, &map_a, kb * G_BK, m0, &full[s]);
                    }
                    if (CONV && B_MN) {
                        for (int j = 0; j < b_boxes; ++j) {
                            const int n = n0 + 32 * j, tap = n / g.cv_c;
                            tma_load_3d(st + G_TILE + j * G_BOX, &map_b, n - tap * g.cv_c,
                                        t0 + (tap / 3) * g.cv_fp + tap % 3, bt, &full[s]);
                        }
                    } else if (B_MN) {
                        for (int j = 0; j < b_boxes; ++j)
                            tma_load_3d(st + G_TILE + j * G_BOX, &map_b, n0 + 32 * j, t0 + g.b_shift, bt, &full[s]);
                    } else {
                        tma_load_2d(st + G_TILE, &map_b, kb * G_BK, n0, &full[s]);
                        if (B_PRE) tma_load_2d(st + L::B_LO, &map_blo, kb * G_BK, n0, &full[s]);
                    }
                }
            }
        } else if (B_PREP) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % L::STAGES;
                mbar_wait(&full[s], (uint32_t)((i / L::STAGES) & 1));
                uint8_t* st = smem + s * L::STAGE;
                if (B_MN) split_mn_tile(st + G_TILE, st + L::B_HI, st + L::B_LO, b_boxes, warp - 1, lane);
                else split_k_tile(st + G_TILE, st + L::B_LO, tid - 32);
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> the tensor core
                g_arrive(&ready[s]);
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(G_CONSUMER_REGS) : "memory");
        const int nkb = slice_blocks();
        const int wg = (warp >> 2) - 1;
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);     // this thread's MMA rows: r0, r0 + 8
        const AFragAddr<A_MN> ad(r0);
        float acc[64], d[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[e] = 0.f;
        for (int i = 0; i < nkb; i += g.ch) {                        // chunks of g.ch blocks, the last one may be shorter
            const int len = min(g.ch, nkb - i);
            if (len == 4) mma_chunk<4, A_MN, B_PREP, L>(d, i, smem, full, ready, empty, ad, lane);
            else if (len == 3) mma_chunk<3, A_MN, B_PREP, L>(d, i, smem, full, ready, empty, ad, lane);
            else if (len == 2) mma_chunk<2, A_MN, B_PREP, L>(d, i, smem, full, ready, empty, ad, lane);
            else mma_chunk<1, A_MN, B_PREP, L>(d, i, smem, full, ready, empty, ad, lane);
#pragma unroll
            for (int e = 0; e < 64; ++e) acc[e] += d[e];            // IEEE-add the chunk
        }
        if (CONV && !A_MN)
            conv_store(acc, g, m0 + r0, m0 + r0 + 8, n0, lane);
        else
            store_acc(acc, g.bias, g.C, g.partial, M, N, g.ldc, g.accumulate, g.perm,
                      m0 + (A_MN ? mn_row(r0) : r0), m0 + (A_MN ? mn_row(r0 + 8) : r0 + 8), n0, lane);
    }
}

template <bool A_MN, bool B_MN, bool B_PRE>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm3x_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
              const __grid_constant__ CUtensorMap map_blo, const GemmArgs g) {
    gemm3x_body<A_MN, B_MN, B_PRE, false>(map_a, map_b, map_blo, g);
}

// Conv mode: WGRAD = false is the tn form (forward / input gradient), true the nt form (weight gradient).
template <bool WGRAD>
__global__ void __launch_bounds__(G_THREADS, 1)
conv3x3_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                    const __grid_constant__ CUtensorMap map_blo, const GemmArgs g) {
    gemm3x_body<WGRAD, WGRAD, false, true>(map_a, map_b, map_blo, g);
}

// C[perm(m)][n] (+)= bias[n] + sum_s partial[s][m][n]   (fixed summation order)
__global__ void gemm3x_reduce_kernel(const float* __restrict__ partial, int nsplit, const float* __restrict__ bias,
                                     float* __restrict__ C, int M, int N, int ldc, int accumulate, int perm) {
    const long long total = (long long)M * N;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / N), n = (int)(i - (long long)m * N);
        float s = partial[i];
        for (int k = 1; k < nsplit; ++k) s += partial[(long long)k * total + i];
        if (bias) s += bias[n];
        const int orow = perm ? (m & 3) * (M >> 2) + (m >> 2) : m;
        float* c = C + (size_t)orow * ldc + n;
        *c = accumulate ? *c + s : s;
    }
}

// lo = x - trunc_tf32(x): the residual the tensor core does not see when it reads the raw fp32 bit pattern.
// Four 128-bit loads in flight per thread (one per thread ran at ~2/3 of the HBM rate).
constexpr int RES_UNROLL = 4;
__global__ void __launch_bounds__(256) tf32_residual_kernel(const float* __restrict__ x, float* __restrict__ lo, long long n) {
    const long long base = (long long)blockIdx.x * (256 * RES_UNROLL * 4) + threadIdx.x * 4;
    if (base + (RES_UNROLL - 1) * 1024 + 3 < n && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(lo)) & 15) == 0) {
        float4 v[RES_UNROLL];
#pragma unroll
        for (int k = 0; k < RES_UNROLL; ++k) v[k] = __ldcs(reinterpret_cast<const float4*>(x + base + k * 1024));
#pragma unroll
        for (int k = 0; k < RES_UNROLL; ++k)
            *reinterpret_cast<float4*>(lo + base + k * 1024) =
                make_float4(tf32_residual(v[k].x), tf32_residual(v[k].y), tf32_residual(v[k].z), tf32_residual(v[k].w));
    } else {
        for (int k = 0; k < RES_UNROLL; ++k)
            for (long long i = base + k * 1024; i < n && i < base + k * 1024 + 4; ++i) lo[i] = tf32_residual(x[i]);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// K-major operand: row-major fp32 matrix [rows, K] with row pitch ld (floats; rows may overlap when ld < K: the im2col
// view of a strided convolution) -> 2-D tensor map with boxes of 32 (K) x box_rows, 128-byte swizzle
int make_map_k(CUtensorMap* map, const float* ptr, int rows, int K, int ld, int box_rows) {
    EncodeTiledFn enc = encode_fn();
    B200_REQUIRE(enc != nullptr, "gemm: cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)G_BK, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "gemm: cuTensorMapEncodeTiled failed (%d) for a [%d x %d] matrix", (int)r, rows, K);
    return B200_OK;
}

// MN-major operand: element (batch b, time t, column c) at ptr[b * bstride + t * ld + c] -> 3-D tensor map (c, t, b)
// with boxes of 32 columns x 32 rows x 1 (128-byte swizzle if `swizzle`); reads outside [0,cols) x [0,T) are zero-filled
int make_map_mn(CUtensorMap* map, const float* ptr, int cols, int T, int batches, long long ld, long long bstride,
                bool swizzle) {
    EncodeTiledFn enc = encode_fn();
    B200_REQUIRE(enc != nullptr, "gemm: cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)T, (cuuint64_t)batches};
    const cuuint64_t strides[2] = {(cuuint64_t)ld * sizeof(float), (cuuint64_t)(batches > 1 ? bstride : ld * (long long)T) * sizeof(float)};
    const cuuint32_t box[3] = {32, (cuuint32_t)G_BK, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "gemm: cuTensorMapEncodeTiled failed (%d) for a [%d x %d x %d] operand", (int)r,
                 batches, T, cols);
    return B200_OK;
}

// Split-K factor.  Few tiles (skinny products): one slice per idle SM.  A tile grid that is neither small nor a
// multiple of the SM count is cut so that the CTA count lands just below a multiple of the SM count - as long as a
// slice keeps >= 64 K blocks and the partial tiles stay below 160 MB.
int max_split(int M, int N) {
    const long long per = (long long)M * N * (long long)sizeof(float);
    long long s = (160LL << 20) / (per > 0 ? per : 1);
    if (s > G_MAX_SPLIT) s = G_MAX_SPLIT;
    return s < 1 ? 1 : (int)s;
}

// Which rule decided the split count (b200asr_debug_gemm_plan reports it).
enum SplitRule { SPLIT_ONE = 0, SPLIT_SM_FILL = 1, SPLIT_EFFICIENCY = 2, SPLIT_WORKSPACE = 3 };

int pick_split(int M, int N, int KB, int* rule) {
    const int tiles = ((M + G_BM - 1) / G_BM) * ((N + G_BN - 1) / G_BN);
    const int sms = sm_count();
    int s = sms / tiles;
    if (s > KB / 8) s = KB / 8;           // at least 8 K blocks per slice
    if (s > G_MAX_SPLIT) s = G_MAX_SPLIT;
    if (s < 1) s = 1;
    *rule = s > 1 ? SPLIT_SM_FILL : SPLIT_ONE;
    auto eff = [&](int q) {
        const long long ctas = (long long)tiles * q;
        return (double)ctas / (double)(((ctas + sms - 1) / sms) * sms);
    };
    if (2 * tiles <= sms && eff(s) < 0.93) {
        const int cap = max_split(M, N);
        for (int q = s + 1; q <= cap && KB / q >= 64; ++q)
            if (eff(q) >= 0.97) { *rule = SPLIT_EFFICIENCY; return q; }
    }
    return s;
}

// The split-K plan of one launch, for both kernels: the count pick_split asks for (counted in K blocks of 32 k, so the
// f16x3 kernel's 64-k blocks count twice), one slice when the workspace cannot hold the partial tiles, slices of whole
// units of `unit` K blocks (f16x3: one scale chunk), and no empty slices.
struct SplitPlan {
    int rule, requested, nsplit, kb_per_split;
};

SplitPlan plan_split(int M, int N, int KB, int unit, int rule_kb, size_t ws_bytes) {
    SplitPlan p;
    p.requested = pick_split(M, N, rule_kb, &p.rule);
    int nsplit = p.requested;
    if (nsplit > 1 && ws_bytes < (size_t)nsplit * M * N * sizeof(float)) {
        nsplit = 1;
        p.rule = SPLIT_WORKSPACE;
    }
    const int units = KB / unit;
    p.kb_per_split = (units + nsplit - 1) / nsplit * unit;
    p.nsplit = (KB + p.kb_per_split - 1) / p.kb_per_split;
    return p;
}

// K blocks per accumulation chunk: B200ASR_GEMM_CHUNK = 1 | 2 | 4 (read once).  The tensor core truncates on every
// accumulate (bias towards zero, growing with the chain length): shorter chunks = less bias, more drains.
int gemm_chunk() {
    static int ch = 0;
    if (!ch) {
        const char* e = getenv("B200ASR_GEMM_CHUNK");
        const int v = e ? atoi(e) : G_CH_DEFAULT;
        ch = (v == 1 || v == 2 || v == 4) ? v : G_CH_DEFAULT;
    }
    return ch;
}

template <bool A_MN, bool B_MN, bool B_PRE = false, bool CONV = false>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, GemmArgs g, void* ws, size_t ws_bytes, cudaStream_t stream,
           const CUtensorMap* mblo = nullptr) {
    const SplitPlan p = plan_split(g.M, g.N, g.KB, 1, g.KB, ws ? ws_bytes : 0);
    const int nsplit = p.nsplit;
    g.kb_per_split = p.kb_per_split;
    g.partial = reinterpret_cast<float*>(ws);
    g.ch = gemm_chunk();
    const size_t smem = (size_t)GemmSmem<B_MN>::STAGES * GemmSmem<B_MN>::STAGE + 256;
    static_assert(!CONV || (A_MN == B_MN && !B_PRE), "conv mode: tn or nt, no pre-split B");
    auto fn = CONV ? conv3x3_gemm_kernel<A_MN> : gemm3x_kernel<A_MN, B_MN, B_PRE>;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((g.N + G_BN - 1) / G_BN, (g.M + G_BM - 1) / G_BM, nsplit);
    fn<<<grid, G_THREADS, smem, stream>>>(ma, mb, mblo ? *mblo : mb, g);
    B200_LAUNCH_CHECK(CONV ? "conv3x3_gemm_kernel" : "gemm3x_kernel");
    if (nsplit > 1) {
        const long long total = (long long)g.M * g.N;
        int blocks = (int)((total + 255) / 256);
        if (blocks > 16 * sm_count()) blocks = 16 * sm_count();
        gemm3x_reduce_kernel<<<blocks, 256, 0, stream>>>(g.partial, nsplit, g.bias, g.C, g.M, g.N, g.ldc, g.accumulate,
                                                         g.perm);
        B200_LAUNCH_CHECK("gemm3x_reduce_kernel");
    }
    return B200_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---------------------------------------------------------------------------------------------------------------------
// f16x3: the LSTM layer contractions on scaled fp16 hi/lo images (DESIGN.md 2.2).  An operand X[outer][k] (k = the
// contraction index) is stored as two K-major fp16 images [outer][Kp] (Kp = K rounded up to F_CK, zero-filled) and one
// power-of-two scale per (outer index, chunk of F_CK k): s = 2^e brings the chunk's largest magnitude to [2^13, 2^14),
//   hi = f16_rn(x s),  lo = f16_rn(x s - hi),  sinv[chunk][outer] = 2^-e.
// x s is exact (power of two), |lo| <= 4 and lo stays an fp16 normal down to 2^-28 of the chunk maximum, so hi + lo
// carries x to ~2^-24 of its chunk maximum with one fp32 accumulator (no x2048 lo and cross-term accumulator needed).
// Per K block of 64 k each consumer warpgroup issues A_hi.B_hi + A_hi.B_lo + A_lo.B_hi (m64n128k16, both operands
// from shared memory) into d; the accumulation chunk is the scale chunk, and its fold  acc += d sa[m] sb[n]  is exact
// (powers of two).  Weight-gradient forms get their operands transposed by the split pass (f16_split_cols_kernel),
// so every GEMM is the same K-major x K-major kernel.
// Non-finite values: the chunk maximum is an integer max over the magnitude bit patterns, so a NaN (bits above Inf)
// or an Inf is seen (fmaxf would drop a NaN); such a chunk gets scale 1, its NaN / Inf reaches hi or lo and poisons
// exactly the outputs of its outer index, as in an fp32 GEMM (finite values of that chunk that overflow fp16 only
// touch the same, already poisoned, outputs).  An all-zero chunk gets scale 1.
constexpr int F_BK = 64;                  // fp16 k per K block: one 128-byte swizzle row
constexpr int F_CK = 128;                 // k per scale chunk = per accumulation chunk
constexpr int F_CH = F_CK / F_BK;         // K blocks per chunk
constexpr int F_TILE = G_BM * F_BK * 2;   // 16 KB: one image tile (G_BM == G_BN)
constexpr int F_STAGE = 4 * F_TILE;       // A hi | A lo | B hi | B lo
constexpr int F_STAGES = 3;               // 192 KB

struct F16Args {
    const float* bias;
    const float* sa;       // inverse scales of A [Kp / F_CK][M]
    const float* sb;       // inverse scales of B [Kp / F_CK][N]
    float* C;
    float* partial;        // [nsplit][M][N] when nsplit > 1
    int M, N, ldc, accumulate, perm;
    int KB, kb_per_split;  // K blocks of F_BK, both multiples of F_CH
};

// floor(log2) of the largest magnitude (bit pattern, sign cleared) -> scale exponent, clamped so that 2^e and 2^-e
// are fp32 normals
__device__ __forceinline__ int f16_scale_exp(uint32_t amax) {
    if (amax == 0u || amax >= 0x7f800000u) return 0;
    const int E = amax >= 0x00800000u ? (int)(amax >> 23) - 127 : (31 - __clz((int)amax)) - 149;
    return min(126, max(-126, 13 - E));
}
__device__ __forceinline__ float pow2f(int e) { return __uint_as_float((uint32_t)(127 + e) << 23); }
__device__ __forceinline__ uint32_t abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }
__device__ __forceinline__ void f16_split2(float x0, float x1, float s, __half2& hi, __half2& lo) {
    const float y0 = x0 * s, y1 = x1 * s;
    hi = __floats2half2_rn(y0, y1);
    lo = __floats2half2_rn(y0 - __low2float(hi), y1 - __high2float(hi));
}

// K-major operand x[row][k] (pitch ld floats): one warp per (row, chunk), 4 k per lane
__global__ void __launch_bounds__(256) f16_split_rows_kernel(const float* __restrict__ x, long long ld, int rows, int K,
                                                             int Kp, __half* __restrict__ hi, __half* __restrict__ lo,
                                                             float* __restrict__ sinv) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, c = blockIdx.y;
    if (row >= rows) return;
    const int k = c * F_CK + 4 * lane;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < K) v = *reinterpret_cast<const float4*>(x + (size_t)row * ld + k);      // K % 4 == 0
    const uint32_t a = __reduce_max_sync(0xffffffffu, max(max(abs_bits(v.x), abs_bits(v.y)), max(abs_bits(v.z), abs_bits(v.w))));
    const int e = f16_scale_exp(a);
    const float s = pow2f(e);
    __half2 h[2], l[2];
    f16_split2(v.x, v.y, s, h[0], l[0]);
    f16_split2(v.z, v.w, s, h[1], l[1]);
    const size_t o = (size_t)row * Kp + k;
    *reinterpret_cast<uint2*>(hi + o) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(lo + o) = *reinterpret_cast<const uint2*>(l);
    if (lane == 0) sinv[(size_t)c * rows + row] = pow2f(-e);
}

// MN-major operand -> transposed image [col][r], r = b T + t over the contraction rows, element x[b bstride + (t + shift)
// ld + col] (zero outside [0, T): the h_prev of a direction, shifted per utterance).  One CTA per (chunk of F_CK rows,
// 64 columns) through shared memory; warp w then writes columns 8w .. 8w + 7, one 256-byte image row per column.
__global__ void __launch_bounds__(256) f16_split_cols_kernel(const float* __restrict__ x, long long ld, long long bstride,
                                                             int shift, int T, int R, int cols, int Rp,
                                                             __half* __restrict__ hi, __half* __restrict__ lo,
                                                             float* __restrict__ sinv) {
    __shared__ float tile[F_CK][65];
    const int r0 = blockIdx.y * F_CK, c0 = blockIdx.x * 64, tid = threadIdx.x;
    const int cq = 4 * (tid & 15);
#pragma unroll
    for (int i = 0; i < F_CK / 16; ++i) {
        const int rr = (tid >> 4) + 16 * i, r = r0 + rr;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < R && c0 + cq < cols) {                  // cols % 4 == 0
            const int b = r / T, t = r - b * T + shift;
            if (t >= 0 && t < T) v = *reinterpret_cast<const float4*>(x + b * bstride + (long long)t * ld + c0 + cq);
        }
        tile[rr][cq] = v.x; tile[rr][cq + 1] = v.y; tile[rr][cq + 2] = v.z; tile[rr][cq + 3] = v.w;
    }
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    for (int j = 0; j < 8; ++j) {
        const int cc = 8 * warp + j, col = c0 + cc;
        if (col >= cols) break;
        const float v0 = tile[2 * lane][cc], v1 = tile[2 * lane + 1][cc];
        const float v2 = tile[64 + 2 * lane][cc], v3 = tile[65 + 2 * lane][cc];
        const uint32_t a = __reduce_max_sync(0xffffffffu, max(max(abs_bits(v0), abs_bits(v1)), max(abs_bits(v2), abs_bits(v3))));
        const int e = f16_scale_exp(a);
        const float s = pow2f(e);
        __half2 h0, l0, h1, l1;
        f16_split2(v0, v1, s, h0, l0);
        f16_split2(v2, v3, s, h1, l1);
        const size_t o = (size_t)col * Rp + r0 + 2 * lane;
        *reinterpret_cast<__half2*>(hi + o) = h0;
        *reinterpret_cast<__half2*>(hi + o + 64) = h1;
        *reinterpret_cast<__half2*>(lo + o) = l0;
        *reinterpret_cast<__half2*>(lo + o + 64) = l1;
        if (lane == 0) sinv[(size_t)blockIdx.y * cols + col] = pow2f(-e);
    }
}

// The gate gradient dG of every direction, g[d][r][c] (R = B T rows, cols = 4 H unit-major columns), read once for the
// three things the layer backward needs from it: the transposed images of each direction (dW_ih, dW_hh; as
// f16_split_cols_kernel), optionally the row images of all directions side by side (dX; as f16_split_rows_kernel, with
// direction d in image columns [d Kp, (d + 1) Kp) and scale chunks [d Kp / F_CK, (d + 1) Kp / F_CK)), and the column
// sums of each 128-row tile (the bias gradient, reduced afterwards in a fixed order: no atomics).  One CTA per (128
// rows, 128 columns, direction) staged in shared memory: its 128 columns of a row are one row-image chunk and its 128
// rows of a column one transposed-image chunk, so every scale and image element comes out of the same values through
// the same f16_scale_exp / f16_split2 as in the single-image passes, bit for bit.
constexpr int DG_PITCH = F_CK + 4;        // staged row pitch (floats): float4 stores, conflict-free float4 column reads
constexpr int DG_SMEM = F_CK * DG_PITCH * 4;

__global__ void __launch_bounds__(256, 3) f16_split_dg_kernel(const float* __restrict__ g, int R, int cols, int Kp,
                                                              int Rp, __half* __restrict__ t_hi,
                                                              __half* __restrict__ t_lo, float* __restrict__ t_sinv,
                                                              __half* __restrict__ r_hi, __half* __restrict__ r_lo,
                                                              float* __restrict__ r_sinv, float* __restrict__ colsum) {
    extern __shared__ float4 dg_smem[];
    float* tile = reinterpret_cast<float*>(dg_smem);
    const int r0 = blockIdx.x * F_CK, c0 = blockIdx.y * F_CK, d = blockIdx.z, ndir = gridDim.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* gd = g + (size_t)d * R * cols;
    // rows warp + 8 i, 4 columns per lane: stage them, and write their row images (8 rows per batch of loads in flight)
    const int c = c0 + 4 * lane;
    const size_t ldr = (size_t)ndir * Kp;
#pragma unroll
    for (int i0 = 0; i0 < F_CK / 8; i0 += 8) {
        float4 v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = r0 + warp + 8 * (i0 + i);
            v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < R && c < cols) v[i] = *reinterpret_cast<const float4*>(gd + (size_t)r * cols + c);   // cols % 4 == 0
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int rr = warp + 8 * (i0 + i), r = r0 + rr;
            *reinterpret_cast<float4*>(tile + rr * DG_PITCH + 4 * lane) = v[i];
            if (r_hi != nullptr && r < R) {
                const uint32_t a = __reduce_max_sync(0xffffffffu, max(max(abs_bits(v[i].x), abs_bits(v[i].y)),
                                                                      max(abs_bits(v[i].z), abs_bits(v[i].w))));
                const int e = f16_scale_exp(a);
                const float s = pow2f(e);
                __half2 h[2], l[2];
                f16_split2(v[i].x, v[i].y, s, h[0], l[0]);
                f16_split2(v[i].z, v[i].w, s, h[1], l[1]);
                const size_t o = (size_t)r * ldr + (size_t)d * Kp + c;
                *reinterpret_cast<uint2*>(r_hi + o) = *reinterpret_cast<const uint2*>(h);
                *reinterpret_cast<uint2*>(r_lo + o) = *reinterpret_cast<const uint2*>(l);
                if (lane == 0) r_sinv[(size_t)(d * (Kp / F_CK) + blockIdx.y) * R + r] = pow2f(-e);
            }
        }
    }
    __syncthreads();
    // warp w: column groups 4 (w + 8 j) .. + 3; lane holds rows lane + 32 i of the group's 4 columns
    const size_t t_img = (size_t)d * cols * Rp, t_sc = (size_t)d * (Rp / F_CK) * cols;
    for (int j = 0; j < F_CK / 32; ++j) {
        const int cc = 4 * (warp + 8 * j), col0 = c0 + cc;
        if (col0 >= cols) break;
        float4 u[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) u[i] = *reinterpret_cast<const float4*>(tile + (lane + 32 * i) * DG_PITCH + cc);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float x0 = (&u[0].x)[q], x1 = (&u[1].x)[q], x2 = (&u[2].x)[q], x3 = (&u[3].x)[q];
            const int col = col0 + q;
            const uint32_t a = __reduce_max_sync(0xffffffffu, max(max(abs_bits(x0), abs_bits(x1)),
                                                                  max(abs_bits(x2), abs_bits(x3))));
            const int e = f16_scale_exp(a);
            const float s = pow2f(e);
            __half2 h01, l01, h23, l23;                 // (rows lane, lane + 32), (lane + 64, lane + 96)
            f16_split2(x0, x1, s, h01, l01);
            f16_split2(x2, x3, s, h23, l23);
            const size_t o = t_img + (size_t)col * Rp + r0 + lane;
            t_hi[o] = __low2half(h01); t_hi[o + 32] = __high2half(h01);
            t_hi[o + 64] = __low2half(h23); t_hi[o + 96] = __high2half(h23);
            t_lo[o] = __low2half(l01); t_lo[o + 32] = __high2half(l01);
            t_lo[o + 64] = __low2half(l23); t_lo[o + 96] = __high2half(l23);
            float sum = (x0 + x1) + (x2 + x3);
#pragma unroll
            for (int m = 16; m > 0; m >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, m);
            if (lane == 0) {
                t_sinv[t_sc + (size_t)blockIdx.x * cols + col] = pow2f(-e);
                colsum[(size_t)blockIdx.x * ndir * cols + (size_t)d * cols + col] = sum;
            }
        }
    }
}

// One accumulation chunk (F_CH K blocks, starting at block i0 of the slice) into d (overwritten): block j + 1 is issued
// before block j is waited for, the wait that retires a block releases its stage, the chunk ends in the only drain.
__device__ __forceinline__ void f16_chunk(float (&d)[64], int i0, const uint8_t* smem, uint64_t* full, uint64_t* empty,
                                          uint32_t a_off, int lane) {
#pragma unroll
    for (int j = 0; j < F_CH; ++j) {
        const int i = i0 + j, s = i % F_STAGES;
        mbar_wait(&full[s], (uint32_t)((i / F_STAGES) & 1));
        const uint32_t st = smem_u32(smem + s * F_STAGE);
        const uint32_t ahi = st + a_off, alo = ahi + F_TILE, bhi = st + 2 * F_TILE, blo = st + 3 * F_TILE;
        wgmma::fence_operand(d);
        wgmma::fence();
#pragma unroll
        for (int k = 0; k < F_BK / 16; ++k) {
            const uint64_t dah = wgmma::desc_k_sw128(ahi + 32 * k), dbh = wgmma::desc_k_sw128(bhi + 32 * k);
            wgmma::mma_f16_n128(d, dah, dbh, (j | k) != 0);
            wgmma::mma_f16_n128(d, dah, wgmma::desc_k_sw128(blo + 32 * k), 1);
            wgmma::mma_f16_n128(d, wgmma::desc_k_sw128(alo + 32 * k), dbh, 1);
        }
        wgmma::commit_group();
        if (j + 1 < F_CH) wgmma::wait_group<1>();
        else wgmma::wait_all();
        if (lane == 0 && j > 0) g_arrive(&empty[(i - 1) % F_STAGES]);
    }
    wgmma::fence_operand(d);
    if (lane == 0) g_arrive(&empty[(i0 + F_CH - 1) % F_STAGES]);
}

// C[M,N] (+)= sum_k A[m][k] B[n][k] (+ bias) on f16x3 images; 128 x 128 tile per CTA (x split-K slices), warp 0 lane 0
// issues the TMA loads of the four image tiles, warpgroups 1 and 2 compute 64 rows each.
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_f16x3_kernel(const __grid_constant__ CUtensorMap map_ahi, const __grid_constant__ CUtensorMap map_alo,
                  const __grid_constant__ CUtensorMap map_bhi, const __grid_constant__ CUtensorMap map_blo,
                  const F16Args g) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + F_STAGES * F_STAGE);
    uint64_t* empty = full + F_STAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * G_BM, n0 = blockIdx.x * G_BN;
    const int kb0 = blockIdx.z * g.kb_per_split;
    auto slice_blocks = [&]() { return min(g.KB, kb0 + g.kb_per_split) - kb0; };
    if (tid == 0) {
        for (int s = 0; s < F_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], G_CONSUMERS / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(G_PRODUCER_REGS) : "memory");
        if (warp == 0 && lane == 0) {
            const int nkb = slice_blocks();
            for (int i = 0; i < nkb; ++i) {
                const int s = i % F_STAGES, k = (kb0 + i) * F_BK;
                if (i >= F_STAGES) mbar_wait(&empty[s], (uint32_t)(((i / F_STAGES) - 1) & 1));
                uint8_t* st = smem + s * F_STAGE;
                mbar_expect_tx(&full[s], 4 * F_TILE);
                tma_load_2d(st, &map_ahi, k, m0, &full[s]);
                tma_load_2d(st + F_TILE, &map_alo, k, m0, &full[s]);
                tma_load_2d(st + 2 * F_TILE, &map_bhi, k, n0, &full[s]);
                tma_load_2d(st + 3 * F_TILE, &map_blo, k, n0, &full[s]);
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(G_CONSUMER_REGS) : "memory");
        const int nkb = slice_blocks();
        const int wg = (warp >> 2) - 1;
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
        const int row0 = m0 + r0, row1 = row0 + 8;
        const int M = g.M, N = g.N;
        float acc[64], d[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[e] = 0.f;
        for (int i = 0; i < nkb; i += F_CH) {
            // this chunk's inverse scales, loaded before its MMAs are issued (rows / columns beyond the matrix: 0)
            const size_t c = (size_t)((kb0 + i) / F_CH);
            const float sa0 = row0 < M ? g.sa[c * M + row0] : 0.f, sa1 = row1 < M ? g.sa[c * M + row1] : 0.f;
            float sb[32];
#pragma unroll
            for (int gq = 0; gq < 16; ++gq) {
                const int n = n0 + 8 * gq + 2 * (lane & 3);
                sb[2 * gq] = n < N ? g.sb[c * N + n] : 0.f;
                sb[2 * gq + 1] = n + 1 < N ? g.sb[c * N + n + 1] : 0.f;
            }
            f16_chunk(d, i, smem, full, empty, (uint32_t)(wg * 64 * 128), lane);
#pragma unroll
            for (int gq = 0; gq < 16; ++gq) {
                acc[4 * gq] += d[4 * gq] * sa0 * sb[2 * gq];
                acc[4 * gq + 1] += d[4 * gq + 1] * sa0 * sb[2 * gq + 1];
                acc[4 * gq + 2] += d[4 * gq + 2] * sa1 * sb[2 * gq];
                acc[4 * gq + 3] += d[4 * gq + 3] * sa1 * sb[2 * gq + 1];
            }
        }
        store_acc(acc, g.bias, g.C, g.partial, M, N, g.ldc, g.accumulate, g.perm, row0, row1, n0, lane);
    }
}

// fp16 image [rows][Kp] -> 2-D tensor map with boxes of F_BK (K) x 128 rows, 128-byte swizzle
int make_map_f16(CUtensorMap* map, const void* ptr, int rows, int Kp) {
    EncodeTiledFn enc = encode_fn();
    B200_REQUIRE(enc != nullptr, "gemm: cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dims[2] = {(cuuint64_t)Kp, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)Kp * 2};
    const cuuint32_t box[2] = {(cuuint32_t)F_BK, (cuuint32_t)G_BM};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "gemm_f16x3: cuTensorMapEncodeTiled failed (%d) for a [%d x %d] image", (int)r, rows,
                 Kp);
    return B200_OK;
}

}  // namespace
}  // namespace b200asr

using namespace b200asr;

extern "C" size_t b200asr_gemm3x_workspace_bytes(int M, int N) {
    if (M <= 0 || N <= 0) return 0;
    int s = max_split(M, N);                   // upper bound of what pick_split() may choose for any K
    const int tiles = ((M + G_BM - 1) / G_BM) * ((N + G_BN - 1) / G_BN);
    if (2 * tiles > sm_count()) s = 1;
    return s > 1 ? (size_t)s * M * N * sizeof(float) : 0;
}

extern "C" int b200asr_gemm3x_tn(const float* A, int lda, const float* B, const float* B_lo, const float* bias, float* C,
                                 int M, int N, int K, int ldc, int accumulate, void* workspace, size_t workspace_bytes,
                                 b200asr_stream stream) {
    B200_REQUIRE(A && B && C, "gemm3x_tn: null pointer");
    B200_REQUIRE(lda > 0 && (lda % 4) == 0, "gemm3x_tn: lda %d must be a positive multiple of 4", lda);
    // TMA: 16-byte aligned row pitch; at least one full tile's worth of work is not required (tails are zero-filled)
    B200_REQUIRE(M > 0 && N > 0 && K > 0 && (K % 4) == 0,
                 "gemm3x_tn: unsupported sizes M=%d N=%d K=%d (K %% 4 must be 0)", M, N, K);
    B200_REQUIRE(ldc >= N, "gemm3x_tn: ldc %d < N %d", ldc, N);
    B200_REQUIRE(aligned16(A) && aligned16(B), "gemm3x_tn: operands must be 16-byte aligned");
    CUtensorMap ma, mb;
    int rc = make_map_k(&ma, A, M, K, lda, G_BM);
    if (rc != B200_OK) return rc;
    rc = make_map_k(&mb, B, N, K, K, G_BN);
    if (rc != B200_OK) return rc;
    GemmArgs g = {};
    g.bias = bias; g.C = C; g.M = M; g.N = N; g.ldc = ldc; g.accumulate = accumulate;
    g.KB = (K + G_BK - 1) / G_BK; g.kbt = g.KB;
    if (B_lo) {
        B200_REQUIRE(aligned16(B_lo), "gemm3x_tn: operands must be 16-byte aligned");
        CUtensorMap mlo;
        rc = make_map_k(&mlo, B_lo, N, K, K, G_BN);
        if (rc != B200_OK) return rc;
        return launch<false, false, true>(ma, mb, g, workspace, workspace_bytes, (cudaStream_t)stream, &mlo);
    }
    return launch<false, false>(ma, mb, g, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_gemm3x_nn(const float* A, int lda, const float* B, int ldb, const float* bias, float* C, int M,
                                 int N, int K, int ldc, int accumulate, void* workspace, size_t workspace_bytes,
                                 b200asr_stream stream) {
    B200_REQUIRE(A && B && C, "gemm3x_nn: null pointer");
    B200_REQUIRE(M > 0 && N > 0 && K > 0, "gemm3x_nn: bad sizes M=%d N=%d K=%d", M, N, K);
    B200_REQUIRE(lda >= K && (lda % 4) == 0 && ldb >= N && (ldb % 4) == 0 && ldc >= N,
                 "gemm3x_nn: row pitches must be multiples of 4 floats (lda %d ldb %d ldc %d)", lda, ldb, ldc);
    B200_REQUIRE(aligned16(A) && aligned16(B), "gemm3x_nn: operands must be 16-byte aligned");
    CUtensorMap ma, mb;
    int rc = make_map_k(&ma, A, M, K, lda, G_BM);
    if (rc != B200_OK) return rc;
    rc = make_map_mn(&mb, B, N, K, 1, ldb, 0, false);
    if (rc != B200_OK) return rc;
    GemmArgs g = {};
    g.bias = bias; g.C = C; g.M = M; g.N = N; g.ldc = ldc; g.accumulate = accumulate;
    g.KB = (K + G_BK - 1) / G_BK; g.kbt = g.KB;
    return launch<false, true>(ma, mb, g, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_gemm3x_nt(const float* A, long long lda, long long a_bstride, int a_shift, const float* B,
                                 long long ldb, long long b_bstride, int b_shift, float* C, int M, int N, int T,
                                 int batches, int ldc, int accumulate, int permute_rows, void* workspace,
                                 size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(A && B && C, "gemm3x_nt: null pointer");
    B200_REQUIRE(M > 0 && N > 0 && T > 0 && batches > 0, "gemm3x_nt: bad sizes M=%d N=%d T=%d batches=%d", M, N, T,
                 batches);
    // (a pitch smaller than the row length = overlapping rows: the in-place im2col view of a strided convolution)
    B200_REQUIRE(lda > 0 && (lda % 4) == 0 && ldb > 0 && (ldb % 4) == 0 && (a_bstride % 4) == 0 &&
                     (b_bstride % 4) == 0 && ldc >= N,
                 "gemm3x_nt: pitches must be multiples of 4 floats (lda %lld ldb %lld)", lda, ldb);
    B200_REQUIRE(aligned16(A) && aligned16(B), "gemm3x_nt: operands must be 16-byte aligned");
    B200_REQUIRE(!permute_rows || (M % 4) == 0, "gemm3x_nt: the row permutation needs M %% 4 == 0");
    B200_REQUIRE(a_shift >= -G_BK && a_shift <= G_BK && b_shift >= -G_BK && b_shift <= G_BK, "gemm3x_nt: bad shift");
    // Row r of an operand read with shift s belongs to step t = r - s only.  The last K block of a batch entry runs t
    // up to the next multiple of 32, so with s < 0 the rows from T + s on would meet the other operand at a step t >= T
    // (where it is not zero-filled when its shift is negative too): the tensor maps end at row T + min(s, 0).
    const int Ta = T + (a_shift < 0 ? a_shift : 0), Tb = T + (b_shift < 0 ? b_shift : 0);
    if (Ta <= 0 || Tb <= 0) {                                   // no step has both rows in range: an empty sum
        if (!accumulate) B200_CUDA(cudaMemset2DAsync(C, (size_t)ldc * sizeof(float), 0, (size_t)N * sizeof(float), M,
                                                      (cudaStream_t)stream));
        return B200_OK;
    }
    CUtensorMap ma, mb;
    int rc = make_map_mn(&ma, A, M, Ta, batches, lda, a_bstride, true);
    if (rc != B200_OK) return rc;
    rc = make_map_mn(&mb, B, N, Tb, batches, ldb, b_bstride, false);
    if (rc != B200_OK) return rc;
    GemmArgs g = {};
    g.C = C; g.M = M; g.N = N; g.ldc = ldc; g.accumulate = accumulate; g.perm = permute_rows;
    g.kbt = (T + G_BK - 1) / G_BK; g.KB = g.kbt * batches;
    g.a_shift = a_shift; g.b_shift = b_shift;
    return launch<true, true>(ma, mb, g, workspace, workspace_bytes, (cudaStream_t)stream);
}

// The zero-haloed layout of a 3x3 convolution's operands: grid rows R = batches (T + 2) (F + 2); a buffer holds R + F + 3
// rows, position (b, t, f) of the data at grid row (b (T + 2) + t + 1) (F + 2) + f + 1 = m + F + 3.
static int conv_geometry(const char* what, int C, int taps, int batches, int T, int F, int O, int* R) {
    B200_REQUIRE((taps == 9 && C >= 32 && (C % 32) == 0) || (taps == 1 && C == 32),
                 "%s: needs 9 taps over a multiple of 32 channels, or one tap over a 32-wide im2col (taps %d C %d)", what,
                 taps, C);
    B200_REQUIRE(batches > 0 && T > 0 && F > 0 && O > 0 && (O % 4) == 0,
                 "%s: bad sizes batches=%d T=%d F=%d O=%d (O %% 4 must be 0)", what, batches, T, F, O);
    const long long rows = (long long)batches * (T + 2) * (F + 2);
    B200_REQUIRE(rows + F + 3 < (1LL << 31) - 4 * G_BM, "%s: too many rows (%lld)", what, rows);
    *R = (int)rows;
    return B200_OK;
}

extern "C" int b200asr_conv3x3_fwd(const float* x, int C, int taps, const float* w, const float* bias, const float* mask,
                                   int relu, float* y, int batches, int T, int F, int O, b200asr_stream stream) {
    B200_REQUIRE(x && w && y, "conv3x3_fwd: null pointer");
    int R = 0;
    int rc = conv_geometry("conv3x3_fwd", C, taps, batches, T, F, O, &R);
    if (rc != B200_OK) return rc;
    B200_REQUIRE(aligned16(x) && aligned16(w) && aligned16(y) && (!mask || aligned16(mask)),
                 "conv3x3_fwd: operands must be 16-byte aligned");
    const int K = taps * C, pad = F + 3;
    CUtensorMap ma, mb;
    if ((rc = make_map_k(&ma, x, taps == 9 ? R + pad : R, C, C, G_BM)) != B200_OK) return rc;
    if ((rc = make_map_k(&mb, w, O, K, K, G_BN)) != B200_OK) return rc;
    GemmArgs g = {};
    g.bias = bias; g.C = y + (size_t)pad * O; g.M = R; g.N = O; g.ldc = O;
    g.KB = K / G_BK; g.kbt = g.KB;
    g.cv_c = C; g.cv_fp = F + 2; g.cv_t = T; g.cv_f = F; g.cv_relu = relu != 0;
    g.cv_mask = mask ? mask + (size_t)pad * O : nullptr;
    return launch<false, false, false, true>(ma, mb, g, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int b200asr_conv3x3_wgrad(const float* dy, const float* x, int C, int taps, float* dw, int batches, int T,
                                     int F, int O, void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(dy && x && dw, "conv3x3_wgrad: null pointer");
    int R = 0;
    int rc = conv_geometry("conv3x3_wgrad", C, taps, batches, T, F, O, &R);
    if (rc != B200_OK) return rc;
    B200_REQUIRE(aligned16(dy) && aligned16(x), "conv3x3_wgrad: operands must be 16-byte aligned");
    const int pad = F + 3;
    CUtensorMap ma, mb;
    if ((rc = make_map_mn(&ma, dy + (size_t)pad * O, O, R, 1, O, 0, true)) != B200_OK) return rc;
    if ((rc = make_map_mn(&mb, x, C, taps == 9 ? R + pad : R, 1, C, 0, false)) != B200_OK) return rc;
    GemmArgs g = {};
    g.C = dw; g.M = O; g.N = taps * C; g.ldc = taps * C;
    g.kbt = (R + G_BK - 1) / G_BK; g.KB = g.kbt;
    g.cv_c = C; g.cv_fp = F + 2; g.cv_t = T; g.cv_f = F;
    return launch<true, true, false, true>(ma, mb, g, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_tf32_residual(const float* x, float* lo, long long n, b200asr_stream stream) {
    B200_REQUIRE(x && lo && n >= 0, "tf32_residual: bad arguments");
    if (n == 0) return B200_OK;
    const long long per_block = 256LL * RES_UNROLL * 4;
    tf32_residual_kernel<<<(unsigned)((n + per_block - 1) / per_block), 256, 0, (cudaStream_t)stream>>>(x, lo, n);
    B200_LAUNCH_CHECK("tf32_residual_kernel");
    return B200_OK;
}

extern "C" int b200asr_f16x3_padded_k(int K) { return K > 0 ? (K + F_CK - 1) / F_CK * F_CK : 0; }

extern "C" int b200asr_f16x3_split_rows(const float* x, long long ld, int rows, int K, void* hi, void* lo, float* sinv,
                                        b200asr_stream stream) {
    B200_REQUIRE(x && hi && lo && sinv, "f16x3_split_rows: null pointer");
    B200_REQUIRE(rows > 0 && K > 0 && (K % 4) == 0 && ld >= K && (ld % 4) == 0 && aligned16(x),
                 "f16x3_split_rows: needs K %% 4 == 0, a pitch that is a multiple of 4 floats, 16-byte alignment "
                 "(rows %d K %d ld %lld)", rows, K, ld);
    const int Kp = b200asr_f16x3_padded_k(K);
    dim3 grid((rows + 7) / 8, Kp / F_CK);
    f16_split_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ld, rows, K, Kp, (__half*)hi, (__half*)lo, sinv);
    B200_LAUNCH_CHECK("f16_split_rows_kernel");
    return B200_OK;
}

extern "C" int b200asr_f16x3_split_cols(const float* x, long long ld, long long bstride, int shift, int T, int batches,
                                        int cols, void* hi, void* lo, float* sinv, b200asr_stream stream) {
    B200_REQUIRE(x && hi && lo && sinv, "f16x3_split_cols: null pointer");
    B200_REQUIRE(T > 0 && batches > 0 && cols > 0 && (cols % 4) == 0 && ld >= cols && (ld % 4) == 0 &&
                     (bstride % 4) == 0 && (batches == 1 || bstride >= (long long)T * ld) && aligned16(x),
                 "f16x3_split_cols: needs cols %% 4 == 0, pitches that are multiples of 4 floats, 16-byte alignment "
                 "(cols %d ld %lld bstride %lld)", cols, ld, bstride);
    B200_REQUIRE((long long)T * batches < (1LL << 31) - F_CK, "f16x3_split_cols: too many rows");
    const int R = T * batches, Rp = b200asr_f16x3_padded_k(R);
    dim3 grid((cols + 63) / 64, Rp / F_CK);
    f16_split_cols_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ld, bstride, shift, T, R, cols, Rp, (__half*)hi,
                                                                  (__half*)lo, sinv);
    B200_LAUNCH_CHECK("f16_split_cols_kernel");
    return B200_OK;
}

extern "C" int b200asr_f16x3_split_dg(const float* g, int ndir, int rows, int cols, void* t_hi, void* t_lo,
                                      float* t_sinv, void* r_hi, void* r_lo, float* r_sinv, float* colsum,
                                      b200asr_stream stream) {
    B200_REQUIRE(g && t_hi && t_lo && t_sinv && colsum, "f16x3_split_dg: null pointer");
    B200_REQUIRE((r_hi && r_lo && r_sinv) || (!r_hi && !r_lo && !r_sinv),
                 "f16x3_split_dg: the row images need all of hi, lo and sinv (or none of them)");
    B200_REQUIRE((ndir == 1 || ndir == 2) && rows > 0 && cols > 0 && (cols % 4) == 0 && aligned16(g),
                 "f16x3_split_dg: needs 1 or 2 directions, cols %% 4 == 0, 16-byte alignment (ndir %d rows %d cols %d)",
                 ndir, rows, cols);
    B200_REQUIRE(rows < (1 << 30) && cols < (1 << 30) / ndir, "f16x3_split_dg: too many rows or columns");
    const int Rp = b200asr_f16x3_padded_k(rows), Kp = b200asr_f16x3_padded_k(cols);
    B200_CUDA(cudaFuncSetAttribute(f16_split_dg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DG_SMEM));
    dim3 grid(Rp / F_CK, Kp / F_CK, ndir);
    f16_split_dg_kernel<<<grid, 256, DG_SMEM, (cudaStream_t)stream>>>(g, rows, cols, Kp, Rp, (__half*)t_hi,
                                                                      (__half*)t_lo, t_sinv, (__half*)r_hi,
                                                                      (__half*)r_lo, r_sinv, colsum);
    B200_LAUNCH_CHECK("f16_split_dg_kernel");
    return B200_OK;
}

extern "C" int b200asr_gemm_f16x3(const void* a_hi, const void* a_lo, const float* a_sinv, const void* b_hi,
                                  const void* b_lo, const float* b_sinv, const float* bias, float* C, int M, int N,
                                  int Kp, int ldc, int accumulate, int permute_rows, void* workspace,
                                  size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(a_hi && a_lo && a_sinv && b_hi && b_lo && b_sinv && C, "gemm_f16x3: null pointer");
    B200_REQUIRE(M > 0 && N > 0 && Kp > 0 && (Kp % F_CK) == 0 && ldc >= N,
                 "gemm_f16x3: bad sizes M=%d N=%d Kp=%d ldc=%d (Kp must be b200asr_f16x3_padded_k of K)", M, N, Kp, ldc);
    B200_REQUIRE(aligned16(a_hi) && aligned16(a_lo) && aligned16(b_hi) && aligned16(b_lo),
                 "gemm_f16x3: images must be 16-byte aligned");
    B200_REQUIRE(!permute_rows || (M % 4) == 0, "gemm_f16x3: the row permutation needs M %% 4 == 0");
    CUtensorMap mah, mal, mbh, mbl;
    int rc;
    if ((rc = make_map_f16(&mah, a_hi, M, Kp)) != B200_OK) return rc;
    if ((rc = make_map_f16(&mal, a_lo, M, Kp)) != B200_OK) return rc;
    if ((rc = make_map_f16(&mbh, b_hi, N, Kp)) != B200_OK) return rc;
    if ((rc = make_map_f16(&mbl, b_lo, N, Kp)) != B200_OK) return rc;
    F16Args g = {};
    g.bias = bias; g.sa = a_sinv; g.sb = b_sinv; g.C = C;
    g.M = M; g.N = N; g.ldc = ldc; g.accumulate = accumulate; g.perm = permute_rows;
    g.KB = Kp / F_BK;
    // same split rule (and so the same workspace bound, b200asr_gemm3x_workspace_bytes) as the 3xTF32 kernel, in k
    const SplitPlan p = plan_split(M, N, g.KB, F_CH, Kp / G_BK, workspace ? workspace_bytes : 0);
    const int nsplit = p.nsplit;
    g.kb_per_split = p.kb_per_split;
    g.partial = reinterpret_cast<float*>(workspace);
    const size_t smem = (size_t)F_STAGES * F_STAGE + 256;
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaFuncSetAttribute(gemm_f16x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((N + G_BN - 1) / G_BN, (M + G_BM - 1) / G_BM, nsplit);
    gemm_f16x3_kernel<<<grid, G_THREADS, smem, st>>>(mah, mal, mbh, mbl, g);
    B200_LAUNCH_CHECK("gemm_f16x3_kernel");
    if (nsplit > 1) {
        const long long total = (long long)M * N;
        int blocks = (int)((total + 255) / 256);
        if (blocks > 16 * sm_count()) blocks = 16 * sm_count();
        gemm3x_reduce_kernel<<<blocks, 256, 0, st>>>(g.partial, nsplit, bias, C, M, N, ldc, accumulate, permute_rows);
        B200_LAUNCH_CHECK("gemm3x_reduce_kernel");
    }
    return B200_OK;
}

extern "C" int b200asr_debug_gemm_plan(int form, int M, int N, int K, int batches, size_t workspace_bytes, int* desc) {
    B200_REQUIRE(desc != nullptr && form >= 0 && form <= 4 && M > 0 && N > 0 && K > 0 && batches > 0 &&
                     (form == 3 || batches == 1),
                 "debug_gemm_plan: bad arguments (form %d M %d N %d K %d batches %d)", form, M, N, K, batches);
    SplitPlan p;
    int KB, ch, bk;
    if (form == 4) {                                            // f16x3: 64-k blocks, one scale chunk per accumulation
        bk = F_BK;
        ch = F_CH;
        KB = b200asr_f16x3_padded_k(K) / F_BK;
        p = plan_split(M, N, KB, F_CH, KB * F_BK / G_BK, workspace_bytes);
    } else {                                                    // 3xTF32: 32-k blocks; nt walks (batch, time)
        bk = G_BK;
        ch = gemm_chunk();
        KB = (K + G_BK - 1) / G_BK * (form == 3 ? batches : 1);
        p = plan_split(M, N, KB, 1, KB, workspace_bytes);
    }
    const int first = KB < p.kb_per_split ? KB : p.kb_per_split, last = KB - (p.nsplit - 1) * p.kb_per_split;
    const int d[10] = {p.rule, p.requested, p.nsplit, p.kb_per_split, last, ch, (first - 1) % ch + 1,
                       (last - 1) % ch + 1, KB, bk};
    for (int i = 0; i < 10; ++i) desc[i] = d[i];
    return B200_OK;
}
