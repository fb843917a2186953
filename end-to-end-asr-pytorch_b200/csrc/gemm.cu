// K6 / K9 / K11: the dense contractions of the step on the Hopper tensor cores (wgmma), fp32 in and out, fp32-class
// accuracy ("3xTF32").  ONE kernel template serves the three operand arrangements of a layer y = x . W^T + b:
//   tn :  C[M,N] (+)= A[M,K] . B[N,K]^T + bias      forward  (x . W^T): both operands K-major (K contiguous)
//   nn :  C[M,N] (+)= A[M,K] . B[K,N]               input gradient (dY . W): B is MN-major (N contiguous)
//   nt :  C[M,N] (+)= sum_r A[r,M]^T . B[r,N]       weight gradient (dY^T . X): the contraction runs over the B*T rows,
//                                                    both operands MN-major; rows are addressed as (batch, time) so
//                                                    that B can be read SHIFTED by one time step (dW_hh = dG^T . h_prev
//                                                    without materialising h_prev: the row before the first / after the
//                                                    last step of an utterance is out of bounds = zero-filled by TMA)
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
#include <stdlib.h>
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/b200asr.h"

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

// B_PRE: the residual of a K-major B comes from a pre-computed residual matrix (same shape / layout: the weights, split
// once per step by b200asr_tf32_residual) through its own tensor map.  An MN-major B goes through the transposing
// pass, which makes its residual in the same sweep.
template <bool A_MN, bool B_MN, bool B_PRE>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm3x_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
              const __grid_constant__ CUtensorMap map_blo, const GemmArgs g) {
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
                    if (A_MN) {
                        for (int j = 0; j < a_boxes; ++j)
                            tma_load_3d(st + j * G_BOX, &map_a, m0 + 32 * j, t0 + g.a_shift, bt, &full[s]);
                    } else {
                        tma_load_2d(st, &map_a, kb * G_BK, m0, &full[s]);
                    }
                    if (B_MN) {
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
        // ---------------------------------------------------------------- epilogue: registers -> C
        const bool to_partial = gridDim.z > 1;
        float* Cb = to_partial ? g.partial + (size_t)blockIdx.z * M * N : g.C;
        const int ldc = to_partial ? N : g.ldc;
        const float* bias = to_partial ? nullptr : g.bias;
        const int accumulate = to_partial ? 0 : g.accumulate;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + (A_MN ? mn_row(r0 + 8 * h) : r0 + 8 * h);
            if (row >= M) continue;
            const int orow = (!to_partial && g.perm) ? (row & 3) * (M >> 2) + (row >> 2) : row;
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

int pick_split(int M, int N, int KB) {
    const int tiles = ((M + G_BM - 1) / G_BM) * ((N + G_BN - 1) / G_BN);
    const int sms = sm_count();
    int s = sms / tiles;
    if (s > KB / 8) s = KB / 8;           // at least 8 K blocks per slice
    if (s > G_MAX_SPLIT) s = G_MAX_SPLIT;
    if (s < 1) s = 1;
    auto eff = [&](int q) {
        const long long ctas = (long long)tiles * q;
        return (double)ctas / (double)(((ctas + sms - 1) / sms) * sms);
    };
    if (2 * tiles <= sms && eff(s) < 0.93) {
        const int cap = max_split(M, N);
        for (int q = s + 1; q <= cap && KB / q >= 64; ++q)
            if (eff(q) >= 0.97) return q;
    }
    return s;
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

template <bool A_MN, bool B_MN, bool B_PRE = false>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, GemmArgs g, void* ws, size_t ws_bytes, cudaStream_t stream,
           const CUtensorMap* mblo = nullptr) {
    int nsplit = pick_split(g.M, g.N, g.KB);
    if (nsplit > 1 && (ws == nullptr || ws_bytes < (size_t)nsplit * g.M * g.N * sizeof(float))) nsplit = 1;
    g.kb_per_split = (g.KB + nsplit - 1) / nsplit;
    nsplit = (g.KB + g.kb_per_split - 1) / g.kb_per_split;       // no empty slices
    g.partial = reinterpret_cast<float*>(ws);
    g.ch = gemm_chunk();
    const size_t smem = (size_t)GemmSmem<B_MN>::STAGES * GemmSmem<B_MN>::STAGE + 256;
    auto fn = gemm3x_kernel<A_MN, B_MN, B_PRE>;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((g.N + G_BN - 1) / G_BN, (g.M + G_BM - 1) / G_BM, nsplit);
    fn<<<grid, G_THREADS, smem, stream>>>(ma, mb, mblo ? *mblo : mb, g);
    B200_LAUNCH_CHECK("gemm3x_kernel");
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

}  // namespace
}  // namespace b200asr

using namespace b200asr;

extern "C" int b200asr_gemm3x_supported(int M, int N, int K) {
    // TMA: 16-byte aligned row pitch; at least one full tile's worth of work is not required (tails are zero-filled)
    return (M > 0 && N > 0 && K > 0 && (K % 4) == 0) ? 1 : 0;
}

extern "C" size_t b200asr_gemm3x_workspace_bytes(int M, int N) {
    if (M <= 0 || N <= 0) return 0;
    int s = max_split(M, N);                   // upper bound of what pick_split() may choose for any K
    const int tiles = ((M + G_BM - 1) / G_BM) * ((N + G_BN - 1) / G_BN);
    if (2 * tiles > sm_count()) s = 1;
    return s > 1 ? (size_t)s * M * N * sizeof(float) : 0;
}

extern "C" int b200asr_gemm3x_tn(const float* A, const float* B, const float* bias, float* C, int M, int N, int K,
                                 int ldc, int accumulate, b200asr_stream stream) {
    return b200asr_gemm3x_tn_ld(A, K, B, bias, C, M, N, K, ldc, accumulate, stream);
}

static int gemm3x_tn_impl(const float* A, int lda, const float* B, const float* bias, float* C, int M, int N, int K,
                          int ldc, int accumulate, void* ws, size_t ws_bytes, b200asr_stream stream,
                          const float* B_lo = nullptr, const float* A_lo = nullptr) {
    B200_REQUIRE(A && B && C, "gemm3x_tn: null pointer");
    B200_REQUIRE(!A_lo || B_lo, "gemm3x_tn: a residual of A needs the residual of B as well");
    B200_REQUIRE(lda > 0 && (lda % 4) == 0, "gemm3x_tn: lda %d must be a positive multiple of 4", lda);
    B200_REQUIRE(b200asr_gemm3x_supported(M, N, K), "gemm3x_tn: unsupported sizes M=%d N=%d K=%d (K %% 4 must be 0)", M,
                 N, K);
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
        // A's residual is made in registers from the A fragment (A_lo holds the same values and is not read)
        B200_REQUIRE(!A_lo || aligned16(A_lo), "gemm3x_tn: operands must be 16-byte aligned");
        return launch<false, false, true>(ma, mb, g, ws, ws_bytes, (cudaStream_t)stream, &mlo);
    }
    return launch<false, false>(ma, mb, g, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_gemm3x_tn_ld(const float* A, int lda, const float* B, const float* bias, float* C, int M, int N,
                                    int K, int ldc, int accumulate, b200asr_stream stream) {
    return gemm3x_tn_impl(A, lda, B, bias, C, M, N, K, ldc, accumulate, nullptr, 0, stream);
}

extern "C" int b200asr_gemm3x_tn_ws(const float* A, int lda, const float* B, const float* bias, float* C, int M, int N,
                                    int K, int ldc, int accumulate, void* workspace, size_t workspace_bytes,
                                    b200asr_stream stream) {
    return gemm3x_tn_impl(A, lda, B, bias, C, M, N, K, ldc, accumulate, workspace, workspace_bytes, stream);
}

static int gemm3x_nn_impl(const float* A, int lda, const float* B, int ldb, const float* bias, float* C, int M, int N,
                          int K, int ldc, int accumulate, void* ws, size_t ws_bytes, b200asr_stream stream) {
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
    return launch<false, true>(ma, mb, g, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_gemm3x_nn(const float* A, int lda, const float* B, int ldb, const float* bias, float* C, int M,
                                 int N, int K, int ldc, int accumulate, b200asr_stream stream) {
    return gemm3x_nn_impl(A, lda, B, ldb, bias, C, M, N, K, ldc, accumulate, nullptr, 0, stream);
}

extern "C" int b200asr_gemm3x_nn_ws(const float* A, int lda, const float* B, int ldb, const float* bias, float* C, int M,
                                    int N, int K, int ldc, int accumulate, void* workspace, size_t workspace_bytes,
                                    b200asr_stream stream) {
    return gemm3x_nn_impl(A, lda, B, ldb, bias, C, M, N, K, ldc, accumulate, workspace, workspace_bytes, stream);
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
    CUtensorMap ma, mb;
    int rc = make_map_mn(&ma, A, M, T, batches, lda, a_bstride, true);
    if (rc != B200_OK) return rc;
    rc = make_map_mn(&mb, B, N, T, batches, ldb, b_bstride, false);
    if (rc != B200_OK) return rc;
    GemmArgs g = {};
    g.C = C; g.M = M; g.N = N; g.ldc = ldc; g.accumulate = accumulate; g.perm = permute_rows;
    g.kbt = (T + G_BK - 1) / G_BK; g.KB = g.kbt * batches;
    g.a_shift = a_shift; g.b_shift = b_shift;
    return launch<true, true>(ma, mb, g, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200asr_tf32_residual(const float* x, float* lo, long long n, b200asr_stream stream) {
    B200_REQUIRE(x && lo && n >= 0, "tf32_residual: bad arguments");
    if (n == 0) return B200_OK;
    const long long per_block = 256LL * RES_UNROLL * 4;
    tf32_residual_kernel<<<(unsigned)((n + per_block - 1) / per_block), 256, 0, (cudaStream_t)stream>>>(x, lo, n);
    B200_LAUNCH_CHECK("tf32_residual_kernel");
    return B200_OK;
}

extern "C" int b200asr_gemm3x_tn_pre(const float* A, int lda, const float* B, const float* B_lo, const float* bias,
                                     float* C, int M, int N, int K, int ldc, int accumulate, void* workspace,
                                     size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(B_lo, "gemm3x_tn_pre: null residual");
    return gemm3x_tn_impl(A, lda, B, bias, C, M, N, K, ldc, accumulate, workspace, workspace_bytes, stream, B_lo);
}

extern "C" int b200asr_gemm3x_tn_pre2(const float* A, const float* A_lo, int lda, const float* B, const float* B_lo,
                                      const float* bias, float* C, int M, int N, int K, int ldc, int accumulate,
                                      void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(A_lo && B_lo, "gemm3x_tn_pre2: null residual");
    return gemm3x_tn_impl(A, lda, B, bias, C, M, N, K, ldc, accumulate, workspace, workspace_bytes, stream, B_lo, A_lo);
}

