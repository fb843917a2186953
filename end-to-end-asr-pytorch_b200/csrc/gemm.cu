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
// wgmma .tf32 reads fp32 bit patterns from shared memory and ignores the low 13 mantissa bits (inferred from the fp32-
// class parity tests of the tn form, which only hold if the hardware truncates; not probed in isolation), so a raw
// K-major fp32 tile IS the TF32 "hi" operand; the residual  lo = x - trunc(x)  is a second tile of the same layout.  Per 32-wide K
// block the two consumer warpgroups accumulate  A.B + A_lo.B + A.B_lo  in one fp32 register accumulator.
// wgmma has no MN-major form for 32-bit types: an MN-major operand is loaded as plain [32 k][32 column] boxes and
// transposed into the K-major swizzled image (hi and lo at once) by the same pass that makes the residuals.
//
// One 128 x 128 tile per CTA (x split-K slices when the tile grid alone cannot fill the SMs: partial tiles go to a
// workspace and a second small kernel sums them in a fixed order - deterministic).  Warp roles: 0 = TMA producer
// (cp.async.bulk.tensor, out-of-bounds rows / K tail zero-filled by the hardware), 4..11 = two consumer warpgroups
// (64 rows each): they split K block i+1 while their asynchronous MMAs of K block i run.  The accumulation chain is cut
// every G_CH K blocks and summed with IEEE fp32 adds in a second register tile (the tensor core's fp32 accumulate
// is not IEEE-rounded); the epilogue (+ bias [+ C]) runs from those registers.
//
// Shared-memory images.  K-major operand, R rows: R consecutive 128-byte rows (32 k each), 128-byte swizzle; one MMA
// (8 k) advances the descriptor start by 32 bytes.  MN-major operand as loaded: R/32 boxes of [32 k][32 columns] =
// 4096 bytes each (a TMA box {32 columns, 32 rows}, no swizzle).
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
constexpr int G_THREADS = 128 + G_CONSUMERS;    // warpgroup 0: TMA producer (one lane)
constexpr int G_BOX = 32 * G_BK * 4;            // one MN-major box: 32 columns x 32 k
constexpr int G_MAX_SPLIT = 32;
constexpr int G_CH_DEFAULT = 4;                 // K blocks per accumulation chunk; 1, 2 or 4

// stage: [A as loaded | B as loaded | A lo | B lo | A hi (K-major image, MN-major A only) | B hi (same for B)]
template <bool A_MN, bool B_MN>
struct GemmSmem {
    static constexpr int STAGE = (4 + (A_MN ? 1 : 0) + (B_MN ? 1 : 0)) * G_TILE;
    static constexpr int STAGES = (A_MN || B_MN) ? 2 : 3;
    static constexpr int A_HI = A_MN ? 4 * G_TILE : 0;
    static constexpr int B_HI = B_MN ? (A_MN ? 5 : 4) * G_TILE : G_TILE;
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
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(G_CONSUMERS) : "memory"); }
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ float tf32_residual(float x) { return x - tf32_trunc(x); }

// Residual of a K-major tile (elementwise: the image keeps its layout).
__device__ __forceinline__ void split_k_tile(const uint8_t* raw, uint8_t* lo, int ct) {
    const float4* src = reinterpret_cast<const float4*>(raw);
    float4* dst = reinterpret_cast<float4*>(lo);
#pragma unroll 4
    for (int j = ct; j < G_TILE / 16; j += G_CONSUMERS) {
        const float4 v = src[j];
        dst[j] = make_float4(tf32_residual(v.x), tf32_residual(v.y), tf32_residual(v.z), tf32_residual(v.w));
    }
}
// [32 k][32 column] boxes -> K-major swizzled hi and lo images: warp w moves k = 4w .. 4w+3 of column `lane`.
__device__ __forceinline__ void split_mn_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int boxes, int ct) {
    const int c = ct & 31, k0 = (ct >> 5) * 4;
    for (int j = 0; j < boxes; ++j) {
        const float* b = reinterpret_cast<const float*>(raw + j * G_BOX) + k0 * 32 + c;
        const float x0 = b[0], x1 = b[32], x2 = b[64], x3 = b[96];
        const uint32_t off = wgmma::sw128_offset(32 * j + c, k0 * 4);
        *reinterpret_cast<float4*>(hi + off) = make_float4(tf32_trunc(x0), tf32_trunc(x1), tf32_trunc(x2), tf32_trunc(x3));
        *reinterpret_cast<float4*>(lo + off) =
            make_float4(tf32_residual(x0), tf32_residual(x1), tf32_residual(x2), tf32_residual(x3));
    }
}

// B_PRE / A_PRE: the residual of a K-major operand comes from a pre-computed residual matrix (same shape / layout: the
// weights, split once per step by b200asr_tf32_residual) through its own tensor map, so the consumers do not pass
// over that tile.  K-major operands only: an MN-major operand goes through the transposing pass, which makes its
// residual in the same sweep.
template <bool A_MN, bool B_MN, bool B_PRE, bool A_PRE>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm3x_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
              const __grid_constant__ CUtensorMap map_blo, const __grid_constant__ CUtensorMap map_alo, const GemmArgs g) {
    using L = GemmSmem<A_MN, B_MN>;
    static_assert(!(A_PRE && A_MN) && !(B_PRE && B_MN), "only K-major operands bring a pre-computed residual");
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::STAGES * L::STAGE);      // TMA landed
    uint64_t* empty = full + L::STAGES;                                              // MMAs of the stage retired

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * G_BM, n0 = blockIdx.x * G_BN;
    const int M = g.M, N = g.N;
    const int kb0 = blockIdx.z * g.kb_per_split;
    const int kb1 = min(g.KB, kb0 + g.kb_per_split);
    const int nkb = kb1 - kb0;                                   // >= 1 by construction of the grid
    const int a_boxes = min(G_BM / 32, (M - m0 + 31) / 32);      // MN-major: 32-column boxes that hold real data
    const int b_boxes = min(G_BN / 32, (N - n0 + 31) / 32);
    const uint32_t a_bytes = A_MN ? (uint32_t)a_boxes * G_BOX : (uint32_t)G_TILE;
    const uint32_t b_bytes = B_MN ? (uint32_t)b_boxes * G_BOX : (uint32_t)G_TILE;

    if (tid == 0) {
        for (int s = 0; s < L::STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], G_CONSUMERS / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {
            for (int i = 0; i < nkb; ++i) {
                const int kb = kb0 + i;
                const int s = i % L::STAGES;
                if (i >= L::STAGES) mbar_wait(&empty[s], (uint32_t)(((i / L::STAGES) - 1) & 1));
                uint8_t* st = smem + s * L::STAGE;
                mbar_expect_tx(&full[s], (A_PRE ? 2 * a_bytes : a_bytes) + (B_PRE ? 2 * b_bytes : b_bytes));
                const int bt = kb / g.kbt, t0 = (kb - bt * g.kbt) * G_BK;
                if (A_MN) {
                    for (int j = 0; j < a_boxes; ++j)
                        tma_load_3d(st + j * G_BOX, &map_a, m0 + 32 * j, t0 + g.a_shift, bt, &full[s]);
                } else {
                    tma_load_2d(st, &map_a, kb * G_BK, m0, &full[s]);
                    if (A_PRE) tma_load_2d(st + 2 * G_TILE, &map_alo, kb * G_BK, m0, &full[s]);
                }
                if (B_MN) {
                    for (int j = 0; j < b_boxes; ++j)
                        tma_load_3d(st + G_TILE + j * G_BOX, &map_b, n0 + 32 * j, t0 + g.b_shift, bt, &full[s]);
                } else {
                    tma_load_2d(st + G_TILE, &map_b, kb * G_BK, n0, &full[s]);
                    if (B_PRE) tma_load_2d(st + 3 * G_TILE, &map_blo, kb * G_BK, n0, &full[s]);
                }
            }
        }
    } else if (warp >= 4) {
        const int ct = tid - 128, wg = ct >> 7;
        auto split = [&](int i) {
            const int s = i % L::STAGES;
            mbar_wait(&full[s], (uint32_t)((i / L::STAGES) & 1));
            uint8_t* st = smem + s * L::STAGE;
            if (A_MN) split_mn_tile(st, st + L::A_HI, st + 2 * G_TILE, a_boxes, ct);
            else if (!A_PRE) split_k_tile(st, st + 2 * G_TILE, ct);
            if (B_MN) split_mn_tile(st + G_TILE, st + L::B_HI, st + 3 * G_TILE, b_boxes, ct);
            else if (!B_PRE) split_k_tile(st + G_TILE, st + 3 * G_TILE, ct);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> the tensor core
        };
        float acc[64], d[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[e] = 0.f;
        split(0);
        consumer_sync();
        for (int i = 0; i < nkb; ++i) {
            const int s = i % L::STAGES, j = i % g.ch;
            const uint32_t st = smem_u32(smem + s * L::STAGE);
            const uint32_t a = st + L::A_HI + wg * (64 * 128), alo = st + 2 * G_TILE + wg * (64 * 128);
            const uint32_t b = st + L::B_HI, blo = st + 3 * G_TILE;
            wgmma::fence_operand(d);
            wgmma::fence();
#pragma unroll
            for (int k4 = 0; k4 < G_BK / 8; ++k4) {
                const uint64_t da = wgmma::desc_k_sw128(a + k4 * 32), db = wgmma::desc_k_sw128(b + k4 * 32);
                wgmma::mma_tf32_n128(d, da, db, (j | k4) != 0);
                wgmma::mma_tf32_n128(d, wgmma::desc_k_sw128(alo + k4 * 32), db, 1);
                wgmma::mma_tf32_n128(d, da, wgmma::desc_k_sw128(blo + k4 * 32), 1);
            }
            wgmma::commit_group();
            if (i + 1 < nkb) split(i + 1);                 // overlaps the MMAs of K block i
            wgmma::wait_all();
            wgmma::fence_operand(d);
            if (lane == 0) g_arrive(&empty[s]);
            if (j == g.ch - 1 || i == nkb - 1) {
#pragma unroll
                for (int e = 0; e < 64; ++e) acc[e] += d[e];
            }
            consumer_sync();                               // every thread's split of K block i+1 is in place
        }
        // ---------------------------------------------------------------- epilogue: registers -> C
        const bool to_partial = gridDim.z > 1;
        float* Cb = to_partial ? g.partial + (size_t)blockIdx.z * M * N : g.C;
        const int ldc = to_partial ? N : g.ldc;
        const float* bias = to_partial ? nullptr : g.bias;
        const int accumulate = to_partial ? 0 : g.accumulate;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
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
// with boxes of 32 columns x 32 rows x 1, no swizzle; reads outside [0,cols) x [0,T) are zero-filled
int make_map_mn(CUtensorMap* map, const float* ptr, int cols, int T, int batches, long long ld, long long bstride) {
    EncodeTiledFn enc = encode_fn();
    B200_REQUIRE(enc != nullptr, "gemm: cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)T, (cuuint64_t)batches};
    const cuuint64_t strides[2] = {(cuuint64_t)ld * sizeof(float), (cuuint64_t)(batches > 1 ? bstride : ld * (long long)T) * sizeof(float)};
    const cuuint32_t box[3] = {32, (cuuint32_t)G_BK, 1};     // plain rows: the consumers transpose out of this image
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
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

template <bool A_MN, bool B_MN, bool B_PRE = false, bool A_PRE = false>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, GemmArgs g, void* ws, size_t ws_bytes, cudaStream_t stream,
           const CUtensorMap* mblo = nullptr, const CUtensorMap* malo = nullptr) {
    int nsplit = pick_split(g.M, g.N, g.KB);
    if (nsplit > 1 && (ws == nullptr || ws_bytes < (size_t)nsplit * g.M * g.N * sizeof(float))) nsplit = 1;
    g.kb_per_split = (g.KB + nsplit - 1) / nsplit;
    nsplit = (g.KB + g.kb_per_split - 1) / g.kb_per_split;       // no empty slices
    g.partial = reinterpret_cast<float*>(ws);
    g.ch = gemm_chunk();
    const size_t smem = (size_t)GemmSmem<A_MN, B_MN>::STAGES * GemmSmem<A_MN, B_MN>::STAGE + 256;
    auto fn = gemm3x_kernel<A_MN, B_MN, B_PRE, A_PRE>;
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((g.N + G_BN - 1) / G_BN, (g.M + G_BM - 1) / G_BM, nsplit);
    fn<<<grid, G_THREADS, smem, stream>>>(ma, mb, mblo ? *mblo : mb, malo ? *malo : ma, g);
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
        if (A_lo) {
            B200_REQUIRE(aligned16(A_lo), "gemm3x_tn: operands must be 16-byte aligned");
            CUtensorMap malo;
            rc = make_map_k(&malo, A_lo, M, K, lda, G_BM);
            if (rc != B200_OK) return rc;
            return launch<false, false, true, true>(ma, mb, g, ws, ws_bytes, (cudaStream_t)stream, &mlo, &malo);
        }
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
    rc = make_map_mn(&mb, B, N, K, 1, ldb, 0);
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
    int rc = make_map_mn(&ma, A, M, T, batches, lda, a_bstride);
    if (rc != B200_OK) return rc;
    rc = make_map_mn(&mb, B, N, T, batches, ldb, b_bstride);
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

