// wgmma helpers for the sm_90a kernels: shared-memory matrix descriptors, warpgroup MMA issue (both operands in
// shared memory, fp32 accumulators in registers), commit / wait of the asynchronous groups.
//
// Layout conventions used by every kernel in this library:
//  * operands are K-major with the 128-byte swizzle: a tile of R rows x 128 bytes of K (32 tf32 / 64 f16 elements) is
//    stored as R consecutive 128-byte rows, and inside each 1024-byte group of 8 rows the 16-byte chunk c of row r
//    sits at chunk position c ^ (r & 7).  Tiles that are longer in K are a sequence of such "K atoms", each a
//    separate R x 128 B block.  This is also what a TMA load with CU_TENSOR_MAP_SWIZZLE_128B produces.
//  * one wgmma consumes 32 bytes of K (8 tf32 / 16 f16): inside an atom the descriptor start address advances by 32
//    bytes per MMA.  tf32 operands exist K-major only (wgmma transposes 16-bit types alone).
//  * one warpgroup (4 warps) computes M = 64 rows; the fp32 accumulator fragment of warp w, lane l is
//    d[4g + 0,1] = (row 16w + l/4, columns 8g + 2(l%4) + {0,1}),  d[4g + 2,3] = the same columns of row 16w + l/4 + 8.
#pragma once
#include "common.cuh"

namespace b200asr {
namespace wgmma {

// K-major, SWIZZLE_128B matrix descriptor: start address >> 4 in [0,14), leading byte offset (unused: one swizzle
// atom along K) in [16,30), stride byte offset = 1024 (distance between 8-row groups) in [32,46), layout type
// SWIZZLE_128B = 1 in [62,64).
__device__ __forceinline__ uint64_t desc_k_sw128(uint32_t smem_addr) {
    uint64_t d = static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// Byte offset of element (row, byte-in-row) inside one K atom (R rows x 128 B) with the 128-byte swizzle.
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t byte_in_row) {
    return row * 128u + ((((byte_in_row >> 4) ^ (row & 7u)) << 4) | (byte_in_row & 15u));
}

// Orders earlier register / shared-memory accesses of the warpgroup before the MMAs that follow.
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit_group() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// All groups committed by this warp have completed: their accumulators may be read, their operands overwritten.
__device__ __forceinline__ void wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// The compiler may not move reads of an accumulator above the wait that completes its MMAs (nor writes below the issue).
template <int N>
__device__ __forceinline__ void fence_operand(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- MMA issue (all 128 threads of a warpgroup); accumulate = 0 overwrites d ------------------------------------
__device__ __forceinline__ void mma_tf32_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void mma_f16_n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void mma_f16_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

}  // namespace wgmma
}  // namespace b200asr
