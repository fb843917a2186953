// Embedding backward (the row-gather gradient of nn.Embedding, src/lm.py:17,32 in the reference):
//   dW[ids[n], :] += dY[n, :]   for n in [0, N), added IN PLACE into an existing [V, E] gradient.
//
// Deterministic without float atomics: a one-CTA counting sort of (token, position) by token, stable in the
// position, followed by one pass that sums each present token's rows in ascending position and adds that sum once
// onto dW.  Every float result depends only on (ids, dY, dW), never on the launch configuration.
//
//   embed_sort_kernel (1 CTA):  histogram of the valid ids (integer atomics)  ->  exclusive scan  ->  the list of
//       present tokens (ascending) with their segment offsets  ->  stable placement of the positions by warp 0, 32
//       positions per round (__match_any_sync groups equal ids; the group leader bumps the token's cursor).  The
//       per-token counters live in shared memory when V fits, else in the workspace.
//   embed_acc_kernel: grid-stride over the present tokens (x) and over column blocks (y); each thread owns one column
//       and walks the token's segment in order.
#include "../../include/b200asr.h"
#include "common.cuh"

namespace {

constexpr int SORT_THREADS = 1024;
constexpr int ACC_THREADS = 256;
constexpr int SMEM_COUNTER_LIMIT = 160 * 1024;      // bytes of per-token counters kept in shared memory

__global__ void __launch_bounds__(SORT_THREADS, 1)
embed_sort_kernel(const long long* __restrict__ ids, int N, int V, int* gcount, int use_smem, int* __restrict__ pos,
                  int* __restrict__ tok, int* __restrict__ off, int* __restrict__ n_present) {
    extern __shared__ int dyn[];
    __shared__ int warp_tot[32][2];
    int* cnt = use_smem ? dyn : gcount;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;

    for (int v = tid; v < V; v += blockDim.x) cnt[v] = 0;
    __syncthreads();
    for (int n = tid; n < N; n += blockDim.x) {
        const long long id = ids[n];
        if (id >= 0 && id < V) atomicAdd(&cnt[(int)id], 1);
    }
    __syncthreads();

    // exclusive scan of (count, present) over contiguous per-thread ranges
    const int per = (V + blockDim.x - 1) / blockDim.x;
    const int lo = min(V, tid * per), hi = min(V, lo + per);
    int s = 0, f = 0;
    for (int v = lo; v < hi; ++v) {
        const int c = cnt[v];
        s += c;
        f += c > 0;
    }
    int is = s, iff = f;                                    // warp inclusive scan
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int ts = __shfl_up_sync(0xffffffffu, is, o), tf = __shfl_up_sync(0xffffffffu, iff, o);
        if (lane >= o) { is += ts; iff += tf; }
    }
    if (lane == 31) { warp_tot[warp][0] = is; warp_tot[warp][1] = iff; }
    __syncthreads();
    int bs = 0, bf = 0, ts = 0, tf = 0;
    for (int w = 0; w < nw; ++w) {
        if (w < warp) { bs += warp_tot[w][0]; bf += warp_tot[w][1]; }
        ts += warp_tot[w][0];
        tf += warp_tot[w][1];
    }
    int sb = bs + is - s, fb = bf + iff - f;                // exclusive prefixes of this thread's range
    for (int v = lo; v < hi; ++v) {
        const int c = cnt[v];
        if (c > 0) {
            tok[fb] = v;
            off[fb] = sb;
            ++fb;
        }
        cnt[v] = sb;                                        // becomes the token's placement cursor
        sb += c;
    }
    if (tid == 0) {
        off[tf] = ts;
        *n_present = tf;
    }
    __syncthreads();

    // stable placement: rounds of 32 consecutive positions, in order
    if (warp == 0) {
        for (int base = 0; base < N; base += 32) {
            const int n = base + lane;
            const long long id = n < N ? ids[n] : -1;
            const bool valid = id >= 0 && id < V;
            const int v = valid ? (int)id : -1;
            const unsigned mask = __match_any_sync(0xffffffffu, v);
            const int leader = __ffs(mask) - 1;
            const int rank = __popc(mask & ((1u << lane) - 1u));
            int b = 0;
            if (valid && lane == leader) {
                b = cnt[v];
                cnt[v] = b + __popc(mask);
            }
            b = __shfl_sync(0xffffffffu, b, leader);
            if (valid) pos[b + rank] = n;
            __syncwarp();
        }
    }
}

__global__ void
embed_acc_kernel(const float* __restrict__ dY, int E, const int* __restrict__ pos, const int* __restrict__ tok,
                 const int* __restrict__ off, const int* __restrict__ n_present, float* __restrict__ dW) {
    const int K = *n_present;
    for (int k = blockIdx.x; k < K; k += gridDim.x) {
        const int a = off[k], b = off[k + 1];
        float* wrow = dW + (long long)tok[k] * E;
        for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < E; j += gridDim.y * blockDim.x) {
            float acc = 0.f;
            int i = a;
            for (; i + 4 <= b; i += 4) {        // loads issued together, added strictly in position order
                const int p0 = pos[i], p1 = pos[i + 1], p2 = pos[i + 2], p3 = pos[i + 3];
                const float y0 = __ldg(dY + (long long)p0 * E + j), y1 = __ldg(dY + (long long)p1 * E + j);
                const float y2 = __ldg(dY + (long long)p2 * E + j), y3 = __ldg(dY + (long long)p3 * E + j);
                acc += y0;
                acc += y1;
                acc += y2;
                acc += y3;
            }
            for (; i < b; ++i) acc += __ldg(dY + (long long)pos[i] * E + j);
            wrow[j] += acc;
        }
    }
}

size_t align16(size_t x) { return (x + 15) & ~size_t(15); }

}  // namespace

extern "C" size_t b200asr_embedding_bwd_workspace_bytes(int N, int V) {
    if (N < 0 || V <= 0) return 0;
    // counters [V] (used when they do not fit in shared memory), positions [N], tokens [N], offsets [N + 1], count
    return align16(4 * (size_t)V) + align16(4 * (size_t)N) * 2 + align16(4 * ((size_t)N + 2));
}

extern "C" int b200asr_embedding_bwd(const long long* ids, const float* dY, int N, int V, int E, float* dW,
                                     void* workspace, size_t workspace_bytes, b200asr_stream stream) {
    B200_REQUIRE(N >= 0 && V > 0 && E > 0, "embedding_bwd: bad sizes N=%d V=%d E=%d", N, V, E);
    if (N == 0) return B200_OK;
    B200_REQUIRE(ids && dY && dW && workspace, "embedding_bwd: null pointer");
    B200_REQUIRE(workspace_bytes >= b200asr_embedding_bwd_workspace_bytes(N, V),
                 "embedding_bwd: workspace of %zu bytes < %zu", workspace_bytes,
                 b200asr_embedding_bwd_workspace_bytes(N, V));
    char* ws = (char*)workspace;
    int* gcount = (int*)ws;
    ws += align16(4 * (size_t)V);
    int* pos = (int*)ws;
    ws += align16(4 * (size_t)N);
    int* tok = (int*)ws;
    ws += align16(4 * (size_t)N);
    int* off = (int*)ws;
    int* n_present = off + N + 1;
    const cudaStream_t s = (cudaStream_t)stream;

    const size_t cbytes = 4 * (size_t)V;
    const int use_smem = cbytes <= (size_t)SMEM_COUNTER_LIMIT && cbytes <= (size_t)b200asr::max_optin_smem();
    const size_t smem = use_smem ? cbytes : 0;
    if (smem > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(embed_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    embed_sort_kernel<<<1, SORT_THREADS, smem, s>>>(ids, N, V, gcount, use_smem, pos, tok, off, n_present);
    B200_LAUNCH_CHECK("embed_sort_kernel");

    // at most min(N, V) tokens are present; surplus CTAs exit at once
    const int gx = min(min(N, V), 8 * b200asr::sm_count());
    const int gy = (E + ACC_THREADS - 1) / ACC_THREADS;
    embed_acc_kernel<<<dim3(gx, min(gy, 65535)), ACC_THREADS, 0, s>>>(dY, E, pos, tok, off, n_present, dW);
    B200_LAUNCH_CHECK("embed_acc_kernel");
    return B200_OK;
}
