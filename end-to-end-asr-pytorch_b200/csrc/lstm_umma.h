// Internal interface of the wgmma BiLSTM step kernels (csrc/lstm_umma.cu), used by the C-ABI entry points in lstm.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace b200asr {

bool lstm_umma_fwd_supported(int B, int H, int ndir);
bool lstm_umma_bwd_supported(int B, int H, int ndir, int flags);
int lstm_umma_bwd(float* gates, const float* w_hh, const float* cstate, const float* dout, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, long long* trace, int flags, cudaStream_t stream);
size_t lstm_umma_workspace_bytes(int B, int H, int ndir);
int lstm_umma_plan(int B, int H, int ndir, int* unit_block, int* batch_block, int* n_ctas);
int lstm_umma_fwd(float* gates, const float* w_hh, float* cstate, float* out, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, long long* trace, int flags, cudaStream_t stream);

}  // namespace b200asr
