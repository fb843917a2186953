// Internal interface of the wgmma BiLSTM step kernels (csrc/lstm_umma.cu), used by the C-ABI entry points in lstm.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace b200asr {

// The instance lstm_umma_fwd / lstm_umma_bwd launch for these sizes: unit block, template unit block and number of
// launches.  false: no plan.
bool lstm_umma_fwd_variant(int B, int H, int ndir, int* ub, int* ubp, int* nsplit);
bool lstm_umma_bwd_variant(int B, int H, int ndir, int* ub, int* nsplit);
// Cluster size of the backward's two-level exchange for these sizes on the current device (1: no clusters); < 0: no
// plan.  cap > 0 limits it (debug lstm mode bits 4..6).
int lstm_umma_bwd_cluster(int B, int H, int ndir);
void lstm_umma_set_cluster_cap(int cap);
// cell: CELL_LSTM or CELL_GRU (csrc/rnn_cell.cuh); the plan is the same for both
int lstm_umma_bwd(int cell, float* gates, const float* w_hh, const float* cstate, const float* dout, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t lstm_umma_workspace_bytes(int B, int H, int ndir);
int lstm_umma_plan(int B, int H, int ndir, int* unit_block, int* batch_block, int* n_ctas);
// strict: the formal acquire after each flag poll (debug mode 256)
int lstm_umma_fwd(int cell, float* gates, const float* w_hh, float* cstate, float* out, int B, int T, int H, int ndir,
                  void* workspace, size_t workspace_bytes, bool strict, cudaStream_t stream);

}  // namespace b200asr
