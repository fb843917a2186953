/* Test / measurement switches of libb200asr.so.  NOT part of the drop-in boundary (include/b200asr.h): they exist for
 * tests/ (forcing the fallback kernel generations so that they stay covered) and tools/ (A/B timing). */
#ifndef B200ASR_DEBUG_H
#define B200ASR_DEBUG_H
#include "b200asr.h"
#ifdef __cplusplus
extern "C" {
#endif

/* debug/test: 0 (default) = wgmma step GEMMs where the shape allows, else 3xTF32 mma.sync wherever the planner finds
 * a 16-row-tile decomposition, else fp32 FMA; 1 = always the packed-fp32-FMA step kernels; 3 = never wgmma (the
 * mma.sync generation); 256 = as 0, with the formal acquire (ld.acquire + proxy fence) after each flag poll of the
 * wgmma forward.  All are fp32-class and parity-tested.  Bits 4..6 ((mode >> 4) & 7, 0 = none) cap the cluster size
 * of the wgmma backward's two-level exchange: 16 keeps it at 1 (every partial straight to L2), 32 at <= 2. */
B200ASR_API void b200asr_debug_set_lstm_mode(int mode);
/* test: the cluster size CS of the exchange b200asr_bilstm_bwd (bwd = 1) runs for these sizes under the current lstm
 * mode on the current device: the largest of 4, 2 whose staging buffers fit in shared memory, that divides the unit
 * blocks into a multiple of 4 clusters, and whose clusters the device holds all at once for a cooperative launch; else 1
 * (also without a device, without the cluster occupancy query, after the runtime refused a cooperative cluster launch,
 * and for every kernel but the wgmma backward).  < 0 when the shape has no plan. */
B200ASR_API int b200asr_debug_lstm_cluster(int B, int H, int ndir, int bwd);
/* test: the step-kernel variant b200asr_bilstm_fwd (bwd = 0) / _bwd (bwd = 1) runs for these sizes under the current
 * lstm mode on the current device (132 SMs / 232448 B of shared memory without one).  Fills desc[9] =
 * {generation (1 wgmma, 2 mma.sync 3xTF32, 3 fp32 FMA), unit block UB, template unit block (UBP of the wgmma forward,
 *  else UB), exchange protocol of the wgmma kernels (1 data-is-the-flag polling: the backward, 0 flag + bulk copy: the
 *  forward), strict acquire, nsplit (launches), loop form (mma.sync forward 0 = v2, 1 / 2 = fwd_group_mma<1> / <2>;
 *  mma.sync backward 0; FMA: halves NH), FMA register-tile rows R, vectorised UB % 4 == 0 stores}.  Returns 0, or < 0
 * when the shape has no plan.  The dispatcher makes its choice through the same function. */
B200ASR_API int b200asr_debug_lstm_variant(int B, int H, int ndir, int bwd, int* desc);
/* test: which alpha/beta lattice kernel b200asr_ctc_fwd_bwd(_logits) runs for a padded target width L_max: 1-4 = the
 * warp kernel with that many extended-label positions per lane, 5 = the block kernel with one position per thread,
 * 6 = the block kernel with a strided loop over the positions.  The dispatcher calls the same rule. */
B200ASR_API int b200asr_debug_ctc_variant(int L_max);
/* test: the minimum-blocks-per-SM instance (1 or 2) of the location-attention backward kernel that
 * b200asr_locattn_bwd(_acc) launches for these sizes on the current device; 0 for bad sizes. */
B200ASR_API int b200asr_debug_locattn_bwd_minb(int B, int T, int D, int E);
/* test: the same for the dot-product attention backward b200asr_dotattn_bwd_acc launches for R rows. */
B200ASR_API int b200asr_debug_dotattn_bwd_minb(int R, int T, int E);
/* test: the same for the multi-head location-aware backward b200asr_locattn_heads_bwd_acc launches for B utterances
 * of N heads (one cluster per utterance). */
B200ASR_API int b200asr_debug_locattn_heads_bwd_minb(int B, int N, int T, int D, int E);
/* test: the split-K plan b200asr_gemm3x_tn (form 0; 1 with B_lo), _nn (2), _nt (3) or b200asr_gemm_f16x3 (4) makes
 * for these sizes on the current device (132 SMs without one) with a workspace of workspace_bytes.  K is the
 * contraction length (T for nt, which walks `batches` entries of T; batches must be 1 for the other forms; the
 * unpadded or padded K for f16x3).  Fills desc[10] = {rule (0 one slice, 1 SM fill, 2 efficiency search, 3 workspace
 * fallback), split count the rule asked for, slices launched, K blocks per slice, K blocks of the last slice,
 * accumulation chunk length in K blocks, length of the last chunk of the first slice, of the last slice, K blocks in
 * total, k per K block (32 for 3xTF32, 64 for f16x3)}.  The launchers make their choice through the same function. */
B200ASR_API int b200asr_debug_gemm_plan(int form, int M, int N, int K, int batches, size_t workspace_bytes, int* desc);

#ifdef __cplusplus
}
#endif
#endif /* B200ASR_DEBUG_H */
