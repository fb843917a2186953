/* Test / measurement switches of libb200asr.so.  NOT part of the drop-in boundary (include/b200asr.h): they exist for
 * tests/ (forcing the fallback kernel generations so that they stay covered) and tools/ (clock64 timelines, A/B timing). */
#ifndef B200ASR_DEBUG_H
#define B200ASR_DEBUG_H
#include "b200asr.h"
#ifdef __cplusplus
extern "C" {
#endif

/* debug: when non-NULL, CTA 0 of the next b200asr_bilstm_fwd (or, with mode flag 128, _bwd) calls records clock64 stamps into [T][16] int64 */
B200ASR_API void b200asr_debug_set_lstm_trace(long long* device_buffer);
/* debug/test: 0 (default) = wgmma step GEMMs where the shape allows, else 3xTF32 mma.sync wherever the planner finds
 * a 16-row-tile decomposition, else fp32 FMA; 1 = always the packed-fp32-FMA step kernels; 3 = never wgmma (the
 * mma.sync generation).  All are fp32-class and parity-tested.
 * Upper bits (mode >> 4) are test / measurement switches: 512 = the other backward generation (wgmma <-> mma.sync),
 * 1024 / 2048 = the other state-exchange protocol of the wgmma forward / backward kernel (flag + bulk copy <->
 * data-is-the-flag polling), 128 = trace the backward kernel; see tools/time_lstm.py. */
B200ASR_API void b200asr_debug_set_lstm_mode(int mode);
/* test: which alpha/beta lattice kernel b200asr_ctc_fwd_bwd(_logits) runs for a padded target width L_max: 1-4 = the
 * warp kernel with that many extended-label positions per lane, 5 = the block kernel with one position per thread,
 * 6 = the block kernel with a strided loop over the positions.  The dispatcher calls the same rule. */
B200ASR_API int b200asr_debug_ctc_variant(int L_max);
/* test: the minimum-blocks-per-SM instance (1 or 2) of the location-attention backward kernel that
 * b200asr_locattn_bwd(_acc) launches for these sizes on the current device; 0 for bad sizes. */
B200ASR_API int b200asr_debug_locattn_bwd_minb(int B, int T, int D, int E);

#ifdef __cplusplus
}
#endif
#endif /* B200ASR_DEBUG_H */
