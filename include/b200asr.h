/* libb200asr.so - C ABI of the ASR train-step kernels (H100, sm_90a).
 *
 * The reference (Alexander-H-Liu/End-to-end-ASR-Pytorch) is 100% Python and has no FFI of its own: every
 * "kernel" is a stock torch / torchaudio call.  Each entry point below therefore cites the reference CALL SITE
 * (file:line of the reference checkout, or kaldi.py = torchaudio/compliance/kaldi.py) whose arithmetic it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless stated otherwise; tensors are contiguous row-major fp32,
 *     indices / lengths are int64 ("long long") where the reference passes LongTensors, int32 otherwise;
 *   - the library never allocates, frees or retains device memory: the caller owns inputs, outputs and the
 *     workspaces whose sizes the *_workspace_bytes() helpers return;
 *   - all work is enqueued on `stream` (a cudaStream_t) and the call returns without synchronising;
 *   - return value: 0 = ok, <0 = error (-1 invalid argument, -2 CUDA failure); the message is available
 *     from b200asr_last_error() (thread local).  There is no CPU fallback.
 */
#ifndef B200ASR_H
#define B200ASR_H

#include <stddef.h>

#define B200ASR_VERSION 100

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200ASR_API __attribute__((visibility("default")))
#else
#define B200ASR_API
#endif

typedef void* b200asr_stream; /* cudaStream_t */

B200ASR_API int b200asr_version(void);
B200ASR_API const char* b200asr_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py's gpu_launches) */
B200ASR_API unsigned long long b200asr_launch_count(void);
B200ASR_API void b200asr_launch_count_reset(void);
B200ASR_API int b200asr_device_sm_count(void);

/* ---- K1: fused STFT + mel + log -----------------------------------------------------------------------
 * replaces src/audio.py:104-108 -> kaldi.py:514-646 (fbank), :44-83 (framing), :154-217 (dc / pre-emphasis /
 * window).  wave [B, n_max] (zero padded), wave_len [B] samples.  window [win_size] and the sparse mel
 * filters (filter i covers FFT bins mel_start[i] .. +mel_count[i], weights at mel_w[mel_off[i] ..]) are
 * caller-built tables.  fbank [B, t_max, n_mel] (frames >= n_frames[b] are zeroed), n_frames [B] (int32 out)
 * = min(1 + (n - win_size) / win_shift, t_max) with n = clamp(wave_len[b], 0, n_max) (snip_edges=True; 0 when
 * n < win_size): an utterance is its first min(frames, t_max) frames, and no sample at or beyond n_max of its row is
 * read whatever wave_len says.  n_fft must be 512.                                                          */
B200ASR_API int b200asr_fbank_fwd(const float* wave, const int* wave_len, int B, int n_max, int win_size, int win_shift,
                      int n_fft, float preemph, int remove_dc, const float* window, int n_mel,
                      const int* mel_start, const int* mel_count, const int* mel_off, const float* mel_w,
                      int mel_w_total, int use_log, float log_floor, float* fbank, int t_max, int* n_frames,
                      b200asr_stream stream);
/* same kernel fed with 16-bit PCM [B, n_max] (what the corpus files hold, src/data.py:14-43 -> torchaudio.load): the
 * int16 -> fp32 conversion (sample / 32768) happens on the fly, so the host-to-device copy is half as large */
B200ASR_API int b200asr_fbank_fwd_pcm16(const short* pcm, const int* wave_len, int B, int n_max, int win_size, int win_shift,
                      int n_fft, float preemph, int remove_dc, const float* window, int n_mel,
                      const int* mel_start, const int* mel_count, const int* mel_off, const float* mel_w,
                      int mel_w_total, int use_log, float log_floor, float* fbank, int t_max, int* n_frames,
                      b200asr_stream stream);

/* ---- K2+K3: delta / delta-delta + per-utterance CMVN + channel-major interleave ---------------------------
 * replaces src/audio.py:51-54,57-77 (Delta), :25-27 (CMVN, unbiased std, eps added to std), :85-89
 * (Postprocess).  feat [B, t_max, n_mel*(delta_order+1)], rows >= n_frames[b] are zero (pad_sequence,
 * src/data.py:39).  Utterance b is its first m = clamp(n_frames[b], 0, t_max) fbank rows: the CMVN statistics
 * cover exactly those m frames, the delta taps see zeros beyond them, and rows at or beyond m are never read.     */
B200ASR_API size_t b200asr_delta_cmvn_workspace_bytes(int B, int t_max, int n_mel, int delta_order);
B200ASR_API int b200asr_delta_cmvn_fwd(const float* fbank, const int* n_frames, int B, int t_max, int n_mel,
                                       int delta_order, int delta_window, int apply_cmvn, float cmvn_eps,
                                       float* feat, void* workspace, size_t workspace_bytes, b200asr_stream stream);

/* ---- K9: log-softmax over the vocabulary (src/asr.py:96) -------------------------------------------------
 * log_probs may alias logits.  lse [n_rows] and argmax [n_rows] (int64; util.py:117-118 / test_asr.py:116-118)
 * are optional (NULL); log_probs may be NULL when lse is given (statistics only, see b200asr_ctc_fwd_bwd_logits). */
B200ASR_API int b200asr_log_softmax_fwd(const float* logits, float* log_probs, float* lse, long long* argmax,
                            long long n_rows, int V, b200asr_stream stream);
B200ASR_API int b200asr_log_softmax_bwd(const float* log_probs, const float* grad_out, float* grad_in, long long n_rows,
                            int V, b200asr_stream stream);

/* ---- K10: CTC loss forward + backward in one call ---------------------------------------------------------
 * replaces torch.nn.CTCLoss(blank=0, zero_infinity=False) at bin/train_asr.py:49,123-124 (ATen _ctc_loss +
 * _ctc_loss_backward).  log_probs element (b,t,c) lives at log_probs[b*stride_b + t*stride_t + c]; targets
 * [B, L_max] zero padded int64; input_lengths / target_lengths [B] int64.  nll [B] out (per-utterance negative
 * log likelihood, +inf when infeasible).  If grad != NULL it receives, with the same strides as log_probs,
 * grad_scale[b] * (exp(lp) - exp(log sum_{s: l'_s = c} alpha_t(s) beta_t(s) + nll - lp)) for t < input_length
 * and 0 after it - ATen's convention (SURVEY.md F9).  grad_scale may be NULL (= 1).  An infeasible utterance
 * (nll = +inf) gets ATen's zero_infinity=False gradient: NaN at every element for t < input_length, 0 after it
 * (all 0 when input_length is 0); the NaN grad norm then makes the fused update skip the step.               */
B200ASR_API size_t b200asr_ctc_workspace_bytes(int B, int T, int L_max);
B200ASR_API int b200asr_ctc_fwd_bwd(const float* log_probs, long long stride_b, long long stride_t, const long long* targets,
                        const long long* input_lengths, const long long* target_lengths, int B, int T, int V,
                        int L_max, int blank, float* nll, const float* grad_scale, float* grad, void* workspace,
                        size_t workspace_bytes, b200asr_stream stream);
/* The gradient half alone, for callers that learn the upstream scale only in their backward pass (autograd): run
 * b200asr_ctc_fwd_bwd with grad = NULL in the forward (nll + the alpha/beta lattices stay in `workspace`), then this
 * with the SAME workspace.  `upstream` (device scalar, may be NULL) multiplies every element, so no separate scaling
 * pass over the [T,B,V] gradient is needed.  Out-of-range labels are clamped into [0,V) (torch raises on them). */
B200ASR_API int b200asr_ctc_grad(const float* log_probs, long long stride_b, long long stride_t, const long long* targets,
                     const long long* input_lengths, const long long* target_lengths, int B, int T, int V,
                     int L_max, int blank, const float* nll, const float* grad_scale, const float* upstream,
                     float* grad, void* workspace, size_t workspace_bytes, b200asr_stream stream);

/* The CTC head fused into the loss (src/asr.py:96 + bin/train_asr.py:123-124 in one pass structure): the same two
 * calls on LOGITS plus the per-row log-sum-exp  row_lse[b * T + t]  (b200asr_log_softmax_fwd with log_probs = NULL
 * writes only lse + argmax).  log-prob(b,t,c) = logits[...] - row_lse[b*T + t] is formed on the fly, the V-wide log-prob
 * tensor is never written or re-read, and `grad` IS the logit gradient (exp(x - lse) - occupancy has zero class sum,
 * SURVEY.md F9):  12*T*V bytes per utterance (read logits twice, write the gradient once) instead of 28*T*V.      */
B200ASR_API int b200asr_ctc_fwd_bwd_logits(const float* logits, const float* row_lse, long long stride_b, long long stride_t,
                               const long long* targets, const long long* input_lengths,
                               const long long* target_lengths, int B, int T, int V, int L_max, int blank, float* nll,
                               const float* grad_scale, float* grad, void* workspace, size_t workspace_bytes,
                               b200asr_stream stream);
B200ASR_API int b200asr_ctc_grad_logits(const float* logits, const float* row_lse, long long stride_b, long long stride_t,
                            const long long* targets, const long long* input_lengths, const long long* target_lengths,
                            int B, int T, int V, int L_max, int blank, const float* nll, const float* grad_scale,
                            const float* upstream, float* grad, void* workspace, size_t workspace_bytes,
                            b200asr_stream stream);

/* ---- SURVEY 8(f) rank 3: CTC prefix scoring (joint CTC/attention beam search) ---------------------------------
 * replaces CTCPrefixScore.cheap_compute (src/ctc.py:81-116), called from src/decode.py:129-131 once per hypothesis
 * and step on the host.  Scores N hypotheses x C candidate tokens in one launch.
 *   log_probs  [T, V]      CTC log-probs of the utterance          r_prev   [N, T, 2]  state of each prefix
 *   last_char  [N], prefix_len [N] (int32)                         candidates [N, C] (int32, ids in [0,V))
 *   psi [N, C] out: log P(prefix + c, ...)                         r_out [N, C, T, 2] out: state of prefix + c
 * float32, the reference's finite log-zero (-1e8), numpy.logaddexp formula.  Out-of-range ids are the caller's bug. */
B200ASR_API int b200asr_ctc_prefix_score(const float* log_probs, int T, int V, const float* r_prev, const int* last_char,
                             const int* prefix_len, const int* candidates, int N, int C, int blank, int eos,
                             float* psi, float* r_out, b200asr_stream stream);

/* ---- K7/K8: persistent (Bi)LSTM recurrence -----------------------------------------------------------------
 * replaces the time loop inside torch.nn.LSTM as used by src/module.py:112-113,129-132 (one layer,
 * batch_first, zero initial state, run over the padded frames).  ndir = 1 or 2 (direction 1 = reverse time).
 *   gates  [ndir, B, T, H, 4]  in : input projection x.W_ih^T + b_ih + b_hh, gate-interleaved (i,f,g,o minor)
 *                              out: the activated gates (stash for the backward pass)
 *   w_hh   [ndir, 4H, H]       PyTorch layout (weight_hh_l0 [, weight_hh_l0_reverse])
 *   cstate [ndir, B, T, H]     out: cell state after every step (stash)
 *   out    [B, T, ndir*H]      out: hidden states (the layer output)
 * backward: gates in = stash, out = d(loss)/d(pre-activation) in the same layout; dout [B, T, ndir*H].
 * H must be a multiple of 16; the (unit-block, batch-block) decomposition must fit the SM count
 * (b200asr_bilstm_plan reports it).  Launched cooperatively: all CTAs are co-resident.                       */
B200ASR_API size_t b200asr_bilstm_workspace_bytes(int B, int T, int H, int ndir);
B200ASR_API int b200asr_bilstm_plan(int B, int H, int ndir, int* unit_block, int* batch_block, int* n_ctas);
/* 1 when the step GEMMs of this shape run on the tensor cores (3xTF32 mma), 0 for the packed-fp32-FMA kernels,
 * -1 when the shape has no decomposition */
B200ASR_API int b200asr_bilstm_uses_tensor_cores(int B, int H, int ndir);
/* 1 when the forward recurrence of this shape runs on warpgroup MMAs (wgmma f16 with
 * fp32 accumulators in registers and the fp16 hi/lo "2 x 2 block" split product, csrc/lstm_umma.cu), else 0 */
B200ASR_API int b200asr_bilstm_uses_tcgen05(int B, int H, int ndir);
B200ASR_API int b200asr_bilstm_fwd(float* gates, const float* w_hh, float* cstate, float* out, int B, int T, int H, int ndir,
                       void* workspace, size_t workspace_bytes, b200asr_stream stream);
B200ASR_API int b200asr_bilstm_bwd(float* gates, const float* w_hh, const float* cstate, const float* dout, int B, int T,
                       int H, int ndir, void* workspace, size_t workspace_bytes, b200asr_stream stream);

/* ---- K7/K8 with a GRU cell: persistent (Bi)GRU recurrence -----------------------------------------------------
 * replaces the time loop inside torch.nn.GRU as used by src/module.py:112-113,129-132 (the nn.GRU branch: one layer,
 * batch_first, zero initial state, run over the padded frames).  Same kernels, plan, variants and workspace as the
 * BiLSTM above (b200asr_bilstm_workspace_bytes / _plan / b200asr_debug_lstm_variant answer for both cells); only the
 * pointwise cell differs.  The layer's weights are packed into four gate slots per unit, as ops.pack_decoder_weights
 * ("GRU") packs them:
 *   gates  [ndir, B, T, H, 4]  in : (gi_r + gh_r, gi_z + gh_z, gi_n, gh_n) of the input projection, i.e. x.W_ih4^T + b4
 *                                   with W_ih4 = [W_ir; W_iz; W_in; 0] and b4 = (b_ir + b_hr, b_iz + b_hz, b_in, b_hn)
 *                              out: (r, z, n, gh_n) with gh_n = h_{t-1}.W_hn^T + b_hn (stash for the backward pass)
 *   w_hh   [ndir, 4H, H]       packed [W_hr; W_hz; 0; W_hn] (gate-major rows g*H + j, slot 2 zero)
 *   hstate [ndir, B, T, H]     out: h after every step (stash; the backward reads h_{t-1} from it)
 *   out    [B, T, ndir*H]      out: hidden states (the layer output)
 * r = sigmoid, z = sigmoid, n = tanh(gi_n + r.gh_n), h = (h_prev - n).z + n in ATen's expression order.
 * backward: gates in = stash, out = dG = (d pre_r, d pre_z, d gi_n, d gh_n) in the same layout; dout [B, T, ndir*H].
 * Limits as for the BiLSTM (H a multiple of 16).                                                                  */
B200ASR_API int b200asr_bigru_fwd(float* gates, const float* w_hh, float* hstate, float* out, int B, int T, int H, int ndir,
                      void* workspace, size_t workspace_bytes, b200asr_stream stream);
B200ASR_API int b200asr_bigru_bwd(float* gates, const float* w_hh, const float* hstate, const float* dout, int B, int T,
                      int H, int ndir, void* workspace, size_t workspace_bytes, b200asr_stream stream);


/* ---- K13: one LSTM cell step (decoder, src/asr.py:214-221) -------------------------------------------------
 * preact [B, 4H] gate-major (i,f,g,o) = x.W_ih^T + h.W_hh^T + biases; gates [B,4H] activated (stash).        */
B200ASR_API int b200asr_lstm_cell_fwd(const float* preact, const float* c_prev, float* gates, float* c, float* h, int B,
                          int H, b200asr_stream stream);
B200ASR_API int b200asr_lstm_cell_bwd(const float* gates, const float* c_prev, const float* c, const float* dh,
                          const float* dc_next /* may be NULL */, float* dpreact, float* dc_prev, int B, int H,
                          b200asr_stream stream);

/* ---- K13g: one GRU cell step (decoder with module: 'GRU', src/asr.py:214-221) ----------------------------------
 * preact [B, 4H] = (gi_r + gh_r, gi_z + gh_z, gi_n, gh_n), gi = x.W_ih^T + b_ih, gh = h.W_hh^T + b_hh.
 * r = sigmoid, z = sigmoid, n = tanh(gi_n + r.gh_n), h = (h_prev - n).z + n; gates [B, 4H] = (r, z, n, gh_n) (stash).
 * Backward: dpreact [B, 4H] = (d pre_r, d pre_z, d gi_n, d gh_n), dh_prev = dh.z (the part that bypasses the GEMM).
 * dh may be NULL (no gradient reaches h).                                                                           */
B200ASR_API int b200asr_gru_cell_fwd(const float* preact, const float* h_prev, float* gates, float* h, int B, int H,
                         b200asr_stream stream);
B200ASR_API int b200asr_gru_cell_bwd(const float* gates, const float* h_prev, const float* dh /* may be NULL */,
                         float* dpreact, float* dh_prev, int B, int H, b200asr_stream stream);

/* ---- K12: location-aware attention step, forward and backward, one launch each ----------------------------------
 * replaces src/module.py:234-258 (LocationAwareAttention.forward) + :189-195 (_attend), single head:
 * Conv1d(1->K, 2R+1, pad R, no bias) over prev_att -> Linear(K->D, no bias) -> tanh -> energy = Linear(D->1)(tanh(key +
 * q + loc)) / temperature -> masked softmax over t < enc_len[b] -> context = attn . value.
 *   q [B,D] (already tanh(proj_q(h))), key [B,T,D] (tanh(proj_k(enc))), value [B,T,E], prev_att [B,T], enc_len [B] i64,
 *   w_conv [K,2R+1], w_proj [D,K], w_energy [D], b_energy [1]  ->  attn [B,T], ctx [B,E].
 * backward: dctx [B,E], dattn [B,T] or NULL -> dq_part [B,CS,D] (sum over CS = dq), dkey [B,T,D], dvalue [B,T,E],
 * dprev [B,T], wpart [B*CS, P] with P = D*K + K*(2R+1) + D + 1 laid out (d w_proj | d w_conv | d w_energy | d b_energy);
 * the caller sums wpart over its first axis.  CS = b200asr_locattn_cluster_size(T, E) CTAs cooperate per utterance
 * through distributed shared memory.  K <= 16, E % 4 == 0, D <= 512, E / CS <= 1024 (the cluster rule keeps E / CS
 * <= 1024 for every T whenever E % 16 == 0 and E <= 4096).  An utterance with enc_len 0 gets the reference's masked
 * softmax of no frames: NaN attention, NaN context and NaN d(value); its other gradients are 0.                   */
B200ASR_API int b200asr_locattn_cluster_size(int T, int E);
B200ASR_API size_t b200asr_locattn_wpart_floats(int D, int K, int R);
B200ASR_API int b200asr_locattn_fwd(const float* q, const float* key, const float* value, const float* prev_att,
                                    const long long* enc_len, const float* w_conv, const float* w_proj,
                                    const float* w_energy, const float* b_energy, float temperature, int B, int T,
                                    int D, int E, int K, int R, float* attn, float* ctx, b200asr_stream stream);
B200ASR_API int b200asr_locattn_bwd(const float* q, const float* key, const float* value, const float* prev_att,
                                    const long long* enc_len, const float* w_conv, const float* w_proj,
                                    const float* w_energy, float temperature, const float* attn, const float* dctx,
                                    const float* dattn, int B, int T, int D, int E, int K, int R, float* dq_part,
                                    float* dkey, float* dvalue, float* dprev, float* wpart, b200asr_stream stream);
/* The decode loop's form of the backward (src/asr.py:112-151 calls the attention L times on the SAME key / value):
 * d(key) and the weight-gradient partials are ADDED into per-batch accumulators (zeroed by the caller before the first
 * step) and d(value) is not produced here at all: d(value)[b,t,:] = sum_l attn_l[b,t] * dctx_l[b,:] is formed once after
 * the loop by b200asr_attn_dvalue from the stacked per-step alignments [B,L,T] and context gradients [B,L,E] - instead
 * of a [B,T,E] write per step that autograd then has to re-add L-1 times.                                             */
B200ASR_API int b200asr_locattn_bwd_acc(const float* q, const float* key, const float* value, const float* prev_att,
                                        const long long* enc_len, const float* w_conv, const float* w_proj,
                                        const float* w_energy, float temperature, const float* attn, const float* dctx,
                                        const float* dattn, int B, int T, int D, int E, int K, int R, float* dq_part,
                                        float* dkey_acc, float* dprev, float* wpart_acc, b200asr_stream stream);
B200ASR_API int b200asr_attn_dvalue(const float* attn_steps, const float* dctx_steps, int B, int L, int T, int E,
                                    float* dvalue, int accumulate, b200asr_stream stream);

/* ---- K12d: scaled dot-product attention step, one or more heads, forward and decode-loop backward ----------------
 * replaces src/module.py:198-212 (ScaleDotAttention.forward) + :189-195 (_attend), called from src/asr.py:307.  Rows are
 * R = B * num_head (row r = b * num_head + n), row r masked by len = clamp(enc_len[r / num_head], 0, T):
 *   q [R,D] (already tanh(proj_q(h)) per head), key [R,T,D], value [R,T,E] (the tensor Attention.forward forms,
 *   including its value.repeat(num_head, 1, 1) without a value projection), enc_len [B] i64
 *   ->  e[t] = (q . key[r,t]) / temperature for t < len;  attn [R,T] = softmax(e) over t < len, exactly 0 at t >= len;
 *       ctx [R,E] = sum_t attn[t] value[r,t].
 * backward (the decode loop's form, as b200asr_locattn_bwd_acc): dctx [R,E], dattn [R,T] or NULL;
 *   g[t] = dctx . value[r,t] + dattn[t], de[t] = attn[t] (g[t] - sum attn g) / temperature  ->  dq_part [R,CS,D]
 *   (sum over CS = dq), dkey_acc [R,T,D] += de[t] q for t < len.  No d(value): b200asr_attn_dvalue forms it once after the
 *   loop from the stacked (attn_l, dctx_l).  Frames t >= len are never read and receive nothing.
 * CS = b200asr_locattn_cluster_size(T, E) CTAs cooperate per row.  Limits (b200asr_dotattn_supported): 0 < T <=
 * B200ASR_DOTATTN_MAX_T, D <= 512, E % 4 == 0, E / CS <= 1024.  Deterministic: no float atomics.                 */
#define B200ASR_DOTATTN_MAX_T 8192
B200ASR_API int b200asr_dotattn_supported(int T, int D, int E);
B200ASR_API int b200asr_dotattn_fwd(const float* q, const float* key, const float* value, const long long* enc_len,
                                    int num_head, float temperature, int R, int T, int D, int E, float* attn, float* ctx,
                                    b200asr_stream stream);
B200ASR_API int b200asr_dotattn_bwd_acc(const float* q, const float* key, const float* value, const long long* enc_len,
                                        int num_head, float temperature, const float* attn, const float* dctx,
                                        const float* dattn, int R, int T, int D, int E, float* dq_part, float* dkey_acc,
                                        b200asr_stream stream);

/* ---- K12h: multi-head location-aware attention step, forward and decode-loop backward -----------------------------
 * replaces src/module.py:234-258 (LocationAwareAttention.forward) + :189-195 (_attend) with num_head = N > 1.  ONE
 * location convolution per utterance over the N channels of prev_att, its projection shared by the N heads:
 *   conv[b,k,t] = sum_n sum_j w_conv[k,n,j] prev_att[b,n,t+j-R],  loc[b,t,d] = tanh(sum_k w_proj[d,k] conv[b,k,t]),
 *   e[r,t] = (b_energy + sum_d w_energy[d] tanh(key[r,t,d] + q[r,d] + loc[r/N,t,d])) / temperature for t < len,
 *   attn [R,T] = softmax(e) over t < len (exactly 0 at t >= len), ctx [R,E] = sum_t attn[t] value[r,t],
 * with R = B * N rows (row r = b * N + n), len = clamp(enc_len[r / N], 0, T):
 *   q [R,D], key [R,T,D], value [R,T,E] (the tensor Attention.forward forms, including its value.repeat(N, 1, 1)
 *   without a value projection), prev_att [B,N,T], enc_len [B] i64, w_conv [K,N,2R+1], w_proj [D,K], w_energy [D],
 *   b_energy [1].
 * backward (the decode loop's form, as b200asr_locattn_bwd_acc): dctx [R,E], dattn [R,T] or NULL -> dq_part [R,CS,D]
 *   (sum over CS = dq), dkey_acc [R,T,D] += d(key) for t < len, dprev [B,N,T], wpart_acc [B*CS, P] += the per-CTA
 *   partials, P = b200asr_locattn_heads_wpart_floats(N, D, K, R) = D*K + K*N*(2R+1) + D + 1 laid out (d w_proj |
 *   d w_conv | d w_energy | d b_energy).  No d(value): b200asr_attn_dvalue forms it once after the loop over R rows.
 * One cluster of CS = b200asr_locattn_cluster_size(T, E) CTAs per UTTERANCE covers its N heads.  Frames t >= len of
 * key and value are never read.  Deterministic: no float atomics.  An utterance with enc_len 0 gets the reference's
 * NaN attention, context and d(value).  Limits (b200asr_locattn_heads_supported, checked before any CUDA call):
 * N <= 16, K <= 16, D <= 512, E % 4 == 0, E / CS <= 1024, and both kernels' shared memory within the device's opt-in
 * maximum (it grows as N (T + 2R) + K N (2R+1) + N CS T).                                                           */
B200ASR_API int b200asr_locattn_heads_supported(int N, int T, int D, int E, int K, int R);
B200ASR_API size_t b200asr_locattn_heads_wpart_floats(int N, int D, int K, int R);
B200ASR_API int b200asr_locattn_heads_fwd(const float* q, const float* key, const float* value, const float* prev_att,
                                          const long long* enc_len, const float* w_conv, const float* w_proj,
                                          const float* w_energy, const float* b_energy, float temperature, int B,
                                          int N, int T, int D, int E, int K, int R, float* attn, float* ctx,
                                          b200asr_stream stream);
B200ASR_API int b200asr_locattn_heads_bwd_acc(const float* q, const float* key, const float* value,
                                              const float* prev_att, const long long* enc_len, const float* w_conv,
                                              const float* w_proj, const float* w_energy, float temperature,
                                              const float* attn, const float* dctx, const float* dattn, int B, int N,
                                              int T, int D, int E, int K, int R, float* dq_part, float* dkey_acc,
                                              float* dprev, float* wpart_acc, b200asr_stream stream);

/* ---- K15: cross-entropy (log-softmax + NLL, ignore_index) forward + logit gradient ----------------------
 * replaces torch.nn.CrossEntropyLoss(ignore_index=0) at bin/train_asr.py:47,127-131.  row_loss [n_rows] =
 * lse(x) - x[target] (0 for ignored rows); dlogits (optional) = grad_scale[0] * (softmax(x) - onehot), zero rows
 * for ignored targets; grad_scale is a DEVICE scalar (e.g. 1 / number of non-ignored rows) or NULL (= 1).     */
B200ASR_API int b200asr_ce_fwd_bwd(const float* logits, const long long* target, long long ignore_index,
                                   long long n_rows, int V, const float* grad_scale, float* row_loss,
                                   float* dlogits, b200asr_stream stream);

/* ---- embedding backward: the gradient of the row gather  emb(x)  of the RNN language model (src/lm.py:17,32) ------
 * replaces the backward of nn.Embedding there, which allocates and zero-fills a [V, E] tensor per step, scatters
 * into it and has autograd add it into .grad:
 *   dW[ids[n], :] += dY[n, :]   for n in [0, N), IN PLACE on an existing row-major [V, E] fp32 gradient.
 * Deterministic, without float atomics: each touched row gets the sum of its occurrences taken in ascending n, added
 * once onto its value; the result does not depend on the launch configuration.  Rows whose token does not occur are
 * not touched, and ids outside [0, V) are skipped (neither read nor written).  dY is row-major [N, E];
 * workspace >= b200asr_embedding_bwd_workspace_bytes(N, V) bytes, owned by the caller.                           */
B200ASR_API size_t b200asr_embedding_bwd_workspace_bytes(int N, int V);
B200ASR_API int b200asr_embedding_bwd(const long long* ids, const float* dY, int N, int V, int E, float* dW,
                                      void* workspace, size_t workspace_bytes, b200asr_stream stream);

/* ---- K16: gradient norm, clip and optimizer update on flat buffers (src/solver.py:84-89, src/optim.py) ----
 * The norm is accumulated in fp64 and rounded once to fp32.  grad_norm (device scalar) may be NULL (no clipping,
 * no skip); max_norm <= 0 disables clipping.  A NaN norm skips the update: nothing is written.  An Inf norm does
 * not: the clip coefficient is max_norm / inf = 0, as in clip_grad_norm_.
 * step_count (device int64) is the number of applied updates, torch.optim's state["step"]: each call advances it
 * on the device unless the update is skipped, and Adam's bias corrections are formed from the advanced count in
 * double.  rho / beta1 / beta2 are torch's double hyper-parameters; the kernels use them and their complements
 * 1 - rho, 1 - beta formed in double, each rounded once to fp32.                                               */
B200ASR_API size_t b200asr_grad_norm_scratch_bytes(void);
B200ASR_API int b200asr_grad_norm(const float* grad, long long n, float* norm_out, void* scratch, b200asr_stream stream);
B200ASR_API int b200asr_adadelta_step(float* param, const float* grad, float* square_avg, float* acc_delta, long long n,
                          float lr, double rho, float eps, float weight_decay, const float* grad_norm,
                          float max_norm, long long* step_count, b200asr_stream stream);
B200ASR_API int b200asr_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                      double beta1, double beta2, float eps, float weight_decay, const float* grad_norm,
                      float max_norm, long long* step_count, b200asr_stream stream);

/* ---- K6 / K9 / K11: dense  x . W^T (+ bias)  on the tensor cores at fp32-class accuracy ------------------------------
 * replaces the CTC head (src/asr.py:29,96), the proj_k / char_trans / pj Linear layers (src/asr.py:177,220,242-243;
 * src/module.py:123,155), the decoder LSTM's projections (src/asr.py:214-221) and the Conv1d prenet (src/module.py:75-78),
 * with their input and weight gradients.
 * wgmma tf32 with error compensation: A is split into hi / lo in registers, B's raw fp32 tile is its TF32 hi operand
 * (the tensor core truncates) and B's residual tile is either made on the fly in shared memory or read pre-split; three
 * products per K block into one register accumulator.
 * Common arguments: C row-major with leading dimension ldc >= N; bias may be NULL; accumulate != 0 adds to the existing
 * C.  workspace = NULL runs without split-K; otherwise it holds b200asr_gemm3x_workspace_bytes(M, N) bytes and small
 * M x N tile grids with a long contraction (the decoder's per-step products, 64 rows) are cut along K over all SMs,
 * partial tiles summed in a fixed order by a second launch (bias / accumulate applied there).
 *
 * tn:  C[M,N] (+)= A[M,K] . B[N,K]^T + bias[N]      A, B row-major with K contiguous (16-byte aligned, K % 4 == 0).
 *   lda is A's row pitch (floats, multiple of 4).  lda < K is allowed: overlapping rows are the im2col view of a strided
 *   1-D convolution over a [time, channels] buffer (CNNExtractor, src/module.py:75-78: kernel 4, stride 2 -> K = 4*C,
 *   lda = 2*C), so the convolution runs in this kernel without materialising the windows.
 *   B_lo = B - trunc_tf32(B) (b200asr_tf32_residual; same shape as B, dense rows of K floats) is the weight matrix'
 *   residual computed once per step instead of once per tile by every CTA: its tile arrives by TMA like B's and no
 *   shared-memory split pass runs.  B_lo = NULL: the kernel makes B's residual itself; the result is the same. */
B200ASR_API int b200asr_gemm3x_tn(const float* A, int lda, const float* B, const float* B_lo, const float* bias, float* C,
                      int M, int N, int K, int ldc, int accumulate, void* workspace, size_t workspace_bytes,
                      b200asr_stream stream);
/* nn: input gradient  dX = dY . W  (autograd backward of the layers above):
 *   C[M,N] (+)= A[M,K] . B[K,N] + bias[N]       A row-major with K contiguous (pitch lda), B row-major with N contiguous
 * (pitch ldb): the weight matrix is read in place as an MN-major tensor-core operand - no transposed copy; its residual
 * is made in the kernel's transposing pass. */
B200ASR_API int b200asr_gemm3x_nn(const float* A, int lda, const float* B, int ldb, const float* bias, float* C, int M, int N,
                      int K, int ldc, int accumulate, void* workspace, size_t workspace_bytes, b200asr_stream stream);
/* weight gradient  dW = dY^T . X  (autograd backward of the same layers; contraction over the batch*time rows):
 *   C[m,n] (+)= sum_{b < batches} sum_{t < T}  A[b][t + a_shift][m] * B[b][t + b_shift][n]
 * element (b, t, c) of an operand lives at ptr[b * bstride + t * ld + c] (both operands MN-major); rows outside [0, T)
 * read as zero, so  b_shift = -1 / +1  contracts dG[t] with the hidden state of the PREVIOUS step of the forward /
 * reverse direction (dW_hh of nn.LSTM) straight from the layer output.  permute_rows != 0 writes row m of the result
 * to row (m % 4) * (M / 4) + m / 4: from the kernels' unit-major gate order back to PyTorch's gate-major rows.
 * workspace as above.                                                                                               */
B200ASR_API size_t b200asr_gemm3x_workspace_bytes(int M, int N);
B200ASR_API int b200asr_gemm3x_nt(const float* A, long long lda, long long a_bstride, int a_shift, const float* B,
                      long long ldb, long long b_bstride, int b_shift, float* C, int M, int N, int T, int batches,
                      int ldc, int accumulate, int permute_rows, void* workspace, size_t workspace_bytes,
                      b200asr_stream stream);
/* B_lo of the tn form: lo[i] = x[i] - trunc_tf32(x[i]) over n floats. */
B200ASR_API int b200asr_tf32_residual(const float* x, float* lo, long long n, b200asr_stream stream);

/* ---- VGGExtractor (src/module.py:7-66): 3x3 convolutions as implicit GEMMs on the 3xTF32 kernel ----------------------
 * Activations live in zero-haloed channels-last buffers of their (T, F): grid rows R = batches (T + 2) (F + 2), a buffer
 * holds R + F + 3 rows of C floats, and position (b, t, f) sits at row m + F + 3 with m = (b (T + 2) + t) (F + 2) + f.
 * conv3x3_fwd:  y at position (b, t, f), channel o  =  epilogue( bias[o] + sum_{tap, c} x[m + (tap / 3) (F + 2) + tap % 3][c]
 *   * w[o][tap C + c] ),  tap = 3 dt + df.  taps = 9: x is a zero-haloed buffer, C a multiple of 32; taps = 1: x is the
 *   first layer's im2col [R][32] (C = 32, b200asr_vgg_im2col) read at row m.  Epilogue: ReLU when relu != 0 (NaN stays
 *   NaN); when mask != NULL (a buffer like y) zero where mask <= 0 (the ReLU backward of the layer that made mask).  Every
 *   row from F + 3 on is written: junk grid rows (t >= T or f >= F) as exact zeros, which land on y's halo; the first
 *   F + 3 rows of y must be zero beforehand.  The input gradient is the same call on the padded dY with the weights
 *   flipped and transposed (w'[c][tap' O + o] = w[o][(8 - tap') C + c]).  One launch, no split-K.
 * conv3x3_wgrad:  dw[o][tap C + c] = sum_m dy[m + F + 3][o] x[m + (tap / 3) (F + 2) + tap % 3][c]  (x as in _fwd; dy a
 *   buffer with zeros on its halo), split-K over the rows with the workspace of b200asr_gemm3x_workspace_bytes(O,
 *   taps C) (may be NULL).
 * vgg_im2col: features (b, t, c, f) at feat[b ld_b + t Cin F + c F + f], Cin <= 3 -> the [R][32] im2col of the first
 *   conv (k = tap Cin + c, zero beyond 9 Cin and on junk rows).
 * vgg_pool_fwd: MaxPool2d(2, 2) of the buffer y of (T, F), T even, with ATen's scan order and NaN rule; idx [batches][T/2]
 *   [F/2][C] (bytes) receives the window index 2 dt + df; out is the zero-haloed buffer of (T/2, F/2), every row
 *   written, or when flat != 0 the prenet output [batches][T/2][C (F/2)] with index c (F/2) + f.
 * vgg_pool_bwd: the gradient of the buffer y of (T, F) from dout (laid out as pool_fwd's out) through idx, zero where
 *   y <= 0; every row of dy written.
 * vgg_feat_grad: dfeat [batches][T_in][Cin F] from the first conv's padded dY and its weights w1 [O][Cin][3][3]; frames
 *   t >= T get 0. */
B200ASR_API int b200asr_conv3x3_fwd(const float* x, int C, int taps, const float* w, const float* bias, const float* mask,
                        int relu, float* y, int batches, int T, int F, int O, b200asr_stream stream);
B200ASR_API int b200asr_conv3x3_wgrad(const float* dy, const float* x, int C, int taps, float* dw, int batches, int T, int F,
                          int O, void* workspace, size_t workspace_bytes, b200asr_stream stream);
B200ASR_API int b200asr_vgg_im2col(const float* feat, long long ld_b, int batches, int T, int Cin, int F, float* out,
                       b200asr_stream stream);
B200ASR_API int b200asr_vgg_pool_fwd(const float* y, int batches, int T, int F, int C, float* out, unsigned char* idx,
                         int flat, b200asr_stream stream);
B200ASR_API int b200asr_vgg_pool_bwd(const float* dout, const unsigned char* idx, const float* y, int batches, int T, int F,
                         int C, float* dy, int flat, b200asr_stream stream);
B200ASR_API int b200asr_vgg_feat_grad(const float* dy1, const float* w1, int batches, int T, int T_in, int Cin, int F, int O,
                          float* dfeat, b200asr_stream stream);

/* ---- f16x3: the BiLSTM layer contractions on scaled fp16 hi/lo images (input width a multiple of 4) ----------------
 * An operand X[outer][k] (k = the contraction index) becomes two K-major fp16 images hi, lo [outer][Kp],
 * Kp = b200asr_f16x3_padded_k(K) (K rounded up to the 128-k scale chunk, zero-filled), and inverse scales
 * sinv[Kp / 128][outer]: per (outer index, 128-k chunk) a power of two s brings the chunk maximum to [2^13, 2^14),
 * hi = f16(x s), lo = f16(x s - hi), sinv = 1 / s.  A chunk holding a NaN / Inf, or only zeros, gets s = 1.
 *   _split_rows: K-major x (element (row, k) at x[row * ld + k]; K, ld multiples of 4, 16-byte aligned).
 *   _split_cols: MN-major x, transposed: image row = column c, image column r = b T + t, element at
 *     x[b * bstride + (t + shift) * ld + c], zero where t + shift is outside [0, T) (h_prev of a direction).
 *   _split_dg: the gate gradient of a BiLSTM layer, g[ndir][rows][cols] (contiguous; cols a multiple of 4, 16-byte
 *     aligned), read once: per direction d the _split_cols operand of g[d] (t_hi / t_lo [ndir][cols][Rp], t_sinv
 *     [ndir][Rp / 128][cols], Rp = padded rows); if r_hi / r_lo / r_sinv are given (all or none), one _split_rows
 *     operand of all directions side by side (images [rows][ndir Kp], Kp = padded cols, direction d in columns
 *     [d Kp, (d + 1) Kp); r_sinv [ndir Kp / 128][rows]); and colsum[Rp / 128][ndir][cols], the column sums of each
 *     128-row tile.  Images and scales are bit-identical to the two single-image passes on the same data.
 *   b200asr_gemm_f16x3:  C[M,N] (+)= sum_k A[m][k] B[n][k] (+ bias[N]) over the two operands' images (same Kp):
 *     hi.hi + hi.lo + lo.hi per 16 k on the tensor cores, each 128-k chunk folded with its scales into an fp32
 *     register sum; ldc, accumulate, permute_rows (row m -> (m % 4) * (M / 4) + m / 4) and the split-K workspace
 *     (b200asr_gemm3x_workspace_bytes(M, N), may be NULL) as in b200asr_gemm3x_nt.                                 */
B200ASR_API int b200asr_f16x3_padded_k(int K);
B200ASR_API int b200asr_f16x3_split_rows(const float* x, long long ld, int rows, int K, void* hi, void* lo, float* sinv,
                             b200asr_stream stream);
B200ASR_API int b200asr_f16x3_split_cols(const float* x, long long ld, long long bstride, int shift, int T, int batches,
                             int cols, void* hi, void* lo, float* sinv, b200asr_stream stream);
B200ASR_API int b200asr_f16x3_split_dg(const float* g, int ndir, int rows, int cols, void* t_hi, void* t_lo, float* t_sinv,
                           void* r_hi, void* r_lo, float* r_sinv, float* colsum, b200asr_stream stream);
B200ASR_API int b200asr_gemm_f16x3(const void* a_hi, const void* a_lo, const float* a_sinv, const void* b_hi, const void* b_lo,
                       const float* b_sinv, const float* bias, float* C, int M, int N, int Kp, int ldc, int accumulate,
                       int permute_rows, void* workspace, size_t workspace_bytes, b200asr_stream stream);

/* ---- K6 helper: split fp32 into a TF32-representable high part and the fp32 residual ---------------------------
 * hi = x rounded to TF32, lo = x - hi; used to run the input-projection (src/module.py:131, inside nn.LSTM) and the
 * weight-gradient contractions as three error-compensated TF32 tensor-core GEMMs (3xTF32) at fp32-level accuracy.  */
B200ASR_API int b200asr_split_tf32(const float* x, float* hi, float* lo, long long n, b200asr_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* B200ASR_H */
