/* stablets_b200.h -- C ABI of the H100 (sm_90a) kernel library behind stable-ts's word-timestamp hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  stable-ts is pure Python: the arithmetic of this path lives in the
 * third-party `openai-whisper` package that stable_whisper/whisper_compatibility.py:58-76 imports.  Each entry point
 * below replaces one of those calls (or the tensor post-processing stable-ts itself does around them) and is what a
 * ctypes binding in the reference would load (see INTEGRATION.md for the stub).
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - no allocation inside: the caller (PyTorch) owns inputs, outputs and workspaces;
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*), nothing synchronises;
 *   - return value: STB_OK or an STB_ERR_* code; stb_last_error() gives the thread-local message;
 *   - "split" matrices are fp16 hi/lo plane pairs with hi + lo == fp32 value to ~2^-22; in STB_PREC_FP16 mode the
 *     lo plane pointer is NULL and only one tensor-core pass is issued.
 */
#ifndef STABLETS_B200_H
#define STABLETS_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(STB_BUILDING)
#define STB_API __attribute__((visibility("default")))
#else
#define STB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define STB_OK 0
#define STB_ERR_ARG 1
#define STB_ERR_CUDA 2
#define STB_ERR_UNSUPPORTED 3

#define STB_PREC_FP16 1   /* one fp16 tensor-core pass (what the reference's CUDA transcribe path computes in) */
#define STB_PREC_FP16X3 3 /* hi*hi + hi*lo + lo*hi: fp32-grade products, the parity mode (reference CPU path is fp32) */

#define STB_N_FRAMES 3000      /* mel frames per 30 s window (whisper_compatibility.py:87) */
#define STB_N_AUDIO_CTX 1500   /* encoder positions per window */
#define STB_KPAD 1504          /* 1500 rounded up to a multiple of 8: row pitch of score / probability matrices */

STB_API const char* stb_last_error(void);
STB_API int stb_abi_version(void);
/* measurement hooks (bench.py): kernels launched by this library so far; per-launch CUDA-event timing of every kernel */
STB_API unsigned long long stb_launch_count(void);
STB_API void stb_prof_enable(int on);
/* JSON {"kernel": {"n": launches, "ms": event-timed total, "bytes": algorithmic bytes, "flops": algorithmic FLOPs}} of the
 * launches since the previous report (synchronises the device). */
STB_API int stb_prof_report(char* buf, size_t buf_bytes);

/* ------------------------------------------------------------------------------------------------------------
 * a1  log-mel front-end.  Replaces whisper.audio.log_mel_spectrogram + pad_or_trim
 *     (call sites stable_whisper/alignment.py:411-413, :660-661; original_whisper.py:528-530).
 *     audio [B][n_samples] fp32; samples n_samples..padded_samples-1 are zeros (align: padded_samples = 480000;
 *     refine: padded_samples = n_samples).  Frames = padded_samples/160, frames beyond are written as 0.0 (pad_or_trim).
 *     batch_global_max != 0: the "max - 8" floor uses the max over the whole batch (alignment.py:660), else per item.
 *     mel_out [B][n_mels][3000] fp32.  dft_table [400][2] fp32 (cos,sin of 2*pi*j/400), window [400] fp32,
 *     filters [n_mels][201] fp32 are passed in by the host (computed once).  ws >= B*4 bytes.
 * ---------------------------------------------------------------------------------------------------------- */
STB_API int stb_logmel(const float* audio, int B, int n_samples, int padded_samples, int n_mels, const float* filters,
               const float* window, const float* dft_table, int batch_global_max, float* mel_out, void* ws,
               size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * GEMM core (K3): D[b,h] = epilogue(alpha * A[b,h] * B[b,h]^T), wgmma (fp16 inputs, fp32 accumulate in registers) fed
 * by TMA.  Both operands are K-major split-fp16 4-D views (batch b, head h, row, k); strides in ELEMENTS.
 * Exposed for tests; the model entry points below are sequences of these launches.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
    const void* hi;        /* fp16 plane */
    const void* lo;        /* fp16 plane or NULL (single pass) */
    int rows;              /* rows per (b,h) slice (M for A, N for B) */
    int k;                 /* reduction length (any; tiles beyond are zero-filled by TMA) */
    long long row_stride;  /* elements; may be smaller than k (overlapping rows: conv-as-GEMM) */
    long long h_stride;
    long long b_stride;
} stb_operand;

#define STB_ACT_NONE 0
#define STB_ACT_GELU 1

typedef struct {
    float* out_f32;        /* fp32 output or NULL */
    void* out_hi;          /* split fp16 output planes or NULL */
    void* out_lo;
    long long ld_out;      /* elements; normal: off = m*ld_out + n; transposed: off = n*ld_out + m */
    long long out_h_stride;
    long long out_b_stride;
    int transposed;
    const float* bias;     /* [N] (or [M] when bias_per_row) or NULL */
    int bias_per_row;
    const float* residual; /* fp32, added after the activation; may alias out_f32 */
    long long ld_res;
    long long res_h_stride;
    long long res_b_stride;
    float alpha;
    int act;
} stb_epilogue;

STB_API int stb_gemm(const stb_operand* A, const stb_operand* B, int n_batch, int n_head, const stb_epilogue* ep, void* stream);

/* Fused attention (K4): out[b][m][h*64 + c] = softmax(q k^T / 8) v with the scores and probabilities kept in registers
 * (wgmma, one pass over the keys with an online softmax).  q: rows Mq, k = 64; k: rows Mk, k = 64; vT: rows 64, k >= Mk
 * (zero padded keys).  Output split planes with offsets b*out_b_stride + h*out_h_stride + m*ld_out + c.  Non-causal: the
 * encoder's self-attention and the teacher-forced decoder's cross-attention. */
STB_API int stb_attention(const stb_operand* q, const stb_operand* k, const stb_operand* vT, int n_batch, int n_head, int Mq,
                  int Mk, void* out_hi, void* out_lo, long long ld_out, long long out_h_stride, long long out_b_stride,
                  void* stream);

/* Decode-step linear layer for B <= 64 sequences (batched GEMV, mma.sync + 4-CTA split-K cluster, csrc/gemv.cu):
 * out[b][n] = act(sum_k W[n][k] x[b][k] + bias[n]) + res[b][n].  x split planes [B][K] (row pitch K), W split planes
 * [N][K]; lo planes may be NULL (single pass).  K % 32 == 0.  Replaces torch.nn.functional.linear on the KV-cached decode
 * path (whisper/model.py Linear.forward under stable_whisper/decode.py:27-40). */
STB_API int stb_gemv(const void* x_hi, const void* x_lo, int B, int K, const void* w_hi, const void* w_lo, int N,
                     const float* bias, int act, const float* res, long long ld_res, float* out_f32, void* out_hi,
                     void* out_lo, long long ld_out, void* stream);

/* Decode-step linear layer for 17..128 sequences, the kernel the decode step runs for every Linear at those batch sizes
 * (swapped wgmma GEMM, split-K across a thread-block cluster reduced over distributed shared memory, fused epilogue,
 * csrc/decode_linear.cu).  Exposed for tests.
 *   out[b][n] = act(sum_k W[n][k] x[b][k] + bias[n]) + res[b][n] for b < B, n < N; nothing else of the outputs is written.
 *   x split planes [B][K] (row pitch K), W split planes [N][K]; lo planes for both or neither (single pass).  B in 1..128,
 *   K a multiple of 64.  Outputs: fp32 and/or split planes (out_lo may be NULL), row pitch ld_out >= N; res may alias
 *   out_f32 (row pitch ld_res >= N).  bias, res and out_f32 16-byte aligned; out_hi / out_lo 8-byte aligned.
 * stb_decode_linear_split: the cluster size (1..8) stb_decode_linear uses for an N x K weight on the current device, 0 for
 * a bad shape. */
STB_API int stb_decode_linear(const void* x_hi, const void* x_lo, int B, int K, const void* w_hi, const void* w_lo, int N,
                              const float* bias, int act, const float* res, long long ld_res, float* out_f32, void* out_hi,
                              void* out_lo, long long ld_out, void* stream);
STB_API int stb_decode_linear_split(int n, int k);

/* fp32 [rows][cols] (row pitch src_ld) -> split planes (row pitch dst_ld); lo may be NULL */
STB_API int stb_split_f16(const float* src, long long rows, int cols, long long src_ld, void* hi, void* lo, long long dst_ld,
                  void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Model handle: dims + table of caller-owned device weight pointers (already packed, see stable-ts_b200/model.py).
 * Replaces whisper.model.Whisper (encoder / decoder / cross-attention QK capture), reference call sites
 * stable_whisper/timing.py:50-61, decode.py:27-40, alignment.py:660-667.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
    int n_mels, n_audio_ctx, n_audio_state, n_audio_head, n_audio_layer;
    int n_vocab, n_text_ctx, n_text_state, n_text_head, n_text_layer;
} stb_dims;

typedef struct stb_model stb_model;

/* tensor ids for stb_model_set_tensor; `layer` is ignored for the non-layer tensors */
enum {
    STB_T_ENC_CONV1_W = 0, /* split [d][3*n_mels], k index = tap*n_mels + c_in */
    STB_T_ENC_CONV1_B,     /* f32 [d] */
    STB_T_ENC_CONV2_W,     /* split [d][3*d], k index = tap*d + c_in */
    STB_T_ENC_CONV2_B,
    STB_T_ENC_POS,         /* f32 [1500][d] */
    STB_T_ENC_LNPOST_G,
    STB_T_ENC_LNPOST_B,
    STB_T_DEC_TOKEMB_F32,  /* f32 [V][d] (embedding gather) */
    STB_T_DEC_TOKEMB,      /* split [V][d] (logits GEMM) */
    STB_T_DEC_POS,         /* f32 [n_text_ctx][d] */
    STB_T_DEC_LN_G,
    STB_T_DEC_LN_B,
    STB_T_LAYER_BASE = 32,
    /* per-layer ids (add to STB_T_LAYER_BASE); encoder layers use ENC_*, decoder layers DEC_* */
    STB_L_ATTN_LN_G = 0, STB_L_ATTN_LN_B, STB_L_QKV_W /* split [3d][d]: q,k,v */, STB_L_QKV_B /* f32 [3d], k part 0 */,
    STB_L_OUT_W, STB_L_OUT_B, STB_L_MLP_LN_G, STB_L_MLP_LN_B, STB_L_FC1_W, STB_L_FC1_B, STB_L_FC2_W, STB_L_FC2_B,
    STB_L_CROSS_LN_G, STB_L_CROSS_LN_B, STB_L_CQ_W, STB_L_CQ_B, STB_L_CKV_W /* split [2d][d]: k,v */,
    STB_L_CKV_B /* f32 [2d], k part 0 */, STB_L_COUT_W, STB_L_COUT_B,
    STB_L_COUNT
};

STB_API int stb_model_create(const stb_dims* dims, int precision, stb_model** out);
STB_API void stb_model_destroy(stb_model* m);
/* is_decoder: 0 encoder layer table, 1 decoder layer table (only for ids >= STB_T_LAYER_BASE) */
STB_API int stb_model_set_tensor(stb_model* m, int tensor_id, int is_decoder, int layer, const void* p_hi_or_f32, const void* p_lo);

/* a2 encoder: mel [B][n_mels][3000] fp32 -> xa_f32 [B][1500][d] (+ split planes for the cross K/V GEMMs). */
STB_API size_t stb_encoder_ws_bytes(const stb_model* m, int B);
STB_API int stb_encoder_forward(stb_model* m, const float* mel, int B, float* xa_f32, void* xa_hi, void* xa_lo, void* ws,
                        size_t ws_bytes, void* stream);

/* cross-attention K (head-major) and V^T of every decoder layer, computed once per window (whisper's kv_cache for
 * cross_attn).  decode_layout != 0 additionally writes the head-major copy of V that stb_decode_step streams. */
STB_API size_t stb_cross_kv_bytes(const stb_model* m, int B);
STB_API int stb_cross_kv(stb_model* m, const void* xa_hi, const void* xa_lo, int B, int decode_layout, void* cross_kv, void* stream);

/* a3 teacher-forced decoder with cross-attention capture (stable_whisper/timing.py:50-61 under disable_sdpa).
 *   tokens [B][M] int32.  logits (nullable) [B*M][ld_logits] fp32.
 *   qk_out (nullable) fp32 [B][n_sel][M][STB_KPAD]: scaled PRE-softmax cross-attention scores of the selected
 *   (layer, head) pairs sel_pairs_host[2*n_sel] (host array); n_sel < 0 selects all L*H heads in (layer, head) order.
 *   Columns 1500..STB_KPAD-1 of each qk_out row are not written.
 *   The logits do not depend on qk_out, sel_pairs_host or n_sel: a pass computes them the same way whatever it captures. */
STB_API size_t stb_decoder_ws_bytes(const stb_model* m, int B, int M);
STB_API int stb_decoder_forward(stb_model* m, const int32_t* tokens, int B, int M, const void* cross_kv, float* logits,
                        long long ld_logits, float* qk_out, const int32_t* sel_pairs_host, int n_sel, void* ws,
                        size_t ws_bytes, void* stream);

/* a4 / a10 token probabilities (stable_whisper/timing.py:62-64, alignment.py:669-671, refinement.py:305-325):
 *   per row r: p = softmax(logits[row0 + r][:n_classes])[target[r]]; rank_out (nullable) = number of classes with
 *   probability strictly smaller than the target's (== index of the target in the ascending sort, ties aside). */
STB_API int stb_token_probs(const float* logits, long long ld, int n_rows, int n_classes, const int32_t* targets, float* prob_out,
                    int32_t* rank_out, void* stream);

/* a10, 3-D form of the refine plugin (stable_whisper/alignment.py:669-671 returns softmax(logits[:, S:S+N, :eot]); the
 *   unmodified Refiner derives the target's rank from it, non_whisper/refinement.py:305-325):
 *   out[r][0..n_classes) = softmax(logits[r][:n_classes]), fp32, row pitch ld_out. */
STB_API int stb_softmax_probs(const float* logits, long long ld, int n_rows, int n_classes, float* out, long long ld_out,
                      void* stream);

/* a5 QK post-processing, legacy alignment-head path (stable_whisper/timing.py:105-110,194):
 *   qk [B][A][M][ldq] fp32 (as written by stb_decoder_forward; M = rows per head in memory); rows S..S+R-1
 *   (the reference slices [S:-1], i.e. R = n_text_tokens + 1; smaller R lets windows with fewer tokens share a padded
 *   decoder batch), columns [0,F) ->
 *   softmax(qk*qk_scale) over columns -> z-norm over the R rows of each column (biased std) -> median filter
 *   (width, reflect) along columns -> mean over the A heads -> matrix [B][R][ldm] fp32.
 *   ws >= stb_qkpost_ws_bytes. */
STB_API size_t stb_qkpost_ws_bytes(int B, int A, int R, int F);
STB_API int stb_qk_postprocess(const float* qk, int B, int A, int M, long long ldq, int S, int R, int F, float qk_scale,
                       int medfilt_width, float* matrix, long long ldm, void* ws, size_t ws_bytes, void* stream);

/* a5 variants, both over the scores of ALL L*H heads (qk [B][LH][M][ldq], stb_decoder_forward with n_sel < 0):
 *  - dynamic heads (stable_whisper/timing.py:85-103): softmax -> per token row, the `count` heads with the smallest
 *    distance-weighted mass around the row's peak (argmax on the first call; midpoint of the previous jump interval
 *    when prev_jumps [B][R] is given) -> z-norm -> median -> mean.  reuse_softmax != 0 keeps the softmaxed scores left in
 *    `ws` by the previous call (the reference caches them across dynamic iterations, timing.py:89-92).
 *  - "new" aligner (stable_whisper/timing.py:115-163, arXiv 2509.09987): median filter on the raw scores of every row,
 *    softmax, head score = w_colnorm * sum_f ||W[:,f]|| + w_rownorm * sum_m ||W[m,:]|| - w_coverage * penalty, top-k
 *    heads, column-normalised mean, rows S..S+R-1. */
STB_API size_t stb_qkpost_dynamic_ws_bytes(int B, int LH, int R, int F, int count);
STB_API int stb_qk_postprocess_dynamic(const float* qk, int B, int LH, int M, long long ldq, int S, int R, int F, float qk_scale,
                               int medfilt_width, int count, const int32_t* prev_jumps, int reuse_softmax, float* matrix,
                               long long ldm, void* ws, size_t ws_bytes, void* stream);
STB_API size_t stb_qkpost_new_ws_bytes(int B, int LH, int M, int F, int topk);
STB_API int stb_qk_postprocess_new(const float* qk, int B, int LH, int M, long long ldq, int S, int R, int F, float qk_scale,
                           int medfilt_width, int topk, float w_colnorm, float w_rownorm, float w_coverage, float* matrix,
                           long long ldm, void* ws, size_t ws_bytes, void* stream);

/* y[i] = a * x[i] + b * y[i]: combines the head-averaged attention matrices of several models before the DTW
 * (`extra_models`, stable_whisper/timing.py:177-189: the per-model weights are concatenated over heads and averaged). */
STB_API int stb_axpby(float* y, const float* x, float a, float b, long long n, void* stream);

/* a6 DTW + jump extraction (whisper.timing.dtw CPU semantics + stable_whisper/timing.py:195-198):
 *   x [B][R][ldx] fp32 (cost = -x when negate != 0), path over the R x F grid, strict-'<' tie rule, fp32 cost.
 *   jumps [B][R] int32 = first frame of every row on the path (clipped at 0).
 *   path (nullable) [B][2][R+F] int32 = (text_idx, time_idx) in forward order, path_len [B]. */
STB_API size_t stb_dtw_smem_bytes(int R, int F);
STB_API size_t stb_dtw_ws_bytes(int B, int R, int F);   /* transposed + skewed copy of the cost matrix */
STB_API int stb_dtw(const float* x, int B, int R, int F, long long ldx, int negate, int32_t* jumps, int32_t* path,
            int32_t* path_len, void* ws, size_t ws_bytes, void* stream);

/* Section 8(f) row 1 -- non-VAD silence detection, device part (stable_whisper/stabilization/nonvad.py:16-41 audio2loudness,
 *    :58-76 of wav2mask: moving average, quantisation, -> bool).  Per window of a batch [B][stride] of 16 kHz fp32 samples:
 *    threshold = k-th largest |x| (k = int(n * 0.001), computed by the caller), loudness [token_count] = linear
 *    down-sampling of |x| / min(1, 1.75 threshold) (token_count = round(n / 320) + 1, computed by the caller), mask =
 *    round(avg_pool(loudness, k_size, reflect) * q_levels) != 0  (1 = sound).  Outputs have a row pitch of 1501.
 *    thr_in (nullable): per-window thresholds supplied by the caller instead of the k-th largest (the reference's
 *    quantile branch for windows shorter than 1000 samples).  loudness_out / thr_out may be NULL.
 *    The run-length logic of wav2mask (:76-88) stays with the caller (stable-ts_b200/silence.py). */
STB_API int stb_silence_mask(const float* audio, int B, int n_samples, long long stride, int k, int token_count, int q_levels,
                             int k_size, const float* thr_in, float* loudness_out, uint8_t* mask_out, float* thr_out,
                             void* stream);

/* Section 8(f) row 3 -- audio ingest (replaces the ffmpeg pipe of stable_whisper/audio/utils.py:96-125 for PCM/WAV input):
 *    interleaved PCM [n_frames_in][channels] (sample_format 0 = s16, 1 = s32, 2 = f32) -> mono fp32 at rate * L / M:
 *    equal-weight down-mix, polyphase FIR y[m] = sum_j table[(m M) mod L][j] * x[(m M) div L - taps/2 + j] (zero outside the
 *    input), table [L][taps] fp32 built by the caller (stable-ts_b200/audio_io.py: Kaiser-windowed sinc, DC gain 1), taps odd.
 *    quantize_s16 != 0 rounds the result to the int16 grid, as the reference's `-f s16le` pipe does. */
STB_API int stb_resample_mono(const void* pcm, int sample_format, int channels, long long n_frames_in, int L, int M,
                      const float* table, int taps, float* out, long long n_out, int quantize_s16, void* stream);

/* a9 KV-cached decode (stable_whisper/decode.py:33-65; whisper PyTorchInference.logits + logit filters +
 *    GreedyDecoder.update).  One step = one decoder forward for the newest token of B sequences.
 *    Everything position-dependent is read from the DEVICE counter `pos` (index of the token being fed), which the step
 *    increments at its end, so a single captured CUDA graph can replay every step.
 *    state: self-attention K/V caches fp32 [L][2][B][n_text_ctx][d] (stb_decode_state_bytes).
 *    tokens_in [B] int32 -> logits_out [B][ld_logits] fp32. */
STB_API size_t stb_decode_state_bytes(const stb_model* m, int B);
STB_API size_t stb_decode_ws_bytes(const stb_model* m, int B);
STB_API int stb_decode_step(stb_model* m, const int32_t* tokens_in, int B, int32_t* pos, const void* cross_kv, void* state,
                    float* logits_out, long long ld_logits, void* ws, size_t ws_bytes, void* stream);
/* The same step for a batch whose INITIAL tokens differ in length (per-window prompts: `decode_options["prompt"] =
 *    all_tokens[prompt_reset_since:]`, original_whisper.py:533; whisper DecodingTask._get_initial_tokens).  The sequences are
 *    RIGHT-aligned on the shared counter: sequence b's first token is fed at pos == seq_off[b] (= longest - own length), its own
 *    position (positional embedding row) is pos - seq_off[b], and its self-attention reads cache rows [seq_off[b], pos] only, so
 *    every sequence samples its first token at the same step.  Steps with pos < seq_off[b] are idle for b (any token id).
 *    cache_rows: rows per sequence of the K/V caches, n_text_ctx <= cache_rows <= 2 n_text_ctx (stb_decode_state_bytes_rows).
 *    cross_kv: the block stb_cross_kv built for exactly these B windows (decode layout), sequence b reading window b.
 *    seq_off == NULL and cache_rows == n_text_ctx is stb_decode_step. */
STB_API size_t stb_decode_state_bytes_rows(const stb_model* m, int B, int cache_rows);
STB_API int stb_decode_step_ragged(stb_model* m, const int32_t* tokens_in, int B, int32_t* pos, const int32_t* seq_off,
                           int cache_rows, const void* cross_kv, void* state, float* logits_out, long long ld_logits,
                           void* ws, size_t ws_bytes, void* stream);

/* The two attention kernels of the decode step on their own, exposed for tests (csrc/decode.cu).  d = 64 H; B and H in
 *    1..65535.  Outputs: out_f32 fp32 [B][d] and/or split planes out_hi / out_lo fp16 [B][d] (hi = rn(o), lo = rn(o - hi);
 *    out_lo needs out_hi); at least one of out_f32 / out_hi.
 * stb_decode_self_attn: one head-sliced attention of the newest token over the fp32 self-attention K/V cache.
 *    qkv fp32 [B][3d] (q | k | v of the newest token); k_cache, v_cache fp32 [B][cache_rows][d]; pos a DEVICE int32 counter;
 *    seq_off (nullable) a device int32 [B] of first cache rows (NULL: 0).  The kernel writes the k / v slices of qkv into
 *    cache row `pos` and writes nothing else of the caches; sequence b then attends rows [min(seq_off[b], pos), pos] with
 *    weights softmax(q . K[j] / 8), and never reads any other row.  pos < cache_rows is the caller's duty (the host cannot
 *    read the counter).  qkv and the caches 16-byte aligned.
 * stb_decode_cross_attn: attention of one query per sequence over the window's 1500 cross K / V rows.
 *    q fp32 [B][d]; k_hi, v_hi fp16 head-major [B][H][1500][64] (16-byte aligned: TMA sources), the layout
 *    stb_cross_kv(..., decode_layout = 1) writes.  partial: scratch of B H stb_decode_cross_splits() 66 floats.
 *    tickets: B H int32 that must be zero before the first call; every call leaves them zero again, so one pair of
 *    partial / tickets serves any number of calls on one stream. */
STB_API int stb_decode_self_attn(const float* qkv, float* k_cache, float* v_cache, int B, int H, int cache_rows, const int32_t* pos,
                                 const int32_t* seq_off, float* out_f32, void* out_hi, void* out_lo, void* stream);
STB_API int stb_decode_cross_attn(const float* q, const void* k_hi, const void* v_hi, int B, int H, float* partial, int32_t* tickets,
                                  float* out_f32, void* out_hi, void* out_lo, void* stream);
STB_API int stb_decode_cross_splits(void);

/* The LayerNorm and softmax row kernels of the encoder and the teacher-forced decoder on their own, exposed for tests
 *    (csrc/elementwise.cu).  Split planes are hi = rn(y), lo = rn(y - hi) of the fp32 result y.
 * stb_layernorm: whisper's LayerNorm of rows x fp32 [rows][d] (row pitch d): statistics in fp32, biased variance, eps 1e-5,
 *    y = (x - mean) / sqrt(var + 1e-5) gamma + beta.  d a multiple of 128 in 128..1280, rows >= 0.  Outputs (row pitch d):
 *    out_f32 fp32 and / or the split planes out_hi / out_lo fp16 (out_lo needs out_hi); at least one of out_f32 / out_hi.
 *    Nothing beyond row `rows` is written.  x, gamma, beta and out_f32 16-byte aligned; out_hi / out_lo 8-byte aligned.
 * stb_softmax_rows: softmax of attention-score rows S fp32 [n_rows][ld_s] into split planes p_hi / p_lo fp16 [n_rows][ld_p]
 *    (p_lo may be NULL).  Row r covers its first n_valid(r) columns: min(n_cols, r % rows_per_slice + 1) when causal (the
 *    decoder's mask over slices of rows_per_slice query rows), n_cols otherwise; columns n_valid(r)..ld_p-1 are written as
 *    0 and nothing at or beyond ld_p is.  Only columns below n_valid(r) of S are read.  1 <= n_cols <= 1504,
 *    ld_s >= n_cols, n_cols <= ld_p <= 1504; rows_per_slice >= 1 when causal. */
STB_API int stb_layernorm(const float* x, long long rows, int d, const float* gamma, const float* beta, void* out_hi, void* out_lo,
                          float* out_f32, void* stream);
STB_API int stb_softmax_rows(const float* S, long long n_rows, int n_cols, long long ld_s, int rows_per_slice, int causal,
                             void* p_hi, void* p_lo, long long ld_p, void* stream);

/* per-sequence sampling state kept on the device */
typedef struct {
    int32_t n_sampled;   /* tokens sampled so far (0 at sample_begin) */
    int32_t last_tok;    /* newest sampled token */
    int32_t prev_tok;    /* the one before */
    int32_t last_ts;     /* most recent timestamp token sampled, or -1 */
    int32_t done;        /* newest token is EOT */
    float sum_logprob;   /* GreedyDecoder.sum_logprobs */
} stb_seq_state;

/* Logit filters + greedy pick for one step, in place on logits [B][ld] (decode.py:46-58 + whisper.decoding filters):
 *   suppress_mask [V] uint8 (SuppressTokens), first_step_mask [V] uint8 applied when n_sampled == 0 (SuppressBlank),
 *   ApplyTimestampRules from the per-sequence state (apply_ts_rules, no_timestamps id, max_initial_ts index or -1),
 *   ts_mask (nullable) uint8 silent-timestamp mask: [1501] shared by the batch (ts_mask_stride = 0) or one row per
 *   sequence [B][ts_mask_stride] (the reference computes one per window, original_whisper.py:504-511), NaN -> -inf, argmax (first max index), log-softmax gather,
 *   sum_logprob += logprob unless the sequence already ended, ended sequences keep emitting EOT.
 *   Step tables (nullable, [table_rows][B] int32, row = n_sampled so no per-step host traffic is needed):
 *   forced_table: token appended instead of the argmax (fixed-length benchmark scripts / teacher forcing);
 *   token_table: the appended token; argmax_table: the argmax before forcing.  next_out [B] feeds stb_decode_step. */
STB_API int stb_sample_greedy(float* logits, long long ld, int B, int V, int eot, int ts_begin, int no_timestamps,
                      const uint8_t* suppress_mask, const uint8_t* first_step_mask, const uint8_t* ts_mask,
                      long long ts_mask_stride, int max_initial_ts, int apply_ts_rules, const int32_t* forced_table, stb_seq_state* states,
                      int32_t* next_out, int32_t* token_table, int32_t* argmax_table, int table_rows, void* stream);
/* stb_sample_greedy plus the temperature > 0 branch of whisper's GreedyDecoder.update (`Categorical(logits=logits /
 *   temperature).sample()`, used by the temperature fallback of original_whisper.py:349-393):
 *   temperature > 0: the token is drawn by inverse CDF from p_i ~ exp((l_i - max) / temperature) over the FILTERED logits -- the
 *   first index whose running sum (index order) exceeds uniform_table[n_sampled][b] * total; uniform_table [table_rows][B] fp32
 *   in [0, 1) is the caller's random stream (torch.rand under the caller's generator: the draw is a pure function of it).
 *   sum_logprob accumulates log_softmax(unscaled logits)[drawn token], as the reference does.  temperature == 0: the argmax.
 *   sample_cap (nullable) [B]: a sequence that has sampled sample_cap[b] tokens is treated as ended (EOT from then on, no
 *   log-prob) -- the per-sequence form of the reference's `tokens.shape[-1] > n_ctx` stop when initial tokens are ragged. */
STB_API int stb_sample(float* logits, long long ld, int B, int V, int eot, int ts_begin, int no_timestamps,
               const uint8_t* suppress_mask, const uint8_t* first_step_mask, const uint8_t* ts_mask, long long ts_mask_stride,
               int max_initial_ts, int apply_ts_rules, const int32_t* forced_table, stb_seq_state* states, int32_t* next_out,
               int32_t* token_table, int32_t* argmax_table, int table_rows, float temperature, const float* uniform_table,
               const int32_t* sample_cap, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STABLETS_B200_H */
