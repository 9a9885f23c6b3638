/* sbk.h -- C ABI of libsbk.so: the H100-native (sm_90a) ASR inference hot path behind SpeechBrain's
 * module API.  Plain C: raw pointers + sizes, int error codes (0 = ok, <0 = error; text via
 * sbk_last_error()), an opaque CUDA stream (cudaStream_t passed as void*).  No torch types.
 *
 * The reference (speechbrain v1.1.0) has no FFI for this path -- its seam is nn.Module call
 * signatures (SURVEY.md 8b).  Each entry point below names the reference call it replaces
 * (file:line relative to /root/reference/speechbrain/).  Device pointers are caller-owned
 * (torch tensors); the library owns only repacked weights and its workspace.
 */
#ifndef SBK_H_
#define SBK_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sbk_fbank sbk_fbank; /* opaque */
typedef struct sbk_asr sbk_asr;     /* opaque */

enum { SBK_ATT_ROPE = 0, SBK_ATT_RELPOS = 1 };
enum { SBK_ACT_RELU = 0, SBK_ACT_GELU = 1 };
enum { SBK_PART_FBANK = 1, SBK_PART_CNN = 2, SBK_PART_ENCODER = 4, SBK_PART_DECODER = 8, SBK_PART_ALL = 15, SBK_PART_LM = 16 };

typedef struct {
    const char* name;  /* reference state_dict key with recipe prefix, e.g. "Transformer.encoder.layers.0.norm1.norm.weight" */
    const float* data; /* HOST fp32, contiguous, reference layout */
    int64_t numel;
} sbk_tensor;

typedef struct {
    /* Fbank (lobes/features.py:98-145) -- sizes in samples */
    int n_fft, hop, n_mels;
    /* ConvolutionFrontEnd (lobes/models/convolution.py:162-203): 2 blocks, 3x3, stride 2 */
    int cnn_c1, cnn_c2;
    /* TransformerASR (lobes/models/transformer/TransformerASR.py:247-325) */
    int input_size, d_model, nhead, num_encoder_layers, num_decoder_layers, d_ffn, vocab, kernel_size;
    int attention_type;     /* SBK_ATT_ROPE (RoPEMHA) | SBK_ATT_RELPOS (RelPosMHAXL) */
    int decoder_activation; /* SBK_ACT_RELU | SBK_ACT_GELU (the `activation` ctor kwarg) */
    int max_len;            /* positional tables (ctor kwarg max_length, default 2500) */
    int parts;              /* bitmask of SBK_PART_*: which sub-models the weight table carries */
    /* TransformerLM used as a shallow-fusion scorer (lobes/models/transformer/TransformerLM.py; weights "lm.*") */
    int lm_d_model, lm_nhead, lm_layers, lm_d_ffn, lm_activation;
    /* Filterbank amin / top_db (processing/features.py:437-475) and InputNormalization epsilon (:1360-1455) of the fused
       wav -> features front end; 0 = the reference defaults (1e-10, 80 dB, 1e-10) */
    float fbank_amin, fbank_top_db, norm_eps;
} sbk_asr_config;

typedef struct {
    /* S2SBeamSearcher kwargs (decoders/seq2seq.py:752-804); steps are absolute: int(T * ratio) */
    int beam_size, max_steps, min_steps, bos, eos;
    float temperature;
    int using_eos_threshold;
    float eos_threshold;
    int length_normalization;
    float minus_inf;
    /* ScorerBuilder(full_scorers=[TransformerLMScorer]) (decoders/scorer.py:455-560,1221-1268): 0 weight = no scorer */
    float lm_weight, lm_temperature;
    /* ... and CTCScorer (decoders/scorer.py:183-249, decoders/ctc.py:46-295) as a full scorer; needs "ctc_lin.w.*" weights.
       ctc_weight != 0 also scales the decoder log-probs by 1 - ctc_weight (seq2seq.py:791-804,916-921). */
    float ctc_weight;
    int blank_index;
    /* LengthScorer (decoders/scorer.py:956-1072): this constant is added to every token's log-prob at every step */
    float length_weight;
    /* CoverageScorer (decoders/scorer.py:788-955) on the last decoder layer's head-averaged cross-attention:
       score = -(sum_t max(coverage_t, threshold) - T * threshold) / time_step, weighted; 0 weight = off */
    float coverage_weight, coverage_threshold;
} sbk_beam_params;

const char* sbk_last_error(void); /* thread-local message of the last failing call */
int sbk_version(void);
long long sbk_launch_count(void); /* kernels launched by this library so far (graph replays included) */
/* live per-launch timing of the wgmma GEMMs (CUDA events on the launching stream); read after a sync */
void sbk_gemm_profile_enable(int on);
int sbk_gemm_profile_read(int* n_launches, double* total_ms, double* total_flops);

/* ---- Fbank.forward (lobes/features.py:147-169 = STFT processing/features.py:141-188 + spectral_magnitude
 *      :341-378 + Filterbank.forward :512-586 + _amplitude_to_DB :736-759).  window_host[n_fft] is the (centre-
 *      padded) analysis window and mel_matrix_host[(n_fft/2+1) * n_mels] the dense triangular matrix, both
 *      computed by the caller exactly as the reference does (torch ops), so filter values are bit-identical. */
int sbk_fbank_create(int n_fft, int hop, int n_mels, const float* window_host, const float* mel_matrix_host,
                     float amin, float top_db, sbk_fbank** out);
void sbk_fbank_destroy(sbk_fbank* fb);
int sbk_fbank_num_frames(const sbk_fbank* fb, int n_samples);
/* wav_dev [B, L] fp32 -> out_dev [B, 1 + L/hop, n_mels] fp32; utt_max_scratch_dev: B ints */
int sbk_fbank_forward(const sbk_fbank* fb, const float* wav_dev, int B, int L, float* out_dev,
                      int* utt_max_scratch_dev, void* stream);

/* ---- InputNormalization.forward, eval mode (processing/features.py:1404-1455) */
int sbk_input_norm_global(const float* x_dev, float* out_dev, int B, int T, int F, const float* mean_dev,
                          const float* std_dev, float eps, void* stream);
int sbk_input_norm_sentence(const float* x_dev, float* out_dev, const float* rel_len_dev, int B, int T, int F,
                            int std_norm, int avoid_padding_norm, float eps, void* stream);

/* ---- wgmma GEMM self-test hook: out[M,N] = act(A[M,K] W[N,K]^T + bias) (fp16 in, fp32 accumulate) */
int sbk_gemm_f16_test(const void* A_dev, const void* W_dev, const float* bias_dev, void* out_dev, int out_is_f32,
                      int act, int M, int N, int K, void* stream);
/* same kernel, residual epilogue (every Linear that closes a Conformer sub-block): x[M,N] += alpha * (A W^T + bias), fp32 in place */
int sbk_gemm_f16_resid_test(const void* A_dev, const void* W_dev, const float* bias_dev, float* x_dev, float alpha,
                            int M, int N, int K, void* stream);
/* any fused epilogue of the encoder GEMMs: mode 0 fp16 (act 0 none, 1 SiLU, 2 GELU; kv_heads > 0: cross-attention K/V
 * scatter to [layer][K|V][utt][head][t][64] with the given element strides), 1 fp32, 2 residual (out = resid + alpha *
 * (acc + bias), rows t >= row_lens[utt] get alpha 0; out may alias resid), 3 GLU (fp32 [M, N / 2]; weight rows
 * interleaved [16 values | 16 gates] per 32), 4 RoPE (columns per head [q | k | v], q scaled by alpha; tables [T, dh / 2]) */
int sbk_gemm_epilogue_test(const void* A_dev, const void* W_dev, const float* bias_dev, void* out_dev, int ldo, int mode,
                           int act, float alpha, const float* resid_dev, const int* row_lens_dev, int T,
                           const float* rope_cos_dev, const float* rope_sin_dev, int head_dim, int kv_heads,
                           long long kv_part_stride, long long kv_layer_stride, int M, int N, int K, void* stream);
/* the CTC prefix scorer alone (CTCPrefixScore.forward_step + permute_mem, decoders/ctc.py:80-295), driven by a forced search
 * history in the order the beam search runs it: reset, then per step s the state update of the survivors of step s - 1 and
 * the full-vocabulary score.  logits_dev [B, T, V] fp32 ctc_lin output before log_softmax (copied, not modified);
 * enc_len_dev [B] in [0, T]; hist_tok_dev / hist_pred_dev [n_steps, B * beam]: the token and GLOBAL parent row of every
 * hypothesis after step s (the last row is not read).  scores_dev [n_steps, B * beam, V]: step s writes
 * weight * (psi - psi_prev) for every extension of the prefixes given by history rows < s (accumulate != 0: added to what
 * scores_dev holds).  group_width (may be NULL) receives the hypotheses per score CTA.  Allocates and frees its own
 * buffers and synchronises the stream. */
int sbk_ctc_prefix_test(const float* logits_dev, const int* enc_len_dev, int B, int T, int V, int beam, int blank, int bos,
                        int eos, float weight, int accumulate, const int* hist_tok_dev, const int* hist_pred_dev, int n_steps,
                        float* scores_dev, int* group_width, void* stream);

/* ---- model handle: repacks the reference state_dict once */
int sbk_asr_create(const sbk_asr_config* cfg, const sbk_tensor* weights, int n_weights, sbk_asr** out);
void sbk_asr_destroy(sbk_asr* m);
/* A clone shares the repacked weights and owns its own workspace: one clone ("lane") per batch in flight. */
int sbk_asr_clone(sbk_asr* src, sbk_asr** out);
/* DynChunkTrainConfig(chunk_size, left_context_size) for the following encode calls (TransformerASR.encode(...,
 * dynchunktrain_config=...), TransformerASR.py:46-105,475-544; Conformer.py:190-313): chunked attention (a frame sees its own
 * chunk and `left_context_chunks` chunks before it; < 0 = the whole past) and the Dynamic Chunk Convolution.  chunk_size 0
 * (default) = full-context. */
int sbk_asr_set_dynchunk(sbk_asr* m, int chunk_size, int left_context_chunks);
/* Greedy early-exit (`has_ended.all()`, decoders/seq2seq.py:256) is polled every n steps with a stream sync;
 * 0 = never poll: run exactly max_steps and never block the host (fully asynchronous enqueue). Default 8. */
int sbk_asr_set_poll_interval(sbk_asr* m, int every_n_steps);
/* Decoder pre-norms: 1 (default) = fused into the consuming projection kernel (best single-batch latency);
 * 0 = separate LayerNorm kernel (less total GPU time when several batches are in flight). Same numerics. */
int sbk_asr_set_decoder_ln_fusion(sbk_asr* m, int on);
/* Decode steps with at least `rows` live hypotheses (several batches decoded together, wide beams) run their projections
 * on the wgmma GEMM instead of the weight-streaming kernel (default 64; a huge value = never, 1 = always). */
int sbk_asr_set_decoder_tc_min_rows(sbk_asr* m, int rows);
/* TransformerLMRescorer.rescore_hyps (decoders/scorer.py:1835-1882), device part: tokens_dev [n, L] int32 rows
 * "bos ... eos pad pad", lens_dev [n] int32 (tokens incl. bos/eos) -> scores_dev [n] fp32 = sum of log p(token | prefix) at
 * `temperature` with the pad column excluded from the normalisation.  Needs a handle created with SBK_PART_LM. */
int sbk_asr_lm_rescore(sbk_asr* m, const int* tokens_dev, const int* lens_dev, int n, int L, float temperature, int pad_index,
                       float* scores_dev, void* stream);
/* TransformerLM.forward(src) (lobes/models/transformer/TransformerLM.py:127-169), whole sequences at once: tokens_dev [n, s]
 * int32 ids in [0, vocab), 0 = padding (make_masks' key-padding mask; pad positions still get logits, computed like the
 * reference's) -> logits_dev [n, s, vocab] fp32, written directly.  Causal self-attention with the look-ahead and key-padding
 * masks; every layer runs on all n * s rows at once.  Needs a handle created with SBK_PART_LM, s <= max_len and
 * n <= 65535; the call grows a workspace of its own (14 * d_model + 2 * d_ffn bytes per token row) on first use.  Ids are
 * not checked on the host (that would need a synchronise): an id outside [0, vocab) is never used as a table index, it
 * turns its sequence's logits into NaN (other sequences are unaffected).  Enqueue only. */
int sbk_asr_lm_forward(sbk_asr* m, const int* tokens_dev, int n, int s, float* logits_dev, void* stream);
/* The same logits from the KV-cached TransformerLM step that the beam search's scorer and the rescorer run: position by
 * position, teacher-forced, keys with id 0 masked through the token cache.  tokens_dev [n, L] int32 in [0, vocab) ->
 * logits_dev [n, L, vocab] fp32.  L dependent steps: for checking sbk_asr_lm_forward against the step path, not a fast
 * way to get logits.  Needs SBK_PART_LM and L <= max_len. */
int sbk_asr_lm_step_logits(sbk_asr* m, const int* tokens_dev, int n, int L, float* logits_dev, void* stream);
int sbk_asr_num_frames(const sbk_asr* m, int n_samples, int* T_feat, int* T_enc);

/* ConvolutionFrontEnd.forward (lobes/models/convolution.py:116-320): feats [B,T0,n_mels] -> out [B,T2,F2*C2] fp32 */
int sbk_asr_cnn_forward(sbk_asr* m, const float* feats_dev, int B, int T0, float* out_dev, void* stream);
/* TransformerASR.encode (TransformerASR.py:475-544): src [B,T,input_size] fp32 -> enc_out [B,T,d_model] fp32.
 * rel_len_dev: relative lengths (wav_len) or NULL. */
int sbk_asr_encode_from_cnn(sbk_asr* m, const float* src_dev, const float* rel_len_dev, int B, int T,
                            float* enc_out_dev, void* stream);
/* normalised feats [B,T0,n_mels] -> CNN -> encode in one call (inference/ASR.py:100-128 encode_batch, minus Fbank) */
int sbk_asr_encode_feats(sbk_asr* m, const float* feats_dev, const float* rel_len_dev, int B, int T0,
                         float* cnn_out_dev, float* enc_out_dev, void* stream);
/* S2STransformerGreedySearcher.forward (decoders/seq2seq.py:181-276,360-367), KV-cached.
 * pred_dev/score_dev [B, max_steps]; log_probs_dev [B, max_steps, vocab] or NULL; *steps_done = executed steps. */
int sbk_asr_greedy_from_enc(sbk_asr* m, const float* enc_dev, const float* rel_len_dev, int B, int T, int max_steps,
                            int bos, int eos, int* pred_dev, float* score_dev, float* log_probs_dev, int* steps_done,
                            void* stream);
/* torch.max(x, dim=-1).indices of a [rows, V] fp32 device matrix (ctc_greedy_decode, decoders/ctc.py:375) */
int sbk_rows_argmax_f32(const float* x_dev, int rows, int V, int* idx_dev, void* stream);
/* CTC head of an encoder-only recogniser (EncoderASR.transcribe_batch, inference/ASR.py:325-373; ctc_greedy_decode,
 * decoders/ctc.py:335-378): enc_dev [B, T, d_model] fp32, or NULL for the encoder states the previous encode / transcribe
 * call on this handle left in its workspace -> log_probs_dev [B, T, vocab] fp32 = log_softmax(ctc_lin(enc)) (optional) and
 * argmax_dev [B, T] int32 per-frame arg-max (optional; first index on ties like torch.max).  Needs "ctc_lin.w.*" weights. */
int sbk_asr_ctc_head(sbk_asr* m, const float* enc_dev, int B, int T, float* log_probs_dev, int* argmax_dev, void* stream);
/* TransformerASR.decode(tgt, encoder_out, enc_len) (lobes/models/transformer/TransformerASR.py:426-473), teacher-forced on the
 * KV-cached decoder step: tgt_dev [n, S] int32 (bos first), enc_dev [n, T, d_model] fp32, enc_len_dev [n] int32 ABSOLUTE
 * frame counts or NULL -> out_dev [n, S, d_model] fp32 = decoder.norm(decoder(...)) (the input of seq_lin).  The reference's
 * second return value (last layer's head-averaged cross-attention weights) is not produced. */
int sbk_asr_decode_teacher_forced(sbk_asr* m, const int* tgt_dev, const float* enc_dev, const int* enc_len_dev, int n, int S,
                                  int T, float* out_dev, void* stream);
/* S2STransformerBeamSearcher.forward, scorer=None (decoders/seq2seq.py:1632-1723,1853-1934), KV-cached with a
 * cache-row lineage table instead of index_select copies.  Writes the per-step search history
 * hist_*[max_steps, B * beam_size]: token, predecessor row, length-normalised score, raw log-prob; the host replays
 * the finished-hypothesis bookkeeping (:1371-1476) from it. */
int sbk_asr_beam_from_enc(sbk_asr* m, const float* enc_dev, const float* rel_len_dev, int B, int T,
                          const sbk_beam_params* params, int* hist_tok_dev, int* hist_pred_dev, float* hist_score_dev,
                          float* hist_lp_dev, int* steps_done, void* stream);
/* EncoderDecoderASR.transcribe_batch minus the tokenizer (inference/ASR.py:131-169): wav -> token ids.
 * _dev: wav already on the device; _host: HOST buffers, H2D/D2H inside the call (synchronises the stream). */
int sbk_asr_transcribe_greedy_dev(sbk_asr* m, const float* wav_dev, const float* rel_len_dev, int B, int L,
                                  int max_steps, int bos, int eos, float* enc_out_dev, int* pred_dev,
                                  float* score_dev, float* log_probs_dev, int* steps_done, void* stream);
/* Decode coalescing: G batches (B utterances each, separate device buffers) are encoded batch by batch and decoded
 * by ONE greedy loop over G*B hypotheses; pred_dev[g] receives batch g's [B, max_steps] token ids. */
int sbk_asr_transcribe_greedy_group_dev(sbk_asr* m, int G, const float* const* wav_dev, const float* const* rel_len_dev,
                                        int B, int L, int max_steps, int bos, int eos, int* const* pred_dev,
                                        int* steps_done, void* stream);
int sbk_asr_transcribe_greedy_host(sbk_asr* m, const float* wav_host, const float* rel_len_host, int B, int L,
                                   int max_steps, int bos, int eos, int* pred_host, float* score_host,
                                   int* steps_done, void* stream);

/* The group call from HOST buffers (pinned): per batch g, wav_host[g] [B, L] fp32 and rel_len_host[g] [B] are copied to the
 * device on an internal copy stream (batch g+1's copy overlaps batch g's encoder), pred_host[g] [B, max_steps] receives the
 * token ids; pred_dev (NULL, or an array whose entries may be NULL) additionally keeps them on the device.  Enqueue only:
 * the caller synchronises `stream`.  With poll interval 0 the whole call (copies included) replays one CUDA graph. */
int sbk_asr_transcribe_greedy_group_host_async(sbk_asr* m, int G, const float* const* wav_host,
                                               const float* const* rel_len_host, int B, int L, int max_steps, int bos, int eos,
                                               int* const* pred_host, int* const* pred_dev, int* steps_done, void* stream);

/* as _host, but only enqueues (pinned host buffers required); the caller synchronises the stream */
int sbk_asr_transcribe_greedy_host_async(sbk_asr* m, const float* wav_host, const float* rel_len_host, int B, int L,
                                         int max_steps, int bos, int eos, int* pred_host, float* score_host,
                                         int* steps_done, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SBK_H_ */
