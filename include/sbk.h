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

enum { SBK_ATT_ROPE = 0, SBK_ATT_RELPOS = 1, SBK_ATT_HYPERMIX = 2, SBK_ATT_REGULAR = 3 };
enum { SBK_ACT_RELU = 0, SBK_ACT_GELU = 1, SBK_ACT_SILU = 2 };
enum { SBK_ENC_CONFORMER = 0, SBK_ENC_BRANCHFORMER = 1, SBK_ENC_TRANSFORMER = 2 };
enum { SBK_CONFORMER_ACT_SWISH = 0, SBK_CONFORMER_ACT_GELU = 1 };
enum { SBK_PART_FBANK = 1, SBK_PART_CNN = 2, SBK_PART_ENCODER = 4, SBK_PART_DECODER = 8, SBK_PART_ALL = 15, SBK_PART_LM = 16 };

typedef struct {
    const char* name;  /* reference state_dict key with recipe prefix, e.g. "Transformer.encoder.layers.0.norm1.norm.weight" */
    const float* data; /* HOST fp32, contiguous, reference layout */
    int64_t numel;
} sbk_tensor;

typedef struct {
    /* Fbank (lobes/features.py:98-145) -- sizes in samples */
    int n_fft, hop, n_mels;
    /* ConvolutionFrontEnd (lobes/models/convolution.py:162-203): 2 blocks, 3x3, stride 2 (or 3 blocks), see cnn_blocks */
    int cnn_c1, cnn_c2;
    /* TransformerASR (lobes/models/transformer/TransformerASR.py:247-325) */
    int input_size, d_model, nhead, num_encoder_layers, num_decoder_layers, d_ffn, vocab, kernel_size;
    int attention_type;     /* SBK_ATT_ROPE (RoPEMHA) | SBK_ATT_RELPOS (RelPosMHAXL) | SBK_ATT_HYPERMIX (hypermixing: Conformer
                               encoder only, head width d_model / nhead 32 or 64, hypernetwork width d_ffn / nhead a multiple
                               of 16 up to 256; inputs up to 3000 frames) | SBK_ATT_REGULAR (regularMHA: the Transformer
                               encoder only, head width 64 or 128) */
    int decoder_activation; /* SBK_ACT_RELU | SBK_ACT_GELU | SBK_ACT_SILU (the `activation` ctor kwarg) */
    int max_len;            /* positional tables (ctor kwarg max_length, default 2500) */
    int parts;              /* bitmask of SBK_PART_*: which sub-models the weight table carries */
    /* TransformerLM used as a shallow-fusion scorer (lobes/models/transformer/TransformerLM.py; weights "lm.*"): head width
       64 with lm_d_model % 128 == 0, or the Switchboard LM (lm_d_model 264, 12 heads).  With "lm.embedding_proj.w.weight"
       present (TransformerLM(d_embedding=...)) d_embedding is its numel / lm_d_model and the projection is folded into
       the embedding table */
    int lm_d_model, lm_nhead, lm_layers, lm_d_ffn, lm_activation;
    /* Filterbank amin / top_db (processing/features.py:437-475) and InputNormalization epsilon (:1360-1455) of the fused
       wav -> features front end; 0 = the reference defaults (1e-10, 80 dB, 1e-10) */
    float fbank_amin, fbank_top_db, norm_eps;
    /* TransformerASR encoder_module: SBK_ENC_CONFORMER (0, so a zeroed config stays a Conformer) or SBK_ENC_BRANCHFORMER
       (Branchformer.py:92-234: RelPosMHAXL attention, no FFN modules, d_ffn only sizes the decoder) with the CSGU width
       csgu_linear_units (even, csgu_linear_units / 2 % 8 == 0) and kernel_size the CSGU's odd depthwise kernel (<= 31);
       branchformer_activation (SBK_ACT_RELU | SBK_ACT_GELU) follows pre_channel_proj; or SBK_ENC_TRANSFORMER
       (TransformerEncoderLayer, Transformer.py:311-490: pre-norm, regularMHA, Linear + GELU + Linear, the absolute sine table
       added to the input Linear's output) */
    int encoder_module, csgu_linear_units, branchformer_activation;
    /* ConvolutionFrontEnd blocks: 0 or 2 = 2 x (3x3, stride 2) with channels (cnn_c1, cnn_c2) = (64, 32) (the Conformer
       recipes') or (256, 256) (AISHELL-1's Transformer, up to 80 mels); 3 = the LibriSpeech Transformer recipes' (5x5,
       stride 2), (5x5, stride 2), (1x1 + residual 1x1), 64 channels each; any other pair is refused */
    int cnn_blocks;
    /* The Conformer encoder's conformer_activation (Conformer.py: both FFN modules and the convolution module after its
       LayerNorm): SBK_CONFORMER_ACT_SWISH (0, so a zeroed config stays Swish) or SBK_CONFORMER_ACT_GELU (torch.nn.GELU,
       the exact erf form: the Loquacious recipes).  Other values are rejected by sbk_asr_create. */
    int conformer_activation;
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

/* the Branchformer CSGU alone (ConvolutionalSpatialGatingUnit.forward, lobes/models/convolution.py:22-113, gate Identity):
 * u_dev [B*T, C] fp16 -> out_dev [B*T, C/2] fp16 = u[:, :C/2] * (Conv1d_K(LayerNorm(u[:, C/2:])) + bias), the conv "same" with
 * reflect padding inside the batch-padded T (T > (K-1)/2).  ln_g / ln_b [C/2], taps_dev in the reference layout [C/2, 1, K],
 * bias [C/2] fp32; odd K <= 31, C/2 % 8 == 0.  Allocates and frees its own scratch and synchronises the stream. */
int sbk_csgu_test(const void* u_dev, int B, int T, int C, const float* ln_g_dev, const float* ln_b_dev, const float* taps_dev,
                  const float* bias_dev, int K, void* out_dev, void* stream);

/* the encoder self-attention kernel alone, in the engine's layouts: qkv_dev [B*T, 3*H*head_dim] fp16 in per-head
 * [q | k | v] blocks; lens_dev [B] valid frames (NULL: all T; keys j >= lens[b] are masked, padded query rows are computed
 * like any other row).  relpos == 0 (RoPE / regularMHA): scores = q.k, q already scaled, scale unused.  relpos != 0
 * (RelPosMHAXL, head_dim <= 64): scores = ((q+u).k + (q+v).P[|i-j|]) * scale with pos_u_dev / pos_v_dev [H*head_dim] fp32
 * and P_dev [T, H*head_dim] fp16 (row r = linear_pos of relative distance r).  chunk > 0: Dynamic Chunk attention, query i
 * sees keys [max(0, (i/chunk - left_chunks) * chunk), min(len, (i/chunk + 1) * chunk)), left_chunks < 0 = the whole past.
 * A row that sees no key is 0.  out_dev [B*T, H*head_dim] fp16.  Synchronises the stream. */
int sbk_encoder_attention_test(const void* qkv_dev, int B, int T, int H, int head_dim, const int* lens_dev, int relpos,
                               const float* pos_u_dev, const float* pos_v_dev, const void* P_dev, float scale, int chunk,
                               int left_chunks, void* out_dev, void* stream);

/* one Linear of a decode / TransformerLM step alone, through the engine's step projection: out[rows, N] (row stride ldo) =
 * epilogue(A[rows, K] W[N, K]^T + bias), fp16 operands, fp32 accumulate.  backend 0 = weight streaming, 1 = the wgmma GEMM
 * (each launched with the programmatic-dependent-launch setting the step loops give it).  epilogue: 0 fp16, 1 fp16 GELU
 * (erf), 2 fp16 ReLU, 3 fp32, 4 fp32 residual (out += ...), 5 QKV_CACHE: columns [q | k | v] of width N / 3, q (fp16) to out,
 * k and v to kcache_dev / vcache_dev [rows][S_max][N / 3] fp16 at position step.  fp16 stores saturate at +-65504.  The A
 * operand is either A_dev fp16 (row stride lda; X_dev NULL) or LayerNorm(X_dev) of X_dev fp32 [rows, K] with ln_g / ln_b [K]
 * and eps 1e-6 (A_dev NULL): the decoder's pre-norm, fused into the weight-streaming kernel where it is built for K (256,
 * 512, 768, 1024), otherwise a separate LayerNorm kernel.  K % 16 == 0; the wgmma back end needs K, lda and ldo % 8 == 0
 * and, for QKV_CACHE, N / 3 % 32 == 0.  Allocates and frees its own scratch and synchronises the stream. */
int sbk_step_proj_test(int backend, int epilogue, const void* A_dev, int lda, const float* X_dev, const float* ln_g_dev,
                       const float* ln_b_dev, const void* W_dev, const float* bias_dev, int rows, int N, int K, void* out_dev,
                       int ldo, void* kcache_dev, void* vcache_dev, int S_max, int step, void* stream);

/* the decode-step attention alone (one query per row, nn.MultiheadAttention with the scale folded into q): q_dev fp16, row r
 * head h at q_dev[r * ldq + h * dh]; key j of head h for row block b = r / rows_per_block at kbase_dev / vbase_dev
 * [b * row_stride + h * head_stride + j * key_stride] (head_stride 0 = dh) -> out_dev [r * ldo + h * dh] fp16.  dh 64, 128
 * or a multiple of 4 up to 64 (at most 2560 keys).  step >= 0: self-attention over the step + 1 cached keys [0, step]; with
 * lineage_dev [2][rows][lin_stride] (rows_per_block 1) key j of row r lives in cache row lineage[step % 2][r][j], every
 * entry in [0, rows); with tok_cache_dev [rows][lin_stride] keys whose token tok_cache[cache row][j] == pad_tok are masked.
 * step < 0: cross-attention over the first enc_len_dev[b] of max_keys frames (enc_len_dev NULL: all max_keys), in [0,
 * max_keys].  A row with no visible key is NaN, as in the reference.  Synchronises the stream. */
int sbk_dec_attention_test(const void* q_dev, int ldq, const void* kbase_dev, const void* vbase_dev, long long row_stride,
                           int key_stride, int head_stride, int rows_per_block, int rows, int H, int dh, int max_keys, int step,
                           const int* enc_len_dev, const int* lineage_dev, const int* tok_cache_dev, int lin_stride,
                           int pad_tok, void* out_dev, int ldo, void* stream);

/* TransformerLM.forward's causal self-attention alone: qkv_dev [n * s, 3 d] fp16 with columns [q | k | v], H heads of
 * d / H = 64 or 32 side by side (q pre-scaled), tokens_dev [n, s] int32 (keys whose id == pad_tok are masked, as are keys
 * after the query) -> out_dev [n * s, d] fp16.  A query with no visible key is NaN, as in the reference.  Synchronises
 * the stream. */
int sbk_lm_causal_attention_test(const void* qkv_dev, int n, int s, int d, int H, const int* tokens_dev, int pad_tok,
                                 void* out_dev, void* stream);

/* the folded cross-attention of a decode step alone (rows = utterances, one query row each): the folded query projection
 * (gemm_f16_small, fp16 out), dec_xatt_fold_kernel, and the folded output projection added to x_dev [rows, ldx] fp32 in
 * place (columns [0, d); the others are left alone).  h16_dev [rows, d] fp16 is the LayerNorm output feeding the query
 * projection; in_proj_w / in_proj_b / out_w / out_b are the layer's multihead_attn weights as fp32 HOST arrays ([3d, d],
 * [3d], [d, d], [d]), folded on the host like the weight loader does.  enc16_dev [rows, T, d] fp16, enc_len_dev [rows] in
 * [0, T] (0: the row is NaN).  d = 64 H, d = 256 or 512.  Synchronises the stream. */
int sbk_xatt_fold_test(const void* h16_dev, const float* in_proj_w, const float* in_proj_b, const float* out_w,
                       const float* out_b, const void* enc16_dev, const int* enc_len_dev, int rows, int T, int H, int d,
                       float* x_dev, int ldx, void* stream);

/* the streaming encoder's ring write alone (stream_qkv_kernel): qkv_dev [B*n, 3*H*head_dim] fp32 (per head [q | k | v]) ->
 * q_out_dev [B*n, H*head_dim] fp16 and each row's per-head [k | v] into slot (slot0 + i) % cap of kv_out_dev
 * [B][cap][2*H*head_dim] fp16.  inv_freq_dev [head_dim / 2] fp32: RoPE at stream positions pos0 + i with q scaled by
 * q_scale; NULL: no rotation.  Synchronises the stream. */
int sbk_stream_qkv_test(const float* qkv_dev, int B, int n, int H, int head_dim, const float* inv_freq_dev, long long pos0,
                        float q_scale, void* q_out_dev, void* kv_out_dev, int cap, int slot0, void* stream);

/* the Conformer convolution module's depthwise conv + LayerNorm + Swish alone (Conformer.py:314-330): x_dev [B*T, D] fp32
 * (the GLU output) -> out_dev [B*T, D] fp16 = SiLU(LayerNorm(Conv1d_K(x) + bias)), eps 1e-5, zero padding outside [0, T)
 * only (padded frames inside T are inputs).  taps_dev in the reference layout [D, 1, K], bias / ln_g / ln_b [D] fp32; odd K,
 * D % 4 == 0, D <= 1024.  chunk > 0: Dynamic Chunk Convolution (inputs past the end of the output frame's chunk are zero).
 * Allocates and frees its own scratch and synchronises the stream. */
int sbk_dwconv_test(const float* x_dev, int B, int T, int D, int K, const float* taps_dev, const float* bias_dev,
                    const float* ln_g_dev, const float* ln_b_dev, int chunk, void* out_dev, void* stream);
/* the same with the Conformer activation as an argument: act SBK_CONFORMER_ACT_SWISH (SiLU, as sbk_dwconv_test) or
 * SBK_CONFORMER_ACT_GELU (exact erf GELU) after the LayerNorm. */
int sbk_dwconv_act_test(const float* x_dev, int B, int T, int D, int K, const float* taps_dev, const float* bias_dev,
                        const float* ln_g_dev, const float* ln_b_dev, int chunk, int act, void* out_dev, void* stream);

/* the HyperConformer's HyperMixing block alone (HyperMixing.forward, nnet/hypermixing.py:90-195, tied=False, nhead heads of
 * e = d / nhead in {32, 64} channels, k = d_ffn / nhead a multiple of 16 up to 256): x_dev [B*T, d] fp16 (the norm1 output),
 * lens_dev [B] valid frames (NULL: all T; frames t >= lens[b] are the key_padding_mask) -> out_dev [B*T, d] fp32 =
 * layer_norm(mixing), before the residual add.  Weights fp32 in the reference layout: w{1,2}_gen fc1 [nhead, e, e],
 * fc1 biases [nhead, e], fc2 [nhead, k, e], fc2 biases [nhead, k]; ln_g / ln_b [d].  T <= 3000.  Allocates and frees
 * its own scratch and synchronises the stream. */
int sbk_hypermix_test(const void* x_dev, const int* lens_dev, int B, int T, int d, int nhead, int k, const float* w1_fc1_w_dev,
                      const float* w1_fc1_b_dev, const float* w1_fc2_w_dev, const float* w1_fc2_b_dev, const float* w2_fc1_w_dev,
                      const float* w2_fc1_b_dev, const float* w2_fc2_w_dev, const float* w2_fc2_b_dev, const float* ln_g_dev,
                      const float* ln_b_dev, float* out_dev, void* stream);

/* one beam-search step alone (beam_step: S2SBeamSearcher.search_step, decoders/seq2seq.py:1478-1598, with the scorers'
 * scores precomputed), on caller buffers, n_bh = B * beam_size rows.  From params: beam_size, min_steps, eos, temperature,
 * using_eos_threshold, eos_threshold, length_normalization, minus_inf, length_weight (added to every token), and with
 * ctc_weight != 0 blank_index (masked to minus_inf) and the decoder weight 1 - ctc_weight.  path 0 picks the kernels by
 * width, 1 the rows + merge kernels (beam_size <= 16), 2 the radix select.  logits_dev [n_bh, V]; seq_scores_dev [2][n_bh]
 * and lineage_dev [2][n_bh][S_max] ping-pong by step parity; step_dev [n_bh] (one step per utterance, step + 1 < S_max and
 * step < n_hist; advanced by one); finished_dev [B] (eos hypotheses, capped at beam_size) and n_full_dev (utterances whose
 * counter reached beam_size); hist_{tok,pred,score,lp}_dev [n_hist][n_bh] (row `step` written); add_scores_dev [n_bh, V]
 * and add_row_dev [n_bh] optional; x_next_dev [n_bh, d] = emb_dev[token] * sqrt(d) + pe_dev[step + 1] (pe [S_max, d]).  With
 * lm_emb_dev: lm_x_dev fp32 and lm_x16_dev fp16 (saturating) [n_bh, lm_d] from lm_emb_dev / lm_pe_dev the same way, and the
 * token at tok_cache_dev[row * S_max + step + 1].  Every lineage entry in [0, n_bh).  Synchronises the stream. */
int sbk_beam_step_test(const sbk_beam_params* params, int path, int B, int V, int S_max, int n_hist, const float* logits_dev,
                       float* seq_scores_dev, int* lineage_dev, int* step_dev, int* finished_dev, int* n_full_dev,
                       int* hist_tok_dev, int* hist_pred_dev, float* hist_score_dev, float* hist_lp_dev,
                       const float* add_scores_dev, const float* add_row_dev, const float* emb_dev, const float* pe_dev, int d,
                       float* x_next_dev, const float* lm_emb_dev, const float* lm_pe_dev, int lm_d, float* lm_x_dev,
                       void* lm_x16_dev, int* tok_cache_dev, void* stream);

/* the CoverageScorer step alone (coverage_score, decoders/scorer.py:788-955): row r of utterance u = r / rows_per_utt
 * attends with q_dev fp16 (head h at q_dev[r * ldq + h * 64], scale folded in) to the first enc_len_dev[u] of T keys, key
 * t of head h at kbase_dev[u * utt_stride + h * head_stride + t * key_stride] fp16 (head_stride 0 = 64, 16-byte aligned
 * rows); coverage = the head average of that attention + the coverage of its predecessor hist_pred_dev[(step - 1) * n_bh +
 * r] (step > 0) from cov_dev [2][n_bh][T] (ping-pong by step parity, step from step_dev [n_bh], the same in every row) ->
 * out_dev[r] = weight * -(sum_t max(coverage_t, threshold) - T * threshold) / (step + 1).  A row with no visible key has
 * NaN coverage and score, as in the reference.  T * 8 <= 96 KB.  Synchronises the stream. */
int sbk_coverage_score_test(const void* q_dev, int ldq, const void* kbase_dev, long long utt_stride, int key_stride,
                            int head_stride, const int* enc_len_dev, int rows_per_utt, int T, int H, float* cov_dev,
                            const int* hist_pred_dev, const int* step_dev, int n_bh, float threshold, float weight, float* out_dev,
                            void* stream);

/* ---- model handle: repacks the reference state_dict once */
int sbk_asr_create(const sbk_asr_config* cfg, const sbk_tensor* weights, int n_weights, sbk_asr** out);
void sbk_asr_destroy(sbk_asr* m);
/* A clone is a new lane on the same repacked weights: it owns its workspace, graphs, streams and events, and inherits the
   source's settings (set_decoder_ln_fusion, set_decoder_tc_min_rows, set_poll_interval, set_dynchunk).  One clone per batch
   in flight. */
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
/* Chunk-by-chunk streaming encoder (TransformerASR.encode_streaming, TransformerASR.py:546-643; Conformer.py:501-586) for
 * the Conformer encoder with RoPEMHA or RelPosMHAXL.  A stream holds a batch of B streams that advance together: per layer
 * the attention's left context (the projected keys / values of the last `left_frames` frames; -1 = every frame so far) and
 * the Dynamic Chunk Convolution's carry.  Each chunk costs the same whatever the stream's age.  The outputs equal the
 * masked full-sequence run (sbk_asr_set_dynchunk with left_context_chunks = left_frames / chunk_size).  With RelPosMHAXL an
 * unlimited left context holds at most max_len frames.  The weights are the handle's: use a stream with the handle (or a
 * clone) it was created from. */
typedef struct sbk_asr_stream sbk_asr_stream; /* opaque */
int sbk_asr_stream_create(sbk_asr* m, int B, int chunk_size, int left_frames, sbk_asr_stream** out);
/* cnn_out [B, n, input_size] fp32 -> enc_out [B, n, d_model] fp32, 1 <= n <= chunk_size; only the last chunk may be
 * shorter.  No host synchronisation, except when an unlimited left context outgrows its buffer (it doubles). */
int sbk_asr_stream_encode_chunk(sbk_asr* m, sbk_asr_stream* s, const float* cnn_out_dev, int n_frames, float* enc_out_dev,
                                void* stream);
/* the same with the chunk's frames of row b at cnn_out_dev + b * batch_stride (batch_stride >= n_frames * input_size): a
 * trimmed slice of sbk_asr_stream_frontend_chunk's window output, read in place */
int sbk_asr_stream_encode_chunk_strided(sbk_asr* m, sbk_asr_stream* s, const float* cnn_out_dev, long long batch_stride,
                                        int n_frames, float* enc_out_dev, void* stream);
/* StreamingFeatureWrapper.forward (lobes/features.py:508-670) over LengthsCapableSequential(Fbank, InputNormalization
 * (global, eval), ConvolutionFrontEnd): the stream keeps each row's last 2 * pad samples of audio context on the device
 * (zeros before the first chunk).  wav_chunk_dev [B, n_samples] fp32 -> win_out_dev [B, T2, input_size] fp32, the front
 * end over the whole window [context | chunk] of 2 * pad + n_samples samples (T2 from sbk_asr_num_frames of that count);
 * the wrapper's output is frames [pad / stride, T2 - pad / stride) of each row, *n_frames of them, with stride = 4 * hop.
 * pad: a positive multiple of the stride, the same for every chunk of a stream.  The window's Fbank top_db clamp, STFT
 * centre padding and CNN reflect padding are those of the whole window, as in the reference.  The chunk must give at most
 * chunk_size frames, and only the last chunk of a stream may give fewer.  Enqueue only. */
int sbk_asr_stream_frontend_chunk(sbk_asr* m, sbk_asr_stream* s, const float* wav_chunk_dev, int n_samples, int pad,
                                  float* win_out_dev, int* n_frames, void* stream);
int sbk_asr_stream_reset(sbk_asr_stream* s); /* back to an empty context (encoder caches and front-end audio context) */
void sbk_asr_stream_destroy(sbk_asr_stream* s);
/* Layer `layer`'s context: *n_rows = cached frames; kv_out [B, n_rows, 2 * d_model] fp16 (per head [key | value], keys
 * RoPE-rotated by stream position) and carry_out [B, (kernel_size - 1) / 2, d_model] fp32 (depthwise-conv inputs), each
 * written when non-null. */
int sbk_asr_stream_context(sbk_asr* m, const sbk_asr_stream* s, int layer, void* kv_out_dev, float* carry_out_dev,
                           int* n_rows, void* stream);
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
/* Decode coalescing: G batches (B utterances each, separate device buffers) are encoded several batches per encoder pass
 * (up to 65536 encoder rows, or one batch when a batch alone is larger) and decoded by ONE greedy loop over G*B
 * hypotheses; pred_dev[g] receives batch g's [B, max_steps] token ids. */
int sbk_asr_transcribe_greedy_group_dev(sbk_asr* m, int G, const float* const* wav_dev, const float* const* rel_len_dev,
                                        int B, int L, int max_steps, int bos, int eos, int* const* pred_dev,
                                        int* steps_done, void* stream);
int sbk_asr_transcribe_greedy_host(sbk_asr* m, const float* wav_host, const float* rel_len_host, int B, int L,
                                   int max_steps, int bos, int eos, int* pred_host, float* score_host,
                                   int* steps_done, void* stream);

/* The group call from HOST buffers (pinned): per batch g, wav_host[g] [B, L] fp32 and rel_len_host[g] [B] are copied to the
 * device on an internal copy stream (a later encoder pass's copies overlap an earlier pass), pred_host[g] [B, max_steps] receives the
 * token ids; pred_dev (NULL, or an array whose entries may be NULL) additionally keeps them on the device.  Enqueue only:
 * the caller synchronises `stream`.  With poll interval 0 the whole call (copies included) replays one CUDA graph. */
int sbk_asr_transcribe_greedy_group_host_async(sbk_asr* m, int G, const float* const* wav_host,
                                               const float* const* rel_len_host, int B, int L, int max_steps, int bos, int eos,
                                               int* const* pred_host, int* const* pred_dev, int* steps_done, void* stream);

/* as _host, but only enqueues (pinned host buffers required); the caller synchronises the stream */
int sbk_asr_transcribe_greedy_host_async(sbk_asr* m, const float* wav_host, const float* rel_len_host, int B, int L,
                                         int max_steps, int bos, int eos, int* pred_host, float* score_host,
                                         int* steps_done, void* stream);

/* ---- CTC beam search without a language model: the frame loop of CTCBeamSearcher (decoders/ctc.py:1155-1485).
 * Beams are keyed by polynomial hashes modulo 2^61 - 1 of their text and partial word, with base SBK_CTC_HASH_BASE over
 * (code point + 1) per character, plus the string lengths.  The caller describes vocab_list[0 .. n_vocab) per token:
 * tok_info [n_vocab][3] int32 = kind (SBK_CTC_TOK_*), string id (first index holding the same string), length in code
 * points of the string the token appends (token[1:] for a word start, the token for a plain one, else 0);
 * tok_hash [n_vocab][2] uint64 = hash of that string, base^length mod 2^61 - 1. */
#define SBK_CTC_HASH_BASE 0x1F3D5B79A2C4E6F1ull
enum { SBK_CTC_TOK_PLAIN = 0, SBK_CTC_TOK_BLANK = 1, SBK_CTC_TOK_WORD = 2, SBK_CTC_TOK_SPACE = 3 };
typedef struct {
    int blank, beam_size, prune_history;
    /* float32 thresholds: token_prune_min_logp, beam_prune_logp, log(blank_skip_threshold) */
    float token_prune_min_logp, beam_prune_logp, blank_skip_logp;
} sbk_ctc_beam_params;
/* Workspace for one search: runs the token-count pre-pass over log_probs_dev [B, T, V] fp32 with lens_dev [B] int32
 * absolute frame counts (0..T) and synchronises the stream.  1 <= beam_size <= 256, V <= 8192, n_vocab <= V. */
int sbk_ctc_beam_workspace_bytes(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                                 const sbk_ctc_beam_params* params, size_t* bytes, void* stream);
/* The search, one CTA per utterance.  Outputs: frame_beams [B, T] int32 = beams after frame f (-1: frame skipped;
 * frames >= lens[b] untouched), parent / token [B, T, beam_size] int32 = each surviving beam's parent (rank at the previous
 * processed frame) and token, score [B, beam_size] fp32 = final beam scores, n_final [B] int32 = final beam count (-1: a
 * frame had no candidate token, which the reference fails on).  Synchronises the stream once (the pre-pass), then enqueues. */
int sbk_ctc_beam_search(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                        const int* tok_info_dev, const uint64_t* tok_hash_dev, const sbk_ctc_beam_params* params,
                        void* workspace_dev, size_t workspace_bytes, int* frame_beams_dev, int* parent_dev, int* token_dev,
                        float* score_dev, int* n_final_dev, void* stream);

/* ---- CTC prefix beam search without a language model: the frame loop of CTCPrefixBeamSearcher (decoders/ctc.py:
 * 1488-1905), candidates in CPython's set order, float64 beam probabilities.  Strings are hashed as above.  Per token of
 * vocab_list[0 .. n_vocab): tok_info [n_vocab][SBK_CTC_PREFIX_TOK_INTS] int32 = kind (SBK_CTC_TOK_*), string id, length
 * of the token string, length of the string a new beam appends to its text (" " + token[1:] for a word start, else the
 * token), length of token[1:] (word starts), whether the appended string holds whitespace, length of its part before the
 * first whitespace, of its part after the last whitespace, of its last non-empty word between the two (0: none);
 * tok_hash [n_vocab][SBK_CTC_PREFIX_TOK_WORDS] uint64 = hash and base^length of the token string, hash and base^length
 * of the appended string, hash of token[1:], hash and base^length of the leading part, hash of the trailing part, hash
 * of the inner word. */
#define SBK_CTC_PREFIX_TOK_INTS 9
#define SBK_CTC_PREFIX_TOK_WORDS 9
typedef struct {
    int blank, beam_size, prune_history;
    /* float32 thresholds: token_prune_min_logp, log(blank_skip_threshold); float64 beam_prune_logp */
    float token_prune_min_logp, blank_skip_logp;
    double beam_prune_logp;
} sbk_ctc_prefix_beam_params;
/* Workspace for one search: runs the token-count pre-pass over log_probs_dev [B, T, V] fp32 with lens_dev [B] int32
 * absolute frame counts (0..T) and synchronises the stream.  1 <= beam_size <= 256, V <= 8192, n_vocab <= V. */
int sbk_ctc_prefix_beam_workspace_bytes(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                                        const sbk_ctc_prefix_beam_params* params, size_t* bytes, void* stream);
/* The search, one CTA per utterance.  Outputs: frame_beams [B, T] int32 = beams after frame f (-1: frame skipped;
 * frames >= lens[b] untouched), parent / token [B, T, beam_size] int32 = each surviving beam's origin: its rank at the
 * previous processed frame and the token that created it (-1: the beam was carried over), score [B, beam_size] fp64 =
 * final beam scores, n_final [B] int32 = final beam count.  Synchronises the stream once (the pre-pass), then enqueues. */
int sbk_ctc_prefix_beam_search(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                               const int* tok_info_dev, const uint64_t* tok_hash_dev, const sbk_ctc_prefix_beam_params* params,
                               void* workspace_dev, size_t workspace_bytes, int* frame_beams_dev, int* parent_dev,
                               int* token_dev, double* score_dev, int* n_final_dev, void* stream);

/* ---- Transducer greedy search: TransducerBeamSearcher.transducer_greedy_decode (decoders/transducer.py:156-291) with
 * the prediction network Embedding -> LSTM (1 layer, unidirectional, with biases, gate order i, f, g, o) ->
 * Linear(bias=False), the joint GELU(tn + out_PN) (exact erf form) and the output Linear(bias=False) + log-softmax.
 * Weights (HOST fp32, torch layouts): "emb.weight" [vocab, emb_dim], "lstm.weight_ih" [4 hidden, emb_dim],
 * "lstm.weight_hh" [4 hidden, hidden], "lstm.bias_ih" / "lstm.bias_hh" [4 hidden], "proj_dec.weight" [joint, hidden],
 * "out.weight" [vocab, joint].  hidden and joint are multiples of 64 up to 1024, vocab <= 4096, and the fp16 weight
 * slices must fit the shared memory of the device's SMs. */
typedef struct sbk_transducer sbk_transducer; /* opaque */
typedef struct {
    int vocab, emb_dim, hidden, joint;
} sbk_transducer_config;
int sbk_transducer_create(const sbk_transducer_config* cfg, const sbk_tensor* weights, int n_weights, sbk_transducer** out);
void sbk_transducer_destroy(sbk_transducer* m);
/* CTAs per search call (one per SM) and the shared memory one CTA uses at batch size 1 */
int sbk_transducer_info(const sbk_transducer* m, int* ctas, int* smem_bytes_at_b1);
/* One cooperative kernel for the whole call.  tn_dev [B, T, joint] fp32; every frame is decoded.  State in / out (fp32):
 * h_dev, c_dev [B, hidden] and out_pn_dev [B, joint]; with start_from_blank they are overwritten with PN(blank) from a
 * zero LSTM state first.  Outputs: tokens_dev [B, T * (max_symbols_per_step + 1)] int32 (the first n_tokens_dev[b]
 * entries of row b), frames_dev (same shape, may be null) = the frame each token was emitted at, logp_sum_dev [B] = sum of the emitted tokens' log-probabilities, and, if stats_dev is not null,
 * stats_dev[0..1] = rounds (decisions of the longest row) and grid barriers.  1 <= B <= 1024, 0 <= blank < vocab. */
int sbk_transducer_greedy(sbk_transducer* m, const float* tn_dev, int B, int T, int blank, int max_symbols_per_step,
                          int start_from_blank, float* h_dev, float* c_dev, float* out_pn_dev, int* tokens_dev,
                          int* frames_dev, int* n_tokens_dev, float* logp_sum_dev, int* stats_dev, void* stream);

/* ---- Transducer beam search: TransducerBeamSearcher.transducer_beam_search_decode (decoders/transducer.py:320-476)
 * without a language model, on a handle of sbk_transducer_create.  Every utterance starts from [blank] with score 0 and
 * a zero LSTM state and every frame of tn_dev [B, T, joint] fp32 is decoded.  A frame stops after
 * SBK_TRANSDUCER_BEAM_POP_CAP(beam_size) pops at the most: an utterance that reaches it stops there.
 * Outputs, per utterance b and rank n < nbest (rank order = the reference's sort by score / length):
 *   out_tokens_dev [B, nbest, T * SBK_TRANSDUCER_BEAM_POP_CAP(beam_size)] int32: the first out_lens entries are the
 *     hypothesis without its leading blank;
 *   out_lens_dev [B, nbest] int32: the length, -1 when the last beam held fewer than n + 1 hypotheses, and in
 *     out_lens_dev[b, 0] -2 - t when utterance b stopped at the pop cap in frame t;
 *   out_scores_dev [B, nbest] fp32: score / (length + 1), the reference's normalised score.
 * trace_dev (may be null) [B, T * cap, 6 + 2 beam_size] int32: one record per pop, in pop order per utterance, unused
 * records set to -1: (utterance, frame, index of the popped hypothesis in the frame's list -- the previous beam, then the
 * children in the order they were added --, how the frame ended right after this pop (0: it did not, 1: the state_beam
 * test, 2: the beam is full), bit j = child j kept, the popped hypothesis' raw score (fp32 bits), the top beam_size tokens,
 * their log-probabilities (fp32 bits)).  stats_dev (may be null) [4]: rounds, pops, prediction-network steps, grid
 * barriers.  2 <= beam_size <= SBK_TRANSDUCER_BEAM_MAX, beam_size <= vocab, 1 <= nbest <= beam_size, 1 <= B <= 1024.
 * Memory grows as B * T * cap: the token output (4 * nbest bytes per possible pop), a stream-ordered workspace of about
 * B * (8 T cap + 4 (beam_size + cap) (2 hidden + joint) + 20 beam_size (cap + 1)) bytes, and the trace when requested;
 * long inputs with a wide n-best are best searched in smaller batches. */
#define SBK_TRANSDUCER_BEAM_MAX 32
#define SBK_TRANSDUCER_BEAM_POP_CAP(beam_size) (4 * (beam_size))
int sbk_transducer_beam(sbk_transducer* m, const float* tn_dev, int B, int T, int blank, int beam_size, int nbest,
                        float state_beam, float expand_beam, int* out_tokens_dev, int* out_lens_dev, float* out_scores_dev,
                        int* trace_dev, int* stats_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SBK_H_ */
