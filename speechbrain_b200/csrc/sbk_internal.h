// Internal (C++) interfaces between the kernels' host launchers and the C-ABI layer.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace sbk {

// Lays fields out one after another in a buffer, each at a 256-byte boundary.  A buffer's layout is one function that runs
// twice: with base == nullptr to measure the bytes it needs (`used`), then with the buffer to set the fields.
struct Carver {
    uint8_t* base = nullptr;
    size_t used = 0;
    template <class T>
    void operator()(T*& field, size_t bytes) {
        if (base) field = reinterpret_cast<T*>(base + used);
        used += (bytes + 255) & ~size_t(255);
    }
};

// ---- test_hooks.cu: what the kernel test hooks of the C ABI share
// A hook's device scratch: laid out by one Carver function in a single cudaMalloc, freed when it goes out of scope.
struct TestScratch {
    uint8_t* base = nullptr;
    TestScratch() = default;
    TestScratch(const TestScratch&) = delete;
    TestScratch& operator=(const TestScratch&) = delete;
    ~TestScratch() { cudaFree(base); }
    int reserve(const char* who, size_t bytes);  // no allocation for 0 bytes
    template <class Layout>
    int carve(const char* who, Layout&& layout) {
        Carver measure;
        layout(measure);
        if (int rc = reserve(who, measure.used)) return rc;
        Carver take{base};
        layout(take);
        return 0;
    }
};
// A hook's last step: synchronises the stream; a device error becomes "<who>: device error" unless rc already holds one.
int finish_test(const char* who, int rc, cudaStream_t stream);

enum GemmEpiMode { EPI_F16 = 0, EPI_F32 = 1, EPI_RESID = 2, EPI_GLU = 3, EPI_ROPE = 4, EPI_QKV_CACHE = 5 };
enum GemmAct { ACT_NONE = 0, ACT_SILU = 1, ACT_GELU = 2, ACT_RELU = 3, ACT_SILU_FAST = 4 /* tanh.approx form; for EPI_GLU: fast gate sigmoid */ };

struct GemmEpilogue {
    int mode = EPI_F16;
    int act = ACT_NONE;
    const float* bias = nullptr;   // [N] or null
    void* out = nullptr;           // fp16 or fp32, row stride ldo (elements)
    int ldo = 0;
    const float* resid = nullptr;  // EPI_RESID: fp32 [M, ldo]
    float alpha = 1.0f;            // EPI_RESID scale; EPI_ROPE: scale applied to q
    const int* row_lens = nullptr; // EPI_RESID: rows (b, t >= row_lens[b]) get alpha = 0
    int T = 1;                     // frames per utterance (row = b*T + t)
    const float* rope_cos = nullptr;  // EPI_ROPE: [T, head_dim/2]
    const float* rope_sin = nullptr;
    int head_dim = 64;
    // EPI_QKV_CACHE (decoder self-attention in_proj, columns [q | k | v] of width qkv_d): q -> out (fp16, ldo), k / v ->
    // cache[(row * S_max + step_ptr[row]) * qkv_d + col]
    __half* kcache = nullptr; __half* vcache = nullptr; const int* step_ptr = nullptr; int S_max = 0; int qkv_d = 0;
    // EPI_F16 (wide-tile kernel) scatter of the cross-attention [K | V] projections of one or several decoder layers
    // (N = layers * 2 * kv_heads * 64, row = utt * T + t) to layer[l][K|V][utt][head][t][64]; kv_part_stride = elements
    // between the K part and the V part of a layer, kv_layer_stride = elements between layers.  kv_heads 0 = plain
    // row-major store.
    int kv_heads = 0; size_t kv_part_stride = 0; size_t kv_layer_stride = 0;
};

// out = epilogue(A[M,K] fp16 x W[N,K]^T fp16), wgmma tensor cores. gemm_tc.cu
int gemm_f16(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
             cudaStream_t stream);
// Small-M variant for the decode steps of several batches (M = live hypotheses, 64..512): 64 x 32/64 tiles, deep TMA
// ring; any epilogue mode incl. EPI_QKV_CACHE. gemm_tc.cu
int gemm_f16_small(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
                   cudaStream_t stream);
// 128 x 256 tile variant with the coalesced epilogue, N % 256 == 0. gemm_tc2.cu
int gemm_f16_wide(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
                  cudaStream_t stream);


const char* last_error();
void launch_count_begin_capture();
long long launch_count_end_capture();
void launch_count_add(long long n);
long long launch_count();

// Optional live timing of every wgmma GEMM launch (CUDA events on the launching stream).
struct GemmProfile {
    bool enabled = false;
    std::vector<cudaEvent_t> ev;   // start/stop pairs
    std::vector<double> flops;     // 2*M*N*K per launch
    std::vector<int> shape;        // M, N, K, epilogue mode per launch
};
GemmProfile* gemm_profile();

// ---- fbank.cu
struct Fbank;
int fbank_create(Fbank** out, int n_fft, int hop, int n_mels, const float* window_host, const float* mel_matrix_host,
                 float amin, float top_db);
void fbank_destroy(Fbank* fb);
int fbank_num_frames(const Fbank* fb, int L);
int fbank_forward(const Fbank* fb, const float* wav, int B, int L, float* out, int* utt_max, const float* mean,
                  const float* stdv, float eps, cudaStream_t stream);
int global_norm_forward(const float* x, float* out, int B, int T, int F, const float* mean, const float* stdv,
                        float eps, cudaStream_t stream);
int sentence_norm_forward(const float* x, float* out, const float* rel_len, int B, int T, int F, int std_norm,
                          int avoid_padding_norm, float eps, cudaStream_t stream);

// ---- frontend.cu
// A ConvolutionFrontEnd's weights: 2 blocks of K x K convolutions (K = 3, out_channels (c1, c2) = (64, 32) or (256, 256)),
// or the Transformer recipes' 3 blocks (5x5 / stride 2, 5x5 / stride 2, 1x1 with a residual 1x1), 64 channels.
struct CnnWeights {
    int blocks = 0, c1 = 0, c2 = 0;
    const float *w1 = nullptr, *b1 = nullptr;   // block 1: conv [c1, K, K], bias [c1]
    const float *g1 = nullptr, *be1 = nullptr;  // block 1: LayerNorm [F1, c1]
    const __half* w2 = nullptr;  // block 2: conv [c2][(kf * K + kt) * c1 + ch]; at 256 channels as 128B-swizzled k-blocks
    const float *b2 = nullptr, *g2 = nullptr, *be2 = nullptr;  // block 2: bias [c2], LayerNorm [F2, c2]
    const float *w3 = nullptr, *b3 = nullptr;   // block 3: [convs.conv_0 | reduce_conv.conv] as [128, 64], [128]
    const float *g3 = nullptr, *be3 = nullptr, *gr = nullptr, *ber = nullptr;  // block 3: convs.norm_0, reduce_conv.norm
};
// feats [B, T0, F0] fp32 -> out [B, T2, F2 * c2] fp16 (+ fp32 when out_f is set); act1_h [B, T1, F1, c1] scratch
int cnn_frontend_forward(const float* feats, int B, int T0, int F0, const CnnWeights& w, __half* act1_h, __half* out_h,
                         float* out_f, cudaStream_t stream);

// ---- encoder_ops.cu
// pdl: launched with programmatic stream serialisation (fp16 output only; the decode step's pre-norms)
int layernorm_rows(const float* x, void* out, bool out_half, const float* gamma, const float* beta, int M, int D,
                   float eps, cudaStream_t stream, bool pdl = false);
// y = LN_a(x) (fp32, stored when y_out != null), z = LN_b(y) -> z_out (fp16 or fp32): two chained LayerNorms in one pass
int layernorm2_rows(const float* x, float* y_out, void* z_out, bool z_half, const float* ga, const float* ba, float eps_a,
                    const float* gb, const float* bb, float eps_b, int M, int D, cudaStream_t stream);
// out = LN(x; gamma, beta), out2 = LN(x; gamma2, beta2): two fp16 LayerNorms of the same rows from one pass
int layernorm_rows_dual(const float* x, __half* out, const float* gamma, const float* beta, __half* out2, const float* gamma2,
                        const float* beta2, int M, int D, float eps, cudaStream_t stream);
// rows x n fp32 (row stride ld_in) -> rows x n fp16, packed
int cast_f32_f16(const float* in, __half* out, size_t n, cudaStream_t stream, int rows = 1, size_t ld_in = 0);
// Branchformer CSGU: u [B*T, C] fp16 -> g [B*T, C/2] fp16 = u[:, :C/2] * (dwconv_K(LN(u[:, C/2:])) + bias), reflect padding
// inside T; taps tap-major [31, C/2] as csgu_repack_taps lays them out; stats: B*T float2 of scratch
int csgu_forward(const __half* u, int B, int T, int C, const float* gamma, const float* beta, float eps, const float* taps,
                 const float* bias, int K, float2* stats, __half* g, cudaStream_t stream);
constexpr int CSGU_TAP_ROWS = 31;
void csgu_repack_taps(const float* src, int C2, int K, float* dst);  // (C/2, 1, K) -> [CSGU_TAP_ROWS, C/2] (host)
// HyperConformer token mixing (HyperMixing, tied=False): generator g = 0 (w1_gen) / 1 (w2_gen) with fc1 [M, e, e] and
// fc2 [M, k, e] fp16 in the reference layout, fp32 biases [M, e] / [M, k]; ln_g / ln_b the module's LayerNorm [d]
struct HyperMixWeights {
    const __half *fc1w[2], *fc2w[2];
    const float *fc1b[2], *fc2b[2];
    const float *ln_g, *ln_b;
};
constexpr int HM_PE_ROWS = 3000;  // HyperMixing's own PositionalEncoding(d, max_length=3000)
// x [B*T, d] fp32 += LayerNorm_hm(HyperMixing(h16)), h16 the norm1 output [B*T, d] fp16; M heads of e = d / M in {32, 64},
// KH = d_ffn / M (multiple of 16, <= 256); pe [HM_PE_ROWS, d] fp32 (sine_table); lens device int[B] (null: all T).
// Scratch: part (hypermix_part_floats), G [B * d * KH] fp16, gscale [B * M] fp32.  T <= HM_PE_ROWS.
int hypermix_forward(const __half* h16, int B, int T, int d, int M, int KH, const int* lens, const float* pe,
                     const HyperMixWeights& w, float* part, __half* G, float* gscale, float* x, cudaStream_t stream);
size_t hypermix_part_floats(int B, int T, int d, int KH);
// chunk > 0: Dynamic Chunk Convolution (inputs past the end of the output frame's chunk are zero).  left: [B, (K-1)/2, D]
// inputs of the frames before frame 0 (a stream's carry), null = zero padding.  gelu: exact erf GELU after the LayerNorm,
// else Swish (the Conformer's conformer_activation).
int dwconv_ln_act(const float* glu, int B, int T, int D, int K, const float* wdw, const float* bdw, const float* gamma,
                  const float* beta, float eps, __half* out, cudaStream_t stream, bool gelu, int chunk = 0,
                  const float* left = nullptr);
// carry [B, (K-1)/2, D] <- the last (K-1)/2 rows of [carry; glu [B, n, D]]; has_old false: the old carry counts as zeros
int dwconv_carry(const float* glu, int B, int n, int D, int K, bool has_old, float* carry, cudaStream_t stream);
void dwconv_repack_taps(const float* src, int D, int K, float* dst);  // (D, 1, K) -> tap-major [K, D] (host)
int encoder_attention(const __half* qkv, int ld, int B, int T, int H, int head_dim, const int* lens, bool relpos,
                      const float* pos_u, const float* pos_v, const __half* P, int ldp, float scale, __half* out,
                      int ldo, cudaStream_t stream, int chunk = 0, int left_chunks = -1);
// One chunk of a stream: the window is W rows [cached rows; the chunk's nq rows], all visible to every query.
struct AttStream {
    const __half* q = nullptr; int ldq = 0;  // [B * nq, ldq] the chunk's queries, head h at column h * head_dim
    const __half* kv = nullptr; int ldkv = 0;  // ring [B][cap][ldkv]: head h's [k | v] at column h * 2 * head_dim
    int cap = 0, start = 0;                    // window row r lives in slot (start + r) % cap
    int nq = 0;
};
// out [B * nq, ldo] fp16; RelPos: P [>= W rows, ldp] = linear_pos(pe[|r|]); RoPE: q and k arrive rotated, q scaled
int encoder_attention_stream(const AttStream& sa, int B, int W, int H, int head_dim, bool relpos, const float* pos_u,
                             const float* pos_v, const __half* P, int ldp, float scale, __half* out, int ldo,
                             cudaStream_t stream);
// CTAs per SM of the RelPosMHAXL encoder attention at head_dim, full-sequence or stream form, with the attributes its launch sets
int encoder_attention_occupancy(int head_dim, bool stream, int* ctas);
// qkv [B*n, 3d] fp32 -> q [B*n, d] fp16 and the rows' [k | v] into ring slots (slot0 + i) % cap of kv [B][cap][2d] fp16;
// inv_freq [head_dim / 2] set: RoPE at stream positions pos0 + i, q scaled by q_scale
int stream_qkv(const float* qkv, int B, int n, int H, int DH, const float* inv_freq, long long pos0, float q_scale,
               __half* q, __half* kv, int cap, int slot0, cudaStream_t stream);
// TransformerLM whole-sequence causal self-attention: qkv [n*s, 3d] fp16 ([q | k | v], head_dim d / H of 64 or 32, q
// pre-scaled), tokens
// [n, s] int32 (keys whose id == pad_tok are masked) -> out [n*s, d] fp16
int lm_causal_attention(const __half* qkv, int n, int s, int d, int H, const int* tokens, int pad_tok, __half* out,
                        cudaStream_t stream);

// ---- decoder.cu
enum SkinnyEpi { SK_F16 = 0, SK_F16_GELU = 1, SK_F32 = 2, SK_RESID = 3, SK_QKV_CACHE = 4, SK_F16_RELU = 5, SK_F16_SILU = 6 };
struct SkinnyArgs {
    const __half* A; int lda;
    const __half* W; int ldw;
    const float* bias;
    int n_rows, N, K, epi;
    void* out; int ldo;              // SK_F16/F32: out ; SK_RESID: fp32 x (in place) ; SK_QKV_CACHE: q buffer fp16 [n, d]
    __half* kcache; __half* vcache;  // SK_QKV_CACHE: [n_rows, S_max, d]
    const int* step_ptr; int S_max; int d; float q_scale;
    // LayerNorm-fused variant: A = LayerNorm(X fp32 [n_rows, K]) computed in-kernel (X != nullptr)
    const float* X; const float* ln_g; const float* ln_b; float ln_eps;
};
// programmatic dependent launch of the decode-step kernels launched by decoder.cu (attention, skinny GEMM, greedy /
// beam bookkeeping, TransformerLM helpers)
void set_pdl(bool on);
int skinny_gemm(const SkinnyArgs& a, cudaStream_t stream);
struct DecAttnArgs {
    const __half* q; int ldq;
    const __half* kbase; const __half* vbase;
    size_t row_stride;
    int key_stride;
    int head_stride = 0;  // elements between heads inside a row block; 0 = dh (heads side by side in one key row)
    int rows_per_block;
    const int* n_keys_ptr;
    const int* enc_len;
    int n_keys_fixed;
    int H, dh;
    __half* out; int ldo;
    const int* lineage; int lin_stride;  // beam search: [2][n_rows][lin_stride] cache-row table (null for greedy)
    const int* tok_cache; int pad_tok;   // LM pad mask: keys whose token (tok_cache[phys_row][pos]) == pad_tok are masked
};
int dec_attention(const DecAttnArgs& a, int n_rows, int max_keys, cudaStream_t stream);
// Cross-attention of one query row per utterance over the fp16 encoder states e [n_utt][T][D] with folded weights:
// q [n_utt, ldq] holds the H folded queries W_k,h^T q_h (D each), out [n_utt, ldo] gets the H context vectors
// sum_t p_t e_t (D each).  D = 512 with H <= 8, or D = 256 with H <= 4.
struct XattFoldArgs {
    const __half* q; int ldq;
    const __half* e; const int* enc_len; int T;
    int H, D;
    __half* out; int ldo;
};
int dec_xatt_fold(const XattFoldArgs& a, int n_utt, cudaStream_t stream);
struct BeamLm {  // TransformerLM scorer state the beam step feeds (all null/0 when there is no LM)
    const float* emb = nullptr; const float* pe = nullptr; int d = 0;  // d: the row pitch of emb, pe, x and x16
    float scale = 0.0f;                                                 // x = emb[token] * scale + pe[step]
    float* x = nullptr; __half* x16 = nullptr; int* tok_cache = nullptr;
};
struct BeamStepArgs {
    const float* logits; int V; int beam; int S_max;
    float* seq_scores; int* lineage; int* step_arr; int* finished; int* n_full;
    int* hist_tok; int* hist_pred; float* hist_score; float* hist_lp;
    float temperature, eos_threshold, minus_inf;
    int min_steps, eos, use_eos_threshold, length_norm;
    const float* emb; const float* pe; int d; float* x_next;
    const float* add_scores;  // [n_bh, V] pre-weighted scorer scores or null
    BeamLm lm;
    float attn_weight = 1.0f;  // 1 - ctc_weight (seq2seq.py:803-804, _attn_weight_step)
    int blank = -1;            // CTC blank index, blocked in the log-probs (scorer.py:1248-1250); -1 = no CTC scorer
    float add_const = 0.0f;    // LengthScorer: weight * 1 added to every token (scorer.py:1043-1071)
    const float* add_row = nullptr;  // CoverageScorer: [n_bh] weighted score added to every token of a hypothesis
    float* scratch = nullptr;        // [n_bh * 33] floats: per-row candidates between the two kernels of a step (beam <= 16)
    int path = 0;  // 0: by width (rows + merge up to beam 16, radix select above), 1: rows + merge, 2: radix select
};
// CoverageScorer (decoders/scorer.py:788-955) on the last decoder layer's head-averaged cross-attention
struct CoverageStep {
    const __half* q; int ldq; const __half* kbase; size_t utt_stride; int key_stride; const int* enc_len;
    int head_stride = 0;  // 0 = 64 (heads side by side in a key row)
    int rows_per_utt, T, H; float* cov_base; const int* hist_pred; const int* step_ptr; int n_bh;
    float threshold, weight; float* out;
};
int coverage_score(const CoverageStep& p, cudaStream_t stream);
// CTC prefix scorer (ctc_scorer.cu)
struct CtcStep {
    const float* x; const float* xlin; const float* xb; const int* enc_len;   // xlin = exp(x)
    float* rsum_base; float* rb_base; float* psi_base;  // [2][n_bh, T], [2][n_bh, T], [2][n_bh]: ping-pong by step parity
    float* tab; float* tabM;                            // score-kernel operand tables [n_bh * 2 * (T + 3)], [n_bh * 2]
    const int* hist_tok; const int* hist_pred;
    const int* step_ptr;                                // device step counters [n_bh] (same value in every row)
    int n_bh, bos, T, V, beam, blank, eos;
    float weight; float* out; int accumulate;
};
int ctc_prefix_reset(float* x, float* xlin, float* xb, const int* enc_len, int B, int T, int V, int blank, int beam, float* rsum,
                     float* rb, float* psi_prev, float* tab, float* tabM, cudaStream_t stream);
int ctc_prefix_score(const CtcStep& p, cudaStream_t stream);
int ctc_prefix_group_width(int beam, int T);   // hypotheses per score CTA (the R of ctc_score_kernel<R>)
// x [rows, V] fp32: optional in-place log_softmax per row, arg-max per row -> idx (may be null)
int rows_logsoftmax_argmax(float* x, int rows, int V, bool do_logsoftmax, int* idx, cudaStream_t stream);
int ctc_prefix_update(const CtcStep& p, cudaStream_t stream);
int beam_reset(int n_bh, int beam, int S_max, int bos, int* step_arr, float* seq_scores, int* lineage, int* finished,
               int* n_full, const float* emb, const float* pe, int d, float* x, const BeamLm* lm, cudaStream_t stream);
// x [M, pitch] fp32 rows of D channels and pitch - D zero padding -> LayerNorm over the D channels, in place (write_f32) and
// into x16 [M, pitch] fp16, the padding written as zero; gamma, beta [D]
int layernorm_dual(float* x, __half* x16, const float* gamma, const float* beta, int M, int D, int pitch, float eps,
                   bool write_f32, cudaStream_t stream);
int weighted_log_softmax(const float* logits, float* out, int rows, int V, float temperature, float weight,
                         cudaStream_t stream);
int beam_step(const BeamStepArgs& p, int B, cudaStream_t stream);
int greedy_reset(int* tokens, int tok_stride, int n_rows, int bos, int* step_arr, int* has_ended, int* ended_count,
                 const float* emb, const float* pe, int d, float* x, cudaStream_t stream);
int greedy_select(const float* logits, int n_rows, int V, int* step_arr, int eos, int* tokens, int tok_stride,
                  int* has_ended, int* ended_count, int* pred, float* score, int out_stride, float* log_probs, int L,
                  const float* emb, const float* pe, int d, float* x_next, cudaStream_t stream);

}  // namespace sbk
