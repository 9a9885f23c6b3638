// Model engine: weight repacking, workspace, the encode pipeline (CNN front-end -> Conformer encoder)
// and the KV-cached greedy decode loop.  Host-side orchestration only; all math is in the kernels.
//
// Weights arrive as HOST fp32 arrays named exactly like the reference state_dict (SURVEY.md 8b) with
// the recipe's module prefixes:  "CNN.", "Transformer.", "seq_lin.", plus "normalize.glob_mean/std"
// and "fbank.window" / "fbank.mel_matrix".  They are repacked once (fp16 GEMM operands, interleaved GLU
// rows, concatenated cross-attention K/V projections, pre-scaled decoder queries) into one device arena.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "sbk_internal.h"
#include "../../include/sbk.h"

namespace sbk {

struct EncLayerW {
    const float *ffn1_ln_g, *ffn1_ln_b, *ffn1_b1, *ffn1_b2;
    const __half *ffn1_w1, *ffn1_w2;
    const float *norm1_g, *norm1_b;
    const __half *wqkv, *wo;
    const float* bo;
    const __half* wpos;               // RelPos linear_pos
    const float *pos_u, *pos_v;       // RelPos biases, raw (d_h, H) buffer viewed (H, d_h)
    const float *conv_ln_g, *conv_ln_b;
    const __half* wpw1;               // [2d, d] rows interleaved 16 value / 16 gate
    const float* bpw1;                // interleaved the same way
    const float *wdw, *bdw;           // [d, K], [d]
    const float *aconv_ln_g, *aconv_ln_b;
    const __half* wpw2;
    const float* bpw2;
    const float *ffn2_ln_g, *ffn2_ln_b, *ffn2_b1, *ffn2_b2;
    const __half *ffn2_w1, *ffn2_w2;
    const float *norm2_g, *norm2_b;
};

struct DecLayerW {
    const float *n1g, *n1b, *n2g, *n2b, *n3g, *n3b;
    const __half *w_self_in, *w_self_out, *w_cross_q, *w_cross_out, *w_ffn1, *w_ffn2;
    const float *b_self_in, *b_self_out, *b_cross_q, *b_cross_out, *b_ffn1, *b_ffn2;
};

struct LmLayerW {
    const __half *w_in, *w_out, *w1, *w2;
    const float *b_in, *b_out, *b1, *b2, *n1g, *n1b, *n2g, *n2b;
};

struct Arena {
    uint8_t* base = nullptr;
    size_t cap = 0, used = 0;
    void* take(size_t bytes) {
        const size_t off = (used + 255) & ~size_t(255);
        if (off + bytes > cap) return nullptr;
        used = off + bytes;
        return base + off;
    }
};

struct AsrModel {
    sbk_asr_config cfg;
    Fbank* fbank = nullptr;
    Arena warena;  // weights
    Arena ws;      // workspace (re-carved per shape)
    // frontend
    const float *glob_mean = nullptr, *glob_std = nullptr;
    const float *c1_w, *c1_b, *c1_g, *c1_be, *c2_b, *c2_g, *c2_be;
    const __half* c2_w;
    // encoder
    const __half* w_in; const float* b_in;
    std::vector<EncLayerW> enc;
    const float *enc_norm_g, *enc_norm_b;
    const float *rope_cos = nullptr, *rope_sin = nullptr;  // [max_len, dh/2]
    const __half* relpos_pe = nullptr;                     // [max_len, d] rows = |r|
    int pos_len = 0;
    // decoder
    const float* emb; const float* dec_pe;
    std::vector<DecLayerW> dec;
    const __half* w_ckv; const float* b_ckv;  // [L*2d, d]
    const float *dec_norm_g, *dec_norm_b;
    const __half* w_lin; const float* b_lin;
    const __half* w_ctc = nullptr; const float* b_ctc = nullptr;
    // TransformerLM scorer (optional part)
    bool has_lm = false;
    const float *lm_emb = nullptr, *lm_pe = nullptr;
    std::vector<LmLayerW> lm;
    const float *lm_norm_g, *lm_norm_b, *lm_bp0, *lm_lnp_g, *lm_lnp_b, *lm_bp2;
    const __half *lm_wp0, *lm_wp2;
    // CTC prefix scorer state (allocated on the first beam search that uses it): x [B, T, V] masked log-posteriors,
    // xb [B, T], rsum/rb [2][rows, T] and psi [2][rows] ping-pong by step parity, add [rows, V] when there is no LM buffer
    struct CtcBuf { float* base = nullptr; size_t cap = 0; float *x, *xlin, *xb, *rsum, *rb, *psi, *add, *tab, *tabM; } ctc;
    struct CovBuf { float* base = nullptr; size_t cap = 0; } cov;  // CoverageScorer: [2][rows][T] coverage + [rows] scores
    // TransformerLM whole-sequence forward (run_lm_forward), carved for `rows` = n * s token rows, independent of the
    // decode / beam workspace: residual stream x [rows, d] fp32, its fp16 copy x16, qkv16 [rows, 3d], att16 [rows, d],
    // f16 [rows, d_ffn]
    struct LmFwdBuf {
        uint8_t* base = nullptr; size_t cap = 0; int rows = 0;
        float* x; __half *x16, *qkv16, *att16, *f16;
    } lmf;
    // shapes the workspace is carved for
    int wsB = 0, wsL = 0, ws_rows = 0, ws_steps = 0;
    struct Buf {
        float *wav, *feats, *x, *glu, *enc_out, *act1_f, *cnn_f, *dx, *logits, *score, *seq_scores, *lnout, *beam_scr;
        int *utt_max, *enc_len, *tokens, *step, *has_ended, *ended_count, *pred, *lineage, *finished, *hist_tok, *hist_pred;
        float *hist_score, *hist_lp;
        float* rel_len;
        float *lx, *lh32, *lm_logits, *lm_extra;
        __half *lx16, *lq16, *latt16, *lf16, *lh16, *lkc, *lvc;
        int* tok_cache;
        __half *act1, *a_in, *h16, *f16, *qkv16, *att16, *P16, *enc16, *ckv16, *kcache, *vcache, *dh16, *dq16, *datt16, *df16;
    } b;
    cudaGraphExec_t step_graph = nullptr;
    int graph_rows = -1, graph_T = -1, graph_B = -1, graph_eos = -1, graph_S = -1;
    long long graph_nodes = 0;
    int* host_flag = nullptr;  // pinned
    struct GroupKey { const void *wav[16], *rel[16], *pred[16]; int G, B, L, steps, bos, eos; };
    GroupKey group_key{};
    cudaGraphExec_t group_graph = nullptr;
    long long group_nodes = 0;
    // host-buffer group entry point: device staging of the G batches' wav / lengths, a copy stream forked from the caller's
    // stream (so batch g+1's H2D overlaps batch g's encoder) and its own graph (H2D / D2H memcpy nodes included)
    float* gwav = nullptr; float* grel = nullptr; size_t gwav_cap = 0;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_ready[16] = {};
    cudaStream_t side_stream = nullptr;     // beam search: the LM scorer's branch of a search step
    cudaStream_t dec_stream = nullptr;      // group calls: the decode loop, on a high-priority stream (see transcribe_group_enqueue)
    cudaEvent_t ev_dfork = nullptr, ev_djoin = nullptr;
    cudaEvent_t ev_bfork = nullptr, ev_bjoin = nullptr;
    struct HostGroupKey { const void *wav[16], *rel[16], *pred[16], *pred_dev[16]; int G, B, L, steps, bos, eos; };
    HostGroupKey hgroup_key{};
    cudaGraphExec_t hgroup_graph = nullptr;
    long long hgroup_nodes = 0;
    // beam search: ONE graph of a whole search step (decoder layers + LM step + CTC scorer + beam kernel), replayed per step
    struct BeamKey { sbk_beam_params p; int B, T, rows, S_max, fuse_ln, tc_rows, fork; };
    BeamKey beam_key{};
    cudaGraphExec_t beam_graph = nullptr;
    long long beam_nodes = 0;
    struct PipeKey { const void *wav, *rel, *enc, *pred, *score; int B, L, steps, bos, eos; };
    PipeKey pipe_key{};
    cudaGraphExec_t pipe_graph = nullptr;
    long long pipe_nodes = 0;
    int* weight_refs = nullptr;  // weights (arena + fbank plan) are shared between a handle and its clones (lanes)
    int dec_tc_rows = getenv("SBK_DEC_TC_ROWS") ? atoi(getenv("SBK_DEC_TC_ROWS")) : 64;  // >= this many live hypotheses: wgmma decode GEMMs
    int dyn_chunk = 0, dyn_left = -1;  // DynChunkTrainConfig of the next encode calls (chunk frames, left-context chunks; 0 = off)
    int fuse_dec_ln = 1;         // 1: LayerNorm inside the projection kernel (latency); 0: separate LN kernel (throughput)
    int poll_every = 8;          // greedy early-exit poll interval in steps; 0 = never sync, run exactly max_steps
    bool has_fbank = false, has_cnn = false, has_enc = false, has_dec = false;
    cudaStream_t cap_stream = nullptr;  // private stream for graph capture (the legacy default stream cannot capture)
};

static const float* find(const std::map<std::string, std::pair<const float*, int64_t>>& m, const std::string& k,
                         int64_t numel, bool required = true) {
    auto it = m.find(k);
    if (it == m.end()) {
        if (required) set_error("missing weight '%s'", k.c_str());
        return nullptr;
    }
    if (numel >= 0 && it->second.second != numel) {
        set_error("weight '%s' has %lld elements, expected %lld", k.c_str(), (long long)it->second.second, (long long)numel);
        return nullptr;
    }
    return it->second.first;
}

struct Packer {
    AsrModel* m;
    const std::map<std::string, std::pair<const float*, int64_t>>* w;
    bool ok = true;
    std::vector<float> tmpf;
    std::vector<__half> tmph;
    const float* f32(const std::string& k, int64_t n) {
        const float* src = find(*w, k, n);
        if (!src) { ok = false; return nullptr; }
        return f32_raw(src, n);
    }
    const float* f32_raw(const float* src, int64_t n) {
        void* d = m->warena.take(n * 4);
        if (!d) { ok = false; set_error("weight arena exhausted"); return nullptr; }
        if (cudaMemcpy(d, src, n * 4, cudaMemcpyHostToDevice) != cudaSuccess) { ok = false; set_error("weight upload failed"); }
        return reinterpret_cast<const float*>(d);
    }
    const __half* f16_raw(const float* src, int64_t n, float scale = 1.0f) {
        tmph.resize(n);
        for (int64_t i = 0; i < n; ++i) tmph[i] = __float2half_rn(src[i] * scale);
        void* d = m->warena.take(n * 2);
        if (!d) { ok = false; set_error("weight arena exhausted"); return nullptr; }
        if (cudaMemcpy(d, tmph.data(), n * 2, cudaMemcpyHostToDevice) != cudaSuccess) { ok = false; set_error("weight upload failed"); }
        return reinterpret_cast<const __half*>(d);
    }
    const __half* f16(const std::string& k, int64_t n) {
        const float* src = find(*w, k, n);
        if (!src) { ok = false; return nullptr; }
        return f16_raw(src, n);
    }
};

static size_t weight_arena_bytes(const sbk_asr_config& c) {
    const size_t d = c.d_model, f = c.d_ffn;
    size_t enc = (size_t)c.num_encoder_layers * (4 * d * f + 3 * d * d + d * d + d * d + 2 * d * d + d * d) * 2;
    size_t dec = (size_t)c.num_decoder_layers * (3 * d * d + d * d + 3 * d * d + d * d + 2 * d * f) * 2;
    size_t misc = (size_t)c.vocab * d * (4 + 2 + 2) + (size_t)c.max_len * d * (4 + 2) + (size_t)c.input_size * d * 2;
    size_t lm = 0;
    if (c.parts & SBK_PART_LM) {
        const size_t dl = c.lm_d_model, fl = c.lm_d_ffn;
        lm = (size_t)c.lm_layers * (4 * dl * dl + 2 * dl * fl) * 2 + (size_t)c.vocab * dl * (4 + 2) + dl * dl * 2 +
             (size_t)c.max_len * dl * 4 + (8u << 20);
    }
    return enc + dec + misc + lm + (64u << 20);
}

int asr_create(const sbk_asr_config* cfg, const sbk_tensor* weights, int n_weights, AsrModel** out) {
    SBK_REQUIRE(cfg && weights && out, "asr_create: null argument");
    const sbk_asr_config& c = *cfg;
    SBK_REQUIRE(c.d_model % 8 == 0 && c.d_model % c.nhead == 0, "asr_create: bad d_model/nhead");
    SBK_REQUIRE(c.attention_type == SBK_ATT_ROPE || c.attention_type == SBK_ATT_RELPOS,
                "asr_create: attention_type must be RoPEMHA or RelPosMHAXL");
    const int d = c.d_model, dh = d / c.nhead, F = c.d_ffn, K = c.kernel_size;
    SBK_REQUIRE(dh == 64 || dh == 36 || dh == 32, "asr_create: encoder head_dim=%d not built (64, 36, 32)", dh);
    SBK_REQUIRE(!((c.parts & SBK_PART_DECODER) && c.num_decoder_layers > 0) || (dh <= 64 && dh % 4 == 0 && d % 16 == 0),
                "asr_create: decoder head_dim must be a multiple of 4 up to 64 and d_model a multiple of 16 (got %d, %d)", dh, d);
    SBK_REQUIRE(c.attention_type != SBK_ATT_ROPE || dh % 32 == 0, "asr_create: RoPEMHA needs head_dim %% 32 == 0");
    std::map<std::string, std::pair<const float*, int64_t>> w;
    for (int i = 0; i < n_weights; ++i) w[weights[i].name] = {weights[i].data, weights[i].numel};

    AsrModel* m = new AsrModel();
    m->cfg = c;
    m->warena.cap = weight_arena_bytes(c);
    if (cudaMalloc(&m->warena.base, m->warena.cap) != cudaSuccess) {
        set_error("asr_create: cudaMalloc(%zu) for weights failed", m->warena.cap);
        delete m;
        return SBK_ERR_NOMEM;
    }
    Packer p{m, &w};
    int rc = SBK_OK;
    const bool has_fbank = c.parts & SBK_PART_FBANK, has_cnn = c.parts & SBK_PART_CNN;
    const bool has_enc = (c.parts & SBK_PART_ENCODER) && c.num_encoder_layers >= 0;
    const bool has_dec = (c.parts & SBK_PART_DECODER) && c.num_decoder_layers > 0;
    m->has_fbank = has_fbank; m->has_cnn = has_cnn; m->has_enc = has_enc; m->has_dec = has_dec;
    // ---- Fbank + CMVN
    if (has_fbank) {
        const float* win = find(w, "fbank.window", c.n_fft);
        const float* mel = find(w, "fbank.mel_matrix", (int64_t)(c.n_fft / 2 + 1) * c.n_mels);
        if (!win || !mel) { rc = SBK_ERR_ARG; goto fail; }
        rc = fbank_create(&m->fbank, c.n_fft, c.hop, c.n_mels, win, mel, c.fbank_amin > 0.0f ? c.fbank_amin : 1e-10f,
                          c.fbank_top_db > 0.0f ? c.fbank_top_db : 80.0f);
        if (rc) goto fail;
        if (w.count("normalize.glob_mean")) {
            m->glob_mean = p.f32("normalize.glob_mean", c.n_mels);
            m->glob_std = p.f32("normalize.glob_std", c.n_mels);
        }
    }
    // ---- CNN front-end
    if (has_cnn) {
        const int F1 = (c.n_mels - 1) / 2 + 1, F2 = (F1 - 1) / 2 + 1;
        if (F2 * c.cnn_c2 != c.input_size) { set_error("asr_create: CNN output %d != input_size %d", F2 * c.cnn_c2, c.input_size); rc = SBK_ERR_ARG; goto fail; }
        m->c1_w = p.f32("CNN.convblock_0.convs.conv_0.conv.weight", (int64_t)c.cnn_c1 * 9);
        m->c1_b = p.f32("CNN.convblock_0.convs.conv_0.conv.bias", c.cnn_c1);
        m->c1_g = p.f32("CNN.convblock_0.convs.norm_0.norm.weight", (int64_t)F1 * c.cnn_c1);
        m->c1_be = p.f32("CNN.convblock_0.convs.norm_0.norm.bias", (int64_t)F1 * c.cnn_c1);
        const float* w2 = find(w, "CNN.convblock_1.convs.conv_0.conv.weight", (int64_t)c.cnn_c2 * c.cnn_c1 * 9);
        if (!w2) { rc = SBK_ERR_ARG; goto fail; }
        std::vector<float> w2p((size_t)c.cnn_c2 * 9 * c.cnn_c1);
        for (int o = 0; o < c.cnn_c2; ++o)
            for (int ch = 0; ch < c.cnn_c1; ++ch)
                for (int kf = 0; kf < 3; ++kf)
                    for (int kt = 0; kt < 3; ++kt)
                        w2p[((size_t)o * 9 + kf * 3 + kt) * c.cnn_c1 + ch] = w2[(((size_t)o * c.cnn_c1 + ch) * 3 + kf) * 3 + kt];
        m->c2_w = p.f16_raw(w2p.data(), w2p.size());
        m->c2_b = p.f32("CNN.convblock_1.convs.conv_0.conv.bias", c.cnn_c2);
        m->c2_g = p.f32("CNN.convblock_1.convs.norm_0.norm.weight", (int64_t)F2 * c.cnn_c2);
        m->c2_be = p.f32("CNN.convblock_1.convs.norm_0.norm.bias", (int64_t)F2 * c.cnn_c2);
    }
    // ---- encoder
    if (has_enc) {
    m->w_in = p.f16("Transformer.custom_src_module.layers.0.w.weight", (int64_t)d * c.input_size);
    m->b_in = p.f32("Transformer.custom_src_module.layers.0.w.bias", d);
    m->enc.resize(c.num_encoder_layers);
    for (int l = 0; l < c.num_encoder_layers && p.ok; ++l) {
        const std::string q = "Transformer.encoder.layers." + std::to_string(l) + ".";
        EncLayerW& e = m->enc[l];
        e.ffn1_ln_g = p.f32(q + "ffn_module1.0.weight", d); e.ffn1_ln_b = p.f32(q + "ffn_module1.0.bias", d);
        e.ffn1_w1 = p.f16(q + "ffn_module1.1.ffn.0.weight", (int64_t)F * d); e.ffn1_b1 = p.f32(q + "ffn_module1.1.ffn.0.bias", F);
        e.ffn1_w2 = p.f16(q + "ffn_module1.1.ffn.3.weight", (int64_t)d * F); e.ffn1_b2 = p.f32(q + "ffn_module1.1.ffn.3.bias", d);
        e.norm1_g = p.f32(q + "norm1.norm.weight", d); e.norm1_b = p.f32(q + "norm1.norm.bias", d);
        e.wqkv = p.f16(q + "mha_layer.in_proj_weight", (int64_t)3 * d * d);
        e.wo = p.f16(q + "mha_layer.out_proj.weight", (int64_t)d * d); e.bo = p.f32(q + "mha_layer.out_proj.bias", d);
        e.wpos = nullptr; e.pos_u = e.pos_v = nullptr;
        if (c.attention_type == SBK_ATT_RELPOS) {
            e.wpos = p.f16(q + "mha_layer.linear_pos.weight", (int64_t)d * d);
            e.pos_u = p.f32(q + "mha_layer.pos_bias_u", d); e.pos_v = p.f32(q + "mha_layer.pos_bias_v", d);
        }
        e.conv_ln_g = p.f32(q + "convolution_module.layer_norm.weight", d); e.conv_ln_b = p.f32(q + "convolution_module.layer_norm.bias", d);
        {   // pointwise conv 1 (Conv1d k=1, weight (2d, d, 1)): interleave 16 value rows / 16 gate rows for the GLU epilogue
            const float* src = find(w, q + "convolution_module.bottleneck.0.weight", (int64_t)2 * d * d);
            const float* bs = find(w, q + "convolution_module.bottleneck.0.bias", 2 * d);
            if (!src || !bs) { p.ok = false; break; }
            std::vector<float> wi((size_t)2 * d * d), bi(2 * d);
            for (int ch = 0; ch < d; ++ch) {
                const int blk = ch / 16, j = ch % 16;
                memcpy(&wi[((size_t)blk * 32 + j) * d], &src[(size_t)ch * d], d * 4);
                memcpy(&wi[((size_t)blk * 32 + 16 + j) * d], &src[(size_t)(d + ch) * d], d * 4);
                bi[blk * 32 + j] = bs[ch];
                bi[blk * 32 + 16 + j] = bs[d + ch];
            }
            e.wpw1 = p.f16_raw(wi.data(), wi.size());
            e.bpw1 = p.f32_raw(bi.data(), bi.size());
        }
        {   // depthwise taps (d, 1, K) -> tap-major [K, d] so that a warp's channels read one cache line per tap
            const float* src = find(w, q + "convolution_module.conv.weight", (int64_t)d * K);
            if (!src) { p.ok = false; break; }
            std::vector<float> wt((size_t)K * d);
            for (int ch = 0; ch < d; ++ch)
                for (int k = 0; k < K; ++k) wt[(size_t)k * d + ch] = src[(size_t)ch * K + k];
            e.wdw = p.f32_raw(wt.data(), wt.size());
        }
        e.bdw = p.f32(q + "convolution_module.conv.bias", d);
        e.aconv_ln_g = p.f32(q + "convolution_module.after_conv.0.weight", d); e.aconv_ln_b = p.f32(q + "convolution_module.after_conv.0.bias", d);
        e.wpw2 = p.f16(q + "convolution_module.after_conv.2.weight", (int64_t)d * d); e.bpw2 = p.f32(q + "convolution_module.after_conv.2.bias", d);
        e.ffn2_ln_g = p.f32(q + "ffn_module2.0.weight", d); e.ffn2_ln_b = p.f32(q + "ffn_module2.0.bias", d);
        e.ffn2_w1 = p.f16(q + "ffn_module2.1.ffn.0.weight", (int64_t)F * d); e.ffn2_b1 = p.f32(q + "ffn_module2.1.ffn.0.bias", F);
        e.ffn2_w2 = p.f16(q + "ffn_module2.1.ffn.3.weight", (int64_t)d * F); e.ffn2_b2 = p.f32(q + "ffn_module2.1.ffn.3.bias", d);
        e.norm2_g = p.f32(q + "norm2.norm.weight", d); e.norm2_b = p.f32(q + "norm2.norm.bias", d);
    }
    if (!p.ok) { rc = SBK_ERR_ARG; goto fail; }
    m->enc_norm_g = p.f32("Transformer.encoder.norm.norm.weight", d);
    m->enc_norm_b = p.f32("Transformer.encoder.norm.norm.bias", d);
    // positional tables
    m->pos_len = c.max_len;
    if (c.attention_type == SBK_ATT_ROPE) {
        // nnet/attention.py:1012-1055: angle_{t,i} = t * exp(-2i * ln(1e4) / d_h), computed in fp32 like the reference
        std::vector<float> cs((size_t)c.max_len * dh / 2), sn(cs.size());
        for (int i = 0; i < dh / 2; ++i) {
            const float ang = expf((float)(2 * i) * -(logf(10000.0f) / (float)dh));
            for (int t = 0; t < c.max_len; ++t) {
                const float ta = (float)t * ang;
                cs[(size_t)t * (dh / 2) + i] = cosf(ta);
                sn[(size_t)t * (dh / 2) + i] = sinf(ta);
            }
        }
        m->rope_cos = p.f32_raw(cs.data(), cs.size());
        m->rope_sin = p.f32_raw(sn.data(), sn.size());
    } else {
        // nnet/attention.py:360-408: row |r|: even cols sin(|r| f_i), odd cols cos(|r| f_i)
        std::vector<float> pe((size_t)c.max_len * d);
        for (int i = 0; i < d / 2; ++i) {
            const float fr = expf((float)(2 * i) * -(logf(10000.0f) / (float)d));
            for (int t = 0; t < c.max_len; ++t) {
                pe[(size_t)t * d + 2 * i] = sinf((float)t * fr);
                pe[(size_t)t * d + 2 * i + 1] = cosf((float)t * fr);
            }
        }
        m->relpos_pe = p.f16_raw(pe.data(), pe.size());
    }
    }  // has_enc
    // ---- decoder
    if (has_dec) {
        m->emb = p.f32("Transformer.custom_tgt_module.layers.0.emb.Embedding.weight", (int64_t)c.vocab * d);
        {
            std::vector<float> pe((size_t)c.max_len * d);  // Transformer.py:252-303
            for (int i = 0; i < d / 2; ++i) {
                const float den = expf((float)(2 * i) * -(logf(10000.0f) / (float)d));
                for (int t = 0; t < c.max_len; ++t) {
                    pe[(size_t)t * d + 2 * i] = sinf((float)t * den);
                    pe[(size_t)t * d + 2 * i + 1] = cosf((float)t * den);
                }
            }
            m->dec_pe = p.f32_raw(pe.data(), pe.size());
        }
        const int L = c.num_decoder_layers;
        m->dec.resize(L);
        std::vector<float> wckv((size_t)L * 2 * d * d), bckv((size_t)L * 2 * d);
        const float qs = 1.0f / sqrtf((float)dh);
        for (int l = 0; l < L && p.ok; ++l) {
            const std::string q = "Transformer.decoder.layers." + std::to_string(l) + ".";
            DecLayerW& e = m->dec[l];
            e.n1g = p.f32(q + "norm1.norm.weight", d); e.n1b = p.f32(q + "norm1.norm.bias", d);
            e.n2g = p.f32(q + "norm2.norm.weight", d); e.n2b = p.f32(q + "norm2.norm.bias", d);
            e.n3g = p.f32(q + "norm3.norm.weight", d); e.n3b = p.f32(q + "norm3.norm.bias", d);
            const float* wi = find(w, q + "self_attn.att.in_proj_weight", (int64_t)3 * d * d);
            const float* bi = find(w, q + "self_attn.att.in_proj_bias", 3 * d);
            const float* wc = find(w, q + "multihead_attn.att.in_proj_weight", (int64_t)3 * d * d);
            const float* bc = find(w, q + "multihead_attn.att.in_proj_bias", 3 * d);
            if (!wi || !bi || !wc || !bc) { p.ok = false; break; }
            {   // fold 1/sqrt(d_h) into the query rows
                std::vector<float> ws(wi, wi + (size_t)3 * d * d), bs(bi, bi + 3 * d);
                for (size_t i = 0; i < (size_t)d * d; ++i) ws[i] *= qs;
                for (int i = 0; i < d; ++i) bs[i] *= qs;
                e.w_self_in = p.f16_raw(ws.data(), ws.size());
                e.b_self_in = p.f32_raw(bs.data(), bs.size());
                std::vector<float> wq(wc, wc + (size_t)d * d), bq(bc, bc + d);
                for (auto& v : wq) v *= qs;
                for (auto& v : bq) v *= qs;
                e.w_cross_q = p.f16_raw(wq.data(), wq.size());
                e.b_cross_q = p.f32_raw(bq.data(), bq.size());
            }
            memcpy(&wckv[(size_t)l * 2 * d * d], wc + (size_t)d * d, (size_t)2 * d * d * 4);
            memcpy(&bckv[(size_t)l * 2 * d], bc + d, (size_t)2 * d * 4);
            e.w_self_out = p.f16(q + "self_attn.att.out_proj.weight", (int64_t)d * d); e.b_self_out = p.f32(q + "self_attn.att.out_proj.bias", d);
            e.w_cross_out = p.f16(q + "multihead_attn.att.out_proj.weight", (int64_t)d * d); e.b_cross_out = p.f32(q + "multihead_attn.att.out_proj.bias", d);
            e.w_ffn1 = p.f16(q + "pos_ffn.ffn.0.weight", (int64_t)F * d); e.b_ffn1 = p.f32(q + "pos_ffn.ffn.0.bias", F);
            e.w_ffn2 = p.f16(q + "pos_ffn.ffn.3.weight", (int64_t)d * F); e.b_ffn2 = p.f32(q + "pos_ffn.ffn.3.bias", d);
        }
        if (!p.ok) { rc = SBK_ERR_ARG; goto fail; }
        m->w_ckv = p.f16_raw(wckv.data(), wckv.size());
        m->b_ckv = p.f32_raw(bckv.data(), bckv.size());
        m->dec_norm_g = p.f32("Transformer.decoder.norm.norm.weight", d);
        m->dec_norm_b = p.f32("Transformer.decoder.norm.norm.bias", d);
        m->w_lin = nullptr; m->b_lin = nullptr;
        if (w.count("seq_lin.w.weight")) {  // the output head belongs to the searchers; TransformerASR.decode runs without it
            m->w_lin = p.f16("seq_lin.w.weight", (int64_t)c.vocab * d);
            m->b_lin = p.f32("seq_lin.w.bias", c.vocab);
        }
    }
    if ((c.parts & SBK_PART_LM) && c.lm_layers > 0) {
        const int dl = c.lm_d_model, Fl = c.lm_d_ffn, dhl = dl / c.lm_nhead;
        if (dhl != 64 || dl % 128 != 0) { set_error("asr_create: LM head_dim must be 64 and d_model %% 128 == 0"); rc = SBK_ERR_UNSUPPORTED; goto fail; }
        m->has_lm = true;
        m->lm_emb = p.f32("lm.custom_src_module.emb.Embedding.weight", (int64_t)c.vocab * dl);
        {
            std::vector<float> pe((size_t)c.max_len * dl);
            for (int i = 0; i < dl / 2; ++i) {
                const float den = expf((float)(2 * i) * -(logf(10000.0f) / (float)dl));
                for (int t = 0; t < c.max_len; ++t) {
                    pe[(size_t)t * dl + 2 * i] = sinf((float)t * den);
                    pe[(size_t)t * dl + 2 * i + 1] = cosf((float)t * den);
                }
            }
            m->lm_pe = p.f32_raw(pe.data(), pe.size());
        }
        m->lm.resize(c.lm_layers);
        const float qs = 1.0f / sqrtf((float)dhl);
        for (int l = 0; l < c.lm_layers && p.ok; ++l) {
            const std::string q = "lm.encoder.layers." + std::to_string(l) + ".";
            LmLayerW& e = m->lm[l];
            const float* wi = find(w, q + "self_att.att.in_proj_weight", (int64_t)3 * dl * dl);
            const float* bi = find(w, q + "self_att.att.in_proj_bias", 3 * dl);
            if (!wi || !bi) { p.ok = false; break; }
            std::vector<float> ws(wi, wi + (size_t)3 * dl * dl), bs(bi, bi + 3 * dl);
            for (size_t i = 0; i < (size_t)dl * dl; ++i) ws[i] *= qs;  // fold 1/sqrt(d_h) into the query rows
            for (int i = 0; i < dl; ++i) bs[i] *= qs;
            e.w_in = p.f16_raw(ws.data(), ws.size());
            e.b_in = p.f32_raw(bs.data(), bs.size());
            e.w_out = p.f16(q + "self_att.att.out_proj.weight", (int64_t)dl * dl); e.b_out = p.f32(q + "self_att.att.out_proj.bias", dl);
            e.w1 = p.f16(q + "pos_ffn.ffn.0.weight", (int64_t)Fl * dl); e.b1 = p.f32(q + "pos_ffn.ffn.0.bias", Fl);
            e.w2 = p.f16(q + "pos_ffn.ffn.3.weight", (int64_t)dl * Fl); e.b2 = p.f32(q + "pos_ffn.ffn.3.bias", dl);
            e.n1g = p.f32(q + "norm1.norm.weight", dl); e.n1b = p.f32(q + "norm1.norm.bias", dl);
            e.n2g = p.f32(q + "norm2.norm.weight", dl); e.n2b = p.f32(q + "norm2.norm.bias", dl);
        }
        m->lm_norm_g = p.f32("lm.encoder.norm.norm.weight", dl); m->lm_norm_b = p.f32("lm.encoder.norm.norm.bias", dl);
        m->lm_wp0 = p.f16("lm.output_proj.layers.0.w.weight", (int64_t)dl * dl); m->lm_bp0 = p.f32("lm.output_proj.layers.0.w.bias", dl);
        m->lm_lnp_g = p.f32("lm.output_proj.layers.1.norm.weight", dl); m->lm_lnp_b = p.f32("lm.output_proj.layers.1.norm.bias", dl);
        m->lm_wp2 = p.f16("lm.output_proj.layers.2.w.weight", (int64_t)c.vocab * dl); m->lm_bp2 = p.f32("lm.output_proj.layers.2.w.bias", c.vocab);
        if (!p.ok) { rc = SBK_ERR_ARG; goto fail; }
    }
    if (w.count("ctc_lin.w.weight")) {
        m->w_ctc = p.f16("ctc_lin.w.weight", (int64_t)c.vocab * d);
        m->b_ctc = p.f32("ctc_lin.w.bias", c.vocab);
    }
    if (!p.ok) { rc = SBK_ERR_ARG; goto fail; }
    if (cudaMallocHost(&m->host_flag, 64) != cudaSuccess) { set_error("cudaMallocHost failed"); rc = SBK_ERR_NOMEM; goto fail; }
    m->weight_refs = new int(1);
    if (cudaDeviceSynchronize() != cudaSuccess) { set_error("asr_create: device error after upload"); rc = SBK_ERR_CUDA; goto fail; }
    *out = m;
    return SBK_OK;
fail:
    if (m->fbank) fbank_destroy(m->fbank);
    cudaFree(m->warena.base);
    delete m;
    return rc;
}

// A clone shares the repacked weights but owns its workspace, decode graph and flags: one clone per in-flight
// batch ("lane") lets independent batches overlap on different streams (the decode loop is latency-bound and
// leaves most SMs idle, so concurrent lanes raise throughput without touching per-batch numerics).
int asr_clone(AsrModel* src, AsrModel** out) {
    SBK_REQUIRE(src && out, "asr_clone: null argument");
    AsrModel* m = new AsrModel(*src);
    m->ws = Arena();
    m->wsB = m->wsL = m->ws_rows = m->ws_steps = 0;
    m->b = AsrModel::Buf();
    m->ctc = AsrModel::CtcBuf();
    m->cov = AsrModel::CovBuf();
    m->lmf = AsrModel::LmFwdBuf();
    m->step_graph = nullptr;
    m->pipe_graph = nullptr;
    m->group_graph = nullptr;
    m->hgroup_graph = nullptr;
    m->beam_graph = nullptr;
    m->gwav = m->grel = nullptr; m->gwav_cap = 0;
    m->copy_stream = nullptr; m->ev_fork = nullptr;
    for (auto& e : m->ev_ready) e = nullptr;
    m->graph_rows = m->graph_T = m->graph_B = -1;
    m->cap_stream = nullptr;
    m->host_flag = nullptr;
    if (cudaMallocHost(&m->host_flag, 64) != cudaSuccess) {
        delete m;
        set_error("asr_clone: cudaMallocHost failed");
        return SBK_ERR_NOMEM;
    }
    ++*m->weight_refs;
    *out = m;
    return SBK_OK;
}

void asr_destroy(AsrModel* m) {
    if (!m) return;
    if (m->step_graph) cudaGraphExecDestroy(m->step_graph);
    if (m->pipe_graph) cudaGraphExecDestroy(m->pipe_graph);
    if (m->group_graph) cudaGraphExecDestroy(m->group_graph);
    if (m->hgroup_graph) cudaGraphExecDestroy(m->hgroup_graph);
    if (m->beam_graph) cudaGraphExecDestroy(m->beam_graph);
    cudaFree(m->gwav);
    if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
    if (m->ev_fork) cudaEventDestroy(m->ev_fork);
    for (auto e : m->ev_ready) if (e) cudaEventDestroy(e);
    if (m->weight_refs && --*m->weight_refs == 0) {
        if (m->fbank) fbank_destroy(m->fbank);
        cudaFree(m->warena.base);
        delete m->weight_refs;
    }
    cudaFree(m->ws.base);
    cudaFree(m->ctc.base);
    cudaFree(m->cov.base);
    cudaFree(m->lmf.base);
    if (m->host_flag) cudaFreeHost(m->host_flag);
    if (m->cap_stream) cudaStreamDestroy(m->cap_stream);
    if (m->side_stream) cudaStreamDestroy(m->side_stream);
    if (m->dec_stream) cudaStreamDestroy(m->dec_stream);
    if (m->ev_dfork) cudaEventDestroy(m->ev_dfork);
    if (m->ev_djoin) cudaEventDestroy(m->ev_djoin);
    if (m->ev_bfork) cudaEventDestroy(m->ev_bfork);
    if (m->ev_bjoin) cudaEventDestroy(m->ev_bjoin);
    delete m;
}

// cached graphs bake in workspace pointers / kernel choices: drop them whenever either changes
static void drop_graphs(AsrModel* m) {
    if (m->step_graph) { cudaGraphExecDestroy(m->step_graph); m->step_graph = nullptr; m->graph_rows = -1; }
    if (m->pipe_graph) { cudaGraphExecDestroy(m->pipe_graph); m->pipe_graph = nullptr; }
    if (m->group_graph) { cudaGraphExecDestroy(m->group_graph); m->group_graph = nullptr; }
    if (m->hgroup_graph) { cudaGraphExecDestroy(m->hgroup_graph); m->hgroup_graph = nullptr; }
    if (m->beam_graph) { cudaGraphExecDestroy(m->beam_graph); m->beam_graph = nullptr; }
}

static void frames(const sbk_asr_config& c, int L, int* T0, int* T1, int* T2) {
    *T0 = 1 + L / c.hop;
    *T1 = (*T0 - 1) / 2 + 1;
    *T2 = (*T1 - 1) / 2 + 1;
}

// (Re)carve the workspace for a batch of B utterances of L samples, `rows` decoder hypotheses, `steps` max steps.
static int ensure_workspace(AsrModel* m, int B, int L, int rows, int steps) {
    if (m->ws.base && B <= m->wsB && L <= m->wsL && rows <= m->ws_rows && steps <= m->ws_steps) return SBK_OK;
    B = std::max(B, m->wsB); L = std::max(L, m->wsL); rows = std::max(rows, m->ws_rows); steps = std::max(steps, m->ws_steps);
    const sbk_asr_config& c = m->cfg;
    int T0, T1, T2;
    frames(c, L, &T0, &T1, &T2);
    const int F1 = (c.n_mels - 1) / 2 + 1;
    const size_t M = (size_t)B * T2, d = c.d_model, F = c.d_ffn, Ld = c.num_decoder_layers, S = steps + 1;
    const size_t Md = (size_t)std::max(B, rows) * T2;  // encoder states / cross K,V of every utterance the decoder sees
    size_t need = 0;
    auto sz = [&](size_t bytes) { need += (bytes + 255) & ~size_t(255); };
    sz((size_t)B * L * 4); sz((size_t)B * T0 * c.n_mels * 4); sz(M * d * 4); sz(M * d * 4); sz(Md * d * 4);
    sz((size_t)B * T1 * F1 * c.cnn_c1 * 4); sz(M * c.input_size * 4); sz((size_t)rows * d * 4);
    sz((size_t)rows * c.vocab * 4); sz((size_t)rows * S * 4);
    sz(B * 4); sz((size_t)std::max(B, rows) * 4); sz((size_t)rows * (S + 1) * 4); sz(rows * 4 + 64); sz(rows * 4); sz(64); sz((size_t)rows * S * 4); sz(B * 4);
    sz((size_t)B * T1 * F1 * c.cnn_c1 * 2); sz(M * c.input_size * 2); sz(M * d * 2); sz(M * F * 2); sz(M * 3 * d * 2);
    sz(M * d * 2); sz((size_t)T2 * d * 2); sz(Md * d * 2); sz(Md * Ld * 2 * d * 2);
    sz((size_t)Ld * rows * S * d * 2); sz((size_t)Ld * rows * S * d * 2);
    sz((size_t)rows * d * 2); sz((size_t)rows * d * 2); sz((size_t)rows * d * 2); sz((size_t)rows * F * 2);
    sz((size_t)2 * rows * S * 4); sz(B * 4 + 64); sz((size_t)2 * rows * 4); sz((size_t)rows * d * 4); sz((size_t)rows * 33 * 4);
    sz((size_t)rows * S * 4); sz((size_t)rows * S * 4); sz((size_t)rows * S * 4); sz((size_t)rows * S * 4);
    const size_t dl = m->has_lm ? c.lm_d_model : 0, Fl = m->has_lm ? c.lm_d_ffn : 0, Ll = m->has_lm ? c.lm_layers : 0;
    if (m->has_lm) {
        sz(rows * dl * 4); sz(rows * dl * 4); sz((size_t)rows * c.vocab * 4); sz((size_t)rows * c.vocab * 4);
        sz(rows * dl * 2); sz(rows * dl * 2); sz(rows * dl * 2); sz(rows * Fl * 2); sz(rows * dl * 2);
        sz(Ll * rows * S * dl * 2); sz(Ll * rows * S * dl * 2); sz((size_t)rows * S * 4);
    }
    need += 1 << 20;
    if (need > m->ws.cap) {
        if (m->ws.base) { cudaDeviceSynchronize(); cudaFree(m->ws.base); m->ws.base = nullptr; }
        if (cudaMalloc(&m->ws.base, need) != cudaSuccess) {
            m->ws.cap = 0;
            set_error("workspace cudaMalloc(%zu) failed", need);
            return SBK_ERR_NOMEM;
        }
        m->ws.cap = need;
    }
    drop_graphs(m);
    m->ws.used = 0;
    AsrModel::Buf& b = m->b;
#define TAKE(field, type, bytes) b.field = reinterpret_cast<type*>(m->ws.take(bytes))
    TAKE(wav, float, (size_t)B * L * 4); TAKE(feats, float, (size_t)B * T0 * c.n_mels * 4); TAKE(x, float, M * d * 4);
    TAKE(glu, float, M * d * 4); TAKE(enc_out, float, Md * d * 4); TAKE(act1_f, float, (size_t)B * T1 * F1 * c.cnn_c1 * 4);
    TAKE(cnn_f, float, M * c.input_size * 4); TAKE(dx, float, (size_t)rows * d * 4); TAKE(logits, float, (size_t)rows * c.vocab * 4);
    TAKE(score, float, (size_t)rows * S * 4);
    TAKE(utt_max, int, B * 4); TAKE(enc_len, int, (size_t)std::max(B, rows) * 4); TAKE(tokens, int, (size_t)rows * (S + 1) * 4); TAKE(step, int, rows * 4 + 64);
    TAKE(has_ended, int, rows * 4); TAKE(ended_count, int, 64); TAKE(pred, int, (size_t)rows * S * 4); TAKE(rel_len, float, B * 4);
    TAKE(act1, __half, (size_t)B * T1 * F1 * c.cnn_c1 * 2); TAKE(a_in, __half, M * c.input_size * 2); TAKE(h16, __half, M * d * 2);
    TAKE(f16, __half, M * F * 2); TAKE(qkv16, __half, M * 3 * d * 2); TAKE(att16, __half, M * d * 2);
    TAKE(P16, __half, (size_t)T2 * d * 2); TAKE(enc16, __half, Md * d * 2); TAKE(ckv16, __half, Md * Ld * 2 * d * 2);
    TAKE(kcache, __half, (size_t)Ld * rows * S * d * 2); TAKE(vcache, __half, (size_t)Ld * rows * S * d * 2);
    TAKE(dh16, __half, (size_t)rows * d * 2); TAKE(dq16, __half, (size_t)rows * d * 2); TAKE(datt16, __half, (size_t)rows * d * 2);
    TAKE(df16, __half, (size_t)rows * F * 2);
    TAKE(lineage, int, (size_t)2 * rows * S * 4); TAKE(finished, int, B * 4 + 64); TAKE(seq_scores, float, (size_t)2 * rows * 4);
    TAKE(lnout, float, (size_t)rows * d * 4); TAKE(beam_scr, float, (size_t)rows * 33 * 4);
    TAKE(hist_tok, int, (size_t)rows * S * 4); TAKE(hist_pred, int, (size_t)rows * S * 4);
    TAKE(hist_score, float, (size_t)rows * S * 4); TAKE(hist_lp, float, (size_t)rows * S * 4);
    if (m->has_lm) {
        TAKE(lx, float, rows * dl * 4); TAKE(lh32, float, rows * dl * 4); TAKE(lm_logits, float, (size_t)rows * c.vocab * 4);
        TAKE(lm_extra, float, (size_t)rows * c.vocab * 4);
        TAKE(lx16, __half, rows * dl * 2); TAKE(lq16, __half, rows * dl * 2); TAKE(latt16, __half, rows * dl * 2);
        TAKE(lf16, __half, rows * Fl * 2); TAKE(lh16, __half, rows * dl * 2);
        TAKE(lkc, __half, Ll * rows * S * dl * 2); TAKE(lvc, __half, Ll * rows * S * dl * 2); TAKE(tok_cache, int, (size_t)rows * S * 4);
        if (!b.tok_cache) { set_error("workspace carve failed (LM)"); return SBK_ERR_NOMEM; }
    }
    if (!b.df16 || !b.seq_scores || !b.lnout || !b.hist_lp) { set_error("workspace carve failed"); return SBK_ERR_NOMEM; }
#undef TAKE
    m->wsB = B; m->wsL = L; m->ws_rows = rows; m->ws_steps = steps;
    return SBK_OK;
}

#define RC(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

// feats [B, T0, n_mels] fp32 (already normalised) -> enc_out fp32 [B, T2, d] (+ enc16). enc_len device int[B].
static int run_encoder(AsrModel* m, const float* feats, int B, int T0, const int* enc_len, float* cnn_out_f,
                       float* enc_out, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int T1 = (T0 - 1) / 2 + 1, T = feats ? (T1 - 1) / 2 + 1 : T0;  // feats == nullptr: b.a_in holds [B*T0, input_size]
    const int M = B * T, d = c.d_model, F = c.d_ffn, H = c.nhead, dh = d / H;
    SBK_REQUIRE(m->has_enc, "encode: this handle was created without encoder weights");
    SBK_REQUIRE(feats == nullptr || m->has_cnn, "encode: this handle was created without CNN weights");
    SBK_REQUIRE(T <= m->pos_len, "encode: %d frames exceed max_len=%d", T, m->pos_len);
    if (feats != nullptr)
        RC(cnn_frontend_forward(feats, B, T0, c.n_mels, m->c1_w, m->c1_b, m->c1_g, m->c1_be, c.cnn_c1, m->c2_w, m->c2_b,
                                m->c2_g, m->c2_be, c.cnn_c2, b.act1, nullptr, b.a_in, cnn_out_f, st));
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->b_in; e.out = b.x; e.ldo = d;
    RC(gemm_f16(b.a_in, c.input_size, m->w_in, c.input_size, e, M, d, c.input_size, st));
    const float att_scale = 1.0f / sqrtf((float)d);  // nnet/attention.py:521,1272: 1/sqrt(embed_dim), not head_dim
    for (int l = 0; l < c.num_encoder_layers; ++l) {
        const EncLayerW& w = m->enc[l];
        // --- ffn module 1 (Conformer.py:479); its LayerNorm was fused into the previous layer's norm2 kernel
        if (l == 0) RC(layernorm_rows(b.x, b.h16, true, w.ffn1_ln_g, w.ffn1_ln_b, M, d, 1e-5f, false, st));
        e = GemmEpilogue(); e.mode = EPI_F16; e.act = ACT_SILU; e.bias = w.ffn1_b1; e.out = b.f16; e.ldo = F;
        RC(gemm_f16(b.h16, d, w.ffn1_w1, d, e, M, F, d, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.ffn1_b2; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 0.5f;
        RC(gemm_f16(b.f16, F, w.ffn1_w2, F, e, M, d, F, st));
        // --- self-attention (Conformer.py:481-492)
        RC(layernorm_rows(b.x, b.h16, true, w.norm1_g, w.norm1_b, M, d, 1e-5f, false, st));
        e = GemmEpilogue(); e.out = b.qkv16; e.ldo = 3 * d;
        if (c.attention_type == SBK_ATT_ROPE) {
            e.mode = EPI_ROPE; e.alpha = att_scale; e.T = T; e.rope_cos = m->rope_cos; e.rope_sin = m->rope_sin; e.head_dim = dh;
        } else {
            e.mode = EPI_F16;
        }
        RC(gemm_f16(b.h16, d, w.wqkv, d, e, M, 3 * d, d, st));
        if (c.attention_type == SBK_ATT_RELPOS) {
            e = GemmEpilogue(); e.mode = EPI_F16; e.out = b.P16; e.ldo = d;
            RC(gemm_f16(m->relpos_pe, d, w.wpos, d, e, T, d, d, st));
        }
        RC(encoder_attention(b.qkv16, 3 * d, B, T, H, dh, enc_len, c.attention_type == SBK_ATT_RELPOS, w.pos_u, w.pos_v,
                             b.P16, d, att_scale, b.att16, d, st, m->dyn_chunk, m->dyn_left));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.bo; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 1.0f;
        RC(gemm_f16(b.att16, d, w.wo, d, e, M, d, d, st));
        // --- convolution module (Conformer.py:314-330, 494)
        RC(layernorm_rows(b.x, b.h16, true, w.conv_ln_g, w.conv_ln_b, M, d, 1e-5f, false, st));
        e = GemmEpilogue(); e.mode = EPI_GLU; e.bias = w.bpw1; e.out = b.glu; e.ldo = d;
        RC(gemm_f16(b.h16, d, w.wpw1, d, e, M, 2 * d, d, st));
        RC(dwconv_ln_swish(b.glu, B, T, d, c.kernel_size, w.wdw, w.bdw, w.aconv_ln_g, w.aconv_ln_b, 1e-5f, b.h16, st, m->dyn_chunk));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.bpw2; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 1.0f;
        e.row_lens = enc_len; e.T = T;
        RC(gemm_f16(b.h16, d, w.wpw2, d, e, M, d, d, st));
        // --- ffn module 2 + norm2 (Conformer.py:498)
        RC(layernorm_rows(b.x, b.h16, true, w.ffn2_ln_g, w.ffn2_ln_b, M, d, 1e-5f, false, st));
        e = GemmEpilogue(); e.mode = EPI_F16; e.act = ACT_SILU; e.bias = w.ffn2_b1; e.out = b.f16; e.ldo = F;
        RC(gemm_f16(b.h16, d, w.ffn2_w1, d, e, M, F, d, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.ffn2_b2; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 0.5f;
        RC(gemm_f16(b.f16, F, w.ffn2_w2, F, e, M, d, F, st));
        if (l + 1 < c.num_encoder_layers) {  // norm2 (fp32 residual stream) + the next layer's ffn1 LayerNorm (fp16 operand)
            const EncLayerW& nx = m->enc[l + 1];
            RC(layernorm2_rows(b.x, b.x, b.h16, true, w.norm2_g, w.norm2_b, 1e-5f, nx.ffn1_ln_g, nx.ffn1_ln_b, 1e-5f, M, d, st));
        } else {                             // norm2 + the encoder's final LayerNorm (Conformer.py:700)
            RC(layernorm2_rows(b.x, nullptr, enc_out, false, w.norm2_g, w.norm2_b, 1e-5f, m->enc_norm_g, m->enc_norm_b, 1e-6f, M,
                               d, st));
        }
    }
    if (c.num_encoder_layers == 0)
        RC(layernorm_rows(b.x, enc_out, false, m->enc_norm_g, m->enc_norm_b, M, d, 1e-6f, false, st));
    return SBK_OK;
}

__global__ void abs_len_kernel(const float* rel, int B, int T, int* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    // torch.round (half to even) of rel * T   (TransformerASR.py:148, seq2seq.py:206)
    if (i < B) out[i] = min(T, max(0, __float2int_rn(rel[i] * static_cast<float>(T))));
}

// Decoder pre-norm feeding a projection: either fused into the projection kernel (a.X) or a separate tiny kernel
// writing fp16 (a.A).  Fusion saves a launch per projection (single-batch latency); the separate kernel avoids
// recomputing the same 32-row LayerNorm in ~100-300 CTAs (GPU time when several batches are in flight).
static int dec_ln(AsrModel* m, SkinnyArgs& a, const float* g, const float* bta, int rows, cudaStream_t st) {
    AsrModel::Buf& b = m->b;
    const int d = m->cfg.d_model;
    if (m->fuse_dec_ln && (d == 256 || d == 512 || d == 768 || d == 1024)) {  // widths the LN-fused projection is built for
        a.X = b.dx; a.ln_g = g; a.ln_b = bta; a.ln_eps = 1e-6f;
        return SBK_OK;
    }
    a.A = b.dh16; a.lda = d;
    return layernorm_rows(b.dx, b.dh16, true, g, bta, rows, d, 1e-6f, false, st);
}

// Decode step when many hypotheses are live (several batches decoded together, or a wide beam): the projections run on
// the wgmma GEMM (128 x 32/64 tiles, a handful of CTAs each, so concurrent lanes share the GPU) instead of the
// weight-streaming kernel whose cost grows with every 32 rows.  Same maths: fp16 operands, fp32 accumulate / residual.
// Cross-attention K/V of every decoder layer, projected once per utterance from the encoder states (b.enc16).  Layout per
// layer (default): [K | V] parts, each [utt][head][T][64] -- the decode-step attention of (utterance, head) then streams one
// contiguous T x 128 B block of K and one of V instead of 128-byte pieces 2 KB apart (SBK_XATT_ROWMAJOR=1: the round-1
// [utt * T][K(d) | V(d)] rows).  Needs head_dim 64.
static bool xatt_headmajor(const AsrModel* m) {
    static const bool legacy = getenv("SBK_XATT_ROWMAJOR") != nullptr || getenv("SBK_GEMM_V1") != nullptr;  // (scatter epilogue: wide-tile kernel only)
    return !legacy && m->cfg.d_model / m->cfg.nhead == 64 && m->cfg.d_model % 256 == 0;
}
static int project_cross_kv(AsrModel* m, int M, int T, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, Ld = c.num_decoder_layers;
    RC(cast_f32_f16(b.enc_out, b.enc16, (size_t)M * d, st));
    if (xatt_headmajor(m)) {  // w_ckv / b_ckv are [Ld * 2d] rows: every layer's K and V in ONE GEMM, scattered per layer
        GemmEpilogue e;
        e.mode = EPI_F16; e.bias = m->b_ckv; e.out = b.ckv16; e.ldo = Ld * 2 * d;
        e.kv_heads = c.nhead; e.kv_part_stride = (size_t)M * d; e.kv_layer_stride = (size_t)M * 2 * d; e.T = T;
        return gemm_f16(b.enc16, d, m->w_ckv, d, e, M, Ld * 2 * d, d, st);
    }
    for (int l = 0; l < Ld; ++l) {
        GemmEpilogue e;
        e.mode = EPI_F16; e.bias = m->b_ckv + (size_t)l * 2 * d; e.out = b.ckv16 + (size_t)l * M * 2 * d; e.ldo = 2 * d;
        RC(gemm_f16(b.enc16, d, m->w_ckv + (size_t)l * 2 * d * d, d, e, M, 2 * d, d, st));
    }
    return SBK_OK;
}
// fills the K/V addressing of a cross-attention call for layer l
static void cross_kv_args(const AsrModel* m, DecAttnArgs& t, int l, int n_utt, int T) {
    const int d = m->cfg.d_model;
    const size_t M = (size_t)n_utt * T;
    t.kbase = m->b.ckv16 + (size_t)l * M * 2 * d;
    if (xatt_headmajor(m)) {
        t.vbase = t.kbase + M * d; t.row_stride = (size_t)T * d; t.head_stride = T * 64; t.key_stride = 64;
    } else {
        t.vbase = t.kbase + d; t.row_stride = (size_t)T * 2 * d; t.head_stride = 0; t.key_stride = 2 * d;
    }
}

static int enqueue_decode_layers_tc(AsrModel* m, int rows, int rows_per_utt, int T, int S_max, const int* lineage,
                                    cudaStream_t st, bool with_head) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, F = c.d_ffn, H = c.nhead, dh = d / H, Ld = c.num_decoder_layers;
    const int n_utt = rows / rows_per_utt;
    for (int l = 0; l < Ld; ++l) {
        const DecLayerW& w = m->dec[l];
        __half* kc = b.kcache + (size_t)l * rows * S_max * d;
        __half* vc = b.vcache + (size_t)l * rows * S_max * d;
        RC(layernorm_rows(b.dx, b.dh16, true, w.n1g, w.n1b, rows, d, 1e-6f, false, st, true));
        GemmEpilogue e;
        e.mode = EPI_QKV_CACHE; e.bias = w.b_self_in; e.out = b.dq16; e.ldo = d; e.kcache = kc; e.vcache = vc;
        e.step_ptr = b.step; e.S_max = S_max; e.qkv_d = d;
        RC(gemm_f16_small(b.dh16, d, w.w_self_in, d, e, rows, 3 * d, d, st));
        DecAttnArgs t{};
        t.q = b.dq16; t.ldq = d; t.kbase = kc; t.vbase = vc; t.row_stride = (size_t)S_max * d; t.key_stride = d;
        t.rows_per_block = 1; t.n_keys_ptr = b.step; t.enc_len = nullptr; t.H = H; t.dh = dh; t.out = b.datt16; t.ldo = d;
        t.lineage = lineage; t.lin_stride = S_max;
        RC(dec_attention(t, rows, S_max, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b_self_out; e.out = b.dx; e.resid = b.dx; e.ldo = d;
        RC(gemm_f16_small(b.datt16, d, w.w_self_out, d, e, rows, d, d, st));
        RC(layernorm_rows(b.dx, b.dh16, true, w.n2g, w.n2b, rows, d, 1e-6f, false, st, true));
        e = GemmEpilogue(); e.mode = EPI_F16; e.bias = w.b_cross_q; e.out = b.dq16; e.ldo = d;
        RC(gemm_f16_small(b.dh16, d, w.w_cross_q, d, e, rows, d, d, st));
        t = DecAttnArgs{};
        t.q = b.dq16; t.ldq = d; cross_kv_args(m, t, l, n_utt, T); t.rows_per_block = rows_per_utt;
        t.n_keys_ptr = nullptr; t.enc_len = b.enc_len; t.H = H; t.dh = dh; t.out = b.datt16; t.ldo = d;
        RC(dec_attention(t, rows, T, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b_cross_out; e.out = b.dx; e.resid = b.dx; e.ldo = d;
        RC(gemm_f16_small(b.datt16, d, w.w_cross_out, d, e, rows, d, d, st));
        RC(layernorm_rows(b.dx, b.dh16, true, w.n3g, w.n3b, rows, d, 1e-6f, false, st, true));
        e = GemmEpilogue(); e.mode = EPI_F16; e.act = c.decoder_activation == SBK_ACT_GELU ? ACT_GELU : ACT_RELU;
        e.bias = w.b_ffn1; e.out = b.df16; e.ldo = F;
        RC(gemm_f16_small(b.dh16, d, w.w_ffn1, d, e, rows, F, d, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b_ffn2; e.out = b.dx; e.resid = b.dx; e.ldo = d;
        RC(gemm_f16_small(b.df16, F, w.w_ffn2, F, e, rows, d, F, st));
    }
    if (!with_head) return SBK_OK;
    SBK_REQUIRE(m->w_lin != nullptr, "decode step: this handle was created without the output head (seq_lin.w.*)");
    RC(layernorm_rows(b.dx, b.dh16, true, m->dec_norm_g, m->dec_norm_b, rows, d, 1e-6f, false, st, true));
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->b_lin; e.out = b.logits; e.ldo = c.vocab;
    RC(gemm_f16_small(b.dh16, d, m->w_lin, d, e, rows, c.vocab, d, st));
    return SBK_OK;
}

// the wgmma decode path (enqueue_decode_layers_tc) for `rows` live hypotheses
static bool decode_tc(const AsrModel* m, int rows) {
    return rows >= m->dec_tc_rows && m->cfg.d_model % 32 == 0;  // (the QKV -> cache scatter epilogue works on 32-column chunks)
}
// Programmatic dependent launch is always on for the wgmma decode path (its GEMMs and LayerNorms are launched with it
// unconditionally); on the weight-streaming path it is opt-in (SBK_PDL=1), where it measured no faster.
static void set_decode_pdl(const AsrModel* m, int rows) { set_pdl(decode_tc(m, rows) || getenv("SBK_PDL") != nullptr); }

static int enqueue_decode_layers(AsrModel* m, int rows, int rows_per_utt, int T, int S_max, const int* lineage,
                                 cudaStream_t st, bool with_head = true) {
    if (decode_tc(m, rows))
        return enqueue_decode_layers_tc(m, rows, rows_per_utt, T, S_max, lineage, st, with_head);
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, F = c.d_ffn, H = c.nhead, dh = d / H, Ld = c.num_decoder_layers;
    const int ffn_epi = c.decoder_activation == SBK_ACT_GELU ? SK_F16_GELU : SK_F16_RELU;
    const int n_utt = rows / rows_per_utt;
    // b.dx already holds emb[token] * sqrt(d) + pe[step] (written by greedy_reset / the previous greedy_select)
    for (int l = 0; l < Ld; ++l) {
        const DecLayerW& w = m->dec[l];
        __half* kc = b.kcache + (size_t)l * rows * S_max * d;
        __half* vc = b.vcache + (size_t)l * rows * S_max * d;
        SkinnyArgs a{};  // LN1 + self-attention in_proj; k/v appended to the cache at position step
        RC(dec_ln(m, a, w.n1g, w.n1b, rows, st));
        a.W = w.w_self_in; a.ldw = d; a.bias = w.b_self_in; a.n_rows = rows; a.N = 3 * d; a.K = d;
        a.epi = SK_QKV_CACHE; a.out = b.dq16; a.ldo = d; a.kcache = kc; a.vcache = vc; a.step_ptr = b.step; a.S_max = S_max;
        a.d = d; a.q_scale = 1.0f;
        RC(skinny_gemm(a, st));
        DecAttnArgs t{};
        t.q = b.dq16; t.ldq = d; t.kbase = kc; t.vbase = vc; t.row_stride = (size_t)S_max * d; t.key_stride = d;
        t.rows_per_block = 1; t.n_keys_ptr = b.step; t.enc_len = nullptr; t.H = H; t.dh = dh; t.out = b.datt16; t.ldo = d;
        t.lineage = lineage; t.lin_stride = S_max;
        RC(dec_attention(t, rows, S_max, st));
        a = SkinnyArgs{}; a.A = b.datt16; a.lda = d; a.W = w.w_self_out; a.ldw = d; a.bias = w.b_self_out; a.n_rows = rows;
        a.N = d; a.K = d; a.epi = SK_RESID; a.out = b.dx; a.ldo = d;
        RC(skinny_gemm(a, st));
        // cross attention: LN2 + (pre-scaled) query projection
        a = SkinnyArgs{};
        RC(dec_ln(m, a, w.n2g, w.n2b, rows, st));
        a.W = w.w_cross_q; a.ldw = d; a.bias = w.b_cross_q; a.n_rows = rows;
        a.N = d; a.K = d; a.epi = SK_F16; a.out = b.dq16; a.ldo = d;
        RC(skinny_gemm(a, st));
        t = DecAttnArgs{};
        t.q = b.dq16; t.ldq = d; cross_kv_args(m, t, l, n_utt, T); t.rows_per_block = rows_per_utt;
        t.n_keys_ptr = nullptr; t.enc_len = b.enc_len; t.H = H; t.dh = dh; t.out = b.datt16; t.ldo = d;
        RC(dec_attention(t, rows, T, st));
        a = SkinnyArgs{}; a.A = b.datt16; a.lda = d; a.W = w.w_cross_out; a.ldw = d; a.bias = w.b_cross_out; a.n_rows = rows;
        a.N = d; a.K = d; a.epi = SK_RESID; a.out = b.dx; a.ldo = d;
        RC(skinny_gemm(a, st));
        // feed-forward: LN3 + ffn1 + activation, then ffn2 + residual
        a = SkinnyArgs{};
        RC(dec_ln(m, a, w.n3g, w.n3b, rows, st));
        a.W = w.w_ffn1; a.ldw = d; a.bias = w.b_ffn1; a.n_rows = rows;
        a.N = F; a.K = d; a.epi = ffn_epi; a.out = b.df16; a.ldo = F;
        RC(skinny_gemm(a, st));
        a = SkinnyArgs{}; a.A = b.df16; a.lda = F; a.W = w.w_ffn2; a.ldw = F; a.bias = w.b_ffn2; a.n_rows = rows;
        a.N = d; a.K = F; a.epi = SK_RESID; a.out = b.dx; a.ldo = d;
        RC(skinny_gemm(a, st));
    }
    if (!with_head) return SBK_OK;
    SBK_REQUIRE(m->w_lin != nullptr, "decode step: this handle was created without the output head (seq_lin.w.*)");
    SkinnyArgs a{};  // final LayerNorm + seq_lin
    RC(dec_ln(m, a, m->dec_norm_g, m->dec_norm_b, rows, st));
    a.W = m->w_lin; a.ldw = d; a.bias = m->b_lin; a.n_rows = rows; a.N = c.vocab; a.K = d;
    a.epi = SK_F32; a.out = b.logits; a.ldo = c.vocab;
    RC(skinny_gemm(a, st));
    return SBK_OK;
}

static int enqueue_decode_step(AsrModel* m, int rows, int rows_per_utt, int T, int S_max, int eos, float* log_probs,
                               int L_lp, cudaStream_t st) {
    AsrModel::Buf& b = m->b;
    RC(enqueue_decode_layers(m, rows, rows_per_utt, T, S_max, nullptr, st));
    RC(greedy_select(b.logits, rows, m->cfg.vocab, b.step, eos, b.tokens, S_max + 1, b.has_ended, b.ended_count, b.pred,
                     b.score, S_max, log_probs, L_lp, m->emb, m->dec_pe, m->cfg.d_model, b.dx, st));
    return SBK_OK;
}

// One TransformerLM step over `rows` hypotheses (post-norm encoder layers with a lineage-indexed KV cache), ending in
// b.lm_extra[rows, V] = weight * log_softmax(lm_logits / temperature): TransformerLMScorer.score (scorer.py:510-543)
// scaled by ScorerBuilder's weight.  b.lx / b.lx16 hold emb[token] * sqrt(d) + pe[step] (beam_reset / beam_step).
// The same step with the projections on the wgmma GEMM (128 x 32/64 tiles): used when many hypotheses are live (wide beams,
// B * beam >= dec_tc_rows), where the weight-streaming kernel's cost grows with every 32 rows.
static int enqueue_lm_step_tc(AsrModel* m, int rows, int S_max, float temperature, float weight, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int dl = c.lm_d_model, Fl = c.lm_d_ffn, H = c.lm_nhead;
    for (int l = 0; l < c.lm_layers; ++l) {
        const LmLayerW& w = m->lm[l];
        __half* kc = b.lkc + (size_t)l * rows * S_max * dl;
        __half* vc = b.lvc + (size_t)l * rows * S_max * dl;
        GemmEpilogue e;
        e.mode = EPI_QKV_CACHE; e.bias = w.b_in; e.out = b.lq16; e.ldo = dl; e.kcache = kc; e.vcache = vc;
        e.step_ptr = b.step; e.S_max = S_max; e.qkv_d = dl;
        RC(gemm_f16_small(b.lx16, dl, w.w_in, dl, e, rows, 3 * dl, dl, st));
        DecAttnArgs t{};
        t.q = b.lq16; t.ldq = dl; t.kbase = kc; t.vbase = vc; t.row_stride = (size_t)S_max * dl; t.key_stride = dl;
        t.rows_per_block = 1; t.n_keys_ptr = b.step; t.H = H; t.dh = 64; t.out = b.latt16; t.ldo = dl;
        t.lineage = b.lineage; t.lin_stride = S_max; t.tok_cache = b.tok_cache; t.pad_tok = 0;
        RC(dec_attention(t, rows, S_max, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b_out; e.out = b.lx; e.resid = b.lx; e.ldo = dl;
        RC(gemm_f16_small(b.latt16, dl, w.w_out, dl, e, rows, dl, dl, st));
        RC(layernorm_dual(b.lx, b.lx16, w.n1g, w.n1b, rows, dl, 1e-6f, true, st));
        e = GemmEpilogue(); e.mode = EPI_F16; e.act = c.lm_activation == SBK_ACT_GELU ? ACT_GELU : ACT_RELU;
        e.bias = w.b1; e.out = b.lf16; e.ldo = Fl;
        RC(gemm_f16_small(b.lx16, dl, w.w1, dl, e, rows, Fl, dl, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b2; e.out = b.lx; e.resid = b.lx; e.ldo = dl;
        RC(gemm_f16_small(b.lf16, Fl, w.w2, Fl, e, rows, dl, Fl, st));
        RC(layernorm_dual(b.lx, b.lx16, w.n2g, w.n2b, rows, dl, 1e-6f, true, st));
    }
    RC(layernorm_dual(b.lx, b.lx16, m->lm_norm_g, m->lm_norm_b, rows, dl, 1e-6f, false, st));  // encoder.norm
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->lm_bp0; e.out = b.lh32; e.ldo = dl;
    RC(gemm_f16_small(b.lx16, dl, m->lm_wp0, dl, e, rows, dl, dl, st));
    RC(layernorm_dual(b.lh32, b.lh16, m->lm_lnp_g, m->lm_lnp_b, rows, dl, 1e-6f, false, st));
    e = GemmEpilogue(); e.mode = EPI_F32; e.bias = m->lm_bp2; e.out = b.lm_logits; e.ldo = c.vocab;
    RC(gemm_f16_small(b.lh16, dl, m->lm_wp2, dl, e, rows, c.vocab, dl, st));
    RC(weighted_log_softmax(b.lm_logits, b.lm_extra, rows, c.vocab, temperature, weight, st));
    return SBK_OK;
}

static int enqueue_lm_step(AsrModel* m, int rows, int S_max, float temperature, float weight, cudaStream_t st) {
    if (rows >= m->dec_tc_rows) return enqueue_lm_step_tc(m, rows, S_max, temperature, weight, st);
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int dl = c.lm_d_model, Fl = c.lm_d_ffn, H = c.lm_nhead;
    for (int l = 0; l < c.lm_layers; ++l) {
        const LmLayerW& w = m->lm[l];
        __half* kc = b.lkc + (size_t)l * rows * S_max * dl;
        __half* vc = b.lvc + (size_t)l * rows * S_max * dl;
        SkinnyArgs a{};
        a.A = b.lx16; a.lda = dl; a.W = w.w_in; a.ldw = dl; a.bias = w.b_in; a.n_rows = rows; a.N = 3 * dl; a.K = dl;
        a.epi = SK_QKV_CACHE; a.out = b.lq16; a.ldo = dl; a.kcache = kc; a.vcache = vc; a.step_ptr = b.step; a.S_max = S_max;
        a.d = dl; a.q_scale = 1.0f;
        RC(skinny_gemm(a, st));
        DecAttnArgs t{};
        t.q = b.lq16; t.ldq = dl; t.kbase = kc; t.vbase = vc; t.row_stride = (size_t)S_max * dl; t.key_stride = dl;
        t.rows_per_block = 1; t.n_keys_ptr = b.step; t.H = H; t.dh = 64; t.out = b.latt16; t.ldo = dl;
        t.lineage = b.lineage; t.lin_stride = S_max; t.tok_cache = b.tok_cache; t.pad_tok = 0;
        RC(dec_attention(t, rows, S_max, st));
        a = SkinnyArgs{}; a.A = b.latt16; a.lda = dl; a.W = w.w_out; a.ldw = dl; a.bias = w.b_out; a.n_rows = rows;
        a.N = dl; a.K = dl; a.epi = SK_RESID; a.out = b.lx; a.ldo = dl;
        RC(skinny_gemm(a, st));
        RC(layernorm_dual(b.lx, b.lx16, w.n1g, w.n1b, rows, dl, 1e-6f, true, st));
        a = SkinnyArgs{}; a.A = b.lx16; a.lda = dl; a.W = w.w1; a.ldw = dl; a.bias = w.b1; a.n_rows = rows;
        a.N = Fl; a.K = dl; a.epi = c.lm_activation == SBK_ACT_GELU ? SK_F16_GELU : SK_F16_RELU; a.out = b.lf16; a.ldo = Fl;
        RC(skinny_gemm(a, st));
        a = SkinnyArgs{}; a.A = b.lf16; a.lda = Fl; a.W = w.w2; a.ldw = Fl; a.bias = w.b2; a.n_rows = rows;
        a.N = dl; a.K = Fl; a.epi = SK_RESID; a.out = b.lx; a.ldo = dl;
        RC(skinny_gemm(a, st));
        RC(layernorm_dual(b.lx, b.lx16, w.n2g, w.n2b, rows, dl, 1e-6f, true, st));
    }
    RC(layernorm_dual(b.lx, b.lx16, m->lm_norm_g, m->lm_norm_b, rows, dl, 1e-6f, false, st));  // encoder.norm
    SkinnyArgs a{};
    a.A = b.lx16; a.lda = dl; a.W = m->lm_wp0; a.ldw = dl; a.bias = m->lm_bp0; a.n_rows = rows; a.N = dl; a.K = dl;
    a.epi = SK_F32; a.out = b.lh32; a.ldo = dl;
    RC(skinny_gemm(a, st));
    RC(layernorm_dual(b.lh32, b.lh16, m->lm_lnp_g, m->lm_lnp_b, rows, dl, 1e-6f, false, st));
    a = SkinnyArgs{}; a.A = b.lh16; a.lda = dl; a.W = m->lm_wp2; a.ldw = dl; a.bias = m->lm_bp2; a.n_rows = rows;
    a.N = c.vocab; a.K = dl; a.epi = SK_F32; a.out = b.lm_logits; a.ldo = c.vocab;
    RC(skinny_gemm(a, st));
    RC(weighted_log_softmax(b.lm_logits, b.lm_extra, rows, c.vocab, temperature, weight, st));
    return SBK_OK;
}

// Beam search (decoders/seq2seq.py:1632-1723 with scorer=None): the device runs decoder step + beam_step_kernel and
// records the per-step (token, predecessor, normalised score, log-prob) history; hypothesis bookkeeping is replayed
// on the host from that history (speechbrain_b200/decoders/seq2seq.py).
static int run_beam(AsrModel* m, int B, int T, const sbk_beam_params& p, int* hist_tok_out, int* hist_pred_out,
                    float* hist_score_out, float* hist_lp_out, int* steps_done, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, Ld = c.num_decoder_layers, M = B * T, beam = p.beam_size, rows = B * beam, S_max = m->ws_steps + 1;
    SBK_REQUIRE(m->has_dec, "beam: this handle was created without decoder weights");
    SBK_REQUIRE(p.max_steps <= m->ws_steps && p.max_steps + 1 <= c.max_len, "beam: max_steps=%d too large", p.max_steps);
    *steps_done = 0;
    if (p.max_steps <= 0) return SBK_OK;
    RC(project_cross_kv(m, M, T, st));
    set_decode_pdl(m, rows);
    const bool use_lm = p.lm_weight != 0.0f;
    SBK_REQUIRE(!use_lm || m->has_lm, "beam: lm_weight != 0 but this handle has no TransformerLM weights");
    const bool use_ctc = p.ctc_weight != 0.0f;
    // the search history lives in the workspace (fixed addresses: the step graph bakes them in) and is copied out at the end
    int* hist_tok = b.hist_tok; int* hist_pred = b.hist_pred; float* hist_score = b.hist_score; float* hist_lp = b.hist_lp;
    CtcStep cs{};
    if (use_ctc) {  // CTCScorer.reset_mem (scorer.py:243-249) + CTCPrefixScore.__init__ (ctc.py:46-78)
        SBK_REQUIRE(m->w_ctc, "beam: ctc_weight != 0 but this handle has no ctc_lin weights");
        SBK_REQUIRE(p.blank_index >= 0 && p.blank_index < c.vocab && p.blank_index != p.bos && p.blank_index != p.eos &&
                    p.bos != p.eos, "Set blank, eos and bos to different indexes for joint ATT/CTC or CTC decoding");
        const size_t V = c.vocab;
        auto al = [](size_t n) { return (n * 4 + 255) & ~size_t(255); };
        const size_t need = 2 * al((size_t)M * V) + al(M) + 2 * al((size_t)2 * rows * T) + al(2 * rows) + (use_lm ? 0 : al(rows * V)) +
                            al((size_t)2 * rows * (T + 4)) + al(2 * rows);
        AsrModel::CtcBuf& cb = m->ctc;
        if (need > cb.cap) {
            if (cb.base) { SBK_CUDA_CHECK(cudaStreamSynchronize(st)); cudaFree(cb.base); cb.base = nullptr; cb.cap = 0; }
            if (m->beam_graph) { cudaGraphExecDestroy(m->beam_graph); m->beam_graph = nullptr; }
            if (cudaMalloc(&cb.base, need) != cudaSuccess) { set_error("beam: CTC scorer cudaMalloc(%zu) failed", need); return SBK_ERR_NOMEM; }
            cb.cap = need;
        }
        char* q = reinterpret_cast<char*>(cb.base);
        cb.x = reinterpret_cast<float*>(q); q += al((size_t)M * V);
        cb.xlin = reinterpret_cast<float*>(q); q += al((size_t)M * V);
        cb.xb = reinterpret_cast<float*>(q); q += al(M);
        cb.rsum = reinterpret_cast<float*>(q); q += al((size_t)2 * rows * T);
        cb.rb = reinterpret_cast<float*>(q); q += al((size_t)2 * rows * T);
        cb.psi = reinterpret_cast<float*>(q); q += al(2 * rows);
        cb.tab = reinterpret_cast<float*>(q); q += al((size_t)2 * rows * (T + 4));
        cb.tabM = reinterpret_cast<float*>(q); q += al(2 * rows);
        cb.add = use_lm ? b.lm_extra : reinterpret_cast<float*>(q);
        GemmEpilogue e;
        e.mode = EPI_F32; e.bias = m->b_ctc; e.out = cb.x; e.ldo = c.vocab;
        RC(gemm_f16(b.enc16, d, m->w_ctc, d, e, M, c.vocab, d, st));
        RC(ctc_prefix_reset(cb.x, cb.xlin, cb.xb, b.enc_len, B, T, c.vocab, p.blank_index, beam, cb.rsum, cb.rb, cb.psi, cb.tab, cb.tabM, st));
        cs.x = cb.x; cs.xlin = cb.xlin; cs.xb = cb.xb; cs.enc_len = b.enc_len; cs.hist_tok = hist_tok; cs.hist_pred = hist_pred; cs.n_bh = rows;
        cs.rsum_base = cb.rsum; cs.rb_base = cb.rb; cs.psi_base = cb.psi; cs.step_ptr = b.step; cs.tab = cb.tab; cs.tabM = cb.tabM;
        cs.bos = p.bos; cs.T = T; cs.V = c.vocab; cs.beam = beam; cs.blank = p.blank_index; cs.eos = p.eos;
        cs.weight = p.ctc_weight; cs.out = cb.add; cs.accumulate = use_lm ? 1 : 0;
    }
    const bool use_cov = p.coverage_weight != 0.0f;
    CoverageStep cv{};
    if (use_cov) {  // CoverageScorer (scorer.py:788-955) on the last decoder layer's head-averaged cross-attention
        SBK_REQUIRE(d / c.nhead == 64, "beam: the coverage scorer is built for head_dim 64");
        const size_t need = ((size_t)2 * rows * T + rows) * 4 + 256;
        if (need > m->cov.cap) {
            if (m->cov.base) { SBK_CUDA_CHECK(cudaStreamSynchronize(st)); cudaFree(m->cov.base); m->cov.base = nullptr; m->cov.cap = 0; }
            if (m->beam_graph) { cudaGraphExecDestroy(m->beam_graph); m->beam_graph = nullptr; }
            if (cudaMalloc(&m->cov.base, need) != cudaSuccess) { set_error("beam: coverage scorer cudaMalloc(%zu) failed", need); return SBK_ERR_NOMEM; }
            m->cov.cap = need;
        }
        cv.q = b.dq16; cv.ldq = d; cv.kbase = b.ckv16 + (size_t)(Ld - 1) * M * 2 * d;
        if (xatt_headmajor(m)) { cv.utt_stride = (size_t)T * d; cv.key_stride = 64; cv.head_stride = T * 64; }
        else { cv.utt_stride = (size_t)T * 2 * d; cv.key_stride = 2 * d; cv.head_stride = 64; }
        cv.enc_len = b.enc_len; cv.rows_per_utt = beam; cv.T = T; cv.H = c.nhead;
        cv.cov_base = m->cov.base; cv.hist_pred = hist_pred; cv.step_ptr = b.step; cv.n_bh = rows;
        cv.threshold = p.coverage_threshold; cv.weight = p.coverage_weight; cv.out = m->cov.base + (size_t)2 * rows * T;
    }
    BeamLm lm;
    if (use_lm) { lm.emb = m->lm_emb; lm.pe = m->lm_pe; lm.d = c.lm_d_model; lm.x = b.lx; lm.x16 = b.lx16; lm.tok_cache = b.tok_cache; }
    RC(beam_reset(rows, beam, S_max, p.bos, b.step, b.seq_scores, b.lineage, b.finished, b.ended_count, m->emb, m->dec_pe, d,
                  b.dx, use_lm ? &lm : nullptr, st));
    BeamStepArgs a{};
    a.add_scores = use_lm ? b.lm_extra : (use_ctc ? m->ctc.add : nullptr);
    a.lm = lm;
    if (use_ctc) { a.attn_weight = 1.0f - p.ctc_weight; a.blank = p.blank_index; }
    a.add_const = p.length_weight;
    a.add_row = use_cov ? cv.out : nullptr;
    a.logits = b.logits; a.V = c.vocab; a.beam = beam; a.S_max = S_max; a.seq_scores = b.seq_scores; a.lineage = b.lineage;
    a.step_arr = b.step; a.finished = b.finished; a.n_full = b.ended_count;
    a.hist_tok = hist_tok; a.hist_pred = hist_pred; a.hist_score = hist_score; a.hist_lp = hist_lp;
    a.temperature = p.temperature; a.eos_threshold = p.eos_threshold; a.minus_inf = p.minus_inf; a.min_steps = p.min_steps;
    a.eos = p.eos; a.use_eos_threshold = p.using_eos_threshold; a.length_norm = p.length_normalization;
    a.emb = m->emb; a.pe = m->dec_pe; a.d = d; a.x_next = b.dx; a.scratch = b.beam_scr;
    // One whole search step; every kernel takes the step index from the device counters, so the sequence is the same
    // for every step and can be replayed from a graph.  The scorers that do not read the decoder's output of this step --
    // the TransformerLM step and the CTC state update of the PREVIOUS step's survivors -- run as a second branch beside
    // the decoder layers (both are chains of small kernels that leave most SMs idle) and join before the scores are combined.
    const bool fork = (use_lm || use_ctc) && getenv("SBK_BEAM_SERIAL") == nullptr;
    if (fork && !m->side_stream) {
        SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->side_stream, cudaStreamNonBlocking));
        SBK_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_bfork, cudaEventDisableTiming));
        SBK_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_bjoin, cudaEventDisableTiming));
    }
    auto enqueue_step = [&](cudaStream_t s_) -> int {
        cudaStream_t s2 = s_;
        if (fork) {
            s2 = m->side_stream;
            SBK_CUDA_CHECK(cudaEventRecord(m->ev_bfork, s_));
            SBK_CUDA_CHECK(cudaStreamWaitEvent(s2, m->ev_bfork, 0));
        }
        if (use_ctc) RC(ctc_prefix_update(cs, s2));  // permute_scorer_mem on the previous step's survivors (no-op at step 0)
        if (use_lm) RC(enqueue_lm_step(m, rows, S_max, p.lm_temperature, p.lm_weight, s2));
        RC(enqueue_decode_layers(m, rows, beam, T, S_max, b.lineage, s_));
        if (use_cov) RC(coverage_score(cv, s_));  // reads the last layer's cross-attention query left in b.dq16
        if (fork) {
            SBK_CUDA_CHECK(cudaEventRecord(m->ev_bjoin, s2));
            SBK_CUDA_CHECK(cudaStreamWaitEvent(s_, m->ev_bjoin, 0));
        }
        if (use_ctc) RC(ctc_prefix_score(cs, s_));  // ScorerBuilder.score (ctc after transformerlm)
        RC(beam_step(a, B, s_));
        return SBK_OK;
    };
    const bool use_graph = getenv("SBK_NO_GRAPH") == nullptr;
    if (use_graph) {
        AsrModel::BeamKey key;
        memset(&key, 0, sizeof(key));
        key.p = p; key.B = B; key.T = T; key.rows = rows; key.S_max = S_max; key.fuse_ln = m->fuse_dec_ln; key.tc_rows = m->dec_tc_rows; key.fork = fork ? 1 : 0;
        if (m->beam_graph == nullptr || memcmp(&key, &m->beam_key, sizeof(key)) != 0) {
            if (m->beam_graph) { cudaGraphExecDestroy(m->beam_graph); m->beam_graph = nullptr; }
            if (!m->cap_stream) SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
            cudaGraph_t g;
            SBK_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
            launch_count_begin_capture();
            int rc = enqueue_step(m->cap_stream);
            m->beam_nodes = launch_count_end_capture();
            cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &g);
            if (rc) return rc;
            SBK_CUDA_CHECK(ce);
            SBK_CUDA_CHECK(cudaGraphInstantiate(&m->beam_graph, g, 0));
            cudaGraphDestroy(g);
            m->beam_key = key;
        }
    }
    const int check_every = m->poll_every > 0 ? m->poll_every : p.max_steps;
    int s = 0;
    while (s < p.max_steps) {
        const int chunk = std::min(check_every, p.max_steps - s);
        for (int i = 0; i < chunk; ++i) {
            if (use_graph) { SBK_CUDA_CHECK(cudaGraphLaunch(m->beam_graph, st)); launch_count_add(m->beam_nodes); }
            else RC(enqueue_step(st));
        }
        s += chunk;
        if (s < p.max_steps && m->poll_every > 0) {  // `_check_full_beams` (:806-822), polled once per chunk
            SBK_CUDA_CHECK(cudaMemcpyAsync(m->host_flag, b.ended_count, 4, cudaMemcpyDeviceToHost, st));
            SBK_CUDA_CHECK(cudaStreamSynchronize(st));
            if (*m->host_flag >= B) break;
        }
    }
    const size_t hb = (size_t)s * rows * 4;
    if (hist_tok_out) SBK_CUDA_CHECK(cudaMemcpyAsync(hist_tok_out, hist_tok, hb, cudaMemcpyDeviceToDevice, st));
    if (hist_pred_out) SBK_CUDA_CHECK(cudaMemcpyAsync(hist_pred_out, hist_pred, hb, cudaMemcpyDeviceToDevice, st));
    if (hist_score_out) SBK_CUDA_CHECK(cudaMemcpyAsync(hist_score_out, hist_score, hb, cudaMemcpyDeviceToDevice, st));
    if (hist_lp_out) SBK_CUDA_CHECK(cudaMemcpyAsync(hist_lp_out, hist_lp, hb, cudaMemcpyDeviceToDevice, st));
    *steps_done = s;
    return SBK_OK;
}

// Greedy search over encoder states already in the workspace (b.enc_out / b.enc_len).
static int run_greedy(AsrModel* m, int B, int T, int max_steps, int bos, int eos, float* log_probs, int* steps_done,
                      cudaStream_t st, bool in_capture = false) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, M = B * T, rows = B, S_max = m->ws_steps + 1;
    SBK_REQUIRE(m->has_dec, "greedy: this handle was created without decoder weights");
    SBK_REQUIRE(max_steps <= m->ws_steps && max_steps + 1 <= c.max_len, "greedy: max_steps=%d too large", max_steps);
    *steps_done = 0;
    if (max_steps <= 0) return SBK_OK;
    RC(project_cross_kv(m, M, T, st));  // cross-attention K/V of all layers, once per utterance
    RC(greedy_reset(b.tokens, S_max + 1, rows, bos, b.step, b.has_ended, b.ended_count, m->emb, m->dec_pe, d, b.dx, st));
    set_decode_pdl(m, rows);
    const bool use_graph = !in_capture && getenv("SBK_NO_GRAPH") == nullptr && log_probs == nullptr;
    if (in_capture) {  // the caller is capturing the whole pipeline: enqueue exactly max_steps steps, no polling
        for (int i = 0; i < max_steps; ++i) RC(enqueue_decode_step(m, rows, 1, T, S_max, eos, log_probs, max_steps, st));
        *steps_done = max_steps;
        return SBK_OK;
    }
    if (use_graph && (m->step_graph == nullptr || m->graph_rows != rows || m->graph_T != T || m->graph_B != B ||
                      m->graph_eos != eos || m->graph_S != S_max)) {
        if (m->step_graph) { cudaGraphExecDestroy(m->step_graph); m->step_graph = nullptr; }
        cudaGraph_t g;
        if (!m->cap_stream) SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        SBK_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
        launch_count_begin_capture();
        int rc = enqueue_decode_step(m, rows, 1, T, S_max, eos, nullptr, 0, m->cap_stream);
        m->graph_nodes = launch_count_end_capture();
        cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &g);
        if (rc) return rc;
        SBK_CUDA_CHECK(ce);
        SBK_CUDA_CHECK(cudaGraphInstantiate(&m->step_graph, g, 0));
        cudaGraphDestroy(g);
        m->graph_rows = rows; m->graph_T = T; m->graph_B = B; m->graph_eos = eos; m->graph_S = S_max;
    }
    const int check_every = m->poll_every > 0 ? m->poll_every : max_steps;
    int s = 0;
    while (s < max_steps) {
        const int chunk = std::min(check_every, max_steps - s);
        for (int i = 0; i < chunk; ++i) {
            if (use_graph) { SBK_CUDA_CHECK(cudaGraphLaunch(m->step_graph, st)); launch_count_add(m->graph_nodes); }
            else RC(enqueue_decode_step(m, rows, 1, T, S_max, eos, log_probs, max_steps, st));
        }
        s += chunk;
        if (s < max_steps && m->poll_every > 0) {  // seq2seq.py:256 `has_ended.all()` early exit, polled once per chunk
            SBK_CUDA_CHECK(cudaMemcpyAsync(m->host_flag, b.ended_count, 4, cudaMemcpyDeviceToHost, st));
            SBK_CUDA_CHECK(cudaStreamSynchronize(st));
            if (*m->host_flag >= rows) break;
        }
    }
    *steps_done = s;
    return SBK_OK;
}

// ---------------------------------------------------------------------------- TransformerLMRescorer (scorer.py:1835-1882)
// Teacher-forced scoring of n padded token sequences with the KV-cached LM step: position s feeds tokens[:, s] and adds
// log p(tokens[:, s+1]) -- renormalised without the pad column like the reference -- for the rows whose sequence is longer.
__global__ void lm_teacher_reset_kernel(const int* __restrict__ tokens, int n, int L, int S_max, int pad, int* __restrict__ lineage,
                                        int* __restrict__ tok_cache, float* __restrict__ scores) {
    const int r = blockIdx.x;
    for (int p = threadIdx.x; p < S_max; p += blockDim.x) {
        lineage[static_cast<size_t>(r) * S_max + p] = r;                                   // parity 0
        lineage[static_cast<size_t>(n) * S_max + static_cast<size_t>(r) * S_max + p] = r;  // parity 1
        tok_cache[static_cast<size_t>(r) * S_max + p] = p < L ? tokens[static_cast<size_t>(r) * L + p] : pad;
    }
    if (threadIdx.x == 0) scores[r] = 0.0f;
}
__global__ void lm_teacher_embed_kernel(const int* __restrict__ tokens, int L, int s, const float* __restrict__ emb,
                                        const float* __restrict__ pe, int d, float sqrt_d, float* __restrict__ x,
                                        __half* __restrict__ x16, int* __restrict__ step_arr) {
    const int r = blockIdx.x;
    const int tok = tokens[static_cast<size_t>(r) * L + s];
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        const float v = emb[static_cast<size_t>(tok) * d + i] * sqrt_d + pe[static_cast<size_t>(s) * d + i];
        x[static_cast<size_t>(r) * d + i] = v;
        x16[static_cast<size_t>(r) * d + i] = float2half_sat(v);
    }
    if (threadIdx.x == 0) step_arr[r] = s;
}
__global__ void lm_teacher_score_kernel(const float* __restrict__ log_probs, int V, const int* __restrict__ tokens, int L, int s,
                                        const int* __restrict__ lens, int pad, float* __restrict__ scores, int n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n || s + 1 >= lens[r]) return;
    const float* lp = log_probs + static_cast<size_t>(r) * V;
    const int tgt = tokens[static_cast<size_t>(r) * L + s + 1];
    const float v = (tgt == pad ? -INFINITY : lp[tgt]) - log1pf(-expf(lp[pad]));  // log_softmax over the non-pad entries
    if (v == v) scores[r] += v;  // torch.nansum
}

// ---------------------------------------------------------------------------- TransformerASR.decode (TransformerASR.py:426-473)
// Teacher-forced: position s feeds tgt[:, s] through the KV-cached decoder layers and writes decoder.norm(x) to
// out[:, s, :] -- the same numbers the reference gets from one whole-prefix pass with the causal mask.
__global__ void dec_teacher_embed_kernel(const int* __restrict__ tokens, int S, int s, const float* __restrict__ emb,
                                         const float* __restrict__ pe, int d, float sqrt_d, float* __restrict__ x,
                                         int* __restrict__ step_arr) {
    const int r = blockIdx.x;
    const int tok = tokens[static_cast<size_t>(r) * S + s];
    for (int i = threadIdx.x; i < d; i += blockDim.x)
        x[static_cast<size_t>(r) * d + i] = emb[static_cast<size_t>(tok) * d + i] * sqrt_d + pe[static_cast<size_t>(s) * d + i];
    if (threadIdx.x == 0) step_arr[r] = s;
}

static int run_decode_teacher(AsrModel* m, const int* tokens, int n, int S, int T, float* out, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, M = n * T, S_max = m->ws_steps + 1;
    SBK_REQUIRE(m->has_dec, "decode: this handle was created without decoder weights");
    SBK_REQUIRE(S <= m->ws_steps && S <= c.max_len, "decode: %d target positions exceed the workspace / max_len", S);
    RC(project_cross_kv(m, M, T, st));
    for (int s = 0; s < S; ++s) {
        dec_teacher_embed_kernel<<<n, 128, 0, st>>>(tokens, S, s, m->emb, m->dec_pe, d, sqrtf((float)d), b.dx, b.step);
        SBK_LAUNCH_CHECK();
        RC(enqueue_decode_layers(m, n, 1, T, S_max, nullptr, st, false));
        RC(layernorm_rows(b.dx, b.lnout, false, m->dec_norm_g, m->dec_norm_b, n, d, 1e-6f, false, st));
        SBK_CUDA_CHECK(cudaMemcpy2DAsync(out + (size_t)s * d, (size_t)S * d * 4, b.lnout, (size_t)d * 4, (size_t)d * 4, n,
                                         cudaMemcpyDeviceToDevice, st));
    }
    return SBK_OK;
}

static int run_lm_rescore(AsrModel* m, const int* tokens, const int* lens, int n, int L, float temperature, int pad,
                          float* scores, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int S_max = m->ws_steps + 1, dl = c.lm_d_model;
    lm_teacher_reset_kernel<<<n, 128, 0, st>>>(tokens, n, L, S_max, pad, b.lineage, b.tok_cache, scores);
    SBK_LAUNCH_CHECK();
    for (int s = 0; s + 1 < L; ++s) {
        lm_teacher_embed_kernel<<<n, 128, 0, st>>>(tokens, L, s, m->lm_emb, m->lm_pe, dl, sqrtf((float)dl), b.lx, b.lx16, b.step);
        SBK_LAUNCH_CHECK();
        RC(enqueue_lm_step(m, n, S_max, temperature, 1.0f, st));
        lm_teacher_score_kernel<<<ceil_div(n, 128), 128, 0, st>>>(b.lm_extra, c.vocab, tokens, L, s, lens, pad, scores, n);
        SBK_LAUNCH_CHECK();
    }
    return SBK_OK;
}

// The same teacher-forced step path, keeping each position's raw logits: out[:, s, :] = lm_logits after feeding
// tokens[:, s].  Keys are masked through tok_cache exactly as in the rescorer and the beam search's LM scorer.
static int run_lm_step_logits(AsrModel* m, const int* tokens, int n, int L, float* out, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    AsrModel::Buf& b = m->b;
    const int S_max = m->ws_steps + 1, dl = c.lm_d_model, V = c.vocab;
    lm_teacher_reset_kernel<<<n, 128, 0, st>>>(tokens, n, L, S_max, 0, b.lineage, b.tok_cache, b.score);
    SBK_LAUNCH_CHECK();
    for (int s = 0; s < L; ++s) {
        lm_teacher_embed_kernel<<<n, 128, 0, st>>>(tokens, L, s, m->lm_emb, m->lm_pe, dl, sqrtf((float)dl), b.lx, b.lx16, b.step);
        SBK_LAUNCH_CHECK();
        RC(enqueue_lm_step(m, n, S_max, 1.0f, 1.0f, st));
        SBK_CUDA_CHECK(cudaMemcpy2DAsync(out + (size_t)s * V, (size_t)L * V * 4, b.lm_logits, (size_t)V * 4, (size_t)V * 4, n,
                                         cudaMemcpyDeviceToDevice, st));
    }
    return SBK_OK;
}

// ---------------------------------------------------------------------------- TransformerLM.forward (TransformerLM.py:127-169)
// Whole sequences at once: the n * s token rows go through every layer together on the encoder's wgmma GEMMs, attention is
// the causal flash kernel (lm_causal_attention).  Same weights, epilogues and LayerNorm kernel as the KV-cached step.
// Row r = (sequence r / s, position r % s): x = emb[token] * sqrt(d) + pe[pos], fp32 residual stream + fp16 GEMM operand
// (the whole-sequence counterpart of lm_teacher_embed_kernel).  An id outside [0, vocab) is not read from the table: its
// row becomes NaN (and, through attention, its sequence) instead of an out-of-bounds read.
__global__ void lm_embed_kernel(const int* __restrict__ tokens, int s, int vocab, const float* __restrict__ emb,
                                const float* __restrict__ pe, int d, float sqrt_d, float* __restrict__ x,
                                __half* __restrict__ x16) {
    const int r = blockIdx.x, pos = r % s;
    const int tok = tokens[r];
    const bool ok = tok >= 0 && tok < vocab;
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        const float v = ok ? emb[static_cast<size_t>(tok) * d + i] * sqrt_d + pe[static_cast<size_t>(pos) * d + i] : NAN;
        x[static_cast<size_t>(r) * d + i] = v;
        x16[static_cast<size_t>(r) * d + i] = float2half_sat(v);
    }
}

static int ensure_lm_workspace(AsrModel* m, int rows, cudaStream_t st) {
    AsrModel::LmFwdBuf& w = m->lmf;
    if (w.base && rows <= w.rows) return SBK_OK;
    const size_t R = rows, dl = m->cfg.lm_d_model, Fl = m->cfg.lm_d_ffn;
    auto al = [](size_t bytes) { return (bytes + 255) & ~size_t(255); };
    const size_t need = al(R * dl * 4) + al(R * dl * 2) + al(R * 3 * dl * 2) + al(R * dl * 2) + al(R * Fl * 2);
    if (need > w.cap) {
        if (w.base) { SBK_CUDA_CHECK(cudaStreamSynchronize(st)); cudaFree(w.base); w.base = nullptr; w.cap = 0; w.rows = 0; }
        if (cudaMalloc(&w.base, need) != cudaSuccess) { set_error("lm_forward: workspace cudaMalloc(%zu) failed", need); return SBK_ERR_NOMEM; }
        w.cap = need;
    }
    uint8_t* q = w.base;
    w.x = reinterpret_cast<float*>(q); q += al(R * dl * 4);
    w.x16 = reinterpret_cast<__half*>(q); q += al(R * dl * 2);
    w.qkv16 = reinterpret_cast<__half*>(q); q += al(R * 3 * dl * 2);
    w.att16 = reinterpret_cast<__half*>(q); q += al(R * dl * 2);
    w.f16 = reinterpret_cast<__half*>(q);
    w.rows = rows;
    return SBK_OK;
}

static int run_lm_forward(AsrModel* m, const int* tokens, int n, int s, float* logits, cudaStream_t st) {
    const sbk_asr_config& c = m->cfg;
    const int dl = c.lm_d_model, Fl = c.lm_d_ffn, H = c.lm_nhead, M = n * s;
    RC(ensure_lm_workspace(m, M, st));
    const AsrModel::LmFwdBuf& b = m->lmf;
    lm_embed_kernel<<<M, 128, 0, st>>>(tokens, s, c.vocab, m->lm_emb, m->lm_pe, dl, sqrtf((float)dl), b.x, b.x16);
    SBK_LAUNCH_CHECK();
    for (int l = 0; l < c.lm_layers; ++l) {  // post-norm TransformerEncoderLayer (Transformer.py:466-481)
        const LmLayerW& w = m->lm[l];
        GemmEpilogue e;
        e.mode = EPI_F16; e.bias = w.b_in; e.out = b.qkv16; e.ldo = 3 * dl;
        RC(gemm_f16(b.x16, dl, w.w_in, dl, e, M, 3 * dl, dl, st));
        RC(lm_causal_attention(b.qkv16, n, s, dl, H, tokens, 0, b.att16, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b_out; e.out = b.x; e.resid = b.x; e.ldo = dl;
        RC(gemm_f16(b.att16, dl, w.w_out, dl, e, M, dl, dl, st));
        RC(layernorm_dual(b.x, b.x16, w.n1g, w.n1b, M, dl, 1e-6f, true, st));
        e = GemmEpilogue(); e.mode = EPI_F16; e.act = c.lm_activation == SBK_ACT_GELU ? ACT_GELU : ACT_RELU;
        e.bias = w.b1; e.out = b.f16; e.ldo = Fl;
        RC(gemm_f16(b.x16, dl, w.w1, dl, e, M, Fl, dl, st));
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.b2; e.out = b.x; e.resid = b.x; e.ldo = dl;
        RC(gemm_f16(b.f16, Fl, w.w2, Fl, e, M, dl, Fl, st));
        RC(layernorm_dual(b.x, b.x16, w.n2g, w.n2b, M, dl, 1e-6f, true, st));
    }
    RC(layernorm_dual(b.x, b.x16, m->lm_norm_g, m->lm_norm_b, M, dl, 1e-6f, false, st));  // encoder.norm
    // output_proj: Linear d -> d (fp32, into the free residual buffer), LayerNorm, Linear d -> vocab into the caller's logits
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->lm_bp0; e.out = b.x; e.ldo = dl;
    RC(gemm_f16(b.x16, dl, m->lm_wp0, dl, e, M, dl, dl, st));
    RC(layernorm_dual(b.x, b.x16, m->lm_lnp_g, m->lm_lnp_b, M, dl, 1e-6f, false, st));
    e = GemmEpilogue(); e.mode = EPI_F32; e.bias = m->lm_bp2; e.out = logits; e.ldo = c.vocab;
    RC(gemm_f16(b.x16, dl, m->lm_wp2, dl, e, M, c.vocab, dl, st));
    return SBK_OK;
}

}  // namespace sbk

// ============================================================================ C ABI
using namespace sbk;

extern "C" {

const char* sbk_last_error(void) { return sbk::last_error(); }

int sbk_version(void) { return 100; }

long long sbk_launch_count(void) { return sbk::launch_count(); }

void sbk_gemm_profile_enable(int on) {
    GemmProfile* p = gemm_profile();
    for (cudaEvent_t e : p->ev) cudaEventDestroy(e);
    p->ev.clear();
    p->flops.clear();
    p->shape.clear();
    p->enabled = on != 0;
}
// After a device sync: number of timed GEMM launches, their total milliseconds and total FLOPs.
int sbk_gemm_profile_read(int* n_launches, double* total_ms, double* total_flops) {
    GemmProfile* p = gemm_profile();
    double ms = 0.0, fl = 0.0;
    for (size_t i = 0; i < p->flops.size(); ++i) {
        float t = 0.0f;
        if (cudaEventElapsedTime(&t, p->ev[2 * i], p->ev[2 * i + 1]) != cudaSuccess) {
            set_error("sbk_gemm_profile_read: events not complete (synchronize first)");
            return SBK_ERR_CUDA;
        }
        ms += t;
        fl += p->flops[i];
        if (getenv("SBK_GEMM_TRACE"))
            fprintf(stderr, "gemm M=%d N=%d K=%d epi=%d : %.1f us  %.0f TFLOP/s\n", p->shape[4 * i], p->shape[4 * i + 1],
                    p->shape[4 * i + 2], p->shape[4 * i + 3], t * 1e3, p->flops[i] / (t * 1e-3) / 1e12);
    }
    if (n_launches) *n_launches = (int)p->flops.size();
    if (total_ms) *total_ms = ms;
    if (total_flops) *total_flops = fl;
    return SBK_OK;
}

int sbk_fbank_create(int n_fft, int hop, int n_mels, const float* window_host, const float* mel_matrix_host, float amin,
                     float top_db, sbk_fbank** out) {
    return fbank_create(reinterpret_cast<Fbank**>(out), n_fft, hop, n_mels, window_host, mel_matrix_host, amin, top_db);
}
void sbk_fbank_destroy(sbk_fbank* fb) { fbank_destroy(reinterpret_cast<Fbank*>(fb)); }
int sbk_fbank_num_frames(const sbk_fbank* fb, int n_samples) { return fbank_num_frames(reinterpret_cast<const Fbank*>(fb), n_samples); }
int sbk_fbank_forward(const sbk_fbank* fb, const float* wav_dev, int B, int L, float* out_dev, int* utt_max_scratch_dev,
                      void* stream) {
    return fbank_forward(reinterpret_cast<const Fbank*>(fb), wav_dev, B, L, out_dev, utt_max_scratch_dev, nullptr, nullptr,
                         0.0f, static_cast<cudaStream_t>(stream));
}
int sbk_input_norm_global(const float* x_dev, float* out_dev, int B, int T, int F, const float* mean_dev,
                          const float* std_dev, float eps, void* stream) {
    return global_norm_forward(x_dev, out_dev, B, T, F, mean_dev, std_dev, eps, static_cast<cudaStream_t>(stream));
}
int sbk_input_norm_sentence(const float* x_dev, float* out_dev, const float* rel_len_dev, int B, int T, int F,
                            int std_norm, int avoid_padding_norm, float eps, void* stream) {
    return sentence_norm_forward(x_dev, out_dev, rel_len_dev, B, T, F, std_norm, avoid_padding_norm, eps,
                                 static_cast<cudaStream_t>(stream));
}

int sbk_gemm_f16_test(const void* A_dev, const void* W_dev, const float* bias_dev, void* out_dev, int out_is_f32, int act,
                      int M, int N, int K, void* stream) {
    GemmEpilogue e;
    e.mode = out_is_f32 ? EPI_F32 : EPI_F16;
    e.act = act;
    e.bias = bias_dev;
    e.out = out_dev;
    e.ldo = N;
    return gemm_f16(A_dev, K, W_dev, K, e, M, N, K, static_cast<cudaStream_t>(stream));
}

int sbk_gemm_f16_resid_test(const void* A_dev, const void* W_dev, const float* bias_dev, float* x_dev, float alpha, int M,
                            int N, int K, void* stream) {
    GemmEpilogue e;
    e.mode = EPI_RESID;
    e.bias = bias_dev;
    e.out = x_dev;
    e.resid = x_dev;
    e.alpha = alpha;
    e.ldo = N;
    return gemm_f16(A_dev, K, W_dev, K, e, M, N, K, static_cast<cudaStream_t>(stream));
}

int sbk_gemm_epilogue_test(const void* A_dev, const void* W_dev, const float* bias_dev, void* out_dev, int ldo, int mode,
                           int act, float alpha, const float* resid_dev, const int* row_lens_dev, int T,
                           const float* rope_cos_dev, const float* rope_sin_dev, int head_dim, int kv_heads,
                           long long kv_part_stride, long long kv_layer_stride, int M, int N, int K, void* stream) {
    GemmEpilogue e;
    e.mode = mode; e.act = act; e.bias = bias_dev; e.out = out_dev; e.ldo = ldo; e.alpha = alpha;
    e.resid = resid_dev; e.row_lens = row_lens_dev; e.T = T;
    e.rope_cos = rope_cos_dev; e.rope_sin = rope_sin_dev; e.head_dim = head_dim;
    e.kv_heads = kv_heads; e.kv_part_stride = (size_t)kv_part_stride; e.kv_layer_stride = (size_t)kv_layer_stride;
    if (mode < EPI_F16 || mode > EPI_ROPE) { set_error("sbk_gemm_epilogue_test: mode %d", mode); return SBK_ERR_ARG; }
    return gemm_f16(A_dev, K, W_dev, K, e, M, N, K, static_cast<cudaStream_t>(stream));
}

int sbk_ctc_prefix_test(const float* logits_dev, const int* enc_len_dev, int B, int T, int V, int beam, int blank, int bos,
                        int eos, float weight, int accumulate, const int* hist_tok_dev, const int* hist_pred_dev, int n_steps,
                        float* scores_dev, int* group_width, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(logits_dev && enc_len_dev && hist_tok_dev && hist_pred_dev && scores_dev, "ctc_prefix_test: null pointer");
    SBK_REQUIRE(B >= 1 && T >= 1 && V >= 1 && beam >= 1 && n_steps >= 1, "ctc_prefix_test: bad sizes");
    SBK_REQUIRE(blank >= 0 && blank < V && bos >= 0 && bos < V && eos >= 0 && eos < V, "ctc_prefix_test: bad token ids");
    const int rows = B * beam;
    // the kernels index frames, parents and token columns with these: check them on the host first
    std::vector<int> len(B), tok((size_t)n_steps * rows), pred((size_t)n_steps * rows);
    SBK_CUDA_CHECK(cudaMemcpyAsync(len.data(), enc_len_dev, B * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(tok.data(), hist_tok_dev, tok.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(pred.data(), hist_pred_dev, pred.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int v : len) SBK_REQUIRE(v >= 0 && v <= T, "ctc_prefix_test: enc_len %d outside [0, %d]", v, T);
    for (size_t i = 0; i < tok.size(); ++i)
        SBK_REQUIRE(tok[i] >= 0 && tok[i] < V && pred[i] >= 0 && pred[i] < rows, "ctc_prefix_test: history entry %zu out of range", i);
    struct DevBufs {   // freed on every return path
        std::vector<void*> p;
        ~DevBufs() { for (void* q : p) cudaFree(q); }
    } bufs;
    auto alloc = [&](size_t n4, void** out) -> int {   // n4 4-byte elements
        if (cudaMalloc(out, n4 * 4) != cudaSuccess) { set_error("ctc_prefix_test: cudaMalloc(%zu) failed", n4 * 4); return SBK_ERR_NOMEM; }
        bufs.p.push_back(*out);
        return SBK_OK;
    };
    const size_t M = (size_t)B * T;
    float *x, *xlin, *xb, *rsum, *rb, *psi, *tab, *tabM;
    int* steps;
    RC(alloc(M * V, (void**)&x)); RC(alloc(M * V, (void**)&xlin)); RC(alloc(M, (void**)&xb));
    RC(alloc((size_t)2 * rows * T, (void**)&rsum)); RC(alloc((size_t)2 * rows * T, (void**)&rb)); RC(alloc((size_t)2 * rows, (void**)&psi));
    RC(alloc((size_t)2 * rows * (T + 4), (void**)&tab)); RC(alloc((size_t)2 * rows, (void**)&tabM));
    RC(alloc((size_t)n_steps * rows, (void**)&steps));
    std::vector<int> step_val((size_t)n_steps * rows);   // the beam search's per-row step counters, one row of them per step
    for (size_t i = 0; i < step_val.size(); ++i) step_val[i] = static_cast<int>(i / rows);
    SBK_CUDA_CHECK(cudaMemcpyAsync(steps, step_val.data(), step_val.size() * 4, cudaMemcpyHostToDevice, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(x, logits_dev, M * V * 4, cudaMemcpyDeviceToDevice, st));
    RC(ctc_prefix_reset(x, xlin, xb, enc_len_dev, B, T, V, blank, beam, rsum, rb, psi, tab, tabM, st));
    CtcStep cs{};
    cs.x = x; cs.xlin = xlin; cs.xb = xb; cs.enc_len = enc_len_dev; cs.hist_tok = hist_tok_dev; cs.hist_pred = hist_pred_dev;
    cs.n_bh = rows; cs.rsum_base = rsum; cs.rb_base = rb; cs.psi_base = psi; cs.tab = tab; cs.tabM = tabM;
    cs.bos = bos; cs.T = T; cs.V = V; cs.beam = beam; cs.blank = blank; cs.eos = eos; cs.weight = weight; cs.accumulate = accumulate ? 1 : 0;
    for (int s = 0; s < n_steps; ++s) {   // run_beam's order: update of the previous survivors, then the score
        cs.step_ptr = steps + (size_t)s * rows;
        cs.out = scores_dev + (size_t)s * rows * V;
        RC(ctc_prefix_update(cs, st));
        RC(ctc_prefix_score(cs, st));
    }
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    if (group_width) *group_width = ctc_prefix_group_width(beam, T);
    return SBK_OK;
}

int sbk_asr_create(const sbk_asr_config* cfg, const sbk_tensor* weights, int n_weights, sbk_asr** out) {
    return asr_create(cfg, weights, n_weights, reinterpret_cast<AsrModel**>(out));
}
void sbk_asr_destroy(sbk_asr* m) { asr_destroy(reinterpret_cast<AsrModel*>(m)); }
int sbk_asr_clone(sbk_asr* src, sbk_asr** out) {
    return asr_clone(reinterpret_cast<AsrModel*>(src), reinterpret_cast<AsrModel**>(out));
}
int sbk_asr_set_decoder_ln_fusion(sbk_asr* m, int on) {
    AsrModel* mm = reinterpret_cast<AsrModel*>(m);
    if (mm->fuse_dec_ln != (on != 0)) drop_graphs(mm);  // cached graphs were captured with the other kernel sequence
    mm->fuse_dec_ln = on != 0;
    return SBK_OK;
}
int sbk_asr_set_decoder_tc_min_rows(sbk_asr* m, int rows) {
    AsrModel* mm = reinterpret_cast<AsrModel*>(m);
    if (mm->dec_tc_rows != rows) drop_graphs(mm);
    mm->dec_tc_rows = rows;
    return SBK_OK;
}
int sbk_asr_set_dynchunk(sbk_asr* m, int chunk_size, int left_context_chunks) {
    AsrModel* mm = reinterpret_cast<AsrModel*>(m);
    SBK_REQUIRE(chunk_size >= 0, "set_dynchunk: chunk_size must be >= 0 (0 = full-context attention)");
    const int left = left_context_chunks < 0 ? -1 : left_context_chunks;
    if (mm->dyn_chunk != chunk_size || mm->dyn_left != left) drop_graphs(mm);  // cached graphs bake the kernel arguments in
    mm->dyn_chunk = chunk_size;
    mm->dyn_left = left;
    return SBK_OK;
}
int sbk_asr_set_poll_interval(sbk_asr* m, int every_n_steps) {
    reinterpret_cast<AsrModel*>(m)->poll_every = every_n_steps;
    return SBK_OK;
}

int sbk_asr_num_frames(const sbk_asr* mm, int n_samples, int* T_feat, int* T_enc) {
    const AsrModel* m = reinterpret_cast<const AsrModel*>(mm);
    int T0, T1, T2;
    frames(m->cfg, n_samples, &T0, &T1, &T2);
    if (T_feat) *T_feat = T0;
    if (T_enc) *T_enc = T2;
    return SBK_OK;
}

int sbk_asr_cnn_forward(sbk_asr* mm, const float* feats_dev, int B, int T0, float* out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    const sbk_asr_config& c = m->cfg;
    SBK_REQUIRE(m->has_cnn, "cnn_forward: this handle was created without CNN weights");
    const int L = (T0 - 1) * c.hop;
    RC(ensure_workspace(m, B, L, std::max(B, m->ws_rows), std::max(1, m->ws_steps)));
    return cnn_frontend_forward(feats_dev, B, T0, c.n_mels, m->c1_w, m->c1_b, m->c1_g, m->c1_be, c.cnn_c1, m->c2_w, m->c2_b,
                                m->c2_g, m->c2_be, c.cnn_c2, m->b.act1, nullptr, m->b.a_in, out_dev,
                                static_cast<cudaStream_t>(stream));
}

// src_dev: CNN output [B, T, input_size] fp32 -> enc_out_dev [B, T, d] fp32 (TransformerASR.encode)
int sbk_asr_encode_feats(sbk_asr* mm, const float* feats_dev, const float* rel_len_dev, int B, int T0,
                         float* cnn_out_dev, float* enc_out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->cfg;
    const int L = (T0 - 1) * c.hop;
    RC(ensure_workspace(m, B, L, std::max(B, m->ws_rows), std::max(1, m->ws_steps)));
    const int T1 = (T0 - 1) / 2 + 1, T = (T1 - 1) / 2 + 1;
    const int* enc_len = nullptr;
    if (rel_len_dev) {
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_len_dev, B, T, m->b.enc_len);
        SBK_LAUNCH_CHECK();
        enc_len = m->b.enc_len;
    }
    return run_encoder(m, feats_dev, B, T0, enc_len, cnn_out_dev, enc_out_dev ? enc_out_dev : m->b.enc_out, st);
}

int sbk_asr_encode_from_cnn(sbk_asr* mm, const float* src_dev, const float* rel_len_dev, int B, int T,
                            float* enc_out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->cfg;
    const int L = ((T - 1) * 4) * c.hop;  // any L whose frame count maps to >= T encoder frames
    RC(ensure_workspace(m, B, L, std::max(B, m->ws_rows), std::max(1, m->ws_steps)));
    RC(cast_f32_f16(src_dev, m->b.a_in, (size_t)B * T * c.input_size, st));
    const int* enc_len = nullptr;
    if (rel_len_dev) {
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_len_dev, B, T, m->b.enc_len);
        SBK_LAUNCH_CHECK();
        enc_len = m->b.enc_len;
    }
    return run_encoder(m, nullptr, B, T, enc_len, nullptr, enc_out_dev ? enc_out_dev : m->b.enc_out, st);
}

// Full device pipeline on device-resident wav: Fbank -> global CMVN -> CNN -> encoder -> greedy.
// Outputs (device, optional): enc_out [B,T,d] fp32; pred [B, max_steps] int32; score [B, max_steps] fp32.
static int transcribe_enqueue(AsrModel* m, const float* wav_dev, const float* rel_len_dev, int B, int L, int max_steps,
                              int bos, int eos, float* enc_out_dev, int* pred_dev, float* score_dev, float* log_probs_dev,
                              int* steps_done, cudaStream_t st, bool in_capture) {
    const sbk_asr_config& c = m->cfg;
    int T0, T1, T;
    frames(c, L, &T0, &T1, &T);
    AsrModel::Buf& b = m->b;
    RC(fbank_forward(m->fbank, wav_dev, B, L, b.feats, b.utt_max, m->glob_mean, m->glob_std, c.norm_eps > 0.0f ? c.norm_eps : 1e-10f, st));
    const int* enc_len = nullptr;
    if (rel_len_dev) {
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_len_dev, B, T, b.enc_len);
        SBK_LAUNCH_CHECK();
        enc_len = b.enc_len;
    } else {
        std::vector<int> full(B, T);
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_len, full.data(), B * 4, cudaMemcpyHostToDevice, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
        enc_len = b.enc_len;
    }
    RC(run_encoder(m, b.feats, B, T0, enc_len, nullptr, b.enc_out, st));
    if (enc_out_dev)
        SBK_CUDA_CHECK(cudaMemcpyAsync(enc_out_dev, b.enc_out, (size_t)B * T * c.d_model * 4, cudaMemcpyDeviceToDevice, st));
    int done = 0;
    if (max_steps > 0 && m->has_dec) {
        RC(run_greedy(m, B, T, max_steps, bos, eos, log_probs_dev, &done, st, in_capture));
        const int S_max = m->ws_steps + 1;
        if (pred_dev)
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(pred_dev, (size_t)max_steps * 4, b.pred, (size_t)S_max * 4, (size_t)done * 4, B,
                                             cudaMemcpyDeviceToDevice, st));
        if (score_dev)
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(score_dev, (size_t)max_steps * 4, b.score, (size_t)S_max * 4, (size_t)done * 4, B,
                                             cudaMemcpyDeviceToDevice, st));
    }
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// G independent batches of B utterances: each batch goes through Fbank..encoder on its own (B-utterance kernels),
// then ONE greedy loop decodes all G*B hypotheses together.  A decode step is ~50 dependent, latency-bound kernels
// whose cost barely depends on the row count, so coalescing the decode of the
// batches in flight amortises it G-fold; per-utterance results are unchanged (rows are independent).
static int transcribe_group_enqueue(AsrModel* m, int G, const float* const* wav_dev, const float* const* rel_dev, int B, int L,
                                    int max_steps, int bos, int eos, int* const* pred_dev, int* steps_done, cudaStream_t st,
                                    bool in_capture, const cudaEvent_t* ready = nullptr, int* const* pred_host = nullptr) {
    const sbk_asr_config& c = m->cfg;
    int T0, T1, T;
    frames(c, L, &T0, &T1, &T);
    AsrModel::Buf& b = m->b;
    for (int g = 0; g < G; ++g) {
        if (ready) SBK_CUDA_CHECK(cudaStreamWaitEvent(st, ready[g], 0));  // batch g's wav has landed in the staging buffer
        RC(fbank_forward(m->fbank, wav_dev[g], B, L, b.feats, b.utt_max, m->glob_mean, m->glob_std, c.norm_eps > 0.0f ? c.norm_eps : 1e-10f, st));
        int* enc_len = b.enc_len + (size_t)g * B;
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_dev[g], B, T, enc_len);
        SBK_LAUNCH_CHECK();
        RC(run_encoder(m, b.feats, B, T0, enc_len, nullptr, b.enc_out + (size_t)g * B * T * c.d_model, st));
    }
    // The decode loop is a chain of ~3300 small, latency-bound kernels; the encoders of the other lanes are machine-filling
    // ones.  Its kernels go to a stream of the highest priority (under capture: kernel nodes of that priority), so that a ready
    // decode kernel gets the next free SM slots ahead of the remaining CTAs of an encoder kernel instead of queueing behind
    // them.  SBK_DEC_PRIORITY=0: same stream as the encoders.
    static const bool prio = getenv("SBK_DEC_PRIORITY") == nullptr || atoi(getenv("SBK_DEC_PRIORITY")) != 0;
    cudaStream_t ds = st;
    if (prio) {
        if (!m->dec_stream) {
            int lo = 0, hi = 0;
            SBK_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));  // numerically lowest = highest priority
            SBK_CUDA_CHECK(cudaStreamCreateWithPriority(&m->dec_stream, cudaStreamNonBlocking, hi));
            SBK_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_dfork, cudaEventDisableTiming));
            SBK_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_djoin, cudaEventDisableTiming));
        }
        ds = m->dec_stream;
        SBK_CUDA_CHECK(cudaEventRecord(m->ev_dfork, st));
        SBK_CUDA_CHECK(cudaStreamWaitEvent(ds, m->ev_dfork, 0));
    }
    int done = 0;
    RC(run_greedy(m, G * B, T, max_steps, bos, eos, nullptr, &done, ds, in_capture));
    const int S_max = m->ws_steps + 1;
    for (int g = 0; g < G; ++g) {
        if (pred_dev && pred_dev[g])
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(pred_dev[g], (size_t)max_steps * 4, b.pred + (size_t)g * B * S_max, (size_t)S_max * 4,
                                             (size_t)done * 4, B, cudaMemcpyDeviceToDevice, ds));
        if (pred_host && pred_host[g])
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(pred_host[g], (size_t)max_steps * 4, b.pred + (size_t)g * B * S_max, (size_t)S_max * 4,
                                             (size_t)done * 4, B, cudaMemcpyDeviceToHost, ds));
    }
    if (prio) {
        SBK_CUDA_CHECK(cudaEventRecord(m->ev_djoin, ds));
        SBK_CUDA_CHECK(cudaStreamWaitEvent(st, m->ev_djoin, 0));
    }
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// Host-buffer form of the group call: H2D of every batch on a copy stream forked from `st` (batch g+1's copy overlaps
// batch g's encoder), the group pipeline, D2H of the token ids.  Works both eagerly and under stream capture (the fork /
// join events become graph edges, the copies memcpy nodes).
static int transcribe_group_host_enqueue(AsrModel* m, int G, const float* const* wav_host, const float* const* rel_host, int B,
                                         int L, int max_steps, int bos, int eos, int* const* pred_host, int* const* pred_dev,
                                         int* steps_done, cudaStream_t st, bool in_capture) {
    SBK_CUDA_CHECK(cudaEventRecord(m->ev_fork, st));
    SBK_CUDA_CHECK(cudaStreamWaitEvent(m->copy_stream, m->ev_fork, 0));  // the previous call no longer reads the staging buffers
    const float* wav_dev[16];
    const float* rel_dev[16];
    for (int g = 0; g < G; ++g) {
        float* w = m->gwav + (size_t)g * B * L;
        float* r = m->grel + (size_t)g * B;
        SBK_CUDA_CHECK(cudaMemcpyAsync(w, wav_host[g], (size_t)B * L * 4, cudaMemcpyHostToDevice, m->copy_stream));
        SBK_CUDA_CHECK(cudaMemcpyAsync(r, rel_host[g], (size_t)B * 4, cudaMemcpyHostToDevice, m->copy_stream));
        SBK_CUDA_CHECK(cudaEventRecord(m->ev_ready[g], m->copy_stream));
        wav_dev[g] = w; rel_dev[g] = r;
    }
    return transcribe_group_enqueue(m, G, wav_dev, rel_dev, B, L, max_steps, bos, eos, pred_dev, steps_done, st, in_capture,
                                    m->ev_ready, pred_host);
}

int sbk_asr_transcribe_greedy_group_dev(sbk_asr* mm, int G, const float* const* wav_dev, const float* const* rel_len_dev,
                                        int B, int L, int max_steps, int bos, int eos, int* const* pred_dev, int* steps_done,
                                        void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(G >= 1 && G <= 16, "transcribe_group: G=%d not in [1, 16]", G);
    SBK_REQUIRE(m->has_fbank && m->has_cnn && m->has_enc && m->has_dec, "transcribe_group: handle lacks model parts");
    SBK_REQUIRE(m->glob_mean != nullptr, "transcribe_group: model has no normalize.glob_mean/std weights");
    for (int g = 0; g < G; ++g) SBK_REQUIRE(wav_dev[g] && rel_len_dev[g], "transcribe_group: null batch pointer");
    RC(ensure_workspace(m, B, L, std::max(G * B, m->ws_rows), std::max(max_steps, m->ws_steps)));
    const bool whole_graph = m->poll_every == 0 && getenv("SBK_NO_GRAPH") == nullptr && max_steps > 0;
    if (!whole_graph) return transcribe_group_enqueue(m, G, wav_dev, rel_len_dev, B, L, max_steps, bos, eos, pred_dev, steps_done, st, false);
    AsrModel::GroupKey key;
    memset(&key, 0, sizeof(key));
    key.G = G; key.B = B; key.L = L; key.steps = max_steps; key.bos = bos; key.eos = eos;
    for (int g = 0; g < G; ++g) { key.wav[g] = wav_dev[g]; key.rel[g] = rel_len_dev[g]; key.pred[g] = pred_dev[g]; }
    if (m->group_graph == nullptr || memcmp(&key, &m->group_key, sizeof(key)) != 0) {
        if (m->group_graph) { cudaGraphExecDestroy(m->group_graph); m->group_graph = nullptr; }
        if (!m->cap_stream) SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        cudaGraph_t gr;
        SBK_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
        launch_count_begin_capture();
        int done = 0;
        int rc = transcribe_group_enqueue(m, G, wav_dev, rel_len_dev, B, L, max_steps, bos, eos, pred_dev, &done, m->cap_stream, true);
        m->group_nodes = launch_count_end_capture();
        cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &gr);
        if (rc) return rc;
        SBK_CUDA_CHECK(ce);
        SBK_CUDA_CHECK(cudaGraphInstantiate(&m->group_graph, gr, 0));
        cudaGraphDestroy(gr);
        m->group_key = key;
    }
    SBK_CUDA_CHECK(cudaGraphLaunch(m->group_graph, st));
    launch_count_add(m->group_nodes);
    if (steps_done) *steps_done = max_steps;
    return SBK_OK;
}

// Same pipeline from HOST buffers (pinned): the call EncoderDecoderASR.transcribe_batch makes, for G batches at once.
// Enqueue only; the caller synchronises `stream`.  pred_dev (optional, may be NULL or hold NULLs) also keeps the ids on the
// device (multi-GPU: the hypothesis all-gather reads them).
int sbk_asr_transcribe_greedy_group_host_async(sbk_asr* mm, int G, const float* const* wav_host,
                                               const float* const* rel_len_host, int B, int L, int max_steps, int bos, int eos,
                                               int* const* pred_host, int* const* pred_dev, int* steps_done, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(G >= 1 && G <= 16, "transcribe_group_host: G=%d not in [1, 16]", G);
    SBK_REQUIRE(m->has_fbank && m->has_cnn && m->has_enc && m->has_dec, "transcribe_group_host: handle lacks model parts");
    SBK_REQUIRE(m->glob_mean != nullptr, "transcribe_group_host: model has no normalize.glob_mean/std weights");
    SBK_REQUIRE(wav_host && rel_len_host && pred_host, "transcribe_group_host: null argument");
    for (int g = 0; g < G; ++g) SBK_REQUIRE(wav_host[g] && rel_len_host[g] && pred_host[g], "transcribe_group_host: null batch pointer");
    RC(ensure_workspace(m, B, L, std::max(G * B, m->ws_rows), std::max(max_steps, m->ws_steps)));
    const size_t need = (size_t)G * B * L * 4 + (size_t)G * B * 4 + 256;
    if (need > m->gwav_cap) {
        if (m->gwav) { SBK_CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(m->gwav); m->gwav = nullptr; m->gwav_cap = 0; }
        if (m->hgroup_graph) { cudaGraphExecDestroy(m->hgroup_graph); m->hgroup_graph = nullptr; }
        if (cudaMalloc(&m->gwav, need) != cudaSuccess) { set_error("transcribe_group_host: cudaMalloc(%zu) failed", need); return SBK_ERR_NOMEM; }
        m->gwav_cap = need;
    }
    m->grel = m->gwav + (size_t)G * B * L;  // lengths behind the G waveforms
    if (!m->copy_stream) {
        SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
        SBK_CUDA_CHECK(cudaEventCreateWithFlags(&m->ev_fork, cudaEventDisableTiming));
        for (auto& e : m->ev_ready) SBK_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    const bool whole_graph = m->poll_every == 0 && getenv("SBK_NO_GRAPH") == nullptr && max_steps > 0;
    if (!whole_graph)
        return transcribe_group_host_enqueue(m, G, wav_host, rel_len_host, B, L, max_steps, bos, eos, pred_host, pred_dev,
                                             steps_done, st, false);
    AsrModel::HostGroupKey key;
    memset(&key, 0, sizeof(key));
    key.G = G; key.B = B; key.L = L; key.steps = max_steps; key.bos = bos; key.eos = eos;
    for (int g = 0; g < G; ++g) {
        key.wav[g] = wav_host[g]; key.rel[g] = rel_len_host[g]; key.pred[g] = pred_host[g];
        key.pred_dev[g] = pred_dev ? pred_dev[g] : nullptr;
    }
    if (m->hgroup_graph == nullptr || memcmp(&key, &m->hgroup_key, sizeof(key)) != 0) {
        if (m->hgroup_graph) { cudaGraphExecDestroy(m->hgroup_graph); m->hgroup_graph = nullptr; }
        if (!m->cap_stream) SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        cudaGraph_t gr;
        SBK_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
        launch_count_begin_capture();
        int done = 0;
        int rc = transcribe_group_host_enqueue(m, G, wav_host, rel_len_host, B, L, max_steps, bos, eos, pred_host, pred_dev, &done,
                                               m->cap_stream, true);
        m->hgroup_nodes = launch_count_end_capture();
        cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &gr);
        if (rc) return rc;
        SBK_CUDA_CHECK(ce);
        SBK_CUDA_CHECK(cudaGraphInstantiate(&m->hgroup_graph, gr, 0));
        cudaGraphDestroy(gr);
        m->hgroup_key = key;
    }
    SBK_CUDA_CHECK(cudaGraphLaunch(m->hgroup_graph, st));
    launch_count_add(m->hgroup_nodes);
    if (steps_done) *steps_done = max_steps;
    return SBK_OK;
}

int sbk_asr_transcribe_greedy_dev(sbk_asr* mm, const float* wav_dev, const float* rel_len_dev, int B, int L,
                                  int max_steps, int bos, int eos, float* enc_out_dev, int* pred_dev, float* score_dev,
                                  float* log_probs_dev, int* steps_done, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(m->has_fbank && m->has_cnn && m->has_enc, "transcribe: handle lacks fbank/CNN/encoder weights");
    SBK_REQUIRE(m->glob_mean != nullptr, "transcribe: model has no normalize.glob_mean/std (global CMVN) weights");
    RC(ensure_workspace(m, B, L, std::max(B, m->ws_rows), std::max(max_steps, m->ws_steps)));
    // Fixed-length runs (poll interval 0) replay ONE CUDA graph of the whole pipeline (Fbank .. last decode step):
    // ~2.6k kernel nodes, a single host-side launch per batch.
    const bool whole_graph = m->poll_every == 0 && rel_len_dev != nullptr && log_probs_dev == nullptr &&
                             getenv("SBK_NO_GRAPH") == nullptr && (max_steps == 0 || m->has_dec);
    if (!whole_graph)
        return transcribe_enqueue(m, wav_dev, rel_len_dev, B, L, max_steps, bos, eos, enc_out_dev, pred_dev, score_dev,
                                  log_probs_dev, steps_done, st, false);
    AsrModel::PipeKey key;
    memset(&key, 0, sizeof(key));  // the struct has tail padding and is compared with memcmp
    key.wav = wav_dev; key.rel = rel_len_dev; key.enc = enc_out_dev; key.pred = pred_dev; key.score = score_dev;
    key.B = B; key.L = L; key.steps = max_steps; key.bos = bos; key.eos = eos;
    if (m->pipe_graph == nullptr || memcmp(&key, &m->pipe_key, sizeof(key)) != 0) {
        if (m->pipe_graph) { cudaGraphExecDestroy(m->pipe_graph); m->pipe_graph = nullptr; }
        if (!m->cap_stream) SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        cudaGraph_t g;
        SBK_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
        launch_count_begin_capture();
        int done = 0;
        int rc = transcribe_enqueue(m, wav_dev, rel_len_dev, B, L, max_steps, bos, eos, enc_out_dev, pred_dev, score_dev,
                                    nullptr, &done, m->cap_stream, true);
        m->pipe_nodes = launch_count_end_capture();
        cudaError_t ce = cudaStreamEndCapture(m->cap_stream, &g);
        if (rc) return rc;
        SBK_CUDA_CHECK(ce);
        SBK_CUDA_CHECK(cudaGraphInstantiate(&m->pipe_graph, g, 0));
        cudaGraphDestroy(g);
        m->pipe_key = key;
    }
    SBK_CUDA_CHECK(cudaGraphLaunch(m->pipe_graph, st));
    launch_count_add(m->pipe_nodes);
    if (steps_done) *steps_done = max_steps;
    return SBK_OK;
}

// Greedy search from caller-provided encoder states (S2STransformerGreedySearcher.forward).
int sbk_asr_greedy_from_enc(sbk_asr* mm, const float* enc_dev, const float* rel_len_dev, int B, int T, int max_steps,
                            int bos, int eos, int* pred_dev, float* score_dev, float* log_probs_dev, int* steps_done,
                            void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->cfg;
    // workspace sized from T: pick L such that frames(L) -> T
    const int L = std::max(m->wsL, ((T - 1) * 4) * c.hop);
    RC(ensure_workspace(m, std::max(B, m->wsB), L, std::max(B, m->ws_rows), std::max(max_steps, m->ws_steps)));
    AsrModel::Buf& b = m->b;
    SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_out, enc_dev, (size_t)B * T * c.d_model * 4, cudaMemcpyDeviceToDevice, st));
    if (rel_len_dev) {
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_len_dev, B, T, b.enc_len);
        SBK_LAUNCH_CHECK();
    } else {
        std::vector<int> full(B, T);
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_len, full.data(), B * 4, cudaMemcpyHostToDevice, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    int done = 0;
    RC(run_greedy(m, B, T, max_steps, bos, eos, log_probs_dev, &done, st));
    const int S_max = m->ws_steps + 1;
    if (pred_dev && done > 0)
        SBK_CUDA_CHECK(cudaMemcpy2DAsync(pred_dev, (size_t)max_steps * 4, b.pred, (size_t)S_max * 4, (size_t)done * 4, B,
                                         cudaMemcpyDeviceToDevice, st));
    if (score_dev && done > 0)
        SBK_CUDA_CHECK(cudaMemcpy2DAsync(score_dev, (size_t)max_steps * 4, b.score, (size_t)S_max * 4, (size_t)done * 4, B,
                                         cudaMemcpyDeviceToDevice, st));
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// S2STransformerBeamSearcher.forward device part: history arrays are [max_steps, B * beam_size] (device).
int sbk_asr_beam_from_enc(sbk_asr* mm, const float* enc_dev, const float* rel_len_dev, int B, int T,
                          const sbk_beam_params* params, int* hist_tok_dev, int* hist_pred_dev, float* hist_score_dev,
                          float* hist_lp_dev, int* steps_done, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->cfg;
    SBK_REQUIRE(params && params->beam_size >= 1, "beam: bad params");
    const int rows = B * params->beam_size;
    const int L = std::max(m->wsL, ((T - 1) * 4) * c.hop);
    RC(ensure_workspace(m, std::max(B, m->wsB), L, std::max(rows, m->ws_rows), std::max(params->max_steps, m->ws_steps)));
    AsrModel::Buf& b = m->b;
    SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_out, enc_dev, (size_t)B * T * c.d_model * 4, cudaMemcpyDeviceToDevice, st));
    if (rel_len_dev) {
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_len_dev, B, T, b.enc_len);
        SBK_LAUNCH_CHECK();
    } else {
        std::vector<int> full(B, T);
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_len, full.data(), B * 4, cudaMemcpyHostToDevice, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    int done = 0;
    RC(run_beam(m, B, T, *params, hist_tok_dev, hist_pred_dev, hist_score_dev, hist_lp_dev, &done, st));
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// Host-buffer entry point (the call EncoderDecoderASR.transcribe_batch makes): wav/rel_len/pred are HOST
// (ideally pinned) buffers; H2D and D2H copies are part of the call.
static int transcribe_greedy_host_impl(sbk_asr* mm, const float* wav_host, const float* rel_len_host, int B, int L,
                                       int max_steps, int bos, int eos, int* pred_host, float* score_host, int* steps_done,
                                       void* stream, bool sync) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RC(ensure_workspace(m, B, L, std::max(B, m->ws_rows), std::max(max_steps, m->ws_steps)));
    AsrModel::Buf& b = m->b;
    SBK_CUDA_CHECK(cudaMemcpyAsync(b.wav, wav_host, (size_t)B * L * 4, cudaMemcpyHostToDevice, st));
    const float* rel_dev = nullptr;
    if (rel_len_host) {
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.rel_len, rel_len_host, B * 4, cudaMemcpyHostToDevice, st));
        rel_dev = b.rel_len;
    }
    int done = 0;
    RC(sbk_asr_transcribe_greedy_dev(mm, b.wav, rel_dev, B, L, max_steps, bos, eos, nullptr, nullptr, nullptr, nullptr, &done,
                                     stream));
    const int S_max = m->ws_steps + 1;
    if (done > 0) {
        if (pred_host)
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(pred_host, (size_t)max_steps * 4, b.pred, (size_t)S_max * 4, (size_t)done * 4, B,
                                             cudaMemcpyDeviceToHost, st));
        if (score_host)
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(score_host, (size_t)max_steps * 4, b.score, (size_t)S_max * 4, (size_t)done * 4, B,
                                             cudaMemcpyDeviceToHost, st));
    }
    if (sync) SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

int sbk_asr_transcribe_greedy_host(sbk_asr* mm, const float* wav_host, const float* rel_len_host, int B, int L,
                                   int max_steps, int bos, int eos, int* pred_host, float* score_host, int* steps_done,
                                   void* stream) {
    return transcribe_greedy_host_impl(mm, wav_host, rel_len_host, B, L, max_steps, bos, eos, pred_host, score_host,
                                       steps_done, stream, true);
}
// Same, but only ENQUEUES the copies and kernels (pinned buffers required); the caller synchronises the stream.
int sbk_asr_transcribe_greedy_host_async(sbk_asr* mm, const float* wav_host, const float* rel_len_host, int B, int L,
                                         int max_steps, int bos, int eos, int* pred_host, float* score_host,
                                         int* steps_done, void* stream) {
    return transcribe_greedy_host_impl(mm, wav_host, rel_len_host, B, L, max_steps, bos, eos, pred_host, score_host,
                                       steps_done, stream, false);
}

// torch.max(dim=-1) indices of a [rows, V] fp32 matrix (ctc_greedy_decode's arg-max, decoders/ctc.py:375)
int sbk_rows_argmax_f32(const float* x_dev, int rows, int V, int* idx_dev, void* stream) {
    SBK_REQUIRE(x_dev && idx_dev && rows >= 0 && V >= 1, "rows_argmax: bad arguments");
    return rows_logsoftmax_argmax(const_cast<float*>(x_dev), rows, V, false, idx_dev, static_cast<cudaStream_t>(stream));
}

// CTC head of an encoder-only recogniser (EncoderASR, inference/ASR.py:176-389): enc_dev [B, T, d] fp32 (NULL = the encoder
// states left in the workspace by the previous encode call) -> log_probs_dev [B, T, V] fp32 = log_softmax(ctc_lin(enc)) (optional)
// and argmax_dev [B, T] int32 (optional) -- the per-frame arg-max ctc_greedy_decode (decoders/ctc.py:335-378) starts from.
int sbk_asr_ctc_head(sbk_asr* mm, const float* enc_dev, int B, int T, float* log_probs_dev, int* argmax_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->cfg;
    SBK_REQUIRE(m->w_ctc != nullptr, "ctc_head: this handle was created without ctc_lin.w.* weights");
    SBK_REQUIRE(B >= 1 && T >= 1 && (log_probs_dev || argmax_dev), "ctc_head: bad arguments");
    const int L = std::max(m->wsL, ((T - 1) * 4) * c.hop);
    RC(ensure_workspace(m, std::max(B, m->wsB), L, std::max(B, m->ws_rows), std::max(1, m->ws_steps)));
    AsrModel::Buf& b = m->b;
    const size_t M = (size_t)B * T, V = c.vocab;
    if (enc_dev) SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_out, enc_dev, M * c.d_model * 4, cudaMemcpyDeviceToDevice, st));
    float* logits = log_probs_dev;
    if (!logits) {  // arg-max only: the logits live in the (lazily grown) CTC scratch buffer
        AsrModel::CtcBuf& cb = m->ctc;
        const size_t need = M * V * 4 + 256;
        if (need > cb.cap) {
            if (cb.base) { SBK_CUDA_CHECK(cudaStreamSynchronize(st)); cudaFree(cb.base); cb.base = nullptr; cb.cap = 0; }
            if (cudaMalloc(&cb.base, need) != cudaSuccess) { set_error("ctc_head: cudaMalloc(%zu) failed", need); return SBK_ERR_NOMEM; }
            cb.cap = need;
        }
        logits = cb.base;
    }
    RC(cast_f32_f16(b.enc_out, b.enc16, M * c.d_model, st));
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->b_ctc; e.out = logits; e.ldo = c.vocab;
    RC(gemm_f16(b.enc16, c.d_model, m->w_ctc, c.d_model, e, (int)M, c.vocab, c.d_model, st));
    return rows_logsoftmax_argmax(logits, (int)M, c.vocab, log_probs_dev != nullptr, argmax_dev, st);
}

// TransformerASR.decode(tgt, encoder_out, enc_len) (TransformerASR.py:426-473): tgt_dev [n, S] int32 token ids (teacher
// forcing, bos first), enc_dev [n, T, d] fp32, enc_len_dev [n] int32 ABSOLUTE frame counts (or NULL = all T) ->
// out_dev [n, S, d] fp32 = decoder.norm(decoder(...)).  The attention-weight output of the reference is not produced.
int sbk_asr_decode_teacher_forced(sbk_asr* mm, const int* tgt_dev, const float* enc_dev, const int* enc_len_dev, int n, int S,
                                  int T, float* out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->cfg;
    SBK_REQUIRE(tgt_dev && enc_dev && out_dev && n >= 1 && S >= 1 && T >= 1, "decode: bad arguments");
    const int L = std::max(m->wsL, ((T - 1) * 4) * c.hop);
    RC(ensure_workspace(m, std::max(n, m->wsB), L, std::max(n, m->ws_rows), std::max(S, m->ws_steps)));
    AsrModel::Buf& b = m->b;
    SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_out, enc_dev, (size_t)n * T * c.d_model * 4, cudaMemcpyDeviceToDevice, st));
    if (enc_len_dev) {
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_len, enc_len_dev, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    } else {
        std::vector<int> full(n, T);
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_len, full.data(), n * 4, cudaMemcpyHostToDevice, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    return run_decode_teacher(m, tgt_dev, n, S, T, out_dev, st);
}

// TransformerLMRescorer.rescore_hyps device part: tokens [n, L] int32 (bos ... eos, pad-filled), lens [n] int32 (device) ->
// scores [n] fp32 (device) = sum over the sequence of log p(token | prefix) at `temperature`, pad column excluded.
int sbk_asr_lm_rescore(sbk_asr* mm, const int* tokens_dev, const int* lens_dev, int n, int L, float temperature, int pad_index,
                       float* scores_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(m->has_lm, "lm_rescore: this handle was created without TransformerLM weights");
    SBK_REQUIRE(n >= 1 && L >= 2 && L <= m->cfg.max_len && pad_index >= 0 && pad_index < m->cfg.vocab && temperature > 0.0f,
                "lm_rescore: bad arguments (n=%d L=%d pad=%d)", n, L, pad_index);
    SBK_REQUIRE(pad_index == 0, "lm_rescore: pad_index must be 0 (TransformerLM.make_masks pads with index 0)");
    RC(ensure_workspace(m, std::max(1, m->wsB), std::max(m->wsL, 4 * m->cfg.hop), std::max(n, m->ws_rows), std::max(L, m->ws_steps)));
    return run_lm_rescore(m, tokens_dev, lens_dev, n, L, temperature, pad_index, scores_dev, st);
}

// TransformerLM.forward(src) (TransformerLM.py:127-169): tokens_dev [n, s] int32 (pad id 0) -> logits_dev [n, s, vocab] fp32.
int sbk_asr_lm_forward(sbk_asr* mm, const int* tokens_dev, int n, int s, float* logits_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m != nullptr && tokens_dev && logits_dev, "lm_forward: null argument");
    SBK_REQUIRE(m->has_lm, "lm_forward: this handle was created without TransformerLM weights");
    SBK_REQUIRE(n >= 1 && s >= 1, "lm_forward: bad shape n=%d s=%d", n, s);
    SBK_REQUIRE(n <= 65535, "lm_forward: n=%d sequences exceed the 65535 of one call (attention grid z)", n);
    SBK_REQUIRE(s <= m->cfg.max_len, "lm_forward: s=%d exceeds max_len=%d", s, m->cfg.max_len);
    SBK_REQUIRE((long long)n * s * std::max(m->cfg.vocab, 3 * m->cfg.lm_d_model) < (1LL << 31),
                "lm_forward: n * s = %lld token rows is too many for one call", (long long)n * s);
    return run_lm_forward(m, tokens_dev, n, s, logits_dev, static_cast<cudaStream_t>(stream));
}

// Step-by-step counterpart of sbk_asr_lm_forward on the KV-cached LM step: tokens_dev [n, L] -> logits_dev [n, L, vocab].
int sbk_asr_lm_step_logits(sbk_asr* mm, const int* tokens_dev, int n, int L, float* logits_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m != nullptr && tokens_dev && logits_dev, "lm_step_logits: null argument");
    SBK_REQUIRE(m->has_lm, "lm_step_logits: this handle was created without TransformerLM weights");
    SBK_REQUIRE(n >= 1 && L >= 1 && L <= m->cfg.max_len, "lm_step_logits: bad shape n=%d L=%d (max_len %d)", n, L, m->cfg.max_len);
    RC(ensure_workspace(m, std::max(1, m->wsB), std::max(m->wsL, 4 * m->cfg.hop), std::max(n, m->ws_rows), std::max(L, m->ws_steps)));
    return run_lm_step_logits(m, tokens_dev, n, L, logits_dev, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
