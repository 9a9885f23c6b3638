// Weight loading: the one place that knows the reference's state_dict keys and the device formats the kernels read.
//
// Weights arrive as HOST fp32 arrays named exactly like the reference state_dict (SURVEY.md 8b) with the recipe's module
// prefixes:  "CNN.", "Transformer.", "seq_lin.", "ctc_lin.", "lm.", plus "normalize.glob_mean/std" and "fbank.window" /
// "fbank.mel_matrix".  They are repacked (fp16 GEMM operands, interleaved GLU rows, concatenated cross-attention K/V
// projections, pre-scaled queries, tap-major depthwise taps, sine tables) into one device arena.  The packing is one function,
// pack(), that runs twice through a Carver: once to check every tensor and measure the arena, once to upload.
#include <math.h>
#include <string.h>

#include <map>
#include <string>

#include "asr_weights.h"
#include "common.cuh"

namespace sbk {

using WeightMap = std::map<std::string, std::pair<const float*, int64_t>>;

// Places tensors in the arena one after another.  While carve.base is null it only checks and measures: keys are looked
// up and their element counts validated, nothing is converted or copied, and the device pointers it returns are null.
struct Packer {
    const WeightMap& w;
    Carver carve;
    bool ok = true;
    std::vector<__half> tmph;
    bool has(const std::string& k) const { return w.count(k) != 0; }
    int64_t numel(const std::string& k) const { return has(k) ? w.at(k).second : 0; }
    // the host tensor itself, for a repack (null, with ok cleared and the error set, when it is missing or mis-sized)
    const float* host(const std::string& k, int64_t n) {
        auto it = w.find(k);
        if (it == w.end())
            set_error("missing weight '%s'", k.c_str());
        else if (it->second.second != n)
            set_error("weight '%s' has %lld elements, expected %lld", k.c_str(), (long long)it->second.second, (long long)n);
        else
            return it->second.first;
        ok = false;
        return nullptr;
    }
    // the next `bytes` of the arena, filled from src
    void* place(const void* src, size_t bytes) {
        uint8_t* d = nullptr;
        carve(d, bytes);
        if (d && cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
            ok = false;
            set_error("weight upload failed");
        }
        return d;
    }
    const float* f32_raw(const float* src, int64_t n) { return static_cast<const float*>(place(src, n * 4)); }
    const __half* f16_raw(const float* src, int64_t n) {
        if (carve.base) {
            tmph.resize(n);
            for (int64_t i = 0; i < n; ++i) tmph[i] = __float2half_rn(src[i]);
        }
        return static_cast<const __half*>(place(tmph.data(), n * 2));
    }
    const float* f32_raw(const std::vector<float>& v) { return f32_raw(v.data(), v.size()); }
    const __half* f16_raw(const std::vector<float>& v) { return f16_raw(v.data(), v.size()); }
    // float64 products, rounded once to the stored type
    const float* f32_raw(const std::vector<double>& v) { return f32_raw(std::vector<float>(v.begin(), v.end())); }
    const __half* f16_raw(const std::vector<double>& v) {
        if (carve.base) {
            tmph.resize(v.size());
            for (size_t i = 0; i < v.size(); ++i) tmph[i] = __double2half(v[i]);
        }
        return static_cast<const __half*>(place(tmph.data(), v.size() * 2));
    }
    const float* f32(const std::string& k, int64_t n) {
        const float* src = host(k, n);
        return src ? f32_raw(src, n) : nullptr;
    }
    const __half* f16(const std::string& k, int64_t n) {
        const float* src = host(k, n);
        return src ? f16_raw(src, n) : nullptr;
    }
    // prefix.weight -> fp16 [out, in], prefix.bias -> fp32 [out]
    void linear(const std::string& prefix, int64_t out, int64_t in, const __half** wgt, const float** bias) {
        *wgt = f16(prefix + ".weight", out * in);
        *bias = f32(prefix + ".bias", out);
    }
    // LayerNorm prefix.weight, prefix.bias -> fp32 [n]
    void norm(const std::string& prefix, int64_t n, const float** gamma, const float** beta) {
        *gamma = f32(prefix + ".weight", n);
        *beta = f32(prefix + ".bias", n);
    }
};

// ---- host repacks

std::vector<float> sine_table(int rows, int d) {
    std::vector<float> pe((size_t)rows * d);
    for (int i = 0; i < d / 2; ++i) {
        const float den = expf((float)(2 * i) * -(logf(10000.0f) / (float)d));
        for (int t = 0; t < rows; ++t) {
            pe[(size_t)t * d + 2 * i] = sinf((float)t * den);
            pe[(size_t)t * d + 2 * i + 1] = cosf((float)t * den);
        }
    }
    return pe;
}

// A copy of the leading n elements of an nn.MultiheadAttention in_proj weight or bias ([Wq; Wk; Wv] rows) with 1/sqrt(d_h)
// folded into the query part, its first n_query elements
static std::vector<float> fold_query_scale(const float* src, size_t n, size_t n_query, int dh) {
    std::vector<float> v(src, src + n);
    const float qs = 1.0f / sqrtf((float)dh);
    for (size_t i = 0; i < n_query; ++i) v[i] *= qs;
    return v;
}

// [Wq; Wk; Wv] rows of `cols` elements -> per-head [q | k | v] blocks, the encoder attention's layout
static std::vector<float> qkv_rows_per_head(const std::vector<float>& src, int d, int nhead, int cols) {
    const int dh = d / nhead;
    std::vector<float> dst(src.size());
    for (int h = 0; h < nhead; ++h)
        for (int part = 0; part < 3; ++part)
            for (int j = 0; j < dh; ++j) {
                const size_t s = (size_t)part * d + h * dh + j, t = (size_t)h * 3 * dh + part * dh + j;
                memcpy(&dst[t * cols], &src[s * cols], (size_t)cols * 4);
            }
    return dst;
}

// [value rows 0 .. d-1; gate rows 0 .. d-1] of `cols` elements -> 16 value rows / 16 gate rows interleaved, for the GLU epilogue
static std::vector<float> glu_interleave_rows(const float* src, int d, int cols) {
    std::vector<float> dst((size_t)2 * d * cols);
    for (int ch = 0; ch < d; ++ch) {
        const int blk = ch / 16, j = ch % 16;
        memcpy(&dst[((size_t)blk * 32 + j) * cols], &src[(size_t)ch * cols], (size_t)cols * 4);
        memcpy(&dst[((size_t)blk * 32 + 16 + j) * cols], &src[(size_t)(d + ch) * cols], (size_t)cols * 4);
    }
    return dst;
}

// Conv2d weight (o, ch, kf, kt) with K x K taps -> [o][(kf * K + kt) * Ci + ch], input channels innermost
static std::vector<float> conv_taps_channel_last(const float* src, int Co, int Ci, int K) {
    const int taps = K * K;
    std::vector<float> dst((size_t)Co * taps * Ci);
    for (int o = 0; o < Co; ++o)
        for (int ch = 0; ch < Ci; ++ch)
            for (int t = 0; t < taps; ++t) dst[((size_t)o * taps + t) * Ci + ch] = src[((size_t)o * Ci + ch) * taps + t];
    return dst;
}

// Conv2d weight (o, ch, kf, kt), 3 x 3 taps -> the K-major operand [Co][(kf * 3 + kt) * Ci + ch] as 64-wide k-blocks,
// each the 128B-swizzled shared-memory image the 256-channel conv2 kernel copies into one stage: block kb holds row o
// (k = 64 kb .. 64 kb + 63) at 128 o bytes, with its 16-byte chunk j at chunk j ^ (o % 8)
static std::vector<float> conv_taps_kblocks_sw128(const float* src, int Co, int Ci) {
    const std::vector<float> km = conv_taps_channel_last(src, Co, Ci, 3);
    const int K = 9 * Ci;
    std::vector<float> dst(km.size());
    for (int kb = 0; kb < K / 64; ++kb)
        for (int o = 0; o < Co; ++o)
            for (int k = 0; k < 64; ++k)
                dst[((size_t)kb * Co + o) * 64 + (((k >> 3) ^ (o & 7)) << 3) + (k & 7)] = km[(size_t)o * K + kb * 64 + k];
    return dst;
}

// ---- the parts of a model, each in the order its tensors lie in the arena

static void pack_frontend(Packer& p, AsrWeights& W) {
    const sbk_asr_config& c = W.cfg;
    if (W.has_fbank && p.has("normalize.glob_mean")) {
        W.glob_mean = p.f32("normalize.glob_mean", c.n_mels);
        W.glob_std = p.f32("normalize.glob_std", c.n_mels);
    }
    if (!W.has_cnn) return;
    const int F1 = (c.n_mels - 1) / 2 + 1, F2 = (F1 - 1) / 2 + 1;
    const std::string b0 = "CNN.convblock_0.convs.", b1 = "CNN.convblock_1.convs.", b2 = "CNN.convblock_2.";
    // convolution.py:116-320; 3 blocks: kernel_sizes (5, 5, 1), residuals (False, False, True), 64 channels
    CnnWeights& k = W.cnn;
    k.blocks = c.cnn_blocks == 3 ? 3 : 2;
    k.c1 = c.cnn_c1;
    k.c2 = c.cnn_c2;
    const int K = k.blocks == 3 ? 5 : 3, C = 64;
    k.w1 = p.f32(b0 + "conv_0.conv.weight", (int64_t)k.c1 * K * K);
    k.b1 = p.f32(b0 + "conv_0.conv.bias", k.c1);
    p.norm(b0 + "norm_0.norm", (int64_t)F1 * k.c1, &k.g1, &k.be1);
    const float* w2 = p.host(b1 + "conv_0.conv.weight", (int64_t)k.c2 * k.c1 * K * K);
    const float *w3a = nullptr, *w3r = nullptr, *b3a = nullptr, *b3r = nullptr;
    if (k.blocks == 3) {
        w3a = p.host(b2 + "convs.conv_0.conv.weight", (int64_t)C * C);
        w3r = p.host(b2 + "reduce_conv.conv.conv.weight", (int64_t)C * C);
        b3a = p.host(b2 + "convs.conv_0.conv.bias", C);
        b3r = p.host(b2 + "reduce_conv.conv.conv.bias", C);
        if (!w3a || !w3r || !b3a || !b3r) return;
    }
    if (!w2) return;
    k.w2 = p.f16_raw(k.c1 == 256 ? conv_taps_kblocks_sw128(w2, k.c2, k.c1) : conv_taps_channel_last(w2, k.c2, k.c1, K));
    k.b2 = p.f32(b1 + "conv_0.conv.bias", k.c2);
    p.norm(b1 + "norm_0.norm", (int64_t)F2 * k.c2, &k.g2, &k.be2);
    if (k.blocks != 3) return;
    std::vector<float> w3((size_t)2 * C * C), b3(2 * C);  // [convs.conv_0 | reduce_conv.conv] output channels
    memcpy(w3.data(), w3a, (size_t)C * C * 4);
    memcpy(w3.data() + (size_t)C * C, w3r, (size_t)C * C * 4);
    memcpy(b3.data(), b3a, C * 4);
    memcpy(b3.data() + C, b3r, C * 4);
    k.w3 = p.f32_raw(w3);
    k.b3 = p.f32_raw(b3);
    p.norm(b2 + "convs.norm_0.norm", (int64_t)F2 * C, &k.g3, &k.be3);
    p.norm(b2 + "reduce_conv.norm.norm", (int64_t)F2 * C, &k.gr, &k.ber);
}

// mha_layer of a Conformer or Branchformer layer: RoPEMHA, or RelPosMHAXL with its linear_pos and position biases
static void pack_encoder_mha(Packer& p, const sbk_asr_config& c, const std::string& mha, EncLayerW& e) {
    const int d = c.d_model;
    e.wqkv = p.f16(mha + "in_proj_weight", (int64_t)3 * d * d);
    p.linear(mha + "out_proj", d, d, &e.wo, &e.bo);
    if (c.attention_type == SBK_ATT_RELPOS) {
        e.wpos = p.f16(mha + "linear_pos.weight", (int64_t)d * d);
        e.pos_u = p.f32(mha + "pos_bias_u", d);
        e.pos_v = p.f32(mha + "pos_bias_v", d);
    }
}

static void pack_branchformer_layer(Packer& p, const sbk_asr_config& c, const std::string& q, EncLayerW& e) {
    const std::string cb = q + "convolution_branch.";
    const int d = c.d_model, K = c.kernel_size, C = c.csgu_linear_units, C2 = C / 2;
    p.norm(q + "norm_mhsa.norm", d, &e.norm1_g, &e.norm1_b);
    p.norm(q + "norm_conv.norm", d, &e.nconv_g, &e.nconv_b);
    pack_encoder_mha(p, c, q + "mha_layer.", e);
    p.linear(cb + "pre_channel_proj", C, d, &e.wpre, &e.bpre);
    p.linear(cb + "post_channel_proj", d, C2, &e.wpost, &e.bpost);
    p.norm(cb + "csgu.norm.norm", C2, &e.csgu_ln_g, &e.csgu_ln_b);
    const float* taps = p.host(cb + "csgu.conv.conv.weight", (int64_t)C2 * K);
    if (!taps) return;
    std::vector<float> wt((size_t)CSGU_TAP_ROWS * C2);  // (C/2, 1, K) -> tap-major, K centred in CSGU_TAP_ROWS rows
    csgu_repack_taps(taps, C2, K, wt.data());
    e.csgu_taps = p.f32_raw(wt);
    e.csgu_bias = p.f32(cb + "csgu.conv.conv.bias", C2);
    p.linear(q + "merge_proj", d, 2 * d, &e.wmerge, &e.bmerge);
}

static void pack_transformer_layer(Packer& p, const sbk_asr_config& c, const std::string& q, EncLayerW& e) {
    const int d = c.d_model, dh = d / c.nhead, F = c.d_ffn;
    p.norm(q + "norm1.norm", d, &e.norm1_g, &e.norm1_b);
    p.norm(q + "norm2.norm", d, &e.norm2_g, &e.norm2_b);
    const float* wi = p.host(q + "self_att.att.in_proj_weight", (int64_t)3 * d * d);
    const float* bi = p.host(q + "self_att.att.in_proj_bias", 3 * d);
    if (!wi || !bi) return;
    e.wqkv = p.f16_raw(qkv_rows_per_head(fold_query_scale(wi, (size_t)3 * d * d, (size_t)d * d, dh), d, c.nhead, d));
    e.bqkv = p.f32_raw(qkv_rows_per_head(fold_query_scale(bi, 3 * d, d, dh), d, c.nhead, 1));
    p.linear(q + "self_att.att.out_proj", d, d, &e.wo, &e.bo);
    p.linear(q + "pos_ffn.ffn.0", F, d, &e.ffn1_w1, &e.ffn1_b1);
    p.linear(q + "pos_ffn.ffn.3", d, F, &e.ffn1_w2, &e.ffn1_b2);
}

static void pack_conformer_layer(Packer& p, const sbk_asr_config& c, const std::string& q, EncLayerW& e) {
    const std::string cm = q + "convolution_module.";
    const int d = c.d_model, dh = d / c.nhead, F = c.d_ffn, K = c.kernel_size;
    p.norm(q + "ffn_module1.0", d, &e.ffn1_ln_g, &e.ffn1_ln_b);
    p.linear(q + "ffn_module1.1.ffn.0", F, d, &e.ffn1_w1, &e.ffn1_b1);
    p.linear(q + "ffn_module1.1.ffn.3", d, F, &e.ffn1_w2, &e.ffn1_b2);
    p.norm(q + "norm1.norm", d, &e.norm1_g, &e.norm1_b);
    if (c.attention_type == SBK_ATT_HYPERMIX) {
        // hypermixing.py:52-81, 274-337: w{1,2}_gen fc1 (M, e, e) / fc2 (M, k, e), then layer_norm (d)
        const int Mh = c.nhead, kh = F / c.nhead;
        const char* gen[2] = {"mha_layer.hyper.w1_gen.", "mha_layer.hyper.w2_gen."};
        for (int gi = 0; gi < 2; ++gi) {
            e.hm.fc1w[gi] = p.f16(q + gen[gi] + "fc1_weights", (int64_t)Mh * dh * dh);
            e.hm.fc1b[gi] = p.f32(q + gen[gi] + "fc1_biases", (int64_t)Mh * dh);
            e.hm.fc2w[gi] = p.f16(q + gen[gi] + "fc2_weights", (int64_t)Mh * kh * dh);
            e.hm.fc2b[gi] = p.f32(q + gen[gi] + "fc2_biases", (int64_t)Mh * kh);
        }
        p.norm(q + "mha_layer.layer_norm", d, &e.hm.ln_g, &e.hm.ln_b);
    } else {
        pack_encoder_mha(p, c, q + "mha_layer.", e);
    }
    p.norm(cm + "layer_norm", d, &e.conv_ln_g, &e.conv_ln_b);
    const float* pw1 = p.host(cm + "bottleneck.0.weight", (int64_t)2 * d * d);  // pointwise conv 1 (Conv1d k=1, weight (2d, d, 1))
    const float* pb1 = p.host(cm + "bottleneck.0.bias", 2 * d);
    const float* taps = p.host(cm + "conv.weight", (int64_t)d * K);
    if (!pw1 || !pb1 || !taps) return;
    e.wpw1 = p.f16_raw(glu_interleave_rows(pw1, d, d));
    e.bpw1 = p.f32_raw(glu_interleave_rows(pb1, d, 1));
    // depthwise taps (d, 1, K) -> tap-major [K, d] so that a warp's channels read one cache line per tap
    std::vector<float> wt((size_t)K * d);
    dwconv_repack_taps(taps, d, K, wt.data());
    e.wdw = p.f32_raw(wt);
    e.bdw = p.f32(cm + "conv.bias", d);
    p.norm(cm + "after_conv.0", d, &e.aconv_ln_g, &e.aconv_ln_b);
    p.linear(cm + "after_conv.2", d, d, &e.wpw2, &e.bpw2);
    p.norm(q + "ffn_module2.0", d, &e.ffn2_ln_g, &e.ffn2_ln_b);
    p.linear(q + "ffn_module2.1.ffn.0", F, d, &e.ffn2_w1, &e.ffn2_b1);
    p.linear(q + "ffn_module2.1.ffn.3", d, F, &e.ffn2_w2, &e.ffn2_b2);
    p.norm(q + "norm2.norm", d, &e.norm2_g, &e.norm2_b);
}

static void pack_positional_tables(Packer& p, AsrWeights& W) {
    const sbk_asr_config& c = W.cfg;
    const int d = c.d_model, dh = d / c.nhead;
    W.pos_len = c.max_len;
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
        W.rope_cos = p.f32_raw(cs);
        W.rope_sin = p.f32_raw(sn);
    } else if (c.attention_type == SBK_ATT_REGULAR) {
        W.enc_pe = p.f32_raw(sine_table(c.max_len, d));
    } else if (c.attention_type == SBK_ATT_HYPERMIX) {
        W.hm_pe = p.f32_raw(sine_table(HM_PE_ROWS, d));
        W.pos_len = HM_PE_ROWS;
    } else {
        W.relpos_pe = p.f16_raw(sine_table(c.max_len, d));
    }
}

static void pack_encoder(Packer& p, AsrWeights& W) {
    const sbk_asr_config& c = W.cfg;
    const int d = c.d_model;
    p.linear("Transformer.custom_src_module.layers.0.w", d, c.input_size, &W.w_in, &W.b_in);
    W.enc.assign(c.num_encoder_layers, EncLayerW());
    for (int l = 0; l < c.num_encoder_layers && p.ok; ++l) {
        const std::string q = "Transformer.encoder.layers." + std::to_string(l) + ".";
        switch (c.encoder_module) {
            case SBK_ENC_BRANCHFORMER: pack_branchformer_layer(p, c, q, W.enc[l]); break;
            case SBK_ENC_TRANSFORMER: pack_transformer_layer(p, c, q, W.enc[l]); break;
            default: pack_conformer_layer(p, c, q, W.enc[l]);
        }
    }
    if (!p.ok) return;
    p.norm("Transformer.encoder.norm.norm", d, &W.enc_norm_g, &W.enc_norm_b);
    pack_positional_tables(p, W);
}

bool xatt_foldable(const sbk_asr_config& c) {
    return c.d_model == 64 * c.nhead && c.d_model % 256 == 0 && c.nhead * c.d_model <= 4096;
}

void fold_cross_attention(const float* wc, const float* bc, const float* wo, const float* bo, int d, int H,
                          std::vector<double>* xq, std::vector<double>* bxq, std::vector<double>* xo, std::vector<double>* bxo) {
    const int dh = d / H;
    const std::vector<float> wq = fold_query_scale(wc, (size_t)d * d, (size_t)d * d, dh);  // the unfolded path's W_q, b_q
    const std::vector<float> bq = fold_query_scale(bc, d, d, dh);
    const float *wk = wc + (size_t)d * d, *wv = wc + (size_t)2 * d * d, *bv = bc + 2 * d;
    xq->assign((size_t)H * d * d, 0.0); bxq->assign((size_t)H * d, 0.0);
    xo->assign((size_t)d * H * d, 0.0); bxo->assign(bo, bo + d);
    for (int h = 0; h < H; ++h)
        for (int a = 0; a < dh; ++a) {
            const size_t r = (size_t)h * dh + a;  // row of W_q / W_k / W_v, column of W_o
            const float* q = &wq[r * d];
            for (int i = 0; i < d; ++i) {
                const double k = wk[r * d + i];
                double* row = &(*xq)[((size_t)h * d + i) * d];
                for (int j = 0; j < d; ++j) row[j] += k * q[j];
                (*bxq)[(size_t)h * d + i] += k * bq[r];
            }
            for (int o = 0; o < d; ++o) {
                const double w = wo[(size_t)o * d + r];
                double* row = &(*xo)[(size_t)o * H * d + (size_t)h * d];
                for (int i = 0; i < d; ++i) row[i] += w * wv[r * d + i];
                (*bxo)[o] += w * bv[r];
            }
        }
}

static void pack_decoder(Packer& p, AsrWeights& W) {
    const sbk_asr_config& c = W.cfg;
    const int d = c.d_model, dh = d / c.nhead, F = c.d_ffn, L = c.num_decoder_layers;
    W.emb = p.f32("Transformer.custom_tgt_module.layers.0.emb.Embedding.weight", (int64_t)c.vocab * d);
    W.dec_pe = p.f32_raw(sine_table(c.max_len, d));
    W.dec.resize(L);
    std::vector<float> wckv((size_t)L * 2 * d * d), bckv((size_t)L * 2 * d);  // every layer's cross-attention [Wk; Wv] rows
    for (int l = 0; l < L; ++l) {
        const std::string q = "Transformer.decoder.layers." + std::to_string(l) + ".";
        DecLayerW& e = W.dec[l];
        p.norm(q + "norm1.norm", d, &e.n1g, &e.n1b);
        p.norm(q + "norm2.norm", d, &e.n2g, &e.n2b);
        p.norm(q + "norm3.norm", d, &e.n3g, &e.n3b);
        const float* wi = p.host(q + "self_attn.att.in_proj_weight", (int64_t)3 * d * d);
        const float* bi = p.host(q + "self_attn.att.in_proj_bias", 3 * d);
        const float* wc = p.host(q + "multihead_attn.att.in_proj_weight", (int64_t)3 * d * d);
        const float* bc = p.host(q + "multihead_attn.att.in_proj_bias", 3 * d);
        if (!wi || !bi || !wc || !bc) return;
        e.w_self_in = p.f16_raw(fold_query_scale(wi, (size_t)3 * d * d, (size_t)d * d, dh));
        e.b_self_in = p.f32_raw(fold_query_scale(bi, 3 * d, d, dh));
        e.w_cross_q = p.f16_raw(fold_query_scale(wc, (size_t)d * d, (size_t)d * d, dh));
        e.b_cross_q = p.f32_raw(fold_query_scale(bc, d, d, dh));
        memcpy(&wckv[(size_t)l * 2 * d * d], wc + (size_t)d * d, (size_t)2 * d * d * 4);
        memcpy(&bckv[(size_t)l * 2 * d], bc + d, (size_t)2 * d * 4);
        p.linear(q + "self_attn.att.out_proj", d, d, &e.w_self_out, &e.b_self_out);
        p.linear(q + "multihead_attn.att.out_proj", d, d, &e.w_cross_out, &e.b_cross_out);
        if (xatt_foldable(c)) {  // the products are only formed when the arena is filled; measuring needs their sizes
            const float* wo = p.host(q + "multihead_attn.att.out_proj.weight", (int64_t)d * d);
            const float* bo = p.host(q + "multihead_attn.att.out_proj.bias", d);
            if (!wo || !bo) return;
            std::vector<double> xq((size_t)c.nhead * d * d), bxq((size_t)c.nhead * d), xo((size_t)d * c.nhead * d), bxo(d);
            if (p.carve.base) fold_cross_attention(wc, bc, wo, bo, d, c.nhead, &xq, &bxq, &xo, &bxo);
            e.w_xq = p.f16_raw(xq); e.b_xq = p.f32_raw(bxq);
            e.w_xo = p.f16_raw(xo); e.b_xo = p.f32_raw(bxo);
        }
        p.linear(q + "pos_ffn.ffn.0", F, d, &e.w_ffn1, &e.b_ffn1);
        p.linear(q + "pos_ffn.ffn.3", d, F, &e.w_ffn2, &e.b_ffn2);
        if (!p.ok) return;
    }
    W.w_ckv = p.f16_raw(wckv);
    W.b_ckv = p.f32_raw(bckv);
    p.norm("Transformer.decoder.norm.norm", d, &W.dec_norm_g, &W.dec_norm_b);
    // the output head belongs to the searchers; TransformerASR.decode runs without it
    if (p.has("seq_lin.w.weight")) p.linear("seq_lin.w", c.vocab, d, &W.w_lin, &W.b_lin);
}

bool lm_widths(int d, int H, int* dp, int* dhp) {
    if (H > 0 && d == 64 * H && d % 128 == 0) { *dp = d; *dhp = 64; return true; }
    if (d == 264 && H == 12) { *dp = 272; *dhp = 32; return true; }
    return false;
}

// A [rows.size(), cols.size()] copy of the row-major matrix src (`ld` columns): element (i, j) = src[rows[i]][cols[j]], zero
// where either index is -1.  Places a TransformerLM weight in its padded layout.
static std::vector<float> gather2d(const float* src, int ld, const std::vector<int>& rows, const std::vector<int>& cols) {
    std::vector<float> dst(rows.size() * cols.size(), 0.0f);
    for (size_t i = 0; i < rows.size(); ++i)
        if (rows[i] >= 0)
            for (size_t j = 0; j < cols.size(); ++j)
                if (cols[j] >= 0) dst[i * cols.size() + j] = src[(size_t)rows[i] * ld + cols[j]];
    return dst;
}

static void pack_lm(Packer& p, AsrWeights& W) {
    const sbk_asr_config& c = W.cfg;
    const int dl = c.lm_d_model, Fl = c.lm_d_ffn, H = c.lm_nhead, dhl = dl / H, V = c.vocab;
    int dp = 0, dhp = 0;
    lm_widths(dl, H, &dp, &dhp);  // check_config has refused every other shape
    W.lm_dp = dp; W.lm_dhp = dhp; W.lm_da = H * dhp;
    // index maps into the reference's tensors: the residual stream (dp channels, the first dl real), the attention width
    // (da channels, head h's first dhl real), the in_proj's [q | k | v] rows, and the identity over the FFN / vocabulary
    std::vector<int> res(dp, -1), att(W.lm_da, -1), qkv(3 * W.lm_da, -1), ffn(Fl), voc(V), one{0};
    for (int i = 0; i < dl; ++i) res[i] = i;
    for (int h = 0; h < H; ++h)
        for (int j = 0; j < dhl; ++j) att[h * dhp + j] = h * dhl + j;
    for (int part = 0; part < 3; ++part)
        for (int i = 0; i < W.lm_da; ++i) qkv[part * W.lm_da + i] = att[i] < 0 ? -1 : part * dl + att[i];
    for (int i = 0; i < Fl; ++i) ffn[i] = i;
    for (int i = 0; i < V; ++i) voc[i] = i;
    // Linear prefix.weight [out, in] / prefix.bias [out] with their rows picked by `out` and columns by `in`
    auto linear = [&](const std::string& prefix, const std::vector<int>& out, const std::vector<int>& in, int n_out, int n_in,
                      const __half** wgt, const float** bias) {
        const float* w = p.host(prefix + ".weight", (int64_t)n_out * n_in);
        const float* b = p.host(prefix + ".bias", n_out);
        if (!w || !b) return;
        *wgt = p.f16_raw(gather2d(w, n_in, out, in));
        *bias = p.f32_raw(gather2d(b, 1, out, one));
    };

    // the embedding table the step kernels read one row of, at pitch dp
    const std::string proj = "lm.embedding_proj.w";
    if (p.has(proj + ".weight")) {  // TransformerLM(d_embedding=...): NormalizedEmbedding(d_embedding) -> embedding_proj
        const int64_t de = p.numel(proj + ".weight") / dl;
        if (de < 1 || de * dl != p.numel(proj + ".weight")) {
            set_error("weight '%s.weight' has %lld elements, not a multiple of d_model %d", proj.c_str(),
                      (long long)p.numel(proj + ".weight"), dl);
            p.ok = false;
            return;
        }
        const float* E = p.host("lm.custom_src_module.emb.Embedding.weight", (int64_t)V * de);
        const float* Wp = p.host(proj + ".weight", (int64_t)dl * de);
        const float* bp = p.host(proj + ".bias", dl);
        if (!E || !Wp || !bp) return;
        std::vector<double> table((size_t)V * dp, 0.0);  // embedding_proj(sqrt(d_embedding) E[v]), formed only to upload
        if (p.carve.base) {
            const double s = sqrt((double)de);
            for (int v = 0; v < V; ++v)
                for (int o = 0; o < dl; ++o) {
                    double acc = 0.0;
                    for (int64_t i = 0; i < de; ++i) acc += (double)Wp[(size_t)o * de + i] * (s * E[(size_t)v * de + i]);
                    table[(size_t)v * dp + o] = acc + bp[o];
                }
        }
        W.lm_emb = p.f32_raw(table);
        W.lm_emb_scale = 1.0f;
    } else {
        const float* emb = p.host("lm.custom_src_module.emb.Embedding.weight", (int64_t)V * dl);
        if (!emb) return;
        W.lm_emb = p.f32_raw(gather2d(emb, dl, voc, res));
        W.lm_emb_scale = sqrtf((float)dl);
    }
    std::vector<int> pos(c.max_len);
    for (int t = 0; t < c.max_len; ++t) pos[t] = t;
    W.lm_pe = p.f32_raw(gather2d(sine_table(c.max_len, dl).data(), dl, pos, res));
    W.lm.resize(c.lm_layers);
    for (int l = 0; l < c.lm_layers; ++l) {
        const std::string q = "lm.encoder.layers." + std::to_string(l) + ".";
        LmLayerW& e = W.lm[l];
        const float* wi = p.host(q + "self_att.att.in_proj_weight", (int64_t)3 * dl * dl);
        const float* bi = p.host(q + "self_att.att.in_proj_bias", 3 * dl);
        if (!wi || !bi) return;
        // 1 / sqrt(dh) of the true head width; the padded query dims are zero
        e.w_in = p.f16_raw(gather2d(fold_query_scale(wi, (size_t)3 * dl * dl, (size_t)dl * dl, dhl).data(), dl, qkv, res));
        e.b_in = p.f32_raw(gather2d(fold_query_scale(bi, 3 * dl, dl, dhl).data(), 1, qkv, one));
        linear(q + "self_att.att.out_proj", res, att, dl, dl, &e.w_out, &e.b_out);
        linear(q + "pos_ffn.ffn.0", ffn, res, Fl, dl, &e.w1, &e.b1);
        linear(q + "pos_ffn.ffn.3", res, ffn, dl, Fl, &e.w2, &e.b2);
        p.norm(q + "norm1.norm", dl, &e.n1g, &e.n1b);
        p.norm(q + "norm2.norm", dl, &e.n2g, &e.n2b);
        if (!p.ok) return;
    }
    p.norm("lm.encoder.norm.norm", dl, &W.lm_norm_g, &W.lm_norm_b);
    linear("lm.output_proj.layers.0.w", res, res, dl, dl, &W.lm_wp0, &W.lm_bp0);
    p.norm("lm.output_proj.layers.1.norm", dl, &W.lm_lnp_g, &W.lm_lnp_b);
    linear("lm.output_proj.layers.2.w", voc, res, V, dl, &W.lm_wp2, &W.lm_bp2);
}

// Everything that goes into the arena.  Stops at the first part with a missing or mis-sized tensor (p.ok cleared, the
// error set).
static void pack(Packer& p, AsrWeights& W) {
    pack_frontend(p, W);
    if (p.ok && W.has_enc) pack_encoder(p, W);
    if (p.ok && W.has_dec) pack_decoder(p, W);
    if (p.ok && W.has_lm) pack_lm(p, W);
    if (p.ok && p.has("ctc_lin.w.weight")) p.linear("ctc_lin.w", W.cfg.vocab, W.cfg.d_model, &W.w_ctc, &W.b_ctc);
}

// What the kernels are built for.
static int check_config(const sbk_asr_config& c) {
    SBK_REQUIRE(c.d_model % 8 == 0 && c.d_model % c.nhead == 0, "asr_create: bad d_model/nhead");
    SBK_REQUIRE(c.attention_type == SBK_ATT_ROPE || c.attention_type == SBK_ATT_RELPOS || c.attention_type == SBK_ATT_HYPERMIX ||
                    c.attention_type == SBK_ATT_REGULAR,
                "asr_create: attention_type must be RoPEMHA, RelPosMHAXL, hypermixing or regularMHA");
    const int d = c.d_model, dh = d / c.nhead, F = c.d_ffn, K = c.kernel_size;
    const bool hypermix = c.attention_type == SBK_ATT_HYPERMIX;
    const bool tfm = c.encoder_module == SBK_ENC_TRANSFORMER;
    SBK_REQUIRE(tfm == (c.attention_type == SBK_ATT_REGULAR),
                "asr_create: regularMHA is built for the Transformer encoder only, and the Transformer encoder with regularMHA only");
    SBK_REQUIRE(!tfm || dh == 64 || dh == 128, "asr_create: Transformer encoder head_dim=%d not built (128, 64)", dh);
    SBK_REQUIRE(tfm || hypermix || dh == 64 || dh == 36 || dh == 32 ||
                    ((dh == 80 || dh == 96) && c.encoder_module == SBK_ENC_CONFORMER && c.attention_type == SBK_ATT_RELPOS),
                "asr_create: encoder head_dim=%d not built (64, 36, 32; 80 and 96 for the Conformer with RelPosMHAXL)", dh);
    SBK_REQUIRE(((c.cnn_blocks == 0 || c.cnn_blocks == 2) &&
                 ((c.cnn_c1 == 64 && c.cnn_c2 == 32) || (c.cnn_c1 == 256 && c.cnn_c2 == 256))) ||
                    (c.cnn_blocks == 3 && c.cnn_c1 == 64 && c.cnn_c2 == 64),
                "asr_create: cnn_blocks=%d with channels (%d, %d) not built (2 blocks with (64, 32) or (256, 256), 3 with "
                "(64, 64))", c.cnn_blocks, c.cnn_c1, c.cnn_c2);
    SBK_REQUIRE(!hypermix || (c.encoder_module == SBK_ENC_CONFORMER && (dh == 32 || dh == 64) && F % c.nhead == 0 &&
                              (F / c.nhead) % 16 == 0 && F / c.nhead <= 256),
                "asr_create: hypermixing needs the Conformer encoder, a head width d_model / nhead of 32 or 64 and "
                "k = d_ffn / nhead a multiple of 16 up to 256 (got %d, %d)", dh, c.nhead > 0 ? F / c.nhead : 0);
    SBK_REQUIRE(!((c.parts & SBK_PART_DECODER) && c.num_decoder_layers > 0) ||
                    ((dh <= 64 || dh == 80 || dh == 128) && dh % 4 == 0 && d % 16 == 0),
                "asr_create: decoder head_dim must be 128, 80 or a multiple of 4 up to 64 and d_model a multiple of 16 (got %d, %d)",
                dh, d);
    SBK_REQUIRE(c.attention_type != SBK_ATT_ROPE || dh % 32 == 0, "asr_create: RoPEMHA needs head_dim %% 32 == 0");
    SBK_REQUIRE(c.conformer_activation == SBK_CONFORMER_ACT_SWISH || c.conformer_activation == SBK_CONFORMER_ACT_GELU,
                "asr_create: conformer_activation %d not built (0 Swish, 1 GELU)", c.conformer_activation);
    SBK_REQUIRE(c.conformer_activation == SBK_CONFORMER_ACT_SWISH || c.encoder_module == SBK_ENC_CONFORMER,
                "asr_create: conformer_activation GELU is for the Conformer encoder only");
    SBK_REQUIRE(c.encoder_module == SBK_ENC_CONFORMER || c.encoder_module == SBK_ENC_BRANCHFORMER || tfm,
                "asr_create: encoder_module %d (0 Conformer, 1 Branchformer, 2 Transformer)", c.encoder_module);
    SBK_REQUIRE(c.encoder_module != SBK_ENC_BRANCHFORMER ||
                    (c.attention_type == SBK_ATT_RELPOS && c.csgu_linear_units > 0 && c.csgu_linear_units % 16 == 0 &&
                     (K & 1) == 1 && K <= CSGU_TAP_ROWS),
                "asr_create: the Branchformer needs RelPosMHAXL, csgu_linear_units / 2 %% 8 == 0 and an odd kernel_size <= %d "
                "(got %d, %d)", CSGU_TAP_ROWS, c.csgu_linear_units, K);
    if (c.parts & SBK_PART_CNN) {
        const int F1 = (c.n_mels - 1) / 2 + 1, F2 = (F1 - 1) / 2 + 1;
        SBK_REQUIRE(F2 * c.cnn_c2 == c.input_size, "asr_create: CNN output %d != input_size %d", F2 * c.cnn_c2, c.input_size);
    }
    int lm_dp, lm_dhp;
    if ((c.parts & SBK_PART_LM) && c.lm_layers > 0 && !lm_widths(c.lm_d_model, c.lm_nhead, &lm_dp, &lm_dhp)) {
        set_error("asr_create: LM d_model=%d with %d heads not built (head_dim 64 with d_model %% 128 == 0, or d_model 264 "
                  "with 12 heads of 22)", c.lm_d_model, c.lm_nhead);
        return SBK_ERR_UNSUPPORTED;
    }
    return SBK_OK;
}

int load_asr_weights(const sbk_asr_config& c, const sbk_tensor* weights, int n_weights, std::shared_ptr<const AsrWeights>* out) {
    if (int rc = check_config(c)) return rc;
    WeightMap w;
    for (int i = 0; i < n_weights; ++i) w[weights[i].name] = {weights[i].data, weights[i].numel};

    auto wt = std::make_shared<AsrWeights>();
    wt->cfg = c;
    wt->has_fbank = c.parts & SBK_PART_FBANK;
    wt->has_cnn = c.parts & SBK_PART_CNN;
    wt->has_enc = (c.parts & SBK_PART_ENCODER) && c.num_encoder_layers >= 0;
    wt->has_dec = (c.parts & SBK_PART_DECODER) && c.num_decoder_layers > 0;
    wt->has_lm = (c.parts & SBK_PART_LM) && c.lm_layers > 0;
    Packer measure{w};
    const float* win = wt->has_fbank ? measure.host("fbank.window", c.n_fft) : nullptr;
    const float* mel = wt->has_fbank ? measure.host("fbank.mel_matrix", (int64_t)(c.n_fft / 2 + 1) * c.n_mels) : nullptr;
    if (measure.ok) pack(measure, *wt);
    if (!measure.ok) return SBK_ERR_ARG;
    if (cudaMalloc(&wt->arena, measure.carve.used) != cudaSuccess) {
        set_error("asr_create: cudaMalloc(%zu) for weights failed", measure.carve.used);
        return SBK_ERR_NOMEM;
    }
    if (wt->has_fbank) {
        const int rc = fbank_create(&wt->fbank, c.n_fft, c.hop, c.n_mels, win, mel, c.fbank_amin > 0.0f ? c.fbank_amin : 1e-10f,
                                    c.fbank_top_db > 0.0f ? c.fbank_top_db : 80.0f);
        if (rc) return rc;
    }
    Packer upload{w, Carver{wt->arena}};
    pack(upload, *wt);
    if (!upload.ok) return SBK_ERR_ARG;
    if (cudaDeviceSynchronize() != cudaSuccess) {
        set_error("asr_create: device error after upload");
        return SBK_ERR_CUDA;
    }
    *out = std::move(wt);
    return SBK_OK;
}

}  // namespace sbk
