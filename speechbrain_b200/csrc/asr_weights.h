// The model's weights as the kernels read them, and the loader that builds them from a reference state_dict
// (asr_weights.cu).  engine.cu only reads these structs.
#pragma once
#include <memory>
#include <vector>

#include "sbk_internal.h"
#include "../../include/sbk.h"

namespace sbk {

// Fields a layer family does not use stay null.
struct EncLayerW {
    const float *ffn1_ln_g = nullptr, *ffn1_ln_b = nullptr, *ffn1_b1 = nullptr, *ffn1_b2 = nullptr;
    const __half *ffn1_w1 = nullptr, *ffn1_w2 = nullptr;
    const float *norm1_g = nullptr, *norm1_b = nullptr;
    const __half *wqkv = nullptr, *wo = nullptr;
    const float* bo = nullptr;
    const __half* wpos = nullptr;                         // RelPos linear_pos
    const float *pos_u = nullptr, *pos_v = nullptr;       // RelPos biases, raw (d_h, H) buffer viewed (H, d_h)
    const float *conv_ln_g = nullptr, *conv_ln_b = nullptr;
    const __half* wpw1 = nullptr;                         // [2d, d] rows interleaved 16 value / 16 gate
    const float* bpw1 = nullptr;                          // interleaved the same way
    const float *wdw = nullptr, *bdw = nullptr;           // [d, K], [d]
    const float *aconv_ln_g = nullptr, *aconv_ln_b = nullptr;
    const __half* wpw2 = nullptr;
    const float* bpw2 = nullptr;
    const float *ffn2_ln_g = nullptr, *ffn2_ln_b = nullptr, *ffn2_b1 = nullptr, *ffn2_b2 = nullptr;
    const __half *ffn2_w1 = nullptr, *ffn2_w2 = nullptr;
    const float *norm2_g = nullptr, *norm2_b = nullptr;
    // Branchformer layer (Branchformer.py:92-234; the attention uses norm1_g/b = norm_mhsa and wqkv / wo / bo / wpos / pos_u /
    // pos_v above)
    const float *nconv_g = nullptr, *nconv_b = nullptr;   // norm_conv
    // pre_channel_proj [C, d], post_channel_proj [d, C/2], merge_proj [d, 2d]
    const __half *wpre = nullptr, *wpost = nullptr, *wmerge = nullptr;
    const float *bpre = nullptr, *bpost = nullptr, *bmerge = nullptr;
    // taps tap-major [CSGU_TAP_ROWS, C/2] (csgu_repack_taps)
    const float *csgu_ln_g = nullptr, *csgu_ln_b = nullptr, *csgu_taps = nullptr, *csgu_bias = nullptr;
    HyperMixWeights hm{};             // HyperConformer: mha_layer = HyperMixing (replaces wqkv / wo / bo)
    // Transformer layer (Transformer.py:311-490): self_att.att in_proj bias, repacked like wqkv; norm1 / norm2 and the FFN
    // (ffn1_w1 / ffn1_b1 / ffn1_w2 / ffn1_b2) use the fields above
    const float* bqkv = nullptr;
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

// What load_asr_weights uploads and nothing changes afterwards: the configuration, the Fbank plan and the repacked weights
// in one device arena of exactly the bytes they take.  A handle and its clones (lanes) hold it jointly; the last one to go
// frees it.
struct AsrWeights {
    sbk_asr_config cfg;
    Fbank* fbank = nullptr;
    uint8_t* arena = nullptr;
    // frontend
    const float *glob_mean = nullptr, *glob_std = nullptr;
    const float *c1_w = nullptr, *c1_b = nullptr, *c1_g = nullptr, *c1_be = nullptr;
    const float *c2_b = nullptr, *c2_g = nullptr, *c2_be = nullptr;
    const __half* c2_w = nullptr;
    Cnn3Weights cnn3{};  // cfg.cnn_blocks == 3
    // encoder
    const __half* w_in = nullptr; const float* b_in = nullptr;
    std::vector<EncLayerW> enc;
    const float *enc_norm_g = nullptr, *enc_norm_b = nullptr;
    const float *rope_cos = nullptr, *rope_sin = nullptr;  // [max_len, dh/2]
    const __half* relpos_pe = nullptr;                     // [max_len, d] rows = |r|
    const float* hm_pe = nullptr;                          // HyperMixing's own sine table [HM_PE_ROWS, d]
    const float* enc_pe = nullptr;                         // regularMHA: the absolute sine table [max_len, d]
    int pos_len = 0;
    // decoder
    const float *emb = nullptr, *dec_pe = nullptr;
    std::vector<DecLayerW> dec;
    const __half* w_ckv = nullptr; const float* b_ckv = nullptr;  // [L*2d, d]
    const float *dec_norm_g = nullptr, *dec_norm_b = nullptr;
    const __half* w_lin = nullptr; const float* b_lin = nullptr;  // seq_lin, when the state has it
    const __half* w_ctc = nullptr; const float* b_ctc = nullptr;  // ctc_lin, when the state has it
    // TransformerLM scorer (optional part)
    const float *lm_emb = nullptr, *lm_pe = nullptr;
    std::vector<LmLayerW> lm;
    const float *lm_norm_g = nullptr, *lm_norm_b = nullptr, *lm_lnp_g = nullptr, *lm_lnp_b = nullptr;
    const float *lm_bp0 = nullptr, *lm_bp2 = nullptr;
    const __half *lm_wp0 = nullptr, *lm_wp2 = nullptr;
    bool has_fbank = false, has_cnn = false, has_enc = false, has_dec = false, has_lm = false;
    ~AsrWeights() {
        if (fbank) fbank_destroy(fbank);
        cudaFree(arena);
    }
};

// Checks the configuration, then repacks the host fp32 tensors of a reference state_dict (`weights`, named with the recipe's
// module prefixes) into the device formats above.  A configuration that is not built, a missing tensor or one with the wrong
// element count fails before anything is allocated on the device.
int load_asr_weights(const sbk_asr_config& cfg, const sbk_tensor* weights, int n_weights,
                     std::shared_ptr<const AsrWeights>* out);

// Rows t = 0 .. rows - 1 of the reference's PositionalEncoding(d) (Transformer.py:252-303; row |r| of RelPosEncXL,
// nnet/attention.py:360-408, is the same): even columns sin(t f_i), odd columns cos(t f_i), in fp32 like the reference's
// buffer (host)
std::vector<float> sine_table(int rows, int d);

}  // namespace sbk
