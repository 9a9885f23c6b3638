// Kernel test hooks of the C ABI: each runs one kernel family on caller buffers so that tests can compare it with a float64
// reference.  None of them touches an engine handle.  (sbk_step_proj_test lives in engine.cu, next to the step projections
// it runs.)
#include <vector>

#include "asr_weights.h"
#include "common.cuh"

namespace sbk {

int TestScratch::reserve(const char* who, size_t bytes) {
    if (bytes == 0) return SBK_OK;
    if (cudaMalloc(&base, bytes) != cudaSuccess) {
        set_error("%s: cudaMalloc(%zu) failed", who, bytes);
        return SBK_ERR_NOMEM;
    }
    return SBK_OK;
}

int finish_test(const char* who, int rc, cudaStream_t st) {
    if (cudaStreamSynchronize(st) != cudaSuccess && rc == SBK_OK) {
        set_error("%s: device error", who);
        rc = SBK_ERR_CUDA;
    }
    return rc;
}

}  // namespace sbk

using namespace sbk;

extern "C" {

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
    const size_t M = (size_t)B * T;
    float *x = nullptr, *xlin = nullptr, *xb = nullptr, *rsum = nullptr, *rb = nullptr, *psi = nullptr, *tab = nullptr,
          *tabM = nullptr;
    int* steps = nullptr;
    TestScratch scr;
    RC(scr.carve("ctc_prefix_test", [&](Carver& take) {
        take(x, M * V * 4); take(xlin, M * V * 4); take(xb, M * 4);
        take(rsum, (size_t)2 * rows * T * 4); take(rb, (size_t)2 * rows * T * 4); take(psi, (size_t)2 * rows * 4);
        take(tab, (size_t)2 * rows * (T + 4) * 4); take(tabM, (size_t)2 * rows * 4);
        take(steps, (size_t)n_steps * rows * 4);
    }));
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
    RC(finish_test("ctc_prefix_test", SBK_OK, st));
    if (group_width) *group_width = ctc_prefix_group_width(beam, T);
    return SBK_OK;
}

int sbk_csgu_test(const void* u_dev, int B, int T, int C, const float* ln_g_dev, const float* ln_b_dev, const float* taps_dev,
                  const float* bias_dev, int K, void* out_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(u_dev && ln_g_dev && ln_b_dev && taps_dev && bias_dev && out_dev, "csgu_test: null pointer");
    SBK_REQUIRE(B >= 1 && T >= 1 && C >= 16 && C % 16 == 0 && K >= 1 && (K & 1) && K <= CSGU_TAP_ROWS,
                "csgu_test: bad sizes B=%d T=%d C=%d K=%d", B, T, C, K);
    const int C2 = C / 2;
    std::vector<float> src((size_t)C2 * K), wt((size_t)CSGU_TAP_ROWS * C2);
    SBK_CUDA_CHECK(cudaMemcpyAsync(src.data(), taps_dev, src.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    csgu_repack_taps(src.data(), C2, K, wt.data());
    float* taps = nullptr;
    float2* stats = nullptr;
    TestScratch scr;
    RC(scr.carve("csgu_test", [&](Carver& take) { take(taps, wt.size() * 4); take(stats, (size_t)B * T * 8); }));
    int rc = cudaMemcpyAsync(taps, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice, st) == cudaSuccess ? SBK_OK : SBK_ERR_CUDA;
    if (rc == SBK_OK)
        rc = csgu_forward(static_cast<const __half*>(u_dev), B, T, C, ln_g_dev, ln_b_dev, 1e-5f, taps, bias_dev, K, stats,
                          static_cast<__half*>(out_dev), st);
    return finish_test("csgu_test", rc, st);
}

int sbk_encoder_attention_test(const void* qkv_dev, int B, int T, int H, int head_dim, const int* lens_dev, int relpos,
                               const float* pos_u_dev, const float* pos_v_dev, const void* P_dev, float scale, int chunk,
                               int left_chunks, void* out_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(qkv_dev && out_dev && (!relpos || (pos_u_dev && pos_v_dev && P_dev)), "encoder_attention_test: null pointer");
    SBK_REQUIRE(B >= 1 && T >= 1 && H >= 1 && head_dim >= 1, "encoder_attention_test: bad sizes B=%d T=%d H=%d head_dim=%d", B,
                T, H, head_dim);
    // This hook keeps the head widths it was written for.  Its tests pin what it refuses (head width 96 among them), so a
    // width the kernel gains later goes through sbk_encoder_attention_window_test instead and leaves those checks meaning
    // what they say.
    SBK_REQUIRE(head_dim == 128 || head_dim == 80 || head_dim == 64 || head_dim == 36 || head_dim == 32,
                "encoder_attention_test: head_dim=%d not taken here (128, 80, 64, 36, 32)", head_dim);
    const int d = H * head_dim;
    const int rc = encoder_attention(static_cast<const __half*>(qkv_dev), 3 * d, B, T, H, head_dim, lens_dev, relpos != 0,
                                     pos_u_dev, pos_v_dev, static_cast<const __half*>(P_dev), d, scale,
                                     static_cast<__half*>(out_dev), d, st, chunk, left_chunks);
    return finish_test("encoder_attention_test", rc, st);
}

int sbk_encoder_attention_window_test(const void* qkv_dev, const void* kv_dev, int B, int T, int H, int head_dim,
                                      const int* lens_dev, int relpos, const float* pos_u_dev, const float* pos_v_dev,
                                      const void* P_dev, float scale, int chunk, int left_chunks, int cap, int start, int nq,
                                      void* out_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(qkv_dev && out_dev && (!relpos || (pos_u_dev && pos_v_dev && P_dev)), "encoder_attention_window_test: null pointer");
    SBK_REQUIRE(B >= 1 && T >= 1 && H >= 1 && head_dim >= 1, "encoder_attention_window_test: bad sizes B=%d T=%d H=%d head_dim=%d",
                B, T, H, head_dim);
    const int d = H * head_dim;
    int rc;
    if (!kv_dev) {
        rc = encoder_attention(static_cast<const __half*>(qkv_dev), 3 * d, B, T, H, head_dim, lens_dev, relpos != 0, pos_u_dev,
                               pos_v_dev, static_cast<const __half*>(P_dev), d, scale, static_cast<__half*>(out_dev), d, st,
                               chunk, left_chunks);
    } else {
        SBK_REQUIRE(!lens_dev && chunk == 0, "encoder_attention_window_test: a stream window has no lengths and no chunk mask");
        SBK_REQUIRE(nq >= 1 && nq <= T && T <= cap && start >= 0 && start < cap,
                    "encoder_attention_window_test: bad ring (%d queries, %d rows, ring of %d from %d)", nq, T, cap, start);
        AttStream sa;
        sa.q = static_cast<const __half*>(qkv_dev); sa.ldq = d;
        sa.kv = static_cast<const __half*>(kv_dev); sa.ldkv = 2 * d;
        sa.cap = cap; sa.start = start; sa.nq = nq;
        rc = encoder_attention_stream(sa, B, T, H, head_dim, relpos != 0, pos_u_dev, pos_v_dev, static_cast<const __half*>(P_dev),
                                      d, scale, static_cast<__half*>(out_dev), d, st);
    }
    return finish_test("encoder_attention_window_test", rc, st);
}

int sbk_encoder_attention_occupancy(int head_dim, int stream_form, int* ctas_per_sm) {
    SBK_REQUIRE(ctas_per_sm, "encoder_attention_occupancy: null pointer");
    return encoder_attention_occupancy(head_dim, stream_form != 0, ctas_per_sm);
}

int sbk_lm_causal_attention_test(const void* qkv_dev, int n, int s, int d, int H, const int* tokens_dev, int pad_tok,
                                 void* out_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(qkv_dev && tokens_dev && out_dev && n >= 1 && s >= 1 && n <= 65535, "lm_causal_attention_test: bad arguments");
    return finish_test("lm_causal_attention_test",
                       lm_causal_attention(static_cast<const __half*>(qkv_dev), n, s, d, H, tokens_dev, pad_tok,
                                           static_cast<__half*>(out_dev), st), st);
}

int sbk_dec_attention_test(const void* q_dev, int ldq, const void* kbase_dev, const void* vbase_dev, long long row_stride,
                           int key_stride, int head_stride, int rows_per_block, int rows, int H, int dh, int max_keys, int step,
                           const int* enc_len_dev, const int* lineage_dev, const int* tok_cache_dev, int lin_stride,
                           int pad_tok, void* out_dev, int ldo, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(q_dev && kbase_dev && vbase_dev && out_dev, "dec_attention_test: null pointer");
    SBK_REQUIRE(rows >= 1 && H >= 1 && dh >= 1 && max_keys >= 1 && rows_per_block >= 1 && rows % rows_per_block == 0 &&
                    ldq >= H * dh && ldo >= H * dh && key_stride >= 1 && row_stride >= 0 && head_stride >= 0,
                "dec_attention_test: bad sizes rows=%d rows_per_block=%d H=%d dh=%d max_keys=%d", rows, rows_per_block, H, dh,
                max_keys);
    if (dh == 64 || dh == 80 || dh == 128) {  // 16-byte loads of q, K and V
        const uintptr_t al = reinterpret_cast<uintptr_t>(q_dev) | reinterpret_cast<uintptr_t>(kbase_dev) |
                             reinterpret_cast<uintptr_t>(vbase_dev);
        SBK_REQUIRE((al & 15) == 0 && ldq % 8 == 0 && key_stride % 8 == 0 && row_stride % 8 == 0 && head_stride % 8 == 0,
                    "dec_attention_test: head_dim %d needs 16-byte aligned q / key rows", dh);
    }
    const bool self = step >= 0;
    SBK_REQUIRE(self || (!lineage_dev && !tok_cache_dev), "dec_attention_test: a lineage or token mask needs self-attention");
    SBK_REQUIRE(!lineage_dev || rows_per_block == 1, "dec_attention_test: a lineage table needs one cache row per query row");
    SBK_REQUIRE(!self || step < max_keys, "dec_attention_test: step %d >= max_keys %d", step, max_keys);
    SBK_REQUIRE(!(lineage_dev || tok_cache_dev) || step < lin_stride, "dec_attention_test: step %d >= lin_stride %d", step,
                lin_stride);
    // the kernels index rows and frames with these: check them on the host first
    if (lineage_dev) {
        std::vector<int> lin((size_t)2 * rows * lin_stride);
        SBK_CUDA_CHECK(cudaMemcpyAsync(lin.data(), lineage_dev, lin.size() * 4, cudaMemcpyDeviceToHost, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
        for (size_t i = 0; i < lin.size(); ++i)
            SBK_REQUIRE(lin[i] >= 0 && lin[i] < rows, "dec_attention_test: lineage entry %zu = %d outside [0, %d)", i, lin[i], rows);
    }
    if (!self && enc_len_dev) {
        std::vector<int> len(rows / rows_per_block);
        SBK_CUDA_CHECK(cudaMemcpyAsync(len.data(), enc_len_dev, len.size() * 4, cudaMemcpyDeviceToHost, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
        for (int v : len) SBK_REQUIRE(v >= 0 && v <= max_keys, "dec_attention_test: enc_len %d outside [0, %d]", v, max_keys);
    }
    int* step_dev = nullptr;
    TestScratch scr;
    RC(scr.carve("dec_attention_test", [&](Carver& take) { if (self) take(step_dev, 4); }));
    if (self && cudaMemcpyAsync(step_dev, &step, 4, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        set_error("dec_attention_test: copy failed");
        return SBK_ERR_CUDA;
    }
    DecAttnArgs t{};
    t.q = static_cast<const __half*>(q_dev); t.ldq = ldq;
    t.kbase = static_cast<const __half*>(kbase_dev); t.vbase = static_cast<const __half*>(vbase_dev);
    t.row_stride = (size_t)row_stride; t.key_stride = key_stride; t.head_stride = head_stride; t.rows_per_block = rows_per_block;
    t.n_keys_ptr = step_dev; t.enc_len = self ? nullptr : enc_len_dev; t.H = H; t.dh = dh;
    t.out = static_cast<__half*>(out_dev); t.ldo = ldo;
    t.lineage = lineage_dev; t.tok_cache = tok_cache_dev; t.lin_stride = lin_stride; t.pad_tok = pad_tok;
    return finish_test("dec_attention_test", dec_attention(t, rows, max_keys, st), st);
}

int sbk_xatt_fold_test(const void* h16_dev, const float* in_proj_w, const float* in_proj_b, const float* out_w,
                       const float* out_b, const void* enc16_dev, const int* enc_len_dev, int rows, int T, int H, int d,
                       float* x_dev, int ldx, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(h16_dev && in_proj_w && in_proj_b && out_w && out_b && enc16_dev && enc_len_dev && x_dev,
                "xatt_fold_test: null pointer");
    SBK_REQUIRE(rows >= 1 && T >= 1 && H >= 1 && d == 64 * H && (d == 256 || d == 512) && ldx >= d,
                "xatt_fold_test: bad sizes rows=%d T=%d H=%d d=%d ldx=%d", rows, T, H, d, ldx);
    std::vector<int> len(rows);  // the kernel indexes frames with these: check them on the host first
    SBK_CUDA_CHECK(cudaMemcpyAsync(len.data(), enc_len_dev, rows * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int v : len) SBK_REQUIRE(v >= 0 && v <= T, "xatt_fold_test: enc_len %d outside [0, %d]", v, T);
    std::vector<double> xq, bxq, xo, bxo;
    fold_cross_attention(in_proj_w, in_proj_b, out_w, out_b, d, H, &xq, &bxq, &xo, &bxo);
    std::vector<__half> wq16(xq.size()), wo16(xo.size());
    for (size_t i = 0; i < xq.size(); ++i) wq16[i] = __double2half(xq[i]);
    for (size_t i = 0; i < xo.size(); ++i) wo16[i] = __double2half(xo[i]);
    const std::vector<float> bq32(bxq.begin(), bxq.end()), bo32(bxo.begin(), bxo.end());
    const int Hd = H * d;
    __half *wq = nullptr, *wo = nullptr, *q = nullptr, *ctx = nullptr;
    float *bq = nullptr, *bo = nullptr;
    TestScratch scr;
    RC(scr.carve("xatt_fold_test", [&](Carver& take) {
        take(wq, wq16.size() * 2); take(wo, wo16.size() * 2); take(bq, (size_t)Hd * 4); take(bo, (size_t)d * 4);
        take(q, (size_t)rows * Hd * 2); take(ctx, (size_t)rows * Hd * 2);
    }));
    SBK_CUDA_CHECK(cudaMemcpyAsync(wq, wq16.data(), wq16.size() * 2, cudaMemcpyHostToDevice, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(wo, wo16.data(), wo16.size() * 2, cudaMemcpyHostToDevice, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(bq, bq32.data(), (size_t)Hd * 4, cudaMemcpyHostToDevice, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(bo, bo32.data(), (size_t)d * 4, cudaMemcpyHostToDevice, st));
    GemmEpilogue eq;
    eq.mode = EPI_F16; eq.bias = bq; eq.out = q; eq.ldo = Hd;
    int rc = gemm_f16_small(h16_dev, d, wq, d, eq, rows, Hd, d, st);
    XattFoldArgs x{q, Hd, static_cast<const __half*>(enc16_dev), enc_len_dev, T, H, d, ctx, Hd};
    if (rc == SBK_OK) rc = dec_xatt_fold(x, rows, st);
    GemmEpilogue eo;
    eo.mode = EPI_RESID; eo.bias = bo; eo.out = x_dev; eo.resid = x_dev; eo.ldo = ldx;
    if (rc == SBK_OK) rc = gemm_f16_small(ctx, Hd, wo, Hd, eo, rows, d, Hd, st);
    return finish_test("xatt_fold_test", rc, st);
}

int sbk_stream_qkv_test(const float* qkv_dev, int B, int n, int H, int head_dim, const float* inv_freq_dev, long long pos0,
                        float q_scale, void* q_out_dev, void* kv_out_dev, int cap, int slot0, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(qkv_dev && q_out_dev && kv_out_dev, "stream_qkv_test: null pointer");
    SBK_REQUIRE(B >= 1 && H >= 1 && head_dim >= 2 && pos0 >= 0, "stream_qkv_test: bad sizes");
    const int rc = stream_qkv(qkv_dev, B, n, H, head_dim, inv_freq_dev, pos0, q_scale, static_cast<__half*>(q_out_dev),
                              static_cast<__half*>(kv_out_dev), cap, slot0, st);
    return finish_test("stream_qkv_test", rc, st);
}

static int dwconv_test(const float* x_dev, int B, int T, int D, int K, const float* taps_dev, const float* bias_dev,
                       const float* ln_g_dev, const float* ln_b_dev, int chunk, bool gelu, void* out_dev, cudaStream_t st) {
    SBK_REQUIRE(x_dev && taps_dev && bias_dev && ln_g_dev && ln_b_dev && out_dev, "dwconv_test: null pointer");
    SBK_REQUIRE(B >= 1 && T >= 1 && D >= 1 && K >= 1 && chunk >= 0, "dwconv_test: bad sizes B=%d T=%d D=%d K=%d chunk=%d", B, T,
                D, K, chunk);
    std::vector<float> src((size_t)D * K), wt((size_t)K * D);
    SBK_CUDA_CHECK(cudaMemcpyAsync(src.data(), taps_dev, src.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    dwconv_repack_taps(src.data(), D, K, wt.data());
    float* taps = nullptr;
    TestScratch scr;
    RC(scr.carve("dwconv_test", [&](Carver& take) { take(taps, wt.size() * 4); }));
    int rc = cudaMemcpyAsync(taps, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice, st) == cudaSuccess ? SBK_OK : SBK_ERR_CUDA;
    if (rc == SBK_OK)
        rc = dwconv_ln_act(x_dev, B, T, D, K, taps, bias_dev, ln_g_dev, ln_b_dev, 1e-5f, static_cast<__half*>(out_dev), st, gelu,
                           chunk);
    return finish_test("dwconv_test", rc, st);
}

int sbk_dwconv_test(const float* x_dev, int B, int T, int D, int K, const float* taps_dev, const float* bias_dev,
                    const float* ln_g_dev, const float* ln_b_dev, int chunk, void* out_dev, void* stream) {
    return dwconv_test(x_dev, B, T, D, K, taps_dev, bias_dev, ln_g_dev, ln_b_dev, chunk, false, out_dev,
                       static_cast<cudaStream_t>(stream));
}

int sbk_dwconv_act_test(const float* x_dev, int B, int T, int D, int K, const float* taps_dev, const float* bias_dev,
                        const float* ln_g_dev, const float* ln_b_dev, int chunk, int act, void* out_dev, void* stream) {
    SBK_REQUIRE(act == SBK_CONFORMER_ACT_SWISH || act == SBK_CONFORMER_ACT_GELU, "dwconv_act_test: act %d (0 Swish, 1 GELU)", act);
    return dwconv_test(x_dev, B, T, D, K, taps_dev, bias_dev, ln_g_dev, ln_b_dev, chunk, act == SBK_CONFORMER_ACT_GELU, out_dev,
                       static_cast<cudaStream_t>(stream));
}

int sbk_hypermix_test(const void* x_dev, const int* lens_dev, int B, int T, int d, int nhead, int k, const float* w1_fc1_w_dev,
                      const float* w1_fc1_b_dev, const float* w1_fc2_w_dev, const float* w1_fc2_b_dev, const float* w2_fc1_w_dev,
                      const float* w2_fc1_b_dev, const float* w2_fc2_w_dev, const float* w2_fc2_b_dev, const float* ln_g_dev,
                      const float* ln_b_dev, float* out_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(x_dev && w1_fc1_w_dev && w1_fc1_b_dev && w1_fc2_w_dev && w1_fc2_b_dev && w2_fc1_w_dev && w2_fc1_b_dev &&
                    w2_fc2_w_dev && w2_fc2_b_dev && ln_g_dev && ln_b_dev && out_dev, "hypermix_test: null pointer");
    SBK_REQUIRE(B >= 1 && T >= 1 && nhead >= 1 && d % nhead == 0 && k >= 1, "hypermix_test: bad sizes B=%d T=%d d=%d nhead=%d k=%d",
                B, T, d, nhead, k);
    const int e = d / nhead;
    const size_t n1 = (size_t)nhead * e * e, n2 = (size_t)nhead * k * e;
    const std::vector<float> pe = sine_table(HM_PE_ROWS, d);
    const size_t part_n = hypermix_part_floats(B, T, d, k);
    __half *w16 = nullptr, *G = nullptr;
    float *pe_dev = nullptr, *part = nullptr, *gscale = nullptr;
    TestScratch scr;
    RC(scr.carve("hypermix_test", [&](Carver& take) {
        take(w16, 2 * (n1 + n2) * 2); take(pe_dev, pe.size() * 4); take(part, part_n * 4); take(G, (size_t)B * d * k * 2);
        take(gscale, (size_t)B * nhead * 4);
    }));
    HyperMixWeights w;
    w.fc1w[0] = w16; w.fc2w[0] = w16 + n1; w.fc1w[1] = w16 + n1 + n2; w.fc2w[1] = w16 + 2 * n1 + n2;
    w.fc1b[0] = w1_fc1_b_dev; w.fc2b[0] = w1_fc2_b_dev; w.fc1b[1] = w2_fc1_b_dev; w.fc2b[1] = w2_fc2_b_dev;
    w.ln_g = ln_g_dev; w.ln_b = ln_b_dev;
    int rc = cast_f32_f16(w1_fc1_w_dev, const_cast<__half*>(w.fc1w[0]), n1, st);
    if (rc == SBK_OK) rc = cast_f32_f16(w1_fc2_w_dev, const_cast<__half*>(w.fc2w[0]), n2, st);
    if (rc == SBK_OK) rc = cast_f32_f16(w2_fc1_w_dev, const_cast<__half*>(w.fc1w[1]), n1, st);
    if (rc == SBK_OK) rc = cast_f32_f16(w2_fc2_w_dev, const_cast<__half*>(w.fc2w[1]), n2, st);
    if (rc == SBK_OK && (cudaMemcpyAsync(pe_dev, pe.data(), pe.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                         cudaMemsetAsync(out_dev, 0, (size_t)B * T * d * 4, st) != cudaSuccess)) {
        set_error("hypermix_test: copy failed");
        rc = SBK_ERR_CUDA;
    }
    if (rc == SBK_OK)
        rc = hypermix_forward(static_cast<const __half*>(x_dev), B, T, d, nhead, k, lens_dev,
                              pe_dev, w, part, G, gscale, out_dev, st);
    return finish_test("hypermix_test", rc, st);
}

int sbk_beam_step_test(const sbk_beam_params* params, int path, int B, int V, int S_max, int n_hist, const float* logits_dev,
                       float* seq_scores_dev, int* lineage_dev, int* step_dev, int* finished_dev, int* n_full_dev,
                       int* hist_tok_dev, int* hist_pred_dev, float* hist_score_dev, float* hist_lp_dev,
                       const float* add_scores_dev, const float* add_row_dev, const float* emb_dev, const float* pe_dev, int d,
                       float* x_next_dev, const float* lm_emb_dev, const float* lm_pe_dev, int lm_d, float* lm_x_dev,
                       void* lm_x16_dev, int* tok_cache_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(params && logits_dev && seq_scores_dev && lineage_dev && step_dev && finished_dev && n_full_dev && hist_tok_dev &&
                    hist_pred_dev && hist_score_dev && hist_lp_dev && emb_dev && pe_dev && x_next_dev,
                "beam_step_test: null pointer");
    const sbk_beam_params& p = *params;
    const int beam = p.beam_size;
    SBK_REQUIRE(B >= 1 && V >= 1 && S_max >= 2 && n_hist >= 1 && d >= 1, "beam_step_test: bad sizes B=%d V=%d S_max=%d n_hist=%d d=%d",
                B, V, S_max, n_hist, d);
    SBK_REQUIRE(beam >= 1 && beam <= 128 && beam <= V, "beam_step_test: beam_size %d not in [1, min(128, V = %d)]", beam, V);
    SBK_REQUIRE(path >= 0 && path <= 2 && !(path == 1 && beam > 16), "beam_step_test: path %d at beam_size %d", path, beam);
    SBK_REQUIRE(p.eos >= 0 && p.eos < V, "beam_step_test: eos %d outside [0, %d)", p.eos, V);
    SBK_REQUIRE(p.ctc_weight == 0.0f || (p.blank_index >= 0 && p.blank_index < V && p.blank_index != p.eos),
                "beam_step_test: blank %d must be a token other than eos", p.blank_index);
    const bool lm = lm_emb_dev != nullptr;
    SBK_REQUIRE(!lm || (lm_pe_dev && lm_x_dev && lm_x16_dev && tok_cache_dev && lm_d >= 1), "beam_step_test: incomplete LM buffers");
    const int rows = B * beam;
    // the kernels index the history, the lineage, the positional tables and the token cache with these: check them first
    std::vector<int> step((size_t)rows), lin((size_t)2 * rows * S_max);
    SBK_CUDA_CHECK(cudaMemcpyAsync(step.data(), step_dev, step.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(lin.data(), lineage_dev, lin.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int r = 0; r < rows; ++r) {
        const int s = step[r];
        SBK_REQUIRE(s == step[r - r % beam], "beam_step_test: rows of utterance %d at steps %d and %d", r / beam, step[r - r % beam], s);
        SBK_REQUIRE(s >= 0 && s + 1 < S_max && s < n_hist, "beam_step_test: step %d outside [0, min(S_max - 1 = %d, n_hist = %d))", s,
                    S_max - 1, n_hist);
    }
    for (size_t i = 0; i < lin.size(); ++i)
        SBK_REQUIRE(lin[i] >= 0 && lin[i] < rows, "beam_step_test: lineage entry %zu = %d outside [0, %d)", i, lin[i], rows);
    float* scr = nullptr;
    TestScratch scratch;
    const bool rows_merge = path == 1 || (path == 0 && beam <= 16);
    RC(scratch.carve("beam_step_test", [&](Carver& take) { if (rows_merge) take(scr, (size_t)rows * 33 * 4); }));
    BeamStepArgs a{};   // as run_beam fills it
    a.logits = logits_dev; a.V = V; a.beam = beam; a.S_max = S_max; a.seq_scores = seq_scores_dev; a.lineage = lineage_dev;
    a.step_arr = step_dev; a.finished = finished_dev; a.n_full = n_full_dev;
    a.hist_tok = hist_tok_dev; a.hist_pred = hist_pred_dev; a.hist_score = hist_score_dev; a.hist_lp = hist_lp_dev;
    a.temperature = p.temperature; a.eos_threshold = p.eos_threshold; a.minus_inf = p.minus_inf; a.min_steps = p.min_steps;
    a.eos = p.eos; a.use_eos_threshold = p.using_eos_threshold; a.length_norm = p.length_normalization;
    a.emb = emb_dev; a.pe = pe_dev; a.d = d; a.x_next = x_next_dev;
    a.add_scores = add_scores_dev; a.add_row = add_row_dev; a.add_const = p.length_weight;
    if (p.ctc_weight != 0.0f) { a.attn_weight = 1.0f - p.ctc_weight; a.blank = p.blank_index; }
    if (lm) {
        a.lm.emb = lm_emb_dev; a.lm.pe = lm_pe_dev; a.lm.d = lm_d; a.lm.scale = sqrtf((float)lm_d); a.lm.x = lm_x_dev; a.lm.x16 = static_cast<__half*>(lm_x16_dev);
        a.lm.tok_cache = tok_cache_dev;
    }
    a.scratch = scr; a.path = path;
    return finish_test("beam_step_test", beam_step(a, B, st), st);
}

int sbk_coverage_score_test(const void* q_dev, int ldq, const void* kbase_dev, long long utt_stride, int key_stride,
                            int head_stride, const int* enc_len_dev, int rows_per_utt, int T, int H, float* cov_dev,
                            const int* hist_pred_dev, const int* step_dev, int n_bh, float threshold, float weight, float* out_dev,
                            void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(q_dev && kbase_dev && enc_len_dev && cov_dev && hist_pred_dev && step_dev && out_dev, "coverage_test: null pointer");
    SBK_REQUIRE(n_bh >= 1 && rows_per_utt >= 1 && n_bh % rows_per_utt == 0 && H >= 1 && ldq >= H * 64 && T >= 1 &&
                    utt_stride >= 0 && key_stride >= 1 && head_stride >= 0,
                "coverage_test: bad sizes n_bh=%d rows_per_utt=%d H=%d T=%d", n_bh, rows_per_utt, H, T);
    const uintptr_t al = reinterpret_cast<uintptr_t>(kbase_dev);   // 16-byte key loads
    SBK_REQUIRE((al & 15) == 0 && utt_stride % 8 == 0 && key_stride % 8 == 0 && head_stride % 8 == 0,
                "coverage_test: key rows must be 16-byte aligned");
    // the kernel indexes frames, the coverage rows and the history with these: check them first
    std::vector<int> len(n_bh / rows_per_utt), step(n_bh);
    SBK_CUDA_CHECK(cudaMemcpyAsync(len.data(), enc_len_dev, len.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaMemcpyAsync(step.data(), step_dev, step.size() * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int v : len) SBK_REQUIRE(v >= 0 && v <= T, "coverage_test: enc_len %d outside [0, %d]", v, T);
    for (int s : step) SBK_REQUIRE(s == step[0] && s >= 0, "coverage_test: rows at steps %d and %d", step[0], s);
    if (step[0] > 0) {
        std::vector<int> pred(n_bh);
        SBK_CUDA_CHECK(cudaMemcpyAsync(pred.data(), hist_pred_dev + (size_t)(step[0] - 1) * n_bh, pred.size() * 4,
                                       cudaMemcpyDeviceToHost, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));
        for (int v : pred) SBK_REQUIRE(v >= 0 && v < n_bh, "coverage_test: predecessor %d outside [0, %d)", v, n_bh);
    }
    CoverageStep c{};
    c.q = static_cast<const __half*>(q_dev); c.ldq = ldq; c.kbase = static_cast<const __half*>(kbase_dev);
    c.utt_stride = (size_t)utt_stride; c.key_stride = key_stride; c.head_stride = head_stride; c.enc_len = enc_len_dev;
    c.rows_per_utt = rows_per_utt; c.T = T; c.H = H; c.cov_base = cov_dev; c.hist_pred = hist_pred_dev; c.step_ptr = step_dev;
    c.n_bh = n_bh; c.threshold = threshold; c.weight = weight; c.out = out_dev;
    return finish_test("coverage_test", coverage_score(c, st), st);
}

}  // extern "C"
