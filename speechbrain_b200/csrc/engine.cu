// Model engine: workspace, the encode pipeline (CNN front-end -> Conformer encoder) and the KV-cached greedy decode
// loop.  Host-side orchestration only; all math is in the kernels.  The weights are loaded and repacked by asr_weights.cu.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "asr_weights.h"
#include "common.cuh"

namespace sbk {

// One cached CUDA graph and the key it was captured for.  Keys are compared bytewise, so callers zero their padding.
struct GraphCache {
    cudaGraphExec_t exec = nullptr;
    long long nodes = 0;  // kernel launches the graph replays (bench.py's launch count)
    std::string key;
    GraphCache() = default;
    GraphCache(const GraphCache&) = delete;
    GraphCache& operator=(const GraphCache&) = delete;
    ~GraphCache() { reset(); }
    void reset() {
        if (exec) cudaGraphExecDestroy(exec);
        exec = nullptr;
    }
    // Captures enqueue(cap_stream) (creating cap_stream on first use) unless a graph for the same key exists.
    template <class Key, class Enqueue>
    int ensure(const Key& k, cudaStream_t& cap_stream, Enqueue&& enqueue) {
        if (exec && key.size() == sizeof(Key) && memcmp(key.data(), &k, sizeof(Key)) == 0) return SBK_OK;
        reset();
        if (!cap_stream) SBK_CUDA_CHECK(cudaStreamCreateWithFlags(&cap_stream, cudaStreamNonBlocking));
        cudaGraph_t g;
        SBK_CUDA_CHECK(cudaStreamBeginCapture(cap_stream, cudaStreamCaptureModeThreadLocal));
        launch_count_begin_capture();
        const int rc = enqueue(cap_stream);
        nodes = launch_count_end_capture();
        const cudaError_t ce = cudaStreamEndCapture(cap_stream, &g);
        if (rc) return rc;
        SBK_CUDA_CHECK(ce);
        const cudaError_t ie = cudaGraphInstantiate(&exec, g, 0);
        cudaGraphDestroy(g);
        SBK_CUDA_CHECK(ie);
        key.assign(reinterpret_cast<const char*>(&k), sizeof(Key));
        return SBK_OK;
    }
    int launch(cudaStream_t st) {
        SBK_CUDA_CHECK(cudaGraphLaunch(exec, st));
        launch_count_add(nodes);
        return SBK_OK;
    }
};

// A lane's device buffer that only grows (grow_buffer).  Graphs capture pointers into it.
struct DevBuf {
    void* base = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { cudaFree(base); }
};

// A lane's second stream, created by ensure() on first use, with the events that fork work onto it and join it back.
// Under stream capture the fork and join become graph edges.
struct SideStream {
    cudaStream_t s = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    SideStream() = default;
    SideStream(const SideStream&) = delete;
    SideStream& operator=(const SideStream&) = delete;
    ~SideStream() {
        if (s) cudaStreamDestroy(s);
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
    }
    int ensure(bool top_priority = false) {
        if (s) return SBK_OK;
        int lo = 0, hi = 0;  // numerically lowest = highest priority; 0 = the default
        if (top_priority) SBK_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        SBK_CUDA_CHECK(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, hi));
        SBK_CUDA_CHECK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
        SBK_CUDA_CHECK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
        return SBK_OK;
    }
    // s waits for the work enqueued on `from` so far
    int fork(cudaStream_t from) {
        SBK_CUDA_CHECK(cudaEventRecord(ev_fork, from));
        SBK_CUDA_CHECK(cudaStreamWaitEvent(s, ev_fork, 0));
        return SBK_OK;
    }
    // `into` waits for the work enqueued on s so far
    int join(cudaStream_t into) {
        SBK_CUDA_CHECK(cudaEventRecord(ev_join, s));
        SBK_CUDA_CHECK(cudaStreamWaitEvent(into, ev_join, 0));
        return SBK_OK;
    }
};

// A handle: the shared weights plus one lane's state.  A clone is another lane on the same weights with its own workspace,
// graphs, streams and flags: one clone per in-flight batch lets independent batches overlap on different streams (the
// decode loop is latency-bound and leaves most SMs idle, so concurrent lanes raise throughput without touching per-batch
// numerics).  Streams, events and buffers are created on first use; the destructor releases all of them.
struct AsrModel {
    std::shared_ptr<const AsrWeights> wt;
    DevBuf ws;  // workspace (re-carved per shape)
    // CTC prefix scorer state (grown by the first beam search that uses it, see run_beam), or the logits of an arg-max-only
    // ctc_head call
    DevBuf ctc;
    DevBuf cov;  // CoverageScorer: [2][rows][T] coverage + [rows] scores
    // TransformerLM whole-sequence forward (run_lm_forward), carved for `rows` = n * s token rows, independent of the
    // decode / beam workspace: residual stream x [rows, d] fp32, its fp16 copy x16, qkv16 [rows, 3d], att16 [rows, d],
    // f16 [rows, d_ffn]
    DevBuf lmf_mem;
    struct LmFwdBuf {
        int rows = 0;
        float* x; __half *x16, *qkv16, *att16, *f16;
    } lmf;
    // shapes the workspace is carved for (wsBe: utterances per encoder pass, >= wsB)
    int wsB = 0, wsBe = 0, wsL = 0, ws_rows = 0, ws_steps = 0;
    struct Buf {
        float *wav, *feats, *x, *glu, *enc_out, *dx, *logits, *score, *seq_scores, *lnout, *beam_scr;
        int *utt_max, *enc_len, *tokens, *step, *has_ended, *ended_count, *pred, *lineage, *finished, *hist_tok, *hist_pred;
        float *hist_score, *hist_lp;
        float* rel_len;
        float *lx, *lh32, *lm_logits, *lm_extra;
        __half *lx16, *lq16, *latt16, *lf16, *lh16, *lkc, *lvc;
        int* tok_cache;
        __half *act1, *a_in, *h16, *f16, *qkv16, *att16, *P16, *enc16, *ckv16, *kcache, *vcache, *dh16, *dq16, *datt16, *df16;
        // Branchformer encoder only: norm_conv output [M, d], [attention | conv branch] [M, 2d], CSGU output [M, C/2], CSGU
        // LayerNorm statistics [M]
        __half *hc16, *cat16, *g16;
        float2* csgu_stats;
        // HyperConformer encoder only: per-chunk partial H, G = GELU(H) scaled to fp16 [B, d, k], its scales [B, nhead]
        float *hm_part, *hm_gscale;
        __half* hm_G;
    } b;
    GraphCache step_graph;    // one greedy decode step (run_greedy)
    GraphCache group_graph;   // a whole group call (sbk_asr_transcribe_greedy_group_dev)
    GraphCache hgroup_graph;  // the same from host buffers, H2D / D2H memcpy nodes included
    GraphCache beam_graph;    // one whole beam-search step (run_beam)
    GraphCache pipe_graph;    // the whole Fbank .. last decode step pipeline (sbk_asr_transcribe_greedy_dev)
    int* host_flag = nullptr;  // pinned
    // host-buffer group entry point: device staging of the G batches' wav / lengths, a copy stream forked from the caller's
    // stream (so the H2D of a later encoder pass's batches overlaps an earlier pass)
    DevBuf gwav;
    SideStream copy_stream;
    cudaEvent_t ev_ready[16] = {};  // batch g's staging copies have landed
    SideStream side_stream;  // beam search: the LM scorer's branch of a search step
    SideStream dec_stream;   // group calls: the decode loop, on a high-priority stream (see transcribe_group_enqueue)
    cudaStream_t cap_stream = nullptr;  // private stream for graph capture (the legacy default stream cannot capture)
    int dec_tc_rows = 64;        // >= this many live hypotheses: wgmma decode GEMMs
    int dyn_chunk = 0, dyn_left = -1;  // DynChunkTrainConfig of the next encode calls (chunk frames, left-context chunks; 0 = off)
    int fuse_dec_ln = 1;         // 1: LayerNorm inside the projection kernel (latency); 0: separate LN kernel (throughput)
    int poll_every = 8;          // greedy early-exit poll interval in steps; 0 = never sync, run exactly max_steps

    AsrModel() = default;
    AsrModel(const AsrModel&) = delete;
    AsrModel& operator=(const AsrModel&) = delete;
    ~AsrModel() {
        if (host_flag) cudaFreeHost(host_flag);
        if (cap_stream) cudaStreamDestroy(cap_stream);
        for (cudaEvent_t e : ev_ready)
            if (e) cudaEventDestroy(e);
    }
};

// A whole call as one CUDA graph: replays `graph` for `key` (capturing enqueue(cap_stream, &done, true) first when the key
// is new), which runs exactly max_steps decode steps.  With use_graph false: enqueue(st, steps_done, false), eagerly.
template <class Key, class Enqueue>
static int replay_or_enqueue(AsrModel* m, GraphCache& graph, bool use_graph, const Key& key, int max_steps, int* steps_done,
                             cudaStream_t st, Enqueue&& enqueue) {
    if (!use_graph) return enqueue(st, steps_done, false);
    RC(graph.ensure(key, m->cap_stream, [&](cudaStream_t cs) {
        int done = 0;
        return enqueue(cs, &done, true);
    }));
    RC(graph.launch(st));
    if (steps_done) *steps_done = max_steps;
    return SBK_OK;
}

// A new lane on the weights of `wt`.
static int new_lane(std::shared_ptr<const AsrWeights> wt, AsrModel** out) {
    AsrModel* m = new AsrModel();
    m->wt = std::move(wt);
    if (cudaMallocHost(&m->host_flag, 64) != cudaSuccess) {
        delete m;
        set_error("cudaMallocHost failed");
        return SBK_ERR_NOMEM;
    }
    *out = m;
    return SBK_OK;
}

int asr_create(const sbk_asr_config* cfg, const sbk_tensor* weights, int n_weights, AsrModel** out) {
    SBK_REQUIRE(cfg && weights && out, "asr_create: null argument");
    std::shared_ptr<const AsrWeights> wt;
    RC(load_asr_weights(*cfg, weights, n_weights, &wt));
    return new_lane(std::move(wt), out);
}

// A clone is a new lane on the same weights; it inherits the source's settings.
int asr_clone(AsrModel* src, AsrModel** out) {
    SBK_REQUIRE(src && out, "asr_clone: null argument");
    AsrModel* m = nullptr;
    RC(new_lane(src->wt, &m));
    m->fuse_dec_ln = src->fuse_dec_ln;
    m->dec_tc_rows = src->dec_tc_rows;
    m->poll_every = src->poll_every;
    m->dyn_chunk = src->dyn_chunk;
    m->dyn_left = src->dyn_left;
    *out = m;
    return SBK_OK;
}

// cached graphs bake in workspace pointers / kernel choices: drop them whenever either changes
static void drop_graphs(AsrModel* m) {
    m->step_graph.reset();
    m->pipe_graph.reset();
    m->group_graph.reset();
    m->hgroup_graph.reset();
    m->beam_graph.reset();
}

// Makes `buf` hold at least `need` bytes.  Replacing a buffer waits for the device (work on any of the lane's streams may
// still use it) and drops the lane's graphs, which captured pointers into it.
static int grow_buffer(AsrModel* m, DevBuf& buf, size_t need, const char* what) {
    if (need <= buf.cap) return SBK_OK;
    if (buf.base) {
        SBK_CUDA_CHECK(cudaDeviceSynchronize());
        cudaFree(buf.base);
        buf.base = nullptr;
        buf.cap = 0;
        drop_graphs(m);
    }
    if (cudaMalloc(&buf.base, need) != cudaSuccess) {
        set_error("%s: cudaMalloc(%zu) failed", what, need);
        return SBK_ERR_NOMEM;
    }
    buf.cap = need;
    return SBK_OK;
}

static void frames(const sbk_asr_config& c, int L, int* T0, int* T1, int* T2) {
    *T0 = 1 + L / c.hop;
    *T1 = (*T0 - 1) / 2 + 1;
    *T2 = (*T1 - 1) / 2 + 1;
}

// A sample count whose frames() give T encoder frames: sizes the workspace of entries that start from encoder states.
static int enc_samples(const sbk_asr_config& c, int T) { return (T - 1) * 4 * c.hop; }

// The workspace for calls of B utterances of L samples whose encoder passes take up to Be utterances (Be > B: a group call
// encodes several of its batches in one pass), `rows` decoder hypotheses, `steps` max steps.  Encoder activations are sized
// for Be utterances, the per-call buffers (wav, Fbank scratch, lengths, flags) for B.
static void workspace_layout(const AsrModel* m, int B, int Be, int L, int rows, int steps, AsrModel::Buf& b, Carver& take) {
    const sbk_asr_config& c = m->wt->cfg;
    int T0, T1, T2;
    frames(c, L, &T0, &T1, &T2);
    const int F1 = (c.n_mels - 1) / 2 + 1;
    const size_t M = (size_t)Be * T2, d = c.d_model, F = c.d_ffn, Ld = c.num_decoder_layers, S = steps + 1;
    const bool bfm = c.encoder_module == SBK_ENC_BRANCHFORMER && m->wt->has_enc;
    const bool hmx = c.attention_type == SBK_ATT_HYPERMIX && m->wt->has_enc;
    const size_t Cu = bfm ? (size_t)c.csgu_linear_units : 0, Fu = std::max(F, Cu);  // f16 also holds the CSGU input u
    const int Bd = std::max(Be, rows);          // utterances whose encoder states the decoder sees
    const size_t Md = (size_t)Bd * T2;          // encoder states / cross K,V of those utterances
    take(b.wav, (size_t)B * L * 4); take(b.feats, (size_t)Be * T0 * c.n_mels * 4); take(b.x, M * d * 4);
    take(b.glu, M * d * 4); take(b.enc_out, Md * d * 4); take(b.dx, (size_t)rows * d * 4);
    take(b.logits, (size_t)rows * c.vocab * 4); take(b.score, (size_t)rows * S * 4);
    take(b.utt_max, B * 4); take(b.enc_len, (size_t)Bd * 4); take(b.tokens, (size_t)rows * (S + 1) * 4); take(b.step, rows * 4 + 64);
    take(b.has_ended, rows * 4); take(b.ended_count, 64); take(b.pred, (size_t)rows * S * 4); take(b.rel_len, B * 4);
    take(b.act1, (size_t)Be * T1 * F1 * c.cnn_c1 * 2); take(b.a_in, M * c.input_size * 2); take(b.h16, M * d * 2);
    take(b.f16, M * Fu * 2); take(b.qkv16, M * 3 * d * 2); take(b.att16, M * d * 2);
    take(b.P16, (size_t)T2 * d * 2); take(b.enc16, Md * d * 2); take(b.ckv16, Md * Ld * 2 * d * 2);
    take(b.kcache, (size_t)Ld * rows * S * d * 2); take(b.vcache, (size_t)Ld * rows * S * d * 2);
    // a folded cross-attention keeps its H d-wide queries in dq16 and its context vectors in df16
    const size_t Hd = m->wt->has_dec && m->wt->dec[0].w_xq ? (size_t)c.nhead * d : 0;
    take(b.dh16, (size_t)rows * d * 2); take(b.dq16, (size_t)rows * std::max(d, Hd) * 2); take(b.datt16, (size_t)rows * d * 2);
    take(b.df16, (size_t)rows * std::max(F, Hd) * 2);
    take(b.lineage, (size_t)2 * rows * S * 4); take(b.finished, B * 4 + 64); take(b.seq_scores, (size_t)2 * rows * 4);
    take(b.lnout, (size_t)rows * d * 4); take(b.beam_scr, (size_t)rows * 33 * 4);
    take(b.hist_tok, (size_t)rows * S * 4); take(b.hist_pred, (size_t)rows * S * 4);
    take(b.hist_score, (size_t)rows * S * 4); take(b.hist_lp, (size_t)rows * S * 4);
    if (m->wt->has_lm) {  // the residual stream at pitch lm_dp, queries / attention outputs / KV cache at lm_da
        const size_t dp = m->wt->lm_dp, da = m->wt->lm_da, Fl = c.lm_d_ffn, Ll = c.lm_layers;
        take(b.lx, rows * dp * 4); take(b.lh32, rows * dp * 4); take(b.lm_logits, (size_t)rows * c.vocab * 4);
        take(b.lm_extra, (size_t)rows * c.vocab * 4);
        take(b.lx16, rows * dp * 2); take(b.lq16, rows * da * 2); take(b.latt16, rows * da * 2);
        take(b.lf16, rows * Fl * 2); take(b.lh16, rows * dp * 2);
        take(b.lkc, Ll * rows * S * da * 2); take(b.lvc, Ll * rows * S * da * 2); take(b.tok_cache, (size_t)rows * S * 4);
    }
    if (bfm) {
        take(b.hc16, M * d * 2); take(b.cat16, M * 2 * d * 2); take(b.g16, M * Cu / 2 * 2);
        take(b.csgu_stats, M * 8);
    }
    if (hmx) {
        take(b.hm_part, hypermix_part_floats(Be, T2, c.d_model, c.d_ffn / c.nhead) * 4);
        take(b.hm_G, (size_t)Be * d * (F / c.nhead) * 2);
        take(b.hm_gscale, (size_t)Be * c.nhead * 4);
    }
}

// (Re)carve the workspace for at least the given shapes and the ones it is already carved for, so callers pass only what
// they need.  Be: utterances per encoder pass (0: B).
static int ensure_workspace(AsrModel* m, int B, int L, int rows, int steps, int Be = 0) {
    Be = std::max(Be, B);
    if (m->ws.base && B <= m->wsB && Be <= m->wsBe && L <= m->wsL && rows <= m->ws_rows && steps <= m->ws_steps) return SBK_OK;
    B = std::max(B, m->wsB); Be = std::max(Be, m->wsBe); L = std::max(L, m->wsL); rows = std::max(rows, m->ws_rows);
    steps = std::max(steps, m->ws_steps);
    Carver measure;
    workspace_layout(m, B, Be, L, rows, steps, m->b, measure);
    RC(grow_buffer(m, m->ws, measure.used + (1 << 20), "workspace"));
    drop_graphs(m);
    Carver carve{static_cast<uint8_t*>(m->ws.base)};
    workspace_layout(m, B, Be, L, rows, steps, m->b, carve);
    m->wsB = B; m->wsBe = Be; m->wsL = L; m->ws_rows = rows; m->ws_steps = steps;
    return SBK_OK;
}

// One chunk-by-chunk stream (or a batch of B streams advancing together) of a Conformer encoder: per layer the attention's
// left context as a ring of projected [k | v] rows (RoPE keys rotated by stream position) and the Dynamic Chunk
// Convolution's carry, the last (kernel_size - 1) / 2 depthwise-conv inputs.  The window of a chunk is [cached rows; chunk]:
// exactly the keys the masked full-sequence mode lets the chunk's frames see, so its outputs are the same.
struct AsrStream {
    int B = 0, chunk = 0, left = -1;  // left-context frames (-1: the whole past)
    int cap = 0;                      // ring rows per layer and stream (grows for an infinite left context)
    long long total = 0;              // frames encoded so far
    int clen = 0, start = 0;          // cached rows, ring slot of the oldest
    bool ended = false;               // a chunk shorter than `chunk` was seen: it must be the last
    int prow = 0;                     // RelPos: rows of P
    // StreamingFeatureWrapper's audio context: the last 2 * pad samples of each row's previous front-end window, kept in
    // two buffers that alternate (a chunk reads one and writes the other)
    int pad = 0;                      // samples of padding on each side of a window (0: the front end has not run)
    int fe_chunks = 0;                // front-end windows built since the last reset
    bool fe_ended = false;            // a window gave fewer than `chunk` frames: it must be the last
    DevBuf wav_carry;  // [2][B][2 * pad] fp32
    DevBuf kv;     // [L][B][cap][2d] fp16
    DevBuf carry;  // [L][B][halo][d] fp32
    DevBuf P;      // RelPos: [L][prow][d] fp16 = linear_pos(pe[r])
    DevBuf scr;    // inv_freq [dh/2] fp32 (RoPE), qkv [B*chunk, 3d] fp32, q [B*chunk, d] fp16
    const float* inv_freq = nullptr; float* qkv32 = nullptr; __half* q16 = nullptr;
    __half* kv_layer(const sbk_asr_config& c, int l) const {
        return static_cast<__half*>(kv.base) + (size_t)l * B * cap * 2 * c.d_model;
    }
    float* carry_layer(const sbk_asr_config& c, int l) const {
        return static_cast<float*>(carry.base) + (size_t)l * B * ((c.kernel_size - 1) / 2) * c.d_model;
    }
};

// RelPosMHAXL's positional projection of encoder layer l: P [rows, d] fp16 = linear_pos(pe[r]) for r < rows
static int relpos_project(const AsrModel* m, int l, int rows, __half* P, cudaStream_t st) {
    const int d = m->wt->cfg.d_model;
    GemmEpilogue e; e.mode = EPI_F16; e.out = P; e.ldo = d;
    return gemm_f16(m->wt->relpos_pe, d, m->wt->enc[l].wpos, d, e, rows, d, d, st);
}

// Self-attention of encoder layer l on its pre-norm b.h16 [B*T, d] fp16: the QKV projection, RoPEMHA, RelPosMHAXL or
// regularMHA attention over the whole sequence (DynChunkTrain windows when set) or, with s, over one stream chunk's window,
// then the output projection.  That adds to the residual stream b.x, or with cat16 set writes fp16 cat16[:, :d] (row stride
// 2d, the Branchformer's concatenation).
static int self_attention(AsrModel* m, int l, int B, int T, const int* enc_len, const AsrStream* s, __half* cat16,
                          cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const EncLayerW& w = m->wt->enc[l];
    const int M = B * T, d = c.d_model, H = c.nhead, dh = d / H;
    const bool rope = c.attention_type == SBK_ATT_ROPE, relpos = c.attention_type == SBK_ATT_RELPOS;
    // nnet/attention.py:521,1272: 1/sqrt(embed_dim), not head_dim; regularMHA's 1/sqrt(d_h) is folded into the query rows of
    // wqkv / bqkv
    const float att_scale = c.attention_type == SBK_ATT_REGULAR ? 1.0f : 1.0f / sqrtf((float)d);
    GemmEpilogue e;
    e.bias = w.bqkv; e.ldo = 3 * d;
    if (s) {  // the chunk's q and its [k | v] rows in the ring, then attention over [cached rows; chunk]
        __half* kv = s->kv_layer(c, l);
        e.mode = EPI_F32; e.out = s->qkv32;
        RC(gemm_f16(b.h16, d, w.wqkv, d, e, M, 3 * d, d, st));
        RC(stream_qkv(s->qkv32, B, T, H, dh, rope ? s->inv_freq : nullptr, s->total, att_scale, s->q16, kv, s->cap,
                      (s->start + s->clen) % s->cap, st));
        AttStream sa;
        sa.q = s->q16; sa.ldq = d; sa.kv = kv; sa.ldkv = 2 * d; sa.cap = s->cap; sa.start = s->start; sa.nq = T;
        RC(encoder_attention_stream(sa, B, s->clen + T, H, dh, relpos, w.pos_u, w.pos_v,
                                    relpos ? static_cast<const __half*>(s->P.base) + (size_t)l * s->prow * d : nullptr, d,
                                    att_scale, b.att16, d, st));
    } else {
        e.out = b.qkv16;
        if (rope) {
            e.mode = EPI_ROPE; e.alpha = att_scale; e.T = T; e.rope_cos = m->wt->rope_cos; e.rope_sin = m->wt->rope_sin; e.head_dim = dh;
        } else {
            e.mode = EPI_F16;
        }
        RC(gemm_f16(b.h16, d, w.wqkv, d, e, M, 3 * d, d, st));
        if (relpos) RC(relpos_project(m, l, T, b.P16, st));
        RC(encoder_attention(b.qkv16, 3 * d, B, T, H, dh, enc_len, relpos, w.pos_u, w.pos_v, b.P16, d, att_scale, b.att16, d,
                             st, m->dyn_chunk, m->dyn_left));
    }
    e = GemmEpilogue(); e.bias = w.bo;
    if (cat16) {
        e.mode = EPI_F16; e.out = cat16; e.ldo = 2 * d;
    } else {
        e.mode = EPI_RESID; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 1.0f;
    }
    return gemm_f16(b.att16, d, w.wo, d, e, M, d, d, st);
}

// A feed-forward module on its pre-norm b.h16 [M, d] fp16: x += alpha * (act(h16 W1^T + b1) W2^T + b2), the hidden layer in
// b.f16 [M, d_ffn]
static int feed_forward(AsrModel* m, const __half* W1, const float* b1, const __half* W2, const float* b2, int act, float alpha,
                        int M, cudaStream_t st) {
    const int d = m->wt->cfg.d_model, F = m->wt->cfg.d_ffn;
    GemmEpilogue e;
    e.mode = EPI_F16; e.act = act; e.bias = b1; e.out = m->b.f16; e.ldo = F;
    RC(gemm_f16(m->b.h16, d, W1, d, e, M, F, d, st));
    e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = b2; e.out = m->b.x; e.resid = m->b.x; e.ldo = d; e.alpha = alpha;
    return gemm_f16(m->b.f16, F, W2, F, e, M, d, F, st);
}

// Branchformer layers (Branchformer.py:92-234, 330-410) on the fp32 residual stream b.x [B*T, d]:
//     x1 = RelPosMHAXL(norm_mhsa(x));  x2 = post_channel_proj(CSGU(act(pre_channel_proj(norm_conv(x)))))
//     x  = x + merge_proj(cat[x1, x2])
// Neither branch masks padded frames (the attention masks padded keys only).  x1 and x2 are written into the two column
// halves of one [B*T, 2d] fp16 buffer so that merge_proj is one K = 2d GEMM with the residual epilogue.
static int run_branchformer_layers(AsrModel* m, int B, int T, const int* enc_len, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int M = B * T, d = c.d_model, C = c.csgu_linear_units;
    const int act = c.branchformer_activation == SBK_ACT_RELU ? ACT_RELU : ACT_GELU;
    GemmEpilogue e;
    for (int l = 0; l < c.num_encoder_layers; ++l) {
        const EncLayerW& w = m->wt->enc[l];
        RC(layernorm_rows_dual(b.x, b.h16, w.norm1_g, w.norm1_b, b.hc16, w.nconv_g, w.nconv_b, M, d, 1e-5f, st));
        // --- attention branch -> cat16[:, :d]
        RC(self_attention(m, l, B, T, enc_len, nullptr, b.cat16, st));
        // --- convolution branch -> cat16[:, d:]
        e = GemmEpilogue(); e.mode = EPI_F16; e.act = act; e.bias = w.bpre; e.out = b.f16; e.ldo = C;
        RC(gemm_f16(b.hc16, d, w.wpre, d, e, M, C, d, st));
        RC(csgu_forward(b.f16, B, T, C, w.csgu_ln_g, w.csgu_ln_b, 1e-5f, w.csgu_taps, w.csgu_bias, c.kernel_size, b.csgu_stats,
                        b.g16, st));
        e = GemmEpilogue(); e.mode = EPI_F16; e.bias = w.bpost; e.out = b.cat16 + d; e.ldo = 2 * d;
        RC(gemm_f16(b.g16, C / 2, w.wpost, C / 2, e, M, d, C / 2, st));
        // --- x += merge_proj(cat[x1, x2]): every row, padded frames included
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.bmerge; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 1.0f;
        RC(gemm_f16(b.cat16, 2 * d, w.wmerge, 2 * d, e, M, d, 2 * d, st));
    }
    return SBK_OK;
}

// x [B*T, d] += pe[t]: TransformerASR.encode adds the absolute sine table to the input Linear's output (TransformerASR.py:519)
__global__ void add_pos_table_kernel(float* __restrict__ x, const float* __restrict__ pe, int T, int d, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] += pe[(i / d) % T * d + i % d];
}

// Transformer layers (Transformer.py:311-490, normalize_before=True, regularMHA, Linear + GELU + Linear) on the fp32
// residual stream b.x [B*T, d]:
//     x = x + out_proj(MHA(norm1(x)));  x = x + ffn(norm2(x))
// The attention masks padded keys only (make_transformer_src_tgt_masks), so padded frames are computed like the reference.
static int run_transformer_layers(AsrModel* m, int B, int T, const int* enc_len, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int M = B * T, d = c.d_model;
    const size_t n = (size_t)M * d;
    add_pos_table_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(b.x, m->wt->enc_pe, T, d, n);
    SBK_LAUNCH_CHECK();
    for (int l = 0; l < c.num_encoder_layers; ++l) {
        const EncLayerW& w = m->wt->enc[l];
        RC(layernorm_rows(b.x, b.h16, true, w.norm1_g, w.norm1_b, M, d, 1e-6f, st));
        RC(self_attention(m, l, B, T, enc_len, nullptr, nullptr, st));
        RC(layernorm_rows(b.x, b.h16, true, w.norm2_g, w.norm2_b, M, d, 1e-6f, st));
        RC(feed_forward(m, w.ffn1_w1, w.ffn1_b1, w.ffn1_w2, w.ffn1_b2, ACT_GELU, 1.0f, M, st));
    }
    return SBK_OK;
}

// Conformer layers (Conformer.py:472-500) on the fp32 residual stream b.x [B*T, d]; the last layer's norm2 runs fused with
// the encoder's final LayerNorm into enc_out.  s: one chunk of a stream (attention over s's window, the conv over its carry).
static int run_conformer_layers(AsrModel* m, int B, int T, const int* enc_len, float* enc_out, cudaStream_t st,
                                const AsrStream* s) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int M = B * T, d = c.d_model, F = c.d_ffn, H = c.nhead;
    // conformer_activation: both FFN modules' hidden activation and the convolution module's after the LayerNorm
    const bool gelu = c.conformer_activation == SBK_CONFORMER_ACT_GELU;
    const int ffn_act = gelu ? ACT_GELU : ACT_SILU;
    GemmEpilogue e;
    for (int l = 0; l < c.num_encoder_layers; ++l) {
        const EncLayerW& w = m->wt->enc[l];
        // --- ffn module 1 (Conformer.py:479); its LayerNorm was fused into the previous layer's norm2 kernel
        if (l == 0) RC(layernorm_rows(b.x, b.h16, true, w.ffn1_ln_g, w.ffn1_ln_b, M, d, 1e-5f, st));
        RC(feed_forward(m, w.ffn1_w1, w.ffn1_b1, w.ffn1_w2, w.ffn1_b2, ffn_act, 0.5f, M, st));
        // --- self-attention (Conformer.py:481-492)
        RC(layernorm_rows(b.x, b.h16, true, w.norm1_g, w.norm1_b, M, d, 1e-5f, st));
        if (c.attention_type == SBK_ATT_HYPERMIX)  // x += HyperMixing(norm1(x)) (hypermixing.py:90-195)
            RC(hypermix_forward(b.h16, B, T, d, H, F / H, enc_len, m->wt->hm_pe, w.hm, b.hm_part, b.hm_G, b.hm_gscale, b.x, st));
        else
            RC(self_attention(m, l, B, T, enc_len, s, nullptr, st));
        // --- convolution module (Conformer.py:314-330, 494)
        RC(layernorm_rows(b.x, b.h16, true, w.conv_ln_g, w.conv_ln_b, M, d, 1e-5f, st));
        e = GemmEpilogue(); e.mode = EPI_GLU; e.bias = w.bpw1; e.out = b.glu; e.ldo = d;
        RC(gemm_f16(b.h16, d, w.wpw1, d, e, M, 2 * d, d, st));
        if (s) {  // the chunk after the carry, zeros after the chunk (its right edge); then the carry moves on
            float* carry = s->carry_layer(c, l);
            RC(dwconv_ln_act(b.glu, B, T, d, c.kernel_size, w.wdw, w.bdw, w.aconv_ln_g, w.aconv_ln_b, 1e-5f, b.h16, st, gelu, 0,
                             s->total > 0 ? carry : nullptr));
            RC(dwconv_carry(b.glu, B, T, d, c.kernel_size, s->total > 0, carry, st));
        } else {
            RC(dwconv_ln_act(b.glu, B, T, d, c.kernel_size, w.wdw, w.bdw, w.aconv_ln_g, w.aconv_ln_b, 1e-5f, b.h16, st, gelu,
                             m->dyn_chunk));
        }
        e = GemmEpilogue(); e.mode = EPI_RESID; e.bias = w.bpw2; e.out = b.x; e.resid = b.x; e.ldo = d; e.alpha = 1.0f;
        e.row_lens = enc_len; e.T = T;
        RC(gemm_f16(b.h16, d, w.wpw2, d, e, M, d, d, st));
        // --- ffn module 2 + norm2 (Conformer.py:498)
        RC(layernorm_rows(b.x, b.h16, true, w.ffn2_ln_g, w.ffn2_ln_b, M, d, 1e-5f, st));
        RC(feed_forward(m, w.ffn2_w1, w.ffn2_b1, w.ffn2_w2, w.ffn2_b2, ffn_act, 0.5f, M, st));
        if (l + 1 < c.num_encoder_layers) {  // norm2 (fp32 residual stream) + the next layer's ffn1 LayerNorm (fp16 operand)
            const EncLayerW& nx = m->wt->enc[l + 1];
            RC(layernorm2_rows(b.x, b.x, b.h16, true, w.norm2_g, w.norm2_b, 1e-5f, nx.ffn1_ln_g, nx.ffn1_ln_b, 1e-5f, M, d, st));
        } else {                             // norm2 + the encoder's final LayerNorm (Conformer.py:700)
            RC(layernorm2_rows(b.x, nullptr, enc_out, false, w.norm2_g, w.norm2_b, 1e-5f, m->wt->enc_norm_g, m->wt->enc_norm_b, 1e-6f, M,
                               d, st));
        }
    }
    return SBK_OK;
}

// The fused front-end of the configured ConvolutionFrontEnd: feats [B, T0, n_mels] -> b.a_in [B*T2, input_size] fp16
// (+ cnn_out_f fp32 when set).
static int run_cnn(AsrModel* m, const float* feats, int B, int T0, float* cnn_out_f, cudaStream_t st) {
    return cnn_frontend_forward(feats, B, T0, m->wt->cfg.n_mels, m->wt->cnn, m->b.act1, m->b.a_in, cnn_out_f, st);
}

// feats [B, T0, n_mels] fp32 (already normalised) -> enc_out fp32 [B, T2, d] (+ enc16). enc_len device int[B].
// s: one chunk of a stream (T0 = the chunk's frames, feats null): attention over s's window, the conv over its carry.
static int run_encoder(AsrModel* m, const float* feats, int B, int T0, const int* enc_len, float* cnn_out_f,
                       float* enc_out, cudaStream_t st, const AsrStream* s = nullptr) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int T1 = (T0 - 1) / 2 + 1, T = feats ? (T1 - 1) / 2 + 1 : T0;  // feats == nullptr: b.a_in holds [B*T0, input_size]
    // row counts are int (offsets into the activations are size_t); the CNN, attention and conv kernels launch one grid row
    // or layer per utterance
    SBK_REQUIRE(B <= 65535 && (long long)B * T0 <= INT_MAX, "encode: %d utterances of %d frames exceed the kernels' index range",
                B, T0);
    const int M = B * T, d = c.d_model;
    SBK_REQUIRE(m->wt->has_enc, "encode: this handle was created without encoder weights");
    SBK_REQUIRE(feats == nullptr || m->wt->has_cnn, "encode: this handle was created without CNN weights");
    if (c.attention_type == SBK_ATT_HYPERMIX)  // HyperMixing adds its own 3000-row table: longer inputs fail in the reference
        SBK_REQUIRE(T <= HM_PE_ROWS, "encode: %d frames exceed HyperMixing's %d-row positional table", T, HM_PE_ROWS);
    else
        SBK_REQUIRE(T <= m->wt->pos_len, "encode: %d frames exceed max_len=%d", T, m->wt->pos_len);
    SBK_REQUIRE(c.attention_type != SBK_ATT_HYPERMIX || m->dyn_chunk == 0,
                "encode: HyperMixing has no chunked (DynChunkTrainConfig) mode");
    SBK_REQUIRE(c.encoder_module != SBK_ENC_BRANCHFORMER || T > (c.kernel_size - 1) / 2,
                "encode: the Branchformer's reflect-padded conv needs more than %d frames (got %d)", (c.kernel_size - 1) / 2, T);
    SBK_REQUIRE(c.encoder_module != SBK_ENC_BRANCHFORMER || m->dyn_chunk == 0,
                "encode: the Branchformer has no chunked (DynChunkTrainConfig) mode");
    SBK_REQUIRE(c.encoder_module != SBK_ENC_TRANSFORMER || m->dyn_chunk == 0,
                "encode: the Transformer encoder has no chunked (DynChunkTrainConfig) mode");
    if (feats != nullptr) RC(run_cnn(m, feats, B, T0, cnn_out_f, st));
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->wt->b_in; e.out = b.x; e.ldo = d;
    RC(gemm_f16(b.a_in, c.input_size, m->wt->w_in, c.input_size, e, M, d, c.input_size, st));
    if (c.encoder_module == SBK_ENC_BRANCHFORMER) RC(run_branchformer_layers(m, B, T, enc_len, st));
    else if (c.encoder_module == SBK_ENC_TRANSFORMER) RC(run_transformer_layers(m, B, T, enc_len, st));
    else RC(run_conformer_layers(m, B, T, enc_len, enc_out, st, s));
    // encoder.norm, unless a Conformer layer ran it with its norm2
    if (c.encoder_module != SBK_ENC_CONFORMER || c.num_encoder_layers == 0)
        RC(layernorm_rows(b.x, enc_out, false, m->wt->enc_norm_g, m->wt->enc_norm_b, M, d, 1e-6f, st));
    return SBK_OK;
}

__global__ void abs_len_kernel(const float* rel, int B, int T, int* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    // torch.round (half to even) of rel * T   (TransformerASR.py:148, seq2seq.py:206)
    if (i < B) out[i] = min(T, max(0, __float2int_rn(rel[i] * static_cast<float>(T))));
}

// enc_len [B] = round(rel_len * T), or T for every utterance when rel_len is null
static int set_enc_len(int* enc_len, const float* rel_len, int B, int T, cudaStream_t st) {
    if (rel_len) {
        abs_len_kernel<<<ceil_div(B, 128), 128, 0, st>>>(rel_len, B, T, enc_len);
        SBK_LAUNCH_CHECK();
        return SBK_OK;
    }
    std::vector<int> full(B, T);
    SBK_CUDA_CHECK(cudaMemcpyAsync(enc_len, full.data(), B * 4, cudaMemcpyHostToDevice, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));  // before `full` goes out of scope
    return SBK_OK;
}

// Copies a caller's encoder states enc [n, T, d] fp32 into b.enc_out, where the decoders and the CTC head read them.
static int stage_enc(AsrModel* m, const float* enc, int n, int T, cudaStream_t st) {
    SBK_CUDA_CHECK(cudaMemcpyAsync(m->b.enc_out, enc, (size_t)n * T * m->wt->cfg.d_model * 4, cudaMemcpyDeviceToDevice, st));
    return SBK_OK;
}

// Copies the first `steps` columns of a [rows, S_max] per-step workspace array (b.pred, b.score) into dst [rows, ld];
// nothing when dst is null.
static int copy_steps(const AsrModel* m, void* dst, int ld, const void* src, int steps, int rows, cudaMemcpyKind kind,
                      cudaStream_t st) {
    const size_t S_max = m->ws_steps + 1;
    if (dst) SBK_CUDA_CHECK(cudaMemcpy2DAsync(dst, (size_t)ld * 4, src, S_max * 4, (size_t)steps * 4, rows, kind, st));
    return SBK_OK;
}

// Cross-attention K/V of every decoder layer, projected once per utterance from the encoder states (b.enc16).  At head
// width 64 and d_model a multiple of 256 the layout per layer is [K | V] parts, each [utt][head][T][64] -- the decode-step
// attention of (utterance, head) then streams one contiguous T x 128 B block of K and one of V instead of 128-byte pieces
// 2 KB apart.  Every other shape keeps [utt * T][K(d) | V(d)] rows.
static bool xatt_headmajor(const AsrModel* m) {
    return m->wt->cfg.d_model / m->wt->cfg.nhead == 64 && m->wt->cfg.d_model % 256 == 0;
}
// A folded call (xatt_fold) attends over enc16 itself and needs no K/V.
static int project_cross_kv(AsrModel* m, int M, int T, bool fold, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, Ld = c.num_decoder_layers;
    RC(cast_f32_f16(b.enc_out, b.enc16, (size_t)M * d, st));
    if (fold) return SBK_OK;
    if (xatt_headmajor(m)) {  // w_ckv / b_ckv are [Ld * 2d] rows: every layer's K and V in ONE GEMM, scattered per layer
        GemmEpilogue e;
        e.mode = EPI_F16; e.bias = m->wt->b_ckv; e.out = b.ckv16; e.ldo = Ld * 2 * d;
        e.kv_heads = c.nhead; e.kv_part_stride = (size_t)M * d; e.kv_layer_stride = (size_t)M * 2 * d; e.T = T;
        return gemm_f16(b.enc16, d, m->wt->w_ckv, d, e, M, Ld * 2 * d, d, st);
    }
    for (int l = 0; l < Ld; ++l) {
        GemmEpilogue e;
        e.mode = EPI_F16; e.bias = m->wt->b_ckv + (size_t)l * 2 * d; e.out = b.ckv16 + (size_t)l * M * 2 * d; e.ldo = 2 * d;
        RC(gemm_f16(b.enc16, d, m->wt->w_ckv + (size_t)l * 2 * d * d, d, e, M, 2 * d, d, st));
    }
    return SBK_OK;
}
// fills the K/V addressing of a cross-attention call for layer l
static void cross_kv_args(const AsrModel* m, DecAttnArgs& t, int l, int n_utt, int T) {
    const int d = m->wt->cfg.d_model;
    const size_t M = (size_t)n_utt * T;
    t.kbase = m->b.ckv16 + (size_t)l * M * 2 * d;
    if (xatt_headmajor(m)) {
        t.vbase = t.kbase + M * d; t.row_stride = (size_t)T * d; t.head_stride = T * 64; t.key_stride = 64;
    } else {
        t.vbase = t.kbase + d; t.row_stride = (size_t)T * 2 * d; t.head_stride = 0; t.key_stride = 2 * d;
    }
}

// ---------------------------------------------------------------------------- decode / TransformerLM step projections
// The GEMM that runs a step's Linears.  The weight-streaming kernel (skinny_gemm) suits few live rows, but its cost grows
// with every 32 rows; from dec_tc_rows rows on (several batches decoded together, or a wide beam) the wgmma GEMM
// (gemm_f16_small: 64 x 32/64 tiles, a handful of CTAs each, so concurrent lanes share the GPU) takes over.  The
// whole-sequence LM runs on the encoder's GEMM (gemm_f16).  Same maths on all three: fp16 operands, fp32 accumulate /
// residual.
enum StepGemm { SG_STREAM, SG_SMALL, SG_WIDE };

// The back end of a step over `rows` live rows of width `width` (the wgmma QKV -> cache scatter epilogue works on 32-column
// chunks).
static StepGemm step_gemm(const AsrModel* m, int rows, int width) {
    return rows >= m->dec_tc_rows && width % 32 == 0 ? SG_SMALL : SG_STREAM;
}
// Whether a decode call over n_utt utterances of T frames, one row each (greedy and teacher-forced decoding), runs the folded
// cross-attention (dec_xatt_fold): each layer then streams the fp16 encoder states, 2 d bytes per frame, instead of its
// cross-attention K and V, 4 d bytes per frame, and its query and output projections grow from d x d to H d x d weights;
// the call also skips the K/V GEMM over all encoder frames.  By bytes alone the step would gain from n_utt T = 2 (H - 1) d
// frames on, but the two grown projections cost far more than their extra weight bytes (H100 SXM at 700 W, 224 rows, d 512,
// 8 heads: N = 4096 query projection 8 us, K = 4096 output projection 13 us, against 4 us each at d x d).  A folded
// Conformer-L step at T = 251 measured +45 / +58 / +7 / -6 us against the K/V path at 64 / 96 / 160 / 224 live rows,
// while the skipped K/V GEMM (6.3 MFLOP per frame) saves about 4.3 us per utterance once per call (at 370 TFLOP/s).
// Over a 48-step call that crosses over near 150 utterances: the fold starts at n_utt T >= 11 (H - 1) d (39424 frames
// for Conformer-L, 157 utterances of 10 s; DESIGN.md section 9), so 96 rows keep the K/V path and 160 rows fold.  Only
// on the wgmma step back end, and only for decoders packed with folded weights (xatt_foldable).  Beam search keeps the K/V path: several
// rows share an utterance's keys there, and the coverage scorer reads the last layer's K.
static bool xatt_fold(const AsrModel* m, int n_utt, int T) {
    const sbk_asr_config& c = m->wt->cfg;
    return m->wt->dec[0].w_xq != nullptr && step_gemm(m, n_utt, c.d_model) == SG_SMALL &&
           (size_t)n_utt * T >= (size_t)11 * (c.nhead - 1) * c.d_model;
}
// Programmatic dependent launch is on for the wgmma step (its GEMMs and LayerNorms are launched with it unconditionally)
// and off for weight streaming, where it measured no faster (single_batch, H100 SXM at 400 W: 24.8 / 28.2 ms with it
// against 23.4 / 23.3 ms without).  Every entry that runs a step loop sets it before the loop.
static void set_step_pdl(const AsrModel* m, int rows, int width) { set_pdl(step_gemm(m, rows, width) == SG_SMALL); }

// What a step's Linear writes: fp16 (optionally through GELU / ReLU / SiLU), fp32, fp32 added in place to `out` (the
// residual stream), or the self-attention in_proj's [q | k | v]: q to `out`, k and v into the caches at (row, step_ptr[row]).
// (sbk_step_proj_test takes the codes up to PO_QKV_CACHE.)
enum ProjOut { PO_F16, PO_F16_GELU, PO_F16_RELU, PO_F32, PO_RESID, PO_QKV_CACHE, PO_F16_SILU };
// One Linear of a step: out[rows, N] (row stride ldo) = epilogue(A[rows, K] (row stride lda) x W[N, K]^T + bias).
struct Proj {
    const __half* W; const float* bias; int N, K;
    ProjOut kind; void* out; int ldo;
    const __half* A = nullptr; int lda = 0;
    __half* kcache = nullptr; __half* vcache = nullptr; const int* step_ptr = nullptr; int S_max = 0;  // PO_QKV_CACHE
    const float* X = nullptr; const float* ln_g = nullptr; const float* ln_b = nullptr;  // SG_STREAM: A = LayerNorm(X) in-kernel
};

static int project(StepGemm g, const Proj& p, int rows, cudaStream_t st) {
    if (g == SG_STREAM) {
        static const int skinny_epi[] = {SK_F16, SK_F16_GELU, SK_F16_RELU, SK_F32, SK_RESID, SK_QKV_CACHE, SK_F16_SILU};
        SkinnyArgs a{};
        a.A = p.A; a.lda = p.lda; a.W = p.W; a.ldw = p.K; a.bias = p.bias; a.n_rows = rows; a.N = p.N; a.K = p.K;
        a.epi = skinny_epi[p.kind]; a.out = p.out; a.ldo = p.ldo;
        if (p.kind == PO_QKV_CACHE) {
            a.kcache = p.kcache; a.vcache = p.vcache; a.step_ptr = p.step_ptr; a.S_max = p.S_max; a.d = p.N / 3; a.q_scale = 1.0f;
        }
        if (p.X) { a.X = p.X; a.ln_g = p.ln_g; a.ln_b = p.ln_b; a.ln_eps = 1e-6f; }
        return skinny_gemm(a, st);
    }
    GemmEpilogue e;
    e.mode = p.kind == PO_F32 ? EPI_F32 : p.kind == PO_RESID ? EPI_RESID : p.kind == PO_QKV_CACHE ? EPI_QKV_CACHE : EPI_F16;
    e.act = p.kind == PO_F16_GELU ? ACT_GELU : p.kind == PO_F16_RELU ? ACT_RELU : p.kind == PO_F16_SILU ? ACT_SILU : ACT_NONE;
    e.bias = p.bias; e.out = p.out; e.ldo = p.ldo;
    if (p.kind == PO_RESID) e.resid = static_cast<const float*>(p.out);
    if (p.kind == PO_QKV_CACHE) {
        e.kcache = p.kcache; e.vcache = p.vcache; e.step_ptr = p.step_ptr; e.S_max = p.S_max; e.qkv_d = p.N / 3;
    }
    if (g == SG_SMALL) return gemm_f16_small(p.A, p.lda, p.W, p.K, e, rows, p.N, p.K, st);
    return gemm_f16(p.A, p.lda, p.W, p.K, e, rows, p.N, p.K, st);
}

// A decoder pre-norm LN(x) (x fp32 [rows, p.K], eps 1e-6) and the projection it feeds.  Weight streaming fuses the LayerNorm
// into the projection kernel where that kernel is built for the width, which saves a launch per projection (single-batch
// latency); with fusion off it runs a separate kernel into h16 [rows, p.K], which avoids recomputing the same 32-row LayerNorm
// in ~100-300 CTAs (GPU time when several batches are in flight).  The wgmma step always runs the separate kernel, launched
// with PDL.
static int norm_project(StepGemm g, bool fuse_ln, Proj p, const float* x, const float* gamma, const float* beta, __half* h16,
                        int rows, cudaStream_t st) {
    const int d = p.K;
    if (g == SG_STREAM && fuse_ln && (d == 256 || d == 512 || d == 768 || d == 1024)) {
        p.X = x; p.ln_g = gamma; p.ln_b = beta;
    } else {
        RC(layernorm_rows(x, h16, true, gamma, beta, rows, d, 1e-6f, st, g != SG_STREAM));
        p.A = h16; p.lda = d;
    }
    return project(g, p, rows, st);
}
static int dec_norm_project(AsrModel* m, StepGemm g, Proj p, const float* gamma, const float* beta, int rows, cudaStream_t st) {
    return norm_project(g, m->fuse_dec_ln, p, m->b.dx, gamma, beta, m->b.dh16, rows, st);
}

static int enqueue_decode_layers(AsrModel* m, int rows, int rows_per_utt, int T, int S_max, const int* lineage, bool fold,
                                 cudaStream_t st, bool with_head = true) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, F = c.d_ffn, H = c.nhead, dh = d / H, Ld = c.num_decoder_layers;
    const ProjOut ffn_act = c.decoder_activation == SBK_ACT_GELU   ? PO_F16_GELU
                            : c.decoder_activation == SBK_ACT_SILU ? PO_F16_SILU
                                                                   : PO_F16_RELU;
    const int n_utt = rows / rows_per_utt;
    const StepGemm g = step_gemm(m, rows, d);
    // b.dx already holds emb[token] * sqrt(d) + pe[step] (written by greedy_reset / the previous greedy_select)
    for (int l = 0; l < Ld; ++l) {
        const DecLayerW& w = m->wt->dec[l];
        __half* kc = b.kcache + (size_t)l * rows * S_max * d;
        __half* vc = b.vcache + (size_t)l * rows * S_max * d;
        Proj qkv{w.w_self_in, w.b_self_in, 3 * d, d, PO_QKV_CACHE, b.dq16, d};  // LN1 + self-attention in_proj
        qkv.kcache = kc; qkv.vcache = vc; qkv.step_ptr = b.step; qkv.S_max = S_max;
        RC(dec_norm_project(m, g, qkv, w.n1g, w.n1b, rows, st));
        DecAttnArgs t{};
        t.q = b.dq16; t.ldq = d; t.kbase = kc; t.vbase = vc; t.row_stride = (size_t)S_max * d; t.key_stride = d;
        t.rows_per_block = 1; t.n_keys_ptr = b.step; t.enc_len = nullptr; t.H = H; t.dh = dh; t.out = b.datt16; t.ldo = d;
        t.lineage = lineage; t.lin_stride = S_max;
        RC(dec_attention(t, rows, S_max, st));
        RC(project(g, {w.w_self_out, w.b_self_out, d, d, PO_RESID, b.dx, d, b.datt16, d}, rows, st));
        if (fold) {  // LN2 + folded query projection, attention over enc16, folded output projection (rows_per_utt == 1)
            const int Hd = H * d;
            RC(dec_norm_project(m, g, {w.w_xq, w.b_xq, Hd, d, PO_F16, b.dq16, Hd}, w.n2g, w.n2b, rows, st));
            XattFoldArgs x{b.dq16, Hd, b.enc16, b.enc_len, T, H, d, b.df16, Hd};
            RC(dec_xatt_fold(x, rows, st));
            RC(project(g, {w.w_xo, w.b_xo, d, Hd, PO_RESID, b.dx, d, b.df16, Hd}, rows, st));
        } else {
            // cross attention: LN2 + (pre-scaled) query projection
            RC(dec_norm_project(m, g, {w.w_cross_q, w.b_cross_q, d, d, PO_F16, b.dq16, d}, w.n2g, w.n2b, rows, st));
            t = DecAttnArgs{};
            t.q = b.dq16; t.ldq = d; cross_kv_args(m, t, l, n_utt, T); t.rows_per_block = rows_per_utt;
            t.n_keys_ptr = nullptr; t.enc_len = b.enc_len; t.H = H; t.dh = dh; t.out = b.datt16; t.ldo = d;
            RC(dec_attention(t, rows, T, st));
            RC(project(g, {w.w_cross_out, w.b_cross_out, d, d, PO_RESID, b.dx, d, b.datt16, d}, rows, st));
        }
        // feed-forward: LN3 + ffn1 + activation, then ffn2 + residual
        RC(dec_norm_project(m, g, {w.w_ffn1, w.b_ffn1, F, d, ffn_act, b.df16, F}, w.n3g, w.n3b, rows, st));
        RC(project(g, {w.w_ffn2, w.b_ffn2, d, F, PO_RESID, b.dx, d, b.df16, F}, rows, st));
    }
    if (!with_head) return SBK_OK;
    SBK_REQUIRE(m->wt->w_lin != nullptr, "decode step: this handle was created without the output head (seq_lin.w.*)");
    return dec_norm_project(m, g, {m->wt->w_lin, m->wt->b_lin, c.vocab, d, PO_F32, b.logits, c.vocab}, m->wt->dec_norm_g,
                            m->wt->dec_norm_b, rows, st);  // final LayerNorm + seq_lin
}

static int enqueue_decode_step(AsrModel* m, int rows, int T, int S_max, bool fold, int eos, float* log_probs, int L_lp,
                               cudaStream_t st) {
    AsrModel::Buf& b = m->b;
    RC(enqueue_decode_layers(m, rows, 1, T, S_max, nullptr, fold, st));
    RC(greedy_select(b.logits, rows, m->wt->cfg.vocab, b.step, eos, b.tokens, S_max + 1, b.has_ended, b.ended_count, b.pred,
                     b.score, S_max, log_probs, L_lp, m->wt->emb, m->wt->dec_pe, m->wt->cfg.d_model, b.dx, st));
    return SBK_OK;
}

// A post-norm TransformerLM layer after its self-attention (Transformer.py:466-481): x = norm1(x + out_proj(att)), then
// x = norm2(x + ffn(x)).  x is the fp32 residual stream [rows, lm_dp] and x16 its fp16 copy, att16 [rows, lm_da]; f16
// [rows, d_ffn] is scratch.  The LayerNorms take their statistics over the d_model real channels and write zero padding.
static int lm_layer_tail(const AsrModel* m, StepGemm g, const LmLayerW& w, int rows, const __half* att16, float* x,
                         __half* x16, __half* f16, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    const int dl = c.lm_d_model, dp = m->wt->lm_dp, da = m->wt->lm_da, Fl = c.lm_d_ffn;
    const ProjOut act = c.lm_activation == SBK_ACT_GELU ? PO_F16_GELU : PO_F16_RELU;
    RC(project(g, {w.w_out, w.b_out, dp, da, PO_RESID, x, dp, att16, da}, rows, st));
    RC(layernorm_dual(x, x16, w.n1g, w.n1b, rows, dl, dp, 1e-6f, true, st));
    RC(project(g, {w.w1, w.b1, Fl, dp, act, f16, Fl, x16, dp}, rows, st));
    RC(project(g, {w.w2, w.b2, dp, Fl, PO_RESID, x, dp, f16, Fl}, rows, st));
    return layernorm_dual(x, x16, w.n2g, w.n2b, rows, dl, dp, 1e-6f, true, st);
}

// The LM's encoder.norm, then output_proj: Linear d -> d (fp32 into h32), LayerNorm (fp16 into h16), Linear d -> vocab
// (fp32 into logits).
static int lm_output(const AsrModel* m, StepGemm g, int rows, float* x, __half* x16, float* h32, __half* h16, float* logits,
                     cudaStream_t st) {
    const AsrWeights& W = *m->wt;
    const int dl = W.cfg.lm_d_model, dp = W.lm_dp, V = W.cfg.vocab;
    RC(layernorm_dual(x, x16, W.lm_norm_g, W.lm_norm_b, rows, dl, dp, 1e-6f, false, st));
    RC(project(g, {W.lm_wp0, W.lm_bp0, dp, dp, PO_F32, h32, dp, x16, dp}, rows, st));
    RC(layernorm_dual(h32, h16, W.lm_lnp_g, W.lm_lnp_b, rows, dl, dp, 1e-6f, false, st));
    return project(g, {W.lm_wp2, W.lm_bp2, V, dp, PO_F32, logits, V, h16, dp}, rows, st);
}

// One TransformerLM step over `rows` hypotheses (post-norm encoder layers with a lineage-indexed KV cache), ending in
// b.lm_extra[rows, V] = weight * log_softmax(lm_logits / temperature): TransformerLMScorer.score (scorer.py:510-543)
// scaled by ScorerBuilder's weight.  b.lx / b.lx16 hold emb[token] * scale + pe[step] (beam_reset / beam_step).
static int enqueue_lm_step(AsrModel* m, int rows, int S_max, float temperature, float weight, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int dp = m->wt->lm_dp, da = m->wt->lm_da, H = c.lm_nhead;
    const StepGemm g = step_gemm(m, rows, da);
    for (int l = 0; l < c.lm_layers; ++l) {
        const LmLayerW& w = m->wt->lm[l];
        __half* kc = b.lkc + (size_t)l * rows * S_max * da;
        __half* vc = b.lvc + (size_t)l * rows * S_max * da;
        Proj qkv{w.w_in, w.b_in, 3 * da, dp, PO_QKV_CACHE, b.lq16, da, b.lx16, dp};
        qkv.kcache = kc; qkv.vcache = vc; qkv.step_ptr = b.step; qkv.S_max = S_max;
        RC(project(g, qkv, rows, st));
        DecAttnArgs t{};
        t.q = b.lq16; t.ldq = da; t.kbase = kc; t.vbase = vc; t.row_stride = (size_t)S_max * da; t.key_stride = da;
        t.rows_per_block = 1; t.n_keys_ptr = b.step; t.H = H; t.dh = m->wt->lm_dhp; t.out = b.latt16; t.ldo = da;
        t.lineage = b.lineage; t.lin_stride = S_max; t.tok_cache = b.tok_cache; t.pad_tok = 0;
        RC(dec_attention(t, rows, S_max, st));
        RC(lm_layer_tail(m, g, w, rows, b.latt16, b.lx, b.lx16, b.lf16, st));
    }
    RC(lm_output(m, g, rows, b.lx, b.lx16, b.lh32, b.lh16, b.lm_logits, st));
    return weighted_log_softmax(b.lm_logits, b.lm_extra, rows, c.vocab, temperature, weight, st);
}

// Enqueues up to max_steps search steps, step(st) each.  Every poll_every steps (0: never) the host reads b.ended_count and
// stops once it has reached `target`.  *done: the steps enqueued.
template <class Step>
static int run_steps(AsrModel* m, int max_steps, int target, cudaStream_t st, Step&& step, int* done) {
    const int check_every = m->poll_every > 0 ? m->poll_every : max_steps;
    int s = 0;
    while (s < max_steps) {
        const int chunk = std::min(check_every, max_steps - s);
        for (int i = 0; i < chunk; ++i) RC(step(st));
        s += chunk;
        if (s < max_steps && m->poll_every > 0) {
            SBK_CUDA_CHECK(cudaMemcpyAsync(m->host_flag, m->b.ended_count, 4, cudaMemcpyDeviceToHost, st));
            SBK_CUDA_CHECK(cudaStreamSynchronize(st));
            if (*m->host_flag >= target) break;
        }
    }
    *done = s;
    return SBK_OK;
}

// Beam search (decoders/seq2seq.py:1632-1723 with scorer=None): the device runs decoder step + beam_step_kernel and
// records the per-step (token, predecessor, normalised score, log-prob) history; hypothesis bookkeeping is replayed
// on the host from that history (speechbrain_b200/decoders/seq2seq.py).
static int run_beam(AsrModel* m, int B, int T, const sbk_beam_params& p, int* hist_tok_out, int* hist_pred_out,
                    float* hist_score_out, float* hist_lp_out, int* steps_done, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, Ld = c.num_decoder_layers, M = B * T, beam = p.beam_size, rows = B * beam, S_max = m->ws_steps + 1;
    SBK_REQUIRE(m->wt->has_dec, "beam: this handle was created without decoder weights");
    SBK_REQUIRE(p.max_steps <= m->ws_steps && p.max_steps + 1 <= c.max_len, "beam: max_steps=%d too large", p.max_steps);
    *steps_done = 0;
    if (p.max_steps <= 0) return SBK_OK;
    RC(project_cross_kv(m, M, T, false, st));
    set_step_pdl(m, rows, d);
    const bool use_lm = p.lm_weight != 0.0f;
    SBK_REQUIRE(!use_lm || m->wt->has_lm, "beam: lm_weight != 0 but this handle has no TransformerLM weights");
    const bool use_ctc = p.ctc_weight != 0.0f;
    // the search history lives in the workspace (fixed addresses: the step graph bakes them in) and is copied out at the end
    int* hist_tok = b.hist_tok; int* hist_pred = b.hist_pred; float* hist_score = b.hist_score; float* hist_lp = b.hist_lp;
    CtcStep cs{};
    if (use_ctc) {  // CTCScorer.reset_mem (scorer.py:243-249) + CTCPrefixScore.__init__ (ctc.py:46-78)
        SBK_REQUIRE(m->wt->w_ctc, "beam: ctc_weight != 0 but this handle has no ctc_lin weights");
        SBK_REQUIRE(p.blank_index >= 0 && p.blank_index < c.vocab && p.blank_index != p.bos && p.blank_index != p.eos &&
                    p.bos != p.eos, "Set blank, eos and bos to different indexes for joint ATT/CTC or CTC decoding");
        const size_t V = c.vocab;
        float *x = nullptr, *xlin = nullptr, *xb = nullptr, *rsum = nullptr, *rb = nullptr, *psi = nullptr, *tab = nullptr,
              *tabM = nullptr, *add = b.lm_extra;  // with an LM the CTC scores are added to the LM's
        auto layout = [&](Carver& take) {
            take(x, (size_t)M * V * 4); take(xlin, (size_t)M * V * 4); take(xb, (size_t)M * 4);
            take(rsum, (size_t)2 * rows * T * 4); take(rb, (size_t)2 * rows * T * 4); take(psi, (size_t)2 * rows * 4);
            take(tab, (size_t)2 * rows * (T + 4) * 4); take(tabM, (size_t)2 * rows * 4);
            if (!use_lm) take(add, (size_t)rows * V * 4);
        };
        Carver measure;
        layout(measure);
        RC(grow_buffer(m, m->ctc, measure.used, "beam: CTC scorer"));
        Carver carve{static_cast<uint8_t*>(m->ctc.base)};
        layout(carve);
        GemmEpilogue e;
        e.mode = EPI_F32; e.bias = m->wt->b_ctc; e.out = x; e.ldo = c.vocab;
        RC(gemm_f16(b.enc16, d, m->wt->w_ctc, d, e, M, c.vocab, d, st));
        RC(ctc_prefix_reset(x, xlin, xb, b.enc_len, B, T, c.vocab, p.blank_index, beam, rsum, rb, psi, tab, tabM, st));
        cs.x = x; cs.xlin = xlin; cs.xb = xb; cs.enc_len = b.enc_len; cs.hist_tok = hist_tok; cs.hist_pred = hist_pred; cs.n_bh = rows;
        cs.rsum_base = rsum; cs.rb_base = rb; cs.psi_base = psi; cs.step_ptr = b.step; cs.tab = tab; cs.tabM = tabM;
        cs.bos = p.bos; cs.T = T; cs.V = c.vocab; cs.beam = beam; cs.blank = p.blank_index; cs.eos = p.eos;
        cs.weight = p.ctc_weight; cs.out = add; cs.accumulate = use_lm ? 1 : 0;
    }
    const bool use_cov = p.coverage_weight != 0.0f;
    CoverageStep cv{};
    if (use_cov) {  // CoverageScorer (scorer.py:788-955) on the last decoder layer's head-averaged cross-attention
        SBK_REQUIRE(d / c.nhead == 64, "beam: the coverage scorer is built for head_dim 64");
        RC(grow_buffer(m, m->cov, ((size_t)2 * rows * T + rows) * 4 + 256, "beam: coverage scorer"));
        float* cov = static_cast<float*>(m->cov.base);
        cv.q = b.dq16; cv.ldq = d; cv.kbase = b.ckv16 + (size_t)(Ld - 1) * M * 2 * d;
        if (xatt_headmajor(m)) { cv.utt_stride = (size_t)T * d; cv.key_stride = 64; cv.head_stride = T * 64; }
        else { cv.utt_stride = (size_t)T * 2 * d; cv.key_stride = 2 * d; cv.head_stride = 64; }
        cv.enc_len = b.enc_len; cv.rows_per_utt = beam; cv.T = T; cv.H = c.nhead;
        cv.cov_base = cov; cv.hist_pred = hist_pred; cv.step_ptr = b.step; cv.n_bh = rows;
        cv.threshold = p.coverage_threshold; cv.weight = p.coverage_weight; cv.out = cov + (size_t)2 * rows * T;
    }
    BeamLm lm;
    if (use_lm) {
        lm.emb = m->wt->lm_emb; lm.pe = m->wt->lm_pe; lm.d = m->wt->lm_dp; lm.scale = m->wt->lm_emb_scale;
        lm.x = b.lx; lm.x16 = b.lx16; lm.tok_cache = b.tok_cache;
    }
    RC(beam_reset(rows, beam, S_max, p.bos, b.step, b.seq_scores, b.lineage, b.finished, b.ended_count, m->wt->emb, m->wt->dec_pe, d,
                  b.dx, use_lm ? &lm : nullptr, st));
    BeamStepArgs a{};
    a.add_scores = use_lm ? b.lm_extra : (use_ctc ? cs.out : nullptr);
    a.lm = lm;
    if (use_ctc) { a.attn_weight = 1.0f - p.ctc_weight; a.blank = p.blank_index; }
    a.add_const = p.length_weight;
    a.add_row = use_cov ? cv.out : nullptr;
    a.logits = b.logits; a.V = c.vocab; a.beam = beam; a.S_max = S_max; a.seq_scores = b.seq_scores; a.lineage = b.lineage;
    a.step_arr = b.step; a.finished = b.finished; a.n_full = b.ended_count;
    a.hist_tok = hist_tok; a.hist_pred = hist_pred; a.hist_score = hist_score; a.hist_lp = hist_lp;
    a.temperature = p.temperature; a.eos_threshold = p.eos_threshold; a.minus_inf = p.minus_inf; a.min_steps = p.min_steps;
    a.eos = p.eos; a.use_eos_threshold = p.using_eos_threshold; a.length_norm = p.length_normalization;
    a.emb = m->wt->emb; a.pe = m->wt->dec_pe; a.d = d; a.x_next = b.dx; a.scratch = b.beam_scr;
    // One whole search step; every kernel takes the step index from the device counters, so the sequence is the same
    // for every step and can be replayed from a graph.  The scorers that do not read the decoder's output of this step --
    // the TransformerLM step and the CTC state update of the PREVIOUS step's survivors -- run as a second branch beside
    // the decoder layers (both are chains of small kernels that leave most SMs idle) and join before the scores are combined.
    const bool fork = use_lm || use_ctc;
    if (fork) RC(m->side_stream.ensure());
    auto enqueue_step = [&](cudaStream_t s_) -> int {
        cudaStream_t s2 = s_;
        if (fork) {
            RC(m->side_stream.fork(s_));
            s2 = m->side_stream.s;
        }
        if (use_ctc) RC(ctc_prefix_update(cs, s2));  // permute_scorer_mem on the previous step's survivors (no-op at step 0)
        if (use_lm) RC(enqueue_lm_step(m, rows, S_max, p.lm_temperature, p.lm_weight, s2));
        RC(enqueue_decode_layers(m, rows, beam, T, S_max, b.lineage, false, s_));
        if (use_cov) RC(coverage_score(cv, s_));  // reads the last layer's cross-attention query left in b.dq16
        if (fork) RC(m->side_stream.join(s_));
        if (use_ctc) RC(ctc_prefix_score(cs, s_));  // ScorerBuilder.score (ctc after transformerlm)
        RC(beam_step(a, B, s_));
        return SBK_OK;
    };
    struct BeamKey { sbk_beam_params p; int B, T, rows, S_max; } key;
    memset(&key, 0, sizeof(key));
    key.p = p; key.B = B; key.T = T; key.rows = rows; key.S_max = S_max;
    RC(m->beam_graph.ensure(key, m->cap_stream, enqueue_step));
    int s = 0;  // `_check_full_beams` (:806-822): b.ended_count counts the utterances whose beams are full
    RC(run_steps(m, p.max_steps, B, st, [&](cudaStream_t s_) { return m->beam_graph.launch(s_); }, &s));
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
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, M = B * T, rows = B, S_max = m->ws_steps + 1;
    SBK_REQUIRE(m->wt->has_dec, "greedy: this handle was created without decoder weights");
    SBK_REQUIRE(max_steps <= m->ws_steps && max_steps + 1 <= c.max_len, "greedy: max_steps=%d too large", max_steps);
    *steps_done = 0;
    if (max_steps <= 0) return SBK_OK;
    const bool fold = xatt_fold(m, B, T);
    RC(project_cross_kv(m, M, T, fold, st));  // cross-attention K/V of all layers, once per utterance
    RC(greedy_reset(b.tokens, S_max + 1, rows, bos, b.step, b.has_ended, b.ended_count, m->wt->emb, m->wt->dec_pe, d, b.dx, st));
    set_step_pdl(m, rows, d);
    const bool use_graph = !in_capture && log_probs == nullptr;
    if (in_capture) {  // the caller is capturing the whole pipeline: enqueue exactly max_steps steps, no polling
        for (int i = 0; i < max_steps; ++i) RC(enqueue_decode_step(m, rows, T, S_max, fold, eos, log_probs, max_steps, st));
        *steps_done = max_steps;
        return SBK_OK;
    }
    if (use_graph) {
        const struct StepKey { int rows, T, B, eos, S_max; } key = {rows, T, B, eos, S_max};
        RC(m->step_graph.ensure(key, m->cap_stream, [&](cudaStream_t cs) {
            return enqueue_decode_step(m, rows, T, S_max, fold, eos, nullptr, 0, cs);
        }));
    }
    // seq2seq.py:256 `has_ended.all()` early exit
    return run_steps(m, max_steps, rows, st, [&](cudaStream_t s_) {
        return use_graph ? m->step_graph.launch(s_) : enqueue_decode_step(m, rows, T, S_max, fold, eos, log_probs, max_steps, s_);
    }, steps_done);
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
                                        const float* __restrict__ pe, int d, float scale, float* __restrict__ x,
                                        __half* __restrict__ x16, int* __restrict__ step_arr) {
    const int r = blockIdx.x;
    const int tok = tokens[static_cast<size_t>(r) * L + s];
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        const float v = emb[static_cast<size_t>(tok) * d + i] * scale + pe[static_cast<size_t>(s) * d + i];
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
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int d = c.d_model, M = n * T, S_max = m->ws_steps + 1;
    SBK_REQUIRE(m->wt->has_dec, "decode: this handle was created without decoder weights");
    SBK_REQUIRE(S <= m->ws_steps && S <= c.max_len, "decode: %d target positions exceed the workspace / max_len", S);
    const bool fold = xatt_fold(m, n, T);
    RC(project_cross_kv(m, M, T, fold, st));
    set_step_pdl(m, n, d);
    for (int s = 0; s < S; ++s) {
        dec_teacher_embed_kernel<<<n, 128, 0, st>>>(tokens, S, s, m->wt->emb, m->wt->dec_pe, d, sqrtf((float)d), b.dx, b.step);
        SBK_LAUNCH_CHECK();
        RC(enqueue_decode_layers(m, n, 1, T, S_max, nullptr, fold, st, false));
        RC(layernorm_rows(b.dx, b.lnout, false, m->wt->dec_norm_g, m->wt->dec_norm_b, n, d, 1e-6f, st));
        SBK_CUDA_CHECK(cudaMemcpy2DAsync(out + (size_t)s * d, (size_t)S * d * 4, b.lnout, (size_t)d * 4, (size_t)d * 4, n,
                                         cudaMemcpyDeviceToDevice, st));
    }
    return SBK_OK;
}

static int run_lm_rescore(AsrModel* m, const int* tokens, const int* lens, int n, int L, float temperature, int pad,
                          float* scores, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int S_max = m->ws_steps + 1, dp = m->wt->lm_dp;
    set_step_pdl(m, n, m->wt->lm_da);
    lm_teacher_reset_kernel<<<n, 128, 0, st>>>(tokens, n, L, S_max, pad, b.lineage, b.tok_cache, scores);
    SBK_LAUNCH_CHECK();
    for (int s = 0; s + 1 < L; ++s) {
        lm_teacher_embed_kernel<<<n, 128, 0, st>>>(tokens, L, s, m->wt->lm_emb, m->wt->lm_pe, dp, m->wt->lm_emb_scale, b.lx,
                                                   b.lx16, b.step);
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
    const sbk_asr_config& c = m->wt->cfg;
    AsrModel::Buf& b = m->b;
    const int S_max = m->ws_steps + 1, dp = m->wt->lm_dp, V = c.vocab;
    set_step_pdl(m, n, m->wt->lm_da);
    lm_teacher_reset_kernel<<<n, 128, 0, st>>>(tokens, n, L, S_max, 0, b.lineage, b.tok_cache, b.score);
    SBK_LAUNCH_CHECK();
    for (int s = 0; s < L; ++s) {
        lm_teacher_embed_kernel<<<n, 128, 0, st>>>(tokens, L, s, m->wt->lm_emb, m->wt->lm_pe, dp, m->wt->lm_emb_scale, b.lx,
                                                   b.lx16, b.step);
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
// Row r = (sequence r / s, position r % s): x = emb[token] * scale + pe[pos], fp32 residual stream + fp16 GEMM operand
// (the whole-sequence counterpart of lm_teacher_embed_kernel).  An id outside [0, vocab) is not read from the table: its
// row becomes NaN (and, through attention, its sequence) instead of an out-of-bounds read.
__global__ void lm_embed_kernel(const int* __restrict__ tokens, int s, int vocab, const float* __restrict__ emb,
                                const float* __restrict__ pe, int d, float scale, float* __restrict__ x,
                                __half* __restrict__ x16) {
    const int r = blockIdx.x, pos = r % s;
    const int tok = tokens[r];
    const bool ok = tok >= 0 && tok < vocab;
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        const float v = ok ? emb[static_cast<size_t>(tok) * d + i] * scale + pe[static_cast<size_t>(pos) * d + i] : NAN;
        x[static_cast<size_t>(r) * d + i] = v;
        x16[static_cast<size_t>(r) * d + i] = float2half_sat(v);
    }
}

static int ensure_lm_workspace(AsrModel* m, int rows) {
    AsrModel::LmFwdBuf& w = m->lmf;
    if (m->lmf_mem.base && rows <= w.rows) return SBK_OK;
    const size_t R = rows, dp = m->wt->lm_dp, da = m->wt->lm_da, Fl = m->wt->cfg.lm_d_ffn;
    auto layout = [&](Carver& take) {
        take(w.x, R * dp * 4); take(w.x16, R * dp * 2); take(w.qkv16, R * 3 * da * 2); take(w.att16, R * da * 2);
        take(w.f16, R * Fl * 2);
    };
    Carver measure;
    layout(measure);
    RC(grow_buffer(m, m->lmf_mem, measure.used, "lm_forward: workspace"));
    Carver carve{static_cast<uint8_t*>(m->lmf_mem.base)};
    layout(carve);
    w.rows = rows;
    return SBK_OK;
}

static int run_lm_forward(AsrModel* m, const int* tokens, int n, int s, float* logits, cudaStream_t st) {
    const sbk_asr_config& c = m->wt->cfg;
    const int dp = m->wt->lm_dp, da = m->wt->lm_da, H = c.lm_nhead, M = n * s;
    RC(ensure_lm_workspace(m, M));
    const AsrModel::LmFwdBuf& b = m->lmf;
    lm_embed_kernel<<<M, 128, 0, st>>>(tokens, s, c.vocab, m->wt->lm_emb, m->wt->lm_pe, dp, m->wt->lm_emb_scale, b.x, b.x16);
    SBK_LAUNCH_CHECK();
    for (int l = 0; l < c.lm_layers; ++l) {  // post-norm TransformerEncoderLayer (Transformer.py:466-481)
        const LmLayerW& w = m->wt->lm[l];
        RC(project(SG_WIDE, {w.w_in, w.b_in, 3 * da, dp, PO_F16, b.qkv16, 3 * da, b.x16, dp}, M, st));
        RC(lm_causal_attention(b.qkv16, n, s, da, H, tokens, 0, b.att16, st));
        RC(lm_layer_tail(m, SG_WIDE, w, M, b.att16, b.x, b.x16, b.f16, st));
    }
    // output_proj's fp32 Linear d -> d goes into the free residual buffer, its logits into the caller's
    return lm_output(m, SG_WIDE, M, b.x, b.x16, b.x, b.x16, logits, st);
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

int sbk_step_proj_test(int backend, int epilogue, const void* A_dev, int lda, const float* X_dev, const float* ln_g_dev,
                       const float* ln_b_dev, const void* W_dev, const float* bias_dev, int rows, int N, int K, void* out_dev,
                       int ldo, void* kcache_dev, void* vcache_dev, int S_max, int step, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(backend == 0 || backend == 1, "step_proj_test: backend %d (0 weight streaming, 1 wgmma)", backend);
    SBK_REQUIRE(epilogue >= PO_F16 && epilogue <= PO_QKV_CACHE, "step_proj_test: epilogue %d", epilogue);
    SBK_REQUIRE(W_dev && out_dev && (A_dev != nullptr) != (X_dev != nullptr) && (!X_dev || (ln_g_dev && ln_b_dev)),
                "step_proj_test: null pointer, or not exactly one of A and X");
    SBK_REQUIRE(rows >= 1 && N >= 1 && K >= 16 && K % 16 == 0 && (!A_dev || lda >= K),
                "step_proj_test: bad sizes rows=%d N=%d K=%d lda=%d", rows, N, K, lda);
    const bool qkv = epilogue == PO_QKV_CACHE;
    SBK_REQUIRE(!qkv || (N % 3 == 0 && kcache_dev && vcache_dev && step >= 0 && step < S_max),
                "step_proj_test: QKV_CACHE needs N %% 3 == 0, both caches and 0 <= step < S_max (N=%d step=%d S_max=%d)", N,
                step, S_max);
    SBK_REQUIRE(ldo >= (qkv ? N / 3 : N), "step_proj_test: ldo=%d below the output width", ldo);
    // the wgmma epilogue stores 16-byte vectors
    SBK_REQUIRE(backend == 0 || (ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(out_dev) & 15) == 0),
                "step_proj_test: the wgmma back end needs ldo %% 8 == 0 and a 16-byte aligned out");
    int* steps = nullptr;
    __half* h16 = nullptr;
    TestScratch scr;
    RC(scr.carve("step_proj_test", [&](Carver& take) { take(steps, (size_t)rows * 4); take(h16, X_dev ? (size_t)rows * K * 2 : 0); }));
    // one counter per row, all equal, as b.step holds them: the weight-streaming kernel reads row 0's, the wgmma epilogue
    // each row's
    const std::vector<int> step_val(rows, step);
    int rc = cudaMemcpyAsync(steps, step_val.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, st) == cudaSuccess ? SBK_OK
                                                                                                                 : SBK_ERR_CUDA;
    if (rc == SBK_OK) {
        const StepGemm g = backend == 1 ? SG_SMALL : SG_STREAM;
        set_pdl(g == SG_SMALL);  // what set_step_pdl gives this back end
        Proj p{static_cast<const __half*>(W_dev), bias_dev, N, K, static_cast<ProjOut>(epilogue), out_dev, ldo,
               static_cast<const __half*>(A_dev), lda};
        if (qkv) {
            p.kcache = static_cast<__half*>(kcache_dev); p.vcache = static_cast<__half*>(vcache_dev);
            p.step_ptr = steps; p.S_max = S_max;
        }
        rc = X_dev ? norm_project(g, true, p, X_dev, ln_g_dev, ln_b_dev, h16, rows, st) : project(g, p, rows, st);
    }
    return finish_test("step_proj_test", rc, st);
}

int sbk_asr_create(const sbk_asr_config* cfg, const sbk_tensor* weights, int n_weights, sbk_asr** out) {
    return asr_create(cfg, weights, n_weights, reinterpret_cast<AsrModel**>(out));
}
void sbk_asr_destroy(sbk_asr* m) { delete reinterpret_cast<AsrModel*>(m); }
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
    frames(m->wt->cfg, n_samples, &T0, &T1, &T2);
    if (T_feat) *T_feat = T0;
    if (T_enc) *T_enc = T2;
    return SBK_OK;
}

int sbk_asr_cnn_forward(sbk_asr* mm, const float* feats_dev, int B, int T0, float* out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    const sbk_asr_config& c = m->wt->cfg;
    SBK_REQUIRE(m->wt->has_cnn, "cnn_forward: this handle was created without CNN weights");
    RC(ensure_workspace(m, B, (T0 - 1) * c.hop, B, 1));
    return run_cnn(m, feats_dev, B, T0, out_dev, static_cast<cudaStream_t>(stream));
}

// The encoder of an encode entry: b.enc_len = round(rel_len * T) when rel_len is set (else every frame counts), then
// run_encoder from feats (null: from the CNN output in b.a_in) into enc_out (null: b.enc_out).
static int encode_entry(AsrModel* m, const float* feats, const float* rel_len, int B, int T0, int T, float* cnn_out,
                        float* enc_out, cudaStream_t st) {
    if (rel_len) RC(set_enc_len(m->b.enc_len, rel_len, B, T, st));
    return run_encoder(m, feats, B, T0, rel_len ? m->b.enc_len : nullptr, cnn_out, enc_out ? enc_out : m->b.enc_out, st);
}

// src_dev: CNN output [B, T, input_size] fp32 -> enc_out_dev [B, T, d] fp32 (TransformerASR.encode)
int sbk_asr_encode_feats(sbk_asr* mm, const float* feats_dev, const float* rel_len_dev, int B, int T0,
                         float* cnn_out_dev, float* enc_out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    const int L = (T0 - 1) * m->wt->cfg.hop;
    RC(ensure_workspace(m, B, L, B, 1));
    int T0_, T1, T;
    frames(m->wt->cfg, L, &T0_, &T1, &T);
    return encode_entry(m, feats_dev, rel_len_dev, B, T0, T, cnn_out_dev, enc_out_dev, static_cast<cudaStream_t>(stream));
}

int sbk_asr_encode_from_cnn(sbk_asr* mm, const float* src_dev, const float* rel_len_dev, int B, int T,
                            float* enc_out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const sbk_asr_config& c = m->wt->cfg;
    RC(ensure_workspace(m, B, enc_samples(c, T), B, 1));
    RC(cast_f32_f16(src_dev, m->b.a_in, (size_t)B * T * c.input_size, st));
    return encode_entry(m, nullptr, rel_len_dev, B, T, T, nullptr, enc_out_dev, st);
}

// ---- chunk-by-chunk streaming encoder (AsrStream)
static size_t stream_kv_bytes(const sbk_asr_config& c, int B, int cap) {
    return (size_t)c.num_encoder_layers * B * cap * 2 * c.d_model * 2;
}

int sbk_asr_stream_create(sbk_asr* mm, int B, int chunk_size, int left_frames, sbk_asr_stream** out) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m && out, "stream_create: null argument");
    const sbk_asr_config& c = m->wt->cfg;
    const int d = c.d_model, dh = d / c.nhead, L = c.num_encoder_layers, halo = (c.kernel_size - 1) / 2;
    SBK_REQUIRE(m->wt->has_enc, "stream_create: this handle was created without encoder weights");
    SBK_REQUIRE(c.encoder_module == SBK_ENC_CONFORMER && (c.attention_type == SBK_ATT_ROPE || c.attention_type == SBK_ATT_RELPOS),
                "stream_create: streaming is built for the Conformer encoder with RoPEMHA or RelPosMHAXL");
    SBK_REQUIRE(c.attention_type == SBK_ATT_RELPOS ? (dh == 64 || dh == 36 || dh == 32 || dh == 96) : (dh == 64 || dh == 32),
                "stream_create: head_dim=%d not built for streaming (RoPEMHA 64 or 32, RelPosMHAXL 96, 64, 36 or 32)", dh);
    SBK_REQUIRE(B >= 1 && chunk_size >= 1 && left_frames >= -1, "stream_create: B >= 1, chunk_size >= 1, left_frames >= -1");
    const bool relpos = c.attention_type == SBK_ATT_RELPOS;
    const int cap = left_frames >= 0 ? left_frames + chunk_size : std::max(4 * chunk_size, 256);
    SBK_REQUIRE(!relpos || left_frames < 0 || cap <= m->wt->pos_len,
                "stream_create: a window of %d frames exceeds RelPosMHAXL's max_len=%d", cap, m->wt->pos_len);
    std::unique_ptr<AsrStream> st(new AsrStream());
    st->B = B; st->chunk = chunk_size; st->left = left_frames; st->cap = cap;
    auto alloc = [](DevBuf& buf, size_t bytes) {
        if (cudaMalloc(&buf.base, std::max<size_t>(bytes, 256)) != cudaSuccess) {
            set_error("stream_create: cudaMalloc(%zu) failed", bytes);
            return SBK_ERR_NOMEM;
        }
        buf.cap = bytes;
        return SBK_OK;
    };
    RC(alloc(st->kv, stream_kv_bytes(c, B, cap)));
    RC(alloc(st->carry, (size_t)L * B * halo * d * 4));
    const size_t rows = (size_t)B * chunk_size;
    for (int pass = 0; pass < 2; ++pass) {
        Carver take{pass ? static_cast<uint8_t*>(st->scr.base) : nullptr};
        float* inv = nullptr;
        take(inv, (size_t)dh / 2 * 4); take(st->qkv32, rows * 3 * d * 4); take(st->q16, rows * d * 2);
        st->inv_freq = inv;
        if (!pass) RC(alloc(st->scr, take.used));
    }
    if (!relpos) {  // nnet/attention.py:1012-1055: inv_freq_i = exp(-2i * ln(1e4) / d_h) in fp32, as the full-sequence table
        std::vector<float> inv(dh / 2);
        for (int i = 0; i < dh / 2; ++i) inv[i] = expf((float)(2 * i) * -(logf(10000.0f) / (float)dh));
        SBK_CUDA_CHECK(cudaMemcpy(const_cast<float*>(st->inv_freq), inv.data(), inv.size() * 4, cudaMemcpyHostToDevice));
    } else {  // P = linear_pos(pe[r]) for every row a window can reach, once per stream
        st->prow = left_frames >= 0 ? cap : m->wt->pos_len;
        RC(alloc(st->P, (size_t)L * st->prow * d * 2));
        for (int l = 0; l < L; ++l)
            RC(relpos_project(m, l, st->prow, static_cast<__half*>(st->P.base) + (size_t)l * st->prow * d, 0));
        SBK_CUDA_CHECK(cudaStreamSynchronize(0));
    }
    *out = reinterpret_cast<sbk_asr_stream*>(st.release());
    return SBK_OK;
}

void sbk_asr_stream_destroy(sbk_asr_stream* s) { delete reinterpret_cast<AsrStream*>(s); }

int sbk_asr_stream_reset(sbk_asr_stream* ss) {
    AsrStream* s = reinterpret_cast<AsrStream*>(ss);
    SBK_REQUIRE(s, "stream_reset: null stream");
    s->total = 0; s->clen = 0; s->start = 0; s->ended = false;  // the first chunk reads no cache and a zero carry
    s->fe_chunks = 0; s->fe_ended = false;                        // and the first front-end window zero audio context
    return SBK_OK;
}

static int stream_encode(AsrModel* m, AsrStream* s, const float* cnn_out_dev, long long batch_stride, int n, float* enc_out_dev,
                         cudaStream_t st) {
    SBK_REQUIRE(m && s && cnn_out_dev && enc_out_dev, "stream_encode_chunk: null argument");
    const sbk_asr_config& c = m->wt->cfg;
    SBK_REQUIRE(n >= 1 && n <= s->chunk, "stream_encode_chunk: %d frames, the chunk size is %d", n, s->chunk);
    SBK_REQUIRE(batch_stride >= (long long)n * c.input_size, "stream_encode_chunk: batch stride %lld below %d frames of %d",
                batch_stride, n, c.input_size);
    SBK_REQUIRE(!s->ended, "stream_encode_chunk: only the last chunk of a stream may be shorter than the chunk size");
    const int W = s->clen + n;
    SBK_REQUIRE(s->prow == 0 || W <= s->prow,
                "stream_encode_chunk: an unlimited left context holds at most max_len=%d frames with RelPosMHAXL", s->prow);
    if (W > s->cap) {  // unlimited left context (nothing is ever evicted, so the ring starts at slot 0): grow it
        const int ncap = std::max(W, 2 * s->cap);
        DevBuf nb;
        if (cudaMalloc(&nb.base, stream_kv_bytes(c, s->B, ncap)) != cudaSuccess) {
            set_error("stream_encode_chunk: cudaMalloc(%zu) failed", stream_kv_bytes(c, s->B, ncap));
            return SBK_ERR_NOMEM;
        }
        const size_t row = (size_t)2 * c.d_model * 2;
        if (s->clen > 0)
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(nb.base, ncap * row, s->kv.base, s->cap * row, s->clen * row,
                                             (size_t)c.num_encoder_layers * s->B, cudaMemcpyDeviceToDevice, st));
        SBK_CUDA_CHECK(cudaStreamSynchronize(st));  // the old ring is freed below
        std::swap(nb.base, s->kv.base);
        s->kv.cap = stream_kv_bytes(c, s->B, ncap);
        s->cap = ncap;
    }
    RC(ensure_workspace(m, s->B, enc_samples(c, n), s->B, 1));
    // each row's chunk, possibly inside a longer window of the row (the streaming front end's output)
    RC(cast_f32_f16(cnn_out_dev, m->b.a_in, (size_t)n * c.input_size, st, s->B, batch_stride));
    RC(run_encoder(m, nullptr, s->B, n, nullptr, nullptr, enc_out_dev, st, s));
    s->total += n;
    if (n < s->chunk) s->ended = true;
    if (s->left >= 0) {  // keep the last `left` rows of the window
        const int keep = std::min(W, s->left);
        s->start = (s->start + W - keep) % s->cap;
        s->clen = keep;
    } else {
        s->clen = W;
    }
    return SBK_OK;
}

int sbk_asr_stream_encode_chunk(sbk_asr* mm, sbk_asr_stream* ss, const float* cnn_out_dev, int n, float* enc_out_dev,
                                void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m, "stream_encode_chunk: null argument");
    return stream_encode(m, reinterpret_cast<AsrStream*>(ss), cnn_out_dev, (long long)n * m->wt->cfg.input_size, n,
                         enc_out_dev, static_cast<cudaStream_t>(stream));
}

int sbk_asr_stream_encode_chunk_strided(sbk_asr* mm, sbk_asr_stream* ss, const float* cnn_out_dev, long long batch_stride,
                                        int n, float* enc_out_dev, void* stream) {
    return stream_encode(reinterpret_cast<AsrModel*>(mm), reinterpret_cast<AsrStream*>(ss), cnn_out_dev, batch_stride, n,
                         enc_out_dev, static_cast<cudaStream_t>(stream));
}

// One front-end window per row: win [B][2 * pad + n] = [carry | chunk] (zeros for the carry before a stream's first chunk),
// and the window's last 2 * pad samples into the other carry buffer.  StreamingFeatureWrapper.forward, lobes/features.py:
// 615-660.
__global__ void stream_window_kernel(const float* __restrict__ chunk, int n, int P2, const float* __restrict__ carry_in,
                                     float* __restrict__ carry_out, float* __restrict__ win) {
    const int b = blockIdx.y, Lw = P2 + n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Lw; i += gridDim.x * blockDim.x) {
        const float v = i < P2 ? (carry_in ? carry_in[(size_t)b * P2 + i] : 0.0f) : chunk[(size_t)b * n + i - P2];
        win[(size_t)b * Lw + i] = v;
        if (i >= n) carry_out[(size_t)b * P2 + i - n] = v;
    }
}

int sbk_asr_stream_frontend_chunk(sbk_asr* mm, sbk_asr_stream* ss, const float* wav_chunk_dev, int n_samples, int pad,
                                  float* win_out_dev, int* n_frames, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    AsrStream* s = reinterpret_cast<AsrStream*>(ss);
    SBK_REQUIRE(m && s && wav_chunk_dev && win_out_dev, "stream_frontend_chunk: null argument");
    const sbk_asr_config& c = m->wt->cfg;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(m->wt->has_fbank && m->wt->has_cnn && m->wt->glob_mean,
                "stream_frontend_chunk: the handle needs Fbank, global InputNormalization and CNN weights");
    const int stride = 4 * c.hop;  // the Fbank hop times the front end's two stride-2 blocks
    SBK_REQUIRE(pad > 0 && pad % stride == 0, "stream_frontend_chunk: pad=%d is not a positive multiple of the stride %d",
                pad, stride);
    SBK_REQUIRE(s->pad == 0 || s->pad == pad, "stream_frontend_chunk: pad=%d, the stream was started with pad=%d", pad, s->pad);
    SBK_REQUIRE(n_samples >= 1, "stream_frontend_chunk: empty chunk");
    const int P2 = 2 * pad, Lw = P2 + n_samples, trim = pad / stride;
    int T0, T1, T2;
    frames(c, Lw, &T0, &T1, &T2);
    const int n = T2 - 2 * trim;
    SBK_REQUIRE(n >= 1 && n <= s->chunk, "stream_frontend_chunk: %d samples give %d frames, the chunk size is %d", n_samples,
                n, s->chunk);
    // the encoder's own limits too, so that a chunk it would refuse leaves the audio context where it was
    SBK_REQUIRE(!s->fe_ended && !s->ended,
                "stream_frontend_chunk: only the last chunk of a stream may be shorter than the chunk size");
    SBK_REQUIRE(s->prow == 0 || s->clen + n <= s->prow,
                "stream_frontend_chunk: an unlimited left context holds at most max_len=%d frames with RelPosMHAXL", s->prow);
    if (s->pad == 0) {
        if (cudaMalloc(&s->wav_carry.base, (size_t)2 * s->B * P2 * 4) != cudaSuccess) {
            set_error("stream_frontend_chunk: cudaMalloc(%zu) failed", (size_t)2 * s->B * P2 * 4);
            return SBK_ERR_NOMEM;
        }
        s->wav_carry.cap = (size_t)2 * s->B * P2 * 4;
        s->pad = pad;
    }
    RC(ensure_workspace(m, s->B, Lw, s->B, 1));
    float* carry = static_cast<float*>(s->wav_carry.base);
    const int k = s->fe_chunks & 1;
    dim3 grid(std::min(ceil_div(Lw, 256), 64), s->B);
    stream_window_kernel<<<grid, 256, 0, st>>>(wav_chunk_dev, n_samples, P2, s->fe_chunks ? carry + (size_t)k * s->B * P2 : nullptr,
                                              carry + (size_t)(1 - k) * s->B * P2, m->b.wav);
    SBK_LAUNCH_CHECK();
    AsrModel::Buf& b = m->b;
    RC(fbank_forward(m->wt->fbank, b.wav, s->B, Lw, b.feats, b.utt_max, m->wt->glob_mean, m->wt->glob_std,
                     c.norm_eps > 0.0f ? c.norm_eps : 1e-10f, st));
    RC(run_cnn(m, b.feats, s->B, T0, win_out_dev, st));
    s->fe_chunks += 1;
    if (n < s->chunk) s->fe_ended = true;
    if (n_frames) *n_frames = n;
    return SBK_OK;
}

int sbk_asr_stream_context(sbk_asr* mm, const sbk_asr_stream* ss, int layer, void* kv_out_dev, float* carry_out_dev,
                           int* n_rows, void* stream) {
    const AsrModel* m = reinterpret_cast<const AsrModel*>(mm);
    const AsrStream* s = reinterpret_cast<const AsrStream*>(ss);
    SBK_REQUIRE(m && s, "stream_context: null argument");
    const sbk_asr_config& c = m->wt->cfg;
    SBK_REQUIRE(layer >= 0 && layer < c.num_encoder_layers, "stream_context: layer %d of %d", layer, c.num_encoder_layers);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_rows) *n_rows = s->clen;
    const size_t row = (size_t)2 * c.d_model * 2;
    if (kv_out_dev && s->clen > 0) {  // the ring in window order: slots [start, cap) then [0, ...)
        const uint8_t* src = reinterpret_cast<const uint8_t*>(s->kv_layer(c, layer));
        const int n1 = std::min(s->clen, s->cap - s->start), n2 = s->clen - n1;
        uint8_t* dst = static_cast<uint8_t*>(kv_out_dev);
        SBK_CUDA_CHECK(cudaMemcpy2DAsync(dst, s->clen * row, src + s->start * row, s->cap * row, n1 * row, s->B,
                                         cudaMemcpyDeviceToDevice, st));
        if (n2 > 0)
            SBK_CUDA_CHECK(cudaMemcpy2DAsync(dst + n1 * row, s->clen * row, src, s->cap * row, n2 * row, s->B,
                                             cudaMemcpyDeviceToDevice, st));
    }
    if (carry_out_dev) {
        const size_t bytes = (size_t)s->B * ((c.kernel_size - 1) / 2) * c.d_model * 4;
        if (s->total > 0) SBK_CUDA_CHECK(cudaMemcpyAsync(carry_out_dev, s->carry_layer(c, layer), bytes, cudaMemcpyDeviceToDevice, st));
        else SBK_CUDA_CHECK(cudaMemsetAsync(carry_out_dev, 0, bytes, st));
    }
    return SBK_OK;
}

// Full device pipeline on device-resident wav: Fbank -> global CMVN -> CNN -> encoder -> greedy.
// Outputs (device, optional): enc_out [B,T,d] fp32; pred [B, max_steps] int32; score [B, max_steps] fp32.
static int transcribe_enqueue(AsrModel* m, const float* wav_dev, const float* rel_len_dev, int B, int L, int max_steps,
                              int bos, int eos, float* enc_out_dev, int* pred_dev, float* score_dev, float* log_probs_dev,
                              int* steps_done, cudaStream_t st, bool in_capture) {
    const sbk_asr_config& c = m->wt->cfg;
    int T0, T1, T;
    frames(c, L, &T0, &T1, &T);
    AsrModel::Buf& b = m->b;
    RC(fbank_forward(m->wt->fbank, wav_dev, B, L, b.feats, b.utt_max, m->wt->glob_mean, m->wt->glob_std, c.norm_eps > 0.0f ? c.norm_eps : 1e-10f, st));
    RC(set_enc_len(b.enc_len, rel_len_dev, B, T, st));
    RC(run_encoder(m, b.feats, B, T0, b.enc_len, nullptr, b.enc_out, st));
    if (enc_out_dev)
        SBK_CUDA_CHECK(cudaMemcpyAsync(enc_out_dev, b.enc_out, (size_t)B * T * c.d_model * 4, cudaMemcpyDeviceToDevice, st));
    int done = 0;
    if (max_steps > 0 && m->wt->has_dec) {
        RC(run_greedy(m, B, T, max_steps, bos, eos, log_probs_dev, &done, st, in_capture));
        RC(copy_steps(m, pred_dev, max_steps, b.pred, done, B, cudaMemcpyDeviceToDevice, st));
        RC(copy_steps(m, score_dev, max_steps, b.score, done, B, cudaMemcpyDeviceToDevice, st));
    }
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// Batches per encoder pass of a group call of G >= 1 batches of B >= 1 utterances of L samples: as many batches as fit in
// GROUP_PASS_ROWS encoder rows (at least one), then the batches spread evenly over that many passes, so no pass exceeds
// GROUP_PASS_ROWS rows unless a single batch does.  Conformer-L, 32 x 10 s batches (8032 rows), one H100 SXM at 700 W
// (tools/group_encode.py): the encode per batch falls up to about 7 batches per pass and is flat from 7 to 16, while the
// pass's activations grow with it.
constexpr long long GROUP_PASS_ROWS = 1 << 16;
static int group_encode_batches(const sbk_asr_config& c, int G, int B, int L) {
    int T0, T1, T;
    frames(c, L, &T0, &T1, &T);
    const long long fit = std::max(1LL, GROUP_PASS_ROWS / std::max(1LL, (long long)B * T));
    const int E = (int)std::min<long long>(G, fit);
    return ceil_div(G, ceil_div(G, E));
}

// The argument checks of the group entries `who`: G batches of B utterances of L samples, every batch's wav and lengths
// given (and its output ids, when `pred` is given).
static int check_group_call(const AsrModel* m, const char* who, int G, const float* const* wav, const float* const* rel,
                            int* const* pred, int B, int L) {
    SBK_REQUIRE(G >= 1 && G <= 16, "%s: G=%d not in [1, 16]", who, G);
    SBK_REQUIRE(m->wt->has_fbank && m->wt->has_cnn && m->wt->has_enc && m->wt->has_dec, "%s: handle lacks model parts", who);
    SBK_REQUIRE(m->wt->glob_mean != nullptr, "%s: model has no normalize.glob_mean/std weights", who);
    for (int g = 0; g < G; ++g) SBK_REQUIRE(wav[g] && rel[g] && (!pred || pred[g]), "%s: null batch pointer", who);
    SBK_REQUIRE(B >= 1 && L >= 1, "%s: empty batch (B=%d, L=%d)", who, B, L);
    return SBK_OK;
}

// G independent batches of B utterances: Fbank and the lengths run per batch (each batch is its own waveform pointer), the
// CNN and encoder once per chunk of group_encode_batches() consecutive batches over all of the chunk's utterances, then ONE
// greedy loop decodes all G*B hypotheses together.  Every encoder kernel works per row or per utterance, so an utterance's
// encoder states do not depend on how many batches share its pass.  A decode step is ~50 dependent, latency-bound kernels
// whose cost barely depends on the row count, so coalescing the decode of the batches in flight amortises it G-fold;
// per-utterance results are unchanged (rows are independent).
static int transcribe_group_enqueue(AsrModel* m, int G, const float* const* wav_dev, const float* const* rel_dev, int B, int L,
                                    int max_steps, int bos, int eos, int* const* pred_dev, int* steps_done, cudaStream_t st,
                                    bool in_capture, const cudaEvent_t* ready = nullptr, int* const* pred_host = nullptr) {
    const sbk_asr_config& c = m->wt->cfg;
    int T0, T1, T;
    frames(c, L, &T0, &T1, &T);
    AsrModel::Buf& b = m->b;
    const int E = group_encode_batches(c, G, B, L);
    for (int g0 = 0; g0 < G; g0 += E) {
        const int n = std::min(E, G - g0);
        for (int g = g0; g < g0 + n; ++g) {
            if (ready) SBK_CUDA_CHECK(cudaStreamWaitEvent(st, ready[g], 0));  // batch g's wav has landed in the staging buffer
            RC(fbank_forward(m->wt->fbank, wav_dev[g], B, L, b.feats + (size_t)(g - g0) * B * T0 * c.n_mels, b.utt_max,
                             m->wt->glob_mean, m->wt->glob_std, c.norm_eps > 0.0f ? c.norm_eps : 1e-10f, st));
            RC(set_enc_len(b.enc_len + (size_t)g * B, rel_dev[g], B, T, st));
        }
        RC(run_encoder(m, b.feats, n * B, T0, b.enc_len + (size_t)g0 * B, nullptr, b.enc_out + (size_t)g0 * B * T * c.d_model, st));
    }
    // The decode loop is a chain of ~3300 small, latency-bound kernels; the encoders of the other lanes are machine-filling
    // ones.  Its kernels go to a stream of the highest priority (under capture: kernel nodes of that priority), so that a ready
    // decode kernel gets the next free SM slots ahead of the remaining CTAs of an encoder kernel instead of queueing behind
    // them.
    RC(m->dec_stream.ensure(true));
    RC(m->dec_stream.fork(st));
    const cudaStream_t ds = m->dec_stream.s;
    int done = 0;
    RC(run_greedy(m, G * B, T, max_steps, bos, eos, nullptr, &done, ds, in_capture));
    for (int g = 0; g < G; ++g) {
        const int* pred = b.pred + (size_t)g * B * (m->ws_steps + 1);
        RC(copy_steps(m, pred_dev ? pred_dev[g] : nullptr, max_steps, pred, done, B, cudaMemcpyDeviceToDevice, ds));
        RC(copy_steps(m, pred_host ? pred_host[g] : nullptr, max_steps, pred, done, B, cudaMemcpyDeviceToHost, ds));
    }
    RC(m->dec_stream.join(st));
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// Host-buffer form of the group call: H2D of every batch on a copy stream forked from `st` (batch g's Fbank waits for its
// own copy only, so a later encoder pass's copies overlap an earlier pass), the group pipeline, D2H of the token ids.
// Works both eagerly and under stream capture (the fork / join events become graph edges, the copies memcpy nodes).
static int transcribe_group_host_enqueue(AsrModel* m, int G, const float* const* wav_host, const float* const* rel_host, int B,
                                         int L, int max_steps, int bos, int eos, int* const* pred_host, int* const* pred_dev,
                                         int* steps_done, cudaStream_t st, bool in_capture) {
    RC(m->copy_stream.fork(st));  // the previous call no longer reads the staging buffers
    const cudaStream_t cs = m->copy_stream.s;
    const float* wav_dev[16];
    const float* rel_dev[16];
    float* gwav = static_cast<float*>(m->gwav.base);
    float* grel = gwav + (size_t)G * B * L;  // lengths behind the G waveforms
    for (int g = 0; g < G; ++g) {
        float* w = gwav + (size_t)g * B * L;
        float* r = grel + (size_t)g * B;
        SBK_CUDA_CHECK(cudaMemcpyAsync(w, wav_host[g], (size_t)B * L * 4, cudaMemcpyHostToDevice, cs));
        SBK_CUDA_CHECK(cudaMemcpyAsync(r, rel_host[g], (size_t)B * 4, cudaMemcpyHostToDevice, cs));
        SBK_CUDA_CHECK(cudaEventRecord(m->ev_ready[g], cs));
        wav_dev[g] = w; rel_dev[g] = r;
    }
    return transcribe_group_enqueue(m, G, wav_dev, rel_dev, B, L, max_steps, bos, eos, pred_dev, steps_done, st, in_capture,
                                    m->ev_ready, pred_host);
}

int sbk_asr_transcribe_greedy_group_dev(sbk_asr* mm, int G, const float* const* wav_dev, const float* const* rel_len_dev,
                                        int B, int L, int max_steps, int bos, int eos, int* const* pred_dev, int* steps_done,
                                        void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    RC(check_group_call(m, "transcribe_group", G, wav_dev, rel_len_dev, nullptr, B, L));
    RC(ensure_workspace(m, B, L, G * B, max_steps, group_encode_batches(m->wt->cfg, G, B, L) * B));
    const bool whole_graph = m->poll_every == 0 && max_steps > 0;
    struct GroupKey { const void *wav[16], *rel[16], *pred[16]; int G, B, L, steps, bos, eos; } key;
    memset(&key, 0, sizeof(key));
    key.G = G; key.B = B; key.L = L; key.steps = max_steps; key.bos = bos; key.eos = eos;
    for (int g = 0; g < G; ++g) { key.wav[g] = wav_dev[g]; key.rel[g] = rel_len_dev[g]; key.pred[g] = pred_dev ? pred_dev[g] : nullptr; }
    return replay_or_enqueue(m, m->group_graph, whole_graph, key, max_steps, steps_done, static_cast<cudaStream_t>(stream),
                             [&](cudaStream_t s, int* done, bool in_capture) {
        return transcribe_group_enqueue(m, G, wav_dev, rel_len_dev, B, L, max_steps, bos, eos, pred_dev, done, s, in_capture);
    });
}

// Same pipeline from HOST buffers (pinned): the call EncoderDecoderASR.transcribe_batch makes, for G batches at once.
// Enqueue only; the caller synchronises `stream`.  pred_dev (optional, may be NULL or hold NULLs) also keeps the ids on the
// device (multi-GPU: the hypothesis all-gather reads them).
int sbk_asr_transcribe_greedy_group_host_async(sbk_asr* mm, int G, const float* const* wav_host,
                                               const float* const* rel_len_host, int B, int L, int max_steps, int bos, int eos,
                                               int* const* pred_host, int* const* pred_dev, int* steps_done, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(wav_host && rel_len_host && pred_host, "transcribe_group_host: null argument");
    RC(check_group_call(m, "transcribe_group_host", G, wav_host, rel_len_host, pred_host, B, L));
    RC(ensure_workspace(m, B, L, G * B, max_steps, group_encode_batches(m->wt->cfg, G, B, L) * B));
    RC(grow_buffer(m, m->gwav, (size_t)G * B * L * 4 + (size_t)G * B * 4 + 256, "transcribe_group_host"));
    RC(m->copy_stream.ensure());
    for (auto& e : m->ev_ready)
        if (!e) SBK_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    const bool whole_graph = m->poll_every == 0 && max_steps > 0;
    struct HostGroupKey { const void *wav[16], *rel[16], *pred[16], *pred_dev[16]; int G, B, L, steps, bos, eos; } key;
    memset(&key, 0, sizeof(key));
    key.G = G; key.B = B; key.L = L; key.steps = max_steps; key.bos = bos; key.eos = eos;
    for (int g = 0; g < G; ++g) {
        key.wav[g] = wav_host[g]; key.rel[g] = rel_len_host[g]; key.pred[g] = pred_host[g];
        key.pred_dev[g] = pred_dev ? pred_dev[g] : nullptr;
    }
    return replay_or_enqueue(m, m->hgroup_graph, whole_graph, key, max_steps, steps_done, static_cast<cudaStream_t>(stream),
                             [&](cudaStream_t s, int* done, bool in_capture) {
        return transcribe_group_host_enqueue(m, G, wav_host, rel_len_host, B, L, max_steps, bos, eos, pred_host, pred_dev, done, s,
                                             in_capture);
    });
}

int sbk_asr_transcribe_greedy_dev(sbk_asr* mm, const float* wav_dev, const float* rel_len_dev, int B, int L,
                                  int max_steps, int bos, int eos, float* enc_out_dev, int* pred_dev, float* score_dev,
                                  float* log_probs_dev, int* steps_done, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m->wt->has_fbank && m->wt->has_cnn && m->wt->has_enc, "transcribe: handle lacks fbank/CNN/encoder weights");
    SBK_REQUIRE(m->wt->glob_mean != nullptr, "transcribe: model has no normalize.glob_mean/std (global CMVN) weights");
    RC(ensure_workspace(m, B, L, B, max_steps));
    // Fixed-length runs (poll interval 0) replay ONE CUDA graph of the whole pipeline (Fbank .. last decode step):
    // ~2.6k kernel nodes, a single host-side launch per batch.
    const bool whole_graph = m->poll_every == 0 && rel_len_dev != nullptr && log_probs_dev == nullptr &&
                             (max_steps == 0 || m->wt->has_dec);
    struct PipeKey { const void *wav, *rel, *enc, *pred, *score; int B, L, steps, bos, eos; } key;
    memset(&key, 0, sizeof(key));  // the struct has tail padding and is compared bytewise
    key.wav = wav_dev; key.rel = rel_len_dev; key.enc = enc_out_dev; key.pred = pred_dev; key.score = score_dev;
    key.B = B; key.L = L; key.steps = max_steps; key.bos = bos; key.eos = eos;
    return replay_or_enqueue(m, m->pipe_graph, whole_graph, key, max_steps, steps_done, static_cast<cudaStream_t>(stream),
                             [&](cudaStream_t s, int* done, bool in_capture) {
        return transcribe_enqueue(m, wav_dev, rel_len_dev, B, L, max_steps, bos, eos, enc_out_dev, pred_dev, score_dev,
                                  log_probs_dev, done, s, in_capture);
    });
}

// Greedy search from caller-provided encoder states (S2STransformerGreedySearcher.forward).
int sbk_asr_greedy_from_enc(sbk_asr* mm, const float* enc_dev, const float* rel_len_dev, int B, int T, int max_steps,
                            int bos, int eos, int* pred_dev, float* score_dev, float* log_probs_dev, int* steps_done,
                            void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RC(ensure_workspace(m, B, enc_samples(m->wt->cfg, T), B, max_steps));
    AsrModel::Buf& b = m->b;
    RC(stage_enc(m, enc_dev, B, T, st));
    RC(set_enc_len(b.enc_len, rel_len_dev, B, T, st));
    int done = 0;
    RC(run_greedy(m, B, T, max_steps, bos, eos, log_probs_dev, &done, st));
    if (done > 0) {
        RC(copy_steps(m, pred_dev, max_steps, b.pred, done, B, cudaMemcpyDeviceToDevice, st));
        RC(copy_steps(m, score_dev, max_steps, b.score, done, B, cudaMemcpyDeviceToDevice, st));
    }
    if (steps_done) *steps_done = done;
    return SBK_OK;
}

// S2STransformerBeamSearcher.forward device part: history arrays are [max_steps, B * beam_size] (device).
int sbk_asr_beam_from_enc(sbk_asr* mm, const float* enc_dev, const float* rel_len_dev, int B, int T,
                          const sbk_beam_params* params, int* hist_tok_dev, int* hist_pred_dev, float* hist_score_dev,
                          float* hist_lp_dev, int* steps_done, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(params && params->beam_size >= 1, "beam: bad params");
    RC(ensure_workspace(m, B, enc_samples(m->wt->cfg, T), B * params->beam_size, params->max_steps));
    RC(stage_enc(m, enc_dev, B, T, st));
    RC(set_enc_len(m->b.enc_len, rel_len_dev, B, T, st));
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
    RC(ensure_workspace(m, B, L, B, max_steps));
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
    if (done > 0) {
        RC(copy_steps(m, pred_host, max_steps, b.pred, done, B, cudaMemcpyDeviceToHost, st));
        RC(copy_steps(m, score_host, max_steps, b.score, done, B, cudaMemcpyDeviceToHost, st));
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
    const sbk_asr_config& c = m->wt->cfg;
    SBK_REQUIRE(m->wt->w_ctc != nullptr, "ctc_head: this handle was created without ctc_lin.w.* weights");
    SBK_REQUIRE(B >= 1 && T >= 1 && (log_probs_dev || argmax_dev), "ctc_head: bad arguments");
    RC(ensure_workspace(m, B, enc_samples(c, T), B, 1));
    AsrModel::Buf& b = m->b;
    const size_t M = (size_t)B * T, V = c.vocab;
    if (enc_dev) RC(stage_enc(m, enc_dev, B, T, st));
    float* logits = log_probs_dev;
    if (!logits) {  // arg-max only: the logits live in the (lazily grown) CTC scratch buffer
        RC(grow_buffer(m, m->ctc, M * V * 4 + 256, "ctc_head"));
        logits = static_cast<float*>(m->ctc.base);
    }
    RC(cast_f32_f16(b.enc_out, b.enc16, M * c.d_model, st));
    GemmEpilogue e;
    e.mode = EPI_F32; e.bias = m->wt->b_ctc; e.out = logits; e.ldo = c.vocab;
    RC(gemm_f16(b.enc16, c.d_model, m->wt->w_ctc, c.d_model, e, (int)M, c.vocab, c.d_model, st));
    return rows_logsoftmax_argmax(logits, (int)M, c.vocab, log_probs_dev != nullptr, argmax_dev, st);
}

// TransformerASR.decode(tgt, encoder_out, enc_len) (TransformerASR.py:426-473): tgt_dev [n, S] int32 token ids (teacher
// forcing, bos first), enc_dev [n, T, d] fp32, enc_len_dev [n] int32 ABSOLUTE frame counts (or NULL = all T) ->
// out_dev [n, S, d] fp32 = decoder.norm(decoder(...)).  The attention-weight output of the reference is not produced.
int sbk_asr_decode_teacher_forced(sbk_asr* mm, const int* tgt_dev, const float* enc_dev, const int* enc_len_dev, int n, int S,
                                  int T, float* out_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(tgt_dev && enc_dev && out_dev && n >= 1 && S >= 1 && T >= 1, "decode: bad arguments");
    RC(ensure_workspace(m, n, enc_samples(m->wt->cfg, T), n, S));
    AsrModel::Buf& b = m->b;
    RC(stage_enc(m, enc_dev, n, T, st));
    if (enc_len_dev)
        SBK_CUDA_CHECK(cudaMemcpyAsync(b.enc_len, enc_len_dev, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    else
        RC(set_enc_len(b.enc_len, nullptr, n, T, st));
    return run_decode_teacher(m, tgt_dev, n, S, T, out_dev, st);
}

// TransformerLMRescorer.rescore_hyps device part: tokens [n, L] int32 (bos ... eos, pad-filled), lens [n] int32 (device) ->
// scores [n] fp32 (device) = sum over the sequence of log p(token | prefix) at `temperature`, pad column excluded.
int sbk_asr_lm_rescore(sbk_asr* mm, const int* tokens_dev, const int* lens_dev, int n, int L, float temperature, int pad_index,
                       float* scores_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(m->wt->has_lm, "lm_rescore: this handle was created without TransformerLM weights");
    SBK_REQUIRE(n >= 1 && L >= 2 && L <= m->wt->cfg.max_len && pad_index >= 0 && pad_index < m->wt->cfg.vocab && temperature > 0.0f,
                "lm_rescore: bad arguments (n=%d L=%d pad=%d)", n, L, pad_index);
    SBK_REQUIRE(pad_index == 0, "lm_rescore: pad_index must be 0 (TransformerLM.make_masks pads with index 0)");
    RC(ensure_workspace(m, 1, enc_samples(m->wt->cfg, 2), n, L));  // the LM reads no encoder states
    return run_lm_rescore(m, tokens_dev, lens_dev, n, L, temperature, pad_index, scores_dev, st);
}

// TransformerLM.forward(src) (TransformerLM.py:127-169): tokens_dev [n, s] int32 (pad id 0) -> logits_dev [n, s, vocab] fp32.
int sbk_asr_lm_forward(sbk_asr* mm, const int* tokens_dev, int n, int s, float* logits_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m != nullptr && tokens_dev && logits_dev, "lm_forward: null argument");
    SBK_REQUIRE(m->wt->has_lm, "lm_forward: this handle was created without TransformerLM weights");
    SBK_REQUIRE(n >= 1 && s >= 1, "lm_forward: bad shape n=%d s=%d", n, s);
    SBK_REQUIRE(n <= 65535, "lm_forward: n=%d sequences exceed the 65535 of one call (attention grid z)", n);
    SBK_REQUIRE(s <= m->wt->cfg.max_len, "lm_forward: s=%d exceeds max_len=%d", s, m->wt->cfg.max_len);
    SBK_REQUIRE((long long)n * s * std::max(m->wt->cfg.vocab, 3 * m->wt->lm_da) < (1LL << 31),
                "lm_forward: n * s = %lld token rows is too many for one call", (long long)n * s);
    return run_lm_forward(m, tokens_dev, n, s, logits_dev, static_cast<cudaStream_t>(stream));
}

// Step-by-step counterpart of sbk_asr_lm_forward on the KV-cached LM step: tokens_dev [n, L] -> logits_dev [n, L, vocab].
int sbk_asr_lm_step_logits(sbk_asr* mm, const int* tokens_dev, int n, int L, float* logits_dev, void* stream) {
    AsrModel* m = reinterpret_cast<AsrModel*>(mm);
    SBK_REQUIRE(m != nullptr && tokens_dev && logits_dev, "lm_step_logits: null argument");
    SBK_REQUIRE(m->wt->has_lm, "lm_step_logits: this handle was created without TransformerLM weights");
    SBK_REQUIRE(n >= 1 && L >= 1 && L <= m->wt->cfg.max_len, "lm_step_logits: bad shape n=%d L=%d (max_len %d)", n, L, m->wt->cfg.max_len);
    RC(ensure_workspace(m, 1, enc_samples(m->wt->cfg, 2), n, L));  // the LM reads no encoder states
    return run_lm_step_logits(m, tokens_dev, n, L, logits_dev, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
