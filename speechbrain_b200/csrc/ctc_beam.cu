// CTC beam search without a language model, sm_90a: the frame loop of CTCBeamSearcher.partial_decoding
// (speechbrain/decoders/ctc.py:1298-1485) with merge_beams (:782-809), the beam prune and sort_beams (:811-824) and
// _prune_history (:826-866).
//
// One persistent CTA per utterance walks all of that utterance's frames.  The reference keys a beam by STRINGS
// (text, partial_word, last_token); here a beam carries polynomial hashes modulo 2^61 - 1 of its text and partial word
// together with their lengths, the string id of its last token (the first vocabulary index holding the same string) and
// the hash of the last word of its text (for the history pruning).  Per frame:
//   1. skip the frame if lp[blank] > log(blank_skip_threshold);
//   2. candidate tokens = {t < n_vocab : lp[t] > token_prune_min_logp} + argmax(lp), ascending;
//   3. candidates (token-major, beams in rank order inside a token) extend their parent by the string rules and write
//      their key and score to the workspace;
//   4. an open-addressing table merges equal keys: the merged beam keeps the FIRST candidate's position and the LAST
//      candidate's (parent, token), and its score folds the candidates' scores with np.logaddexp's float32 formula in
//      candidate order;
//   5. beams below max + beam_prune_logp go, the beam_size best stay, ranked by (score desc, position asc) --
//      heapq.nlargest's stable order (prune_and_rank, ctc_search.cuh);
//   6. with prune_history, only the first beam per (last word of the text, partial word, last token) stays.
// The CTA writes, per processed frame, the surviving beams' (parent, token) and their count, and the final scores; the
// host replays the token chains of the final beams with exact strings (decoders/ctc.py in this package).
#include "ctc_search.cuh"
#include "sbk_internal.h"

namespace sbk {

namespace {

constexpr uint64_t HSEP = 33;   // ' ': characters are hashed as code point + 1

struct BeamS {
    uint64_t th, ph, pp, wh;   // hash of text, of partial word, P^len(partial), hash of the text's last word
    int tl, pl, wl, sid;       // their lengths; string id of the last token (-1 = None)
};

// One candidate: beam s extended by token t (decoders/ctc.py:1359-1459).
__device__ __forceinline__ BeamS extend(const BeamS& s, int kind, int tsid, uint64_t thash, uint64_t tpow, int tlen) {
    BeamS n = s;
    n.sid = tsid;
    if (kind == SBK_CTC_TOK_BLANK || tsid == s.sid) return n;   // blank or repeated token: only the last token changes
    if (kind == SBK_CTC_TOK_WORD || kind == SBK_CTC_TOK_SPACE) {   // the partial word is committed: merge_tokens(text, partial)
        if (s.pl > 0) {
            if (s.tl == 0) { n.th = s.ph; n.tl = s.pl; }
            else { n.th = hadd(hmul(hadd(hmul(s.th, HBASE), HSEP), s.pp), s.ph); n.tl = s.tl + 1 + s.pl; }
            n.wh = s.ph; n.wl = s.pl;
        }
        if (kind == SBK_CTC_TOK_WORD) { n.ph = thash; n.pl = tlen; n.pp = tpow; }
        else { n.ph = 0; n.pl = 0; n.pp = 1; }
        return n;
    }
    n.ph = hadd(hmul(s.ph, tpow), thash);
    n.pl = s.pl + tlen;
    n.pp = hmul(s.pp, tpow);
    return n;
}

__device__ __forceinline__ uint32_t key_slot(uint64_t th, uint64_t ph, int tl, int pl, int sid) {
    uint64_t h = th * 0x9E3779B97F4A7C15ull;
    h ^= (ph + 0x632BE59BD9B4E019ull) * 0xC2B2AE3D27D4EB4Full;
    h ^= ((static_cast<uint64_t>(tl) << 40) ^ (static_cast<uint64_t>(pl) << 20) ^ static_cast<uint32_t>(sid)) * 0x165667B19E3779F9ull;
    h ^= h >> 29;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 32;
    return static_cast<uint32_t>(h);
}

struct CbArgs {
    const float* lp; const int* lens;
    int T, V, nv;
    const int* tok_i;          // [nv][3]: kind, string id, length of the appended string
    const uint64_t* tok_u;     // [nv][2]: hash of the appended string, P^length
    int blank, beam, prune_history;
    float tok_thr, beam_thr, skip_thr;
    char* ws; size_t ws_stride; int cmax, hcap;
    int* out_n; int* out_par; int* out_tok; float* out_score; int* out_final;
};

__host__ __device__ inline size_t cb_stride(int cmax, int hcap) {
    return 2 * cb_align(static_cast<size_t>(cmax) * 8) + 9 * cb_align(static_cast<size_t>(cmax) * 4) +
           3 * cb_align(static_cast<size_t>(hcap) * 4);
}

__global__ void __launch_bounds__(CB_THREADS, 1) ctc_beam_kernel(const CbArgs a) {
    extern __shared__ int s_tok[];   // [nv] candidate tokens of the frame, ascending
    __shared__ float s_sc[2][CB_MAX_BEAM];
    __shared__ uint64_t s_th[2][CB_MAX_BEAM], s_ph[2][CB_MAX_BEAM], s_pp[2][CB_MAX_BEAM], s_wh[2][CB_MAX_BEAM];
    __shared__ int s_tl[2][CB_MAX_BEAM], s_pl[2][CB_MAX_BEAM], s_wl[2][CB_MAX_BEAM], s_sid[2][CB_MAX_BEAM];
    __shared__ int s_pos[CB_MAX_BEAM];
    __shared__ int s_w[CB_NW];
    __shared__ float s_f[CB_NW];
    __shared__ int s_i[CB_NW];
    const int b = blockIdx.x, tid = threadIdx.x, T = a.T, V = a.V, beam = a.beam;

    // workspace of this utterance (layout: cb_stride)
    char* w = a.ws + static_cast<size_t>(b) * a.ws_stride;
    const size_t c8 = cb_align(static_cast<size_t>(a.cmax) * 8), c4 = cb_align(static_cast<size_t>(a.cmax) * 4);
    uint64_t* c_th = reinterpret_cast<uint64_t*>(w); w += c8;
    uint64_t* c_ph = reinterpret_cast<uint64_t*>(w); w += c8;
    float* c_sc = reinterpret_cast<float*>(w); w += c4;
    int* c_tl = reinterpret_cast<int*>(w); w += c4;
    int* c_pl = reinterpret_cast<int*>(w); w += c4;
    int* c_sid = reinterpret_cast<int*>(w); w += c4;
    int* c_slot = reinterpret_cast<int*>(w); w += c4;
    int* u_cand = reinterpret_cast<int*>(w); w += c4;
    int* u_last = reinterpret_cast<int*>(w); w += c4;
    float* u_sc = reinterpret_cast<float*>(w); w += c4;
    uint32_t* u_key = reinterpret_cast<uint32_t*>(w); w += c4;
    const size_t h4 = cb_align(static_cast<size_t>(a.hcap) * 4);
    int* tab_idx = reinterpret_cast<int*>(w); w += h4;
    int* tab_first = reinterpret_cast<int*>(w); w += h4;
    int* tab_last = reinterpret_cast<int*>(w);

    const int n = a.lens[b];
    int cur = 0, nb = 1;
    if (tid == 0) {
        s_sc[0][0] = 0.0f;
        s_th[0][0] = 0; s_ph[0][0] = 0; s_pp[0][0] = 1; s_wh[0][0] = 0;
        s_tl[0][0] = 0; s_pl[0][0] = 0; s_wl[0][0] = 0; s_sid[0][0] = -1;
    }
    __syncthreads();
    auto load = [&](int buf, int i) {
        BeamS s;
        s.th = s_th[buf][i]; s.ph = s_ph[buf][i]; s.pp = s_pp[buf][i]; s.wh = s_wh[buf][i];
        s.tl = s_tl[buf][i]; s.pl = s_pl[buf][i]; s.wl = s_wl[buf][i]; s.sid = s_sid[buf][i];
        return s;
    };
    auto store = [&](int buf, int i, const BeamS& s) {
        s_th[buf][i] = s.th; s_ph[buf][i] = s.ph; s_pp[buf][i] = s.pp; s_wh[buf][i] = s.wh;
        s_tl[buf][i] = s.tl; s_pl[buf][i] = s.pl; s_wl[buf][i] = s.wl; s_sid[buf][i] = s.sid;
    };
    auto extend_tok = [&](const BeamS& s, int t) {
        const int* ti = a.tok_i + 3 * t;
        return extend(s, ti[0], ti[1], a.tok_u[2 * t], a.tok_u[2 * t + 1], ti[2]);
    };

    for (int f = 0; f < n; ++f) {
        const float* col = a.lp + (static_cast<size_t>(b) * T + f) * V;
        int* on = a.out_n + static_cast<size_t>(b) * T + f;
        if (col[a.blank] > a.skip_thr) {   // skipped frames still count in the frame numbering
            if (tid == 0) *on = -1;
            continue;
        }
        // ---- 2. candidate tokens
        const int am = block_argmax(col, V, s_f, s_i);
        int ntok = 0;
        for (int base = 0; base < a.nv; base += CB_THREADS) {
            const int j = base + tid;
            const bool fl = j < a.nv && (col[j] > a.tok_thr || j == am);
            int tot;
            const int r = block_rank(fl, s_w, &tot);
            if (fl) s_tok[ntok + r] = j;
            ntok += tot;
        }
        if (ntok == 0) {   // the arg-max lies outside vocab_list and nothing passes the token threshold: no candidate
            if (tid == 0) { *on = -2; a.out_final[b] = -1; }
            return;
        }
        __syncthreads();
        // ---- 3. candidates, token-major
        const int C = ntok * nb;
        int H = 64;
        while (H < 2 * C) H <<= 1;
        for (int c = tid; c < C; c += CB_THREADS) {
            const int q = c / nb, p = c - q * nb, t = s_tok[q];
            const BeamS s = extend_tok(load(cur, p), t);
            c_th[c] = s.th; c_ph[c] = s.ph; c_tl[c] = s.tl; c_pl[c] = s.pl; c_sid[c] = s.sid;
            c_sc[c] = __fadd_rn(s_sc[cur][p], col[t]);
        }
        for (int h = tid; h < H; h += CB_THREADS) { tab_idx[h] = -1; tab_first[h] = 0x7fffffff; tab_last[h] = -1; }
        __syncthreads();
        // ---- 4. merge equal keys
        for (int c = tid; c < C; c += CB_THREADS) {
            const uint64_t th = c_th[c], ph = c_ph[c];
            const int tl = c_tl[c], pl = c_pl[c], sid = c_sid[c];
            uint32_t slot = key_slot(th, ph, tl, pl, sid) & (H - 1);
            for (;;) {
                const int o = atomicCAS(&tab_idx[slot], -1, c);
                if (o == -1 || (c_th[o] == th && c_ph[o] == ph && c_tl[o] == tl && c_pl[o] == pl && c_sid[o] == sid)) break;
                slot = (slot + 1) & (H - 1);
            }
            c_slot[c] = static_cast<int>(slot);
            atomicMin(&tab_first[slot], c);
            atomicMax(&tab_last[slot], c);
        }
        __syncthreads();
        int U = 0;
        for (int base = 0; base < C; base += CB_THREADS) {
            const int c = base + tid;
            const bool fl = c < C && tab_first[c_slot[c]] == c;
            int tot;
            const int r = block_rank(fl, s_w, &tot);
            if (fl) u_cand[U + r] = c;
            U += tot;
        }
        __syncthreads();
        float lmax = -INFINITY;
        for (int u = tid; u < U; u += CB_THREADS) {
            const int r = u_cand[u], slot = c_slot[r], last = tab_last[slot];
            float s = c_sc[r];
            for (int c = r + 1; c <= last; ++c)
                if (c_slot[c] == slot) s = logaddexp_np(s, c_sc[c]);
            u_sc[u] = s;
            u_last[u] = last;
            lmax = fmaxf(lmax, s);
        }
        // ---- 5. prune: score >= max + beam_prune_logp, then the beam_size best (stable)
        const int nk = prune_and_rank(U, beam, lmax, a.beam_thr, [&](int u) { return u_sc[u]; }, u_key, s_w, s_pos);
        // the kept beams in rank order: state from the LAST merged candidate's (parent, token)
        const int nxt = cur ^ 1;
        BeamS ns_state = {};
        float my_sc = 0.0f;
        int my_par = 0, my_tok = 0;
        if (tid < nk) {
            const int u = s_pos[tid], c = u_last[u];
            const int q = c / nb;
            my_par = c - q * nb;
            my_tok = s_tok[q];
            my_sc = u_sc[u];
            ns_state = extend_tok(load(cur, my_par), my_tok);
            store(nxt, tid, ns_state);
        }
        __syncthreads();
        // ---- 6. history pruning: the first beam per (last word of the text, partial word, last token)
        bool keep = tid < nk;
        if (a.prune_history && keep) {
            for (int j = 0; j < tid; ++j)
                if (s_wl[nxt][j] == ns_state.wl && s_wh[nxt][j] == ns_state.wh && s_pl[nxt][j] == ns_state.pl &&
                    s_ph[nxt][j] == ns_state.ph && s_sid[nxt][j] == ns_state.sid) { keep = false; break; }
        }
        int nfin;
        const int r = block_rank(keep, s_w, &nfin);   // (its barriers also separate the reads above from the writes below)
        if (keep) {
            store(nxt, r, ns_state);
            s_sc[nxt][r] = my_sc;
            const size_t o = (static_cast<size_t>(b) * T + f) * beam + r;
            a.out_par[o] = my_par;
            a.out_tok[o] = my_tok;
        }
        if (tid == 0) *on = nfin;
        __syncthreads();
        cur = nxt;
        nb = nfin;
    }
    if (tid < nb) a.out_score[static_cast<size_t>(b) * beam + tid] = s_sc[cur][tid];
    if (tid == 0) a.out_final[b] = nb;
}

// largest candidate-token count over the processed frames (synchronises the stream)
int cb_max_tokens(const float* lp, const int* lens, int B, int T, int V, int nv, const sbk_ctc_beam_params* p, cudaStream_t st,
                  int* out) {
    return ctc_max_tokens(lp, lens, B, T, V, nv, p->blank, p->token_prune_min_logp, p->blank_skip_logp, st, out);
}

void cb_sizes(int max_tok, int beam, int* cmax, int* hcap) {
    *cmax = std::max(1, max_tok * beam);
    int h = 64;
    while (h < 2 * *cmax) h <<= 1;
    *hcap = h;
}

}  // namespace

}  // namespace sbk

extern "C" {

int sbk_ctc_beam_workspace_bytes(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                                 const sbk_ctc_beam_params* p, size_t* bytes, void* stream) {
    using namespace sbk;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(bytes, "ctc_beam: null pointer");
    int rc = ctc_check("ctc_beam", log_probs_dev, lens_dev, B, T, V, n_vocab, p, st);
    if (rc) return rc;
    int mt = 0, cmax, hcap;
    rc = cb_max_tokens(log_probs_dev, lens_dev, B, T, V, n_vocab, p, st, &mt);
    if (rc) return rc;
    cb_sizes(mt, p->beam_size, &cmax, &hcap);
    *bytes = static_cast<size_t>(B) * cb_stride(cmax, hcap);
    return SBK_OK;
}

int sbk_ctc_beam_search(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                        const int* tok_info_dev, const uint64_t* tok_hash_dev, const sbk_ctc_beam_params* p,
                        void* workspace_dev, size_t workspace_bytes, int* frame_beams_dev, int* parent_dev, int* token_dev,
                        float* score_dev, int* n_final_dev, void* stream) {
    using namespace sbk;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(tok_info_dev && tok_hash_dev && workspace_dev && frame_beams_dev && parent_dev && token_dev && score_dev &&
                n_final_dev, "ctc_beam: null pointer");
    int rc = ctc_check("ctc_beam", log_probs_dev, lens_dev, B, T, V, n_vocab, p, st);
    if (rc) return rc;
    int mt = 0, cmax, hcap;
    rc = cb_max_tokens(log_probs_dev, lens_dev, B, T, V, n_vocab, p, st, &mt);
    if (rc) return rc;
    cb_sizes(mt, p->beam_size, &cmax, &hcap);
    const size_t stride = cb_stride(cmax, hcap);
    SBK_REQUIRE(workspace_bytes >= static_cast<size_t>(B) * stride,
                "ctc_beam: workspace of %zu bytes, this input needs %zu (sbk_ctc_beam_workspace_bytes)", workspace_bytes,
                static_cast<size_t>(B) * stride);
    static bool attr = false;
    if (!attr) {
        SBK_CUDA_CHECK(cudaFuncSetAttribute(ctc_beam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CB_MAX_VOCAB * 4));
        attr = true;
    }
    CbArgs a;
    a.lp = log_probs_dev; a.lens = lens_dev; a.T = T; a.V = V; a.nv = n_vocab;
    a.tok_i = tok_info_dev; a.tok_u = tok_hash_dev;
    a.blank = p->blank; a.beam = p->beam_size; a.prune_history = p->prune_history ? 1 : 0;
    a.tok_thr = p->token_prune_min_logp; a.beam_thr = p->beam_prune_logp; a.skip_thr = p->blank_skip_logp;
    a.ws = static_cast<char*>(workspace_dev); a.ws_stride = stride; a.cmax = cmax; a.hcap = hcap;
    a.out_n = frame_beams_dev; a.out_par = parent_dev; a.out_tok = token_dev; a.out_score = score_dev; a.out_final = n_final_dev;
    ctc_beam_kernel<<<B, CB_THREADS, static_cast<size_t>(n_vocab) * 4, st>>>(a);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // extern "C"
