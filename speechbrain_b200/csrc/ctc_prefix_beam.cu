// CTC prefix beam search without a language model, sm_90a: the frame loop of CTCPrefixBeamSearcher.partial_decoding
// (speechbrain/decoders/ctc.py:1784-1905) with _get_new_beam (:1645-1782), CTCBeam.step (:487-492), the beam prune,
// sort_beams (:811-824) and _prune_history (:826-866).
//
// One persistent CTA per utterance walks all of that utterance's frames.  A beam carries polynomial hashes modulo
// 2^61 - 1 of its text, of its partial word and of the last whitespace-separated word of its text (for the history key),
// the string id and the index of its last token, and the prefix-search probabilities.  Per frame:
//   1. skip the frame if lp[blank] > log(blank_skip_threshold);
//   2. thread 0 replays CPython 3.12's set tables for set(np.where(lp > token_prune_min_logp)[0]) | {argmax}
//      & set(range(n_vocab)): the candidates are visited in that set's iteration order, which decides which (beam, token)
//      pair creates a text that two pairs reach and the order of the created beams;
//   3. thread 0 walks the (token, beam) pairs in the reference's order: the blank folds into the beam's n_p_b, a token
//      equal (as a string) to the last one folds p_nb + p into the beam's n_p_nb, then text + token is looked up among
//      all beams (open addressing on (text hash, length), first beam in list order), created on a miss, and receives
//      p_b + p or score + p.  The sums follow the reference's NumPy 2 types: score + p in float64 (float32 on the first
//      processed frame, where the score is still the Python 0.0), p_nb + p and p_b + p in float32;
//   4. every beam steps (score = logaddexp(p_b, p_nb) in float64), beams below max + beam_prune_logp go, the beam_size
//      best stay, ranked by (score desc, position asc) -- heapq.nlargest's stable order (prune_and_rank, ctc_search.cuh);
//      with prune_history only the first beam per (last word, partial word, last token) stays.
// The CTA writes, per processed frame, each surviving beam's origin (previous rank, token or -1 when carried over) and
// the final float64 scores; the host replays the texts and frames with exact strings (decoders/ctc.py in this package).
#include "ctc_search.cuh"
#include "sbk_internal.h"

namespace sbk {

namespace {

// per-token table columns (include/sbk.h)
enum { TI_KIND, TI_SID, TI_LLEN, TI_ALEN, TI_PLEN, TI_WS, TI_LEAD, TI_TAIL, TI_INNER, TI_N };
enum { TU_LHASH, TU_LPOW, TU_AHASH, TU_APOW, TU_PHASH, TU_LEADH, TU_LEADP, TU_TAILH, TU_INNERH, TU_N };
static_assert(TI_N == SBK_CTC_PREFIX_TOK_INTS && TU_N == SBK_CTC_PREFIX_TOK_WORDS, "token table width");

struct PBeam {
    uint64_t th, ph, rh, wh;           // hashes: text, partial word, trailing non-space run of the text, last word before it
    double p_b, p_nb, n_p_b, n_p_nb, score;
    int tl, pl, rl, wl;                // their lengths
    int sid, lidx;                     // string id and index of the last token (-1: None)
    int par, tok;                      // origin in this frame: rank at the previous frame, token (-1: carried over)
};

// np.logaddexp for float64 (npy_logaddexp)
__device__ __forceinline__ double logaddexp_np64(double x, double y) {
    if (x == y) return __dadd_rn(x, 0.693147180559945309417232121458176568);
    const double tmp = __dsub_rn(x, y);
    if (tmp > 0.0) return __dadd_rn(x, log1p(exp(-tmp)));
    if (tmp <= 0.0) return __dadd_rn(y, log1p(exp(tmp)));
    return tmp;
}
// np.logaddexp(python float, float32 value): both cast to float32
__device__ __forceinline__ double lae32(double a, float b) { return logaddexp_np(__double2float_rn(a), b); }

// ---- CPython 3.12 set tables for non-negative int keys (hash(v) == v), no deletions (Objects/setobject.c)
struct PySetT {
    int* t;       // slots, -1 = empty
    int* spare;   // the table a resize moves to
    int mask, used;
};

// set_add_entry / set_insert_clean probe sequence: the first slot holding v (when eq) or empty.  The table is never
// full (it grows at 60 % fill) and once perturb reaches 0 (after 7 rounds for 31-bit keys) i -> 5 i + 1 visits every slot,
// so the walk ends within 7 + mask + 1 rounds.
__device__ int set_probe(const int* t, int mask, int v, bool eq) {
    unsigned perturb = static_cast<unsigned>(v), i = static_cast<unsigned>(v) & static_cast<unsigned>(mask);
    for (int round = 0; round <= mask + 8; ++round) {
        const int n = static_cast<int>(i) + 9 <= mask ? 10 : 1;
        for (int j = 0; j < n; ++j) {
            const int e = t[i + j];
            if (e < 0 || (eq && e == v)) return static_cast<int>(i + j);
        }
        perturb >>= 5;
        i = (i * 5u + 1u + perturb) & static_cast<unsigned>(mask);
    }
    return -1;   // not reached
}

__device__ void set_init(PySetT& s, int* b0, int* b1) {
    s.t = b0; s.spare = b1; s.mask = 7; s.used = 0;
    for (int i = 0; i < 8; ++i) b0[i] = -1;
}

__device__ void set_resize(PySetT& s, int minused) {   // set_table_resize
    int size = 8;
    while (size <= minused) size <<= 1;
    int* nt = s.spare;
    for (int i = 0; i < size; ++i) nt[i] = -1;
    for (int i = 0; i <= s.mask; ++i)
        if (s.t[i] >= 0) nt[set_probe(nt, size - 1, s.t[i], false)] = s.t[i];
    s.spare = s.t; s.t = nt; s.mask = size - 1;
}

__device__ void set_add(PySetT& s, int v) {   // set_add_entry
    const int i = set_probe(s.t, s.mask, v, true);
    if (s.t[i] == v) return;
    s.t[i] = v;
    ++s.used;
    if (s.used * 5 >= s.mask * 3) set_resize(s, s.used > 50000 ? s.used * 2 : s.used * 4);
}

__device__ void set_merge(PySetT& s, const PySetT& o) {   // set_merge: set(o), s | o
    if (o.used == 0) return;
    if ((s.used + o.used) * 5 >= s.mask * 3) set_resize(s, (s.used + o.used) * 2);
    if (s.used == 0) {
        if (s.mask == o.mask) {
            for (int i = 0; i <= o.mask; ++i) s.t[i] = o.t[i];
        } else {
            for (int i = 0; i <= o.mask; ++i)
                if (o.t[i] >= 0) s.t[set_probe(s.t, s.mask, o.t[i], false)] = o.t[i];
        }
        s.used = o.used;
        return;
    }
    for (int i = 0; i <= o.mask; ++i)
        if (o.t[i] >= 0) set_add(s, o.t[i]);
}

// list(set(above) | {am} & set(range(nv))) -> ord; returns its length.  bufs: 4 tables of scap ints.
__device__ int candidate_order(const int* above, int nab, int am, int nv, const float* col, float thr, int* bufs, int scap,
                               int* ord) {
    PySetT a, u, m, r;
    set_init(a, bufs, bufs + scap);
    for (int k = 0; k < nab; ++k) set_add(a, above[k]);
    set_init(u, bufs + 2 * scap, bufs + 3 * scap);
    set_merge(u, a);
    int one[8];
    m.t = one; m.spare = nullptr; m.mask = 7; m.used = 1;
    for (int i = 0; i < 8; ++i) one[i] = -1;
    one[am & 7] = am;
    set_merge(u, m);
    set_init(r, bufs, bufs + scap);   // a is no longer needed
    if (nv > u.used) {   // set_intersection walks the smaller operand
        for (int i = 0; i <= u.mask; ++i)
            if (u.t[i] >= 0 && u.t[i] < nv) set_add(r, u.t[i]);
    } else {             // set(range(nv)) holds v in slot v: it is walked in ascending order
        for (int v = 0; v < nv; ++v)
            if (col[v] > thr || v == am) set_add(r, v);
    }
    int n = 0;
    for (int i = 0; i <= r.mask; ++i)
        if (r.t[i] >= 0) ord[n++] = r.t[i];
    return n;
}

// ---- beam lookup by (text hash, length): open addressing, first beam in list order wins
__device__ __forceinline__ uint32_t text_slot(uint64_t th, int tl) {
    uint64_t h = th * 0x9E3779B97F4A7C15ull ^ (static_cast<uint64_t>(tl) * 0xC2B2AE3D27D4EB4Full);
    h ^= h >> 29;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 32;
    return static_cast<uint32_t>(h);
}
// the table holds at most H / 2 beams, so a probe meets an empty slot within H steps
__device__ int text_find(const int* tab, int H, const PBeam* bm, uint64_t th, int tl, int* slot) {
    uint32_t s = text_slot(th, tl) & (H - 1);
    for (int k = 0; k < H; ++k) {
        const int e = tab[s];
        if (e < 0 || (bm[e].th == th && bm[e].tl == tl)) { *slot = static_cast<int>(s); return e; }
        s = (s + 1) & (H - 1);
    }
    *slot = -1;
    return -1;
}

// the beam _get_new_beam creates from o and token t at frame f
__device__ PBeam new_beam(const PBeam& o, int t, const int* ti, const uint64_t* tu) {
    PBeam n;
    n.th = hadd(hmul(o.th, tu[TU_APOW]), tu[TU_AHASH]);
    n.tl = o.tl + ti[TI_ALEN];
    if (!ti[TI_WS]) {   // the appended string has no whitespace: it extends the trailing run
        n.rh = hadd(hmul(o.rh, tu[TU_APOW]), tu[TU_AHASH]); n.rl = o.rl + ti[TI_ALEN];
        n.wh = o.wh; n.wl = o.wl;
    } else {            // run + lead ends a word, then the inner words, then the tail starts the new run
        const int l1 = o.rl + ti[TI_LEAD];
        n.wh = o.wh; n.wl = o.wl;
        if (l1 > 0) { n.wh = hadd(hmul(o.rh, tu[TU_LEADP]), tu[TU_LEADH]); n.wl = l1; }
        if (ti[TI_INNER] > 0) { n.wh = tu[TU_INNERH]; n.wl = ti[TI_INNER]; }
        n.rh = tu[TU_TAILH]; n.rl = ti[TI_TAIL];
    }
    const int kind = ti[TI_KIND];
    if (kind == SBK_CTC_TOK_SPACE) { n.ph = 0; n.pl = 0; }
    else if (kind == SBK_CTC_TOK_WORD) { n.ph = tu[TU_PHASH]; n.pl = ti[TI_PLEN]; }
    else if (t == o.lidx) { n.ph = o.ph; n.pl = o.pl; }
    else { n.ph = hadd(hmul(o.ph, tu[TU_LPOW]), tu[TU_LHASH]); n.pl = o.pl + ti[TI_LLEN]; }
    n.sid = ti[TI_SID]; n.lidx = t;
    n.p_b = n.p_nb = n.n_p_b = n.n_p_nb = n.score = -INFINITY;
    return n;
}

struct PbArgs {
    const float* lp; const int* lens;
    int T, V, nv;
    const int* tok_i; const uint64_t* tok_u;
    int blank, beam, prune_history;
    float tok_thr, skip_thr;
    double beam_thr;
    char* ws; size_t ws_stride; int bcap, hcap, scap;
    int* out_n; int* out_par; int* out_tok; double* out_score; int* out_final;
};

__host__ __device__ inline size_t pb_stride(int beam, int bcap, int hcap, int scap) {
    return cb_align(static_cast<size_t>(bcap) * sizeof(PBeam)) + cb_align(static_cast<size_t>(beam) * sizeof(PBeam)) +
           cb_align(static_cast<size_t>(bcap) * 8) + cb_align(static_cast<size_t>(hcap) * 4) + 4 * cb_align(static_cast<size_t>(scap) * 4);
}

__global__ void __launch_bounds__(CB_THREADS, 1) ctc_prefix_beam_kernel(const PbArgs a) {
    extern __shared__ int s_dyn[];
    int* s_above = s_dyn;          // [V] tokens above the threshold, ascending
    int* s_ord = s_dyn + a.V;      // [nv] candidate tokens in set order
    __shared__ int s_pos[CB_MAX_BEAM];
    __shared__ int s_w[CB_NW];
    __shared__ float s_f[CB_NW];
    __shared__ int s_i[CB_NW];
    const int b = blockIdx.x, tid = threadIdx.x, T = a.T, V = a.V, beam = a.beam;

    char* w = a.ws + static_cast<size_t>(b) * a.ws_stride;
    PBeam* bm = reinterpret_cast<PBeam*>(w); w += cb_align(static_cast<size_t>(a.bcap) * sizeof(PBeam));
    PBeam* nx = reinterpret_cast<PBeam*>(w); w += cb_align(static_cast<size_t>(beam) * sizeof(PBeam));
    uint64_t* key = reinterpret_cast<uint64_t*>(w); w += cb_align(static_cast<size_t>(a.bcap) * 8);
    int* tab = reinterpret_cast<int*>(w); w += cb_align(static_cast<size_t>(a.hcap) * 4);
    int* sets = reinterpret_cast<int*>(w);

    const int n = a.lens[b];
    int nb = 1;
    bool first = true;   // the start beam's score is the Python 0.0 until its first step
    if (tid == 0) {
        PBeam s;
        s.th = s.ph = s.rh = s.wh = 0;
        s.tl = s.pl = s.rl = s.wl = 0;
        s.sid = s.lidx = -1;
        s.p_b = 0.0; s.p_nb = s.n_p_b = s.n_p_nb = -INFINITY; s.score = 0.0;
        s.par = 0; s.tok = -1;
        bm[0] = s;
    }
    __syncthreads();

    for (int f = 0; f < n; ++f) {
        const float* col = a.lp + (static_cast<size_t>(b) * T + f) * V;
        int* on = a.out_n + static_cast<size_t>(b) * T + f;
        if (col[a.blank] > a.skip_thr) {   // skipped frames still count in the frame numbering
            if (tid == 0) *on = -1;
            continue;
        }
        // ---- 2. tokens above the threshold over all V columns (ascending) and the arg-max
        const int am = block_argmax(col, V, s_f, s_i);
        int nab = 0;
        for (int base = 0; base < V; base += CB_THREADS) {
            const int j = base + tid;
            const bool fl = j < V && col[j] > a.tok_thr;
            int tot;
            const int r = block_rank(fl, s_w, &tot);
            if (fl) s_above[nab + r] = j;
            nab += tot;
        }
        const int C = min(a.nv, nab + (col[am] > a.tok_thr ? 0 : 1)) * nb;   // candidate pairs, at most beam x pre-pass count
        int H = 64;
        while (H < 2 * (nb + C)) H <<= 1;
        for (int h = tid; h < H; h += CB_THREADS) tab[h] = -1;
        __syncthreads();
        // ---- 3. the extension, in the reference's order
        if (tid == 0) {
            const int ntok = candidate_order(s_above, nab, am, a.nv, col, a.tok_thr, sets, a.scap, s_ord);
            int slot;
            for (int i = 0; i < nb; ++i)
                if (text_find(tab, H, bm, bm[i].th, bm[i].tl, &slot) < 0) tab[slot] = i;
            int U = nb;
            for (int q = 0; q < ntok; ++q) {
                const int t = s_ord[q];
                const float p = col[t];
                const int* ti = a.tok_i + TI_N * t;
                const uint64_t* tu = a.tok_u + TU_N * t;
                for (int i = 0; i < nb; ++i) {
                    PBeam* o = bm + i;
                    const float sc32 = __fadd_rn(__double2float_rn(o->score), p);
                    const double sc = first ? static_cast<double>(sc32) : __dadd_rn(o->score, static_cast<double>(p));
                    if (t == a.blank) {
                        o->n_p_b = first ? lae32(o->n_p_b, sc32) : logaddexp_np64(o->n_p_b, sc);
                        continue;
                    }
                    if (ti[TI_SID] == o->sid) o->n_p_nb = lae32(o->n_p_nb, __fadd_rn(__double2float_rn(o->p_nb), p));
                    int j = text_find(tab, H, bm, hadd(hmul(o->th, tu[TU_LPOW]), tu[TU_LHASH]), o->tl + ti[TI_LLEN], &slot);
                    if (j < 0) {
                        j = U++;
                        PBeam nbm = new_beam(*o, t, ti, tu);
                        nbm.par = i; nbm.tok = t;
                        bm[j] = nbm;
                        if (text_find(tab, H, bm, nbm.th, nbm.tl, &slot) < 0) tab[slot] = j;   // a word start's text may exist
                    }
                    PBeam* d = bm + j;
                    if (t == o->lidx) {
                        if (o->p_b > -INFINITY) d->n_p_nb = lae32(d->n_p_nb, __fadd_rn(__double2float_rn(o->p_b), p));
                    } else {
                        d->n_p_nb = first ? lae32(d->n_p_nb, sc32) : logaddexp_np64(d->n_p_nb, sc);
                    }
                }
            }
            s_i[0] = U;
        }
        __syncthreads();
        const int U = s_i[0];
        __syncthreads();
        // ---- 4. step, prune: score >= max + beam_prune_logp, then the beam_size best (stable)
        double lmax = -INFINITY;
        for (int u = tid; u < U; u += CB_THREADS) {
            PBeam* x = bm + u;
            x->p_b = x->n_p_b; x->p_nb = x->n_p_nb;
            x->n_p_b = x->n_p_nb = -INFINITY;
            x->score = logaddexp_np64(x->p_b, x->p_nb);
            lmax = fmax(lmax, x->score);
        }
        const int nk = prune_and_rank(U, beam, lmax, a.beam_thr, [&](int u) { return bm[u].score; }, key, s_w, s_pos);
        PBeam me;
        if (tid < nk) {
            me = bm[s_pos[tid]];
            nx[tid] = me;
        }
        __syncthreads();
        // ---- history pruning: the first beam per (last word of the text, partial word, last token)
        bool keep = tid < nk;
        if (a.prune_history && keep) {
            const uint64_t mwh = me.rl > 0 ? me.rh : me.wh;
            const int mwl = me.rl > 0 ? me.rl : me.wl;
            for (int j = 0; j < tid; ++j) {
                const PBeam& o = nx[j];
                if ((o.rl > 0 ? o.rl : o.wl) == mwl && (o.rl > 0 ? o.rh : o.wh) == mwh && o.pl == me.pl && o.ph == me.ph &&
                    o.sid == me.sid) { keep = false; break; }
            }
        }
        int nfin;
        const int r = block_rank(keep, s_w, &nfin);   // (its barriers also separate the reads of bm above from the writes below)
        if (keep) {
            const size_t o = (static_cast<size_t>(b) * T + f) * beam + r;
            a.out_par[o] = me.par;
            a.out_tok[o] = me.tok;
            me.par = r; me.tok = -1;
            bm[r] = me;
        }
        if (tid == 0) *on = nfin;
        __syncthreads();
        nb = nfin;
        first = false;
    }
    if (tid < nb) a.out_score[static_cast<size_t>(b) * beam + tid] = bm[tid].score;
    if (tid == 0) a.out_final[b] = nb;
}

// Workspace shape from the pre-pass over all V columns: a frame has at most mt candidates, so at most beam * mt created
// beams; the set tables of mt + 1 keys stay below 8 (mt + 1) slots.
int pb_sizes(const float* lp, const int* lens, int B, int T, int V, int nv, const sbk_ctc_prefix_beam_params* p, cudaStream_t st,
             int* bcap, int* hcap, int* scap, size_t* stride) {
    int rc = ctc_check("ctc_prefix_beam", lp, lens, B, T, V, nv, p, st);
    if (rc) return rc;
    int mt = 0;
    rc = ctc_max_tokens(lp, lens, B, T, V, V, p->blank, p->token_prune_min_logp, p->blank_skip_logp, st, &mt);
    if (rc) return rc;
    *bcap = p->beam_size + std::max(1, mt) * p->beam_size;
    int h = 64;
    while (h < 2 * *bcap) h <<= 1;
    *hcap = h;
    int s = 8;
    while (s < 8 * (mt + 1)) s <<= 1;
    *scap = s;
    *stride = pb_stride(p->beam_size, *bcap, *hcap, *scap);
    return SBK_OK;
}

}  // namespace

}  // namespace sbk

extern "C" {

int sbk_ctc_prefix_beam_workspace_bytes(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                                        const sbk_ctc_prefix_beam_params* p, size_t* bytes, void* stream) {
    using namespace sbk;
    SBK_REQUIRE(bytes, "ctc_prefix_beam: null pointer");
    int bcap, hcap, scap;
    size_t stride;
    const int rc = pb_sizes(log_probs_dev, lens_dev, B, T, V, n_vocab, p, static_cast<cudaStream_t>(stream), &bcap, &hcap, &scap,
                            &stride);
    if (rc) return rc;
    *bytes = static_cast<size_t>(B) * stride;
    return SBK_OK;
}

int sbk_ctc_prefix_beam_search(const float* log_probs_dev, const int* lens_dev, int B, int T, int V, int n_vocab,
                               const int* tok_info_dev, const uint64_t* tok_hash_dev, const sbk_ctc_prefix_beam_params* p,
                               void* workspace_dev, size_t workspace_bytes, int* frame_beams_dev, int* parent_dev,
                               int* token_dev, double* score_dev, int* n_final_dev, void* stream) {
    using namespace sbk;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(tok_info_dev && tok_hash_dev && workspace_dev && frame_beams_dev && parent_dev && token_dev && score_dev &&
                n_final_dev, "ctc_prefix_beam: null pointer");
    int bcap, hcap, scap;
    size_t stride;
    const int rc = pb_sizes(log_probs_dev, lens_dev, B, T, V, n_vocab, p, st, &bcap, &hcap, &scap, &stride);
    if (rc) return rc;
    SBK_REQUIRE(workspace_bytes >= static_cast<size_t>(B) * stride,
                "ctc_prefix_beam: workspace of %zu bytes, this input needs %zu (sbk_ctc_prefix_beam_workspace_bytes)",
                workspace_bytes, static_cast<size_t>(B) * stride);
    static bool attr = false;
    if (!attr) {
        SBK_CUDA_CHECK(cudaFuncSetAttribute(ctc_prefix_beam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * CB_MAX_VOCAB * 4));
        attr = true;
    }
    PbArgs a;
    a.lp = log_probs_dev; a.lens = lens_dev; a.T = T; a.V = V; a.nv = n_vocab;
    a.tok_i = tok_info_dev; a.tok_u = tok_hash_dev;
    a.blank = p->blank; a.beam = p->beam_size; a.prune_history = p->prune_history ? 1 : 0;
    a.tok_thr = p->token_prune_min_logp; a.skip_thr = p->blank_skip_logp; a.beam_thr = p->beam_prune_logp;
    a.ws = static_cast<char*>(workspace_dev); a.ws_stride = stride; a.bcap = bcap; a.hcap = hcap; a.scap = scap;
    a.out_n = frame_beams_dev; a.out_par = parent_dev; a.out_tok = token_dev; a.out_score = score_dev; a.out_final = n_final_dev;
    ctc_prefix_beam_kernel<<<B, CB_THREADS, static_cast<size_t>(V + n_vocab) * 4, st>>>(a);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // extern "C"
