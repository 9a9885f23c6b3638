// Transducer greedy search, sm_90a: TransducerBeamSearcher.transducer_greedy_decode (speechbrain/decoders/transducer.py
// :156-291) for the recipe prediction network Embedding -> 1-layer LSTM -> Linear(bias=False), the joint
// GELU(tn + out_PN) and the output Linear(bias=False) + log-softmax.
//
// Rows of the reference's batched frame loop are independent (a row that produced blank keeps identical inputs, so it
// keeps producing blank until the frame ends), so every row walks its own frames here: row b keeps a frame index t_b and
// a symbol count, and one ROUND advances every unfinished row by one decision.  A decision is blank (next frame) or a
// token; the (max_symbols_per_step + 1)-th token of a frame also ends the frame, as the reference's `count <= max` loop
// does.  Rounds per call = max_b (T + emitted_b).
//
// One persistent cooperative kernel runs the whole call, one CTA per SM, weight-stationary: CTA g keeps in shared memory
// (fp16) its contiguous slice of W_out rows (vocabulary), of W_hh (all four gates of its hidden units, so the cell update
// stays local) and of W_pd rows (joint units).  Per round:
//   A. z = GELU(tn[b, t_b] + p_b) for the live rows (fp32), the CTA's logits slice and its partial (max, first arg-max,
//      sum exp) per row -> global partials (double-buffered by round parity);
//   grid barrier;
//   B. every CTA reduces the G partials of every row in the same fixed order (so all CTAs agree on the decision without
//      another exchange), records the decision, and for the rows that emitted computes gates = U[tok] + W_hh h and the
//      cell update of its hidden units -> h_next, c;
//   grid barrier (only when some row emitted; the same in every CTA);
//   C. p = W_pd h_next for the emitting rows and the CTA's joint units; h <- h_next for its hidden units;
//   grid barrier.
// U[v] = W_ih E[v] + b_ih + b_hh ([V, 4H] fp32) is built once at create time and replaces the embedding lookup and the
// input product.  Reductions run in a fixed order and no values go through atomics: reruns are bit-identical and a row's
// results do not depend on the other rows of the batch.
//
// The beam search (transducer_beam_search_decode, decoders/transducer.py:320-476, no language model) is a second kernel on
// the same handle, weights and phases: one popped hypothesis per live utterance per round (see transducer_beam_kernel).
#include <cooperative_groups.h>

#include <climits>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "sbk_internal.h"
#include "transducer_merge.cuh"
#include "../../include/sbk.h"

namespace cg = cooperative_groups;

struct sbk_transducer {
    int V, E, H, J;
    int G;            // CTAs per call (one per SM)
    int nv, nh, nj;   // slice sizes per CTA (vocabulary rows, hidden units, joint rows)
    int device;
    float* U = nullptr;      // [V, 4H]
    __half* Whh = nullptr;   // [4H, H]
    __half* Wpd = nullptr;   // [J, H]
    __half* Wout = nullptr;  // [V, J]
};

namespace sbk {

namespace {

constexpr int TD_THREADS = 512;
constexpr int TD_NW = TD_THREADS / 32;
constexpr int TD_RB = 8;           // rows per phase-A chunk
constexpr int TD_MAX_B = 1024;
constexpr int TD_MAX_HJ = 1024;
constexpr int TD_MAX_V = 4096;
constexpr int TB_MAX_G = 256;      // CTAs the beam search's top-K merge follows (8 partial lists per lane)

struct TdArgs {
    const float* U; const __half* Whh; const __half* Wpd; const __half* Wout;
    const float* tn; int B, T, V, H, J, blank, maxsym, start;
    float* h; float* c; float* p; float* hn;
    float* pmax; int* parg; float* psum;   // [2][G][B]
    int* tokens; int* frames; long long tok_stride; int* ntok; float* lsum; int* stats;
    int nv, nh, nj;
};

__host__ __device__ inline size_t align16(size_t x) { return (x + 15) & ~size_t(15); }

struct TdSmem {
    size_t wout, whh, wpd, z, lg, st, total;
    __host__ __device__ TdSmem(int nv, int nh, int nj, int H, int J, int B) {
        wout = 0;
        whh = wout + align16(size_t(nv) * J * 2);
        wpd = whh + align16(size_t(4) * nh * H * 2);
        z = wpd + align16(size_t(nj) * H * 2);
        lg = z + align16(size_t(TD_RB) * J * 4);
        st = lg + align16(size_t(TD_RB) * (nv > 0 ? nv : 1) * 4);
        total = st + align16(size_t(B) * 20);
    }
};

// IEEE expf and division (sigmoid_f in common.cuh is the approximate one)
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// One prediction-network step of a row: the input token (< 0: the row does not step), the (h, c) it starts from and
// where the new (h, c) go.  The greedy search keeps one state per utterance, the beam search one slot per step.
struct PnRow {
    int tok;
    const float* h; const float* c;   // [H]
    float* h_out; float* c_out;       // [H]
};

// gates = U[tok] + W_hh h for this CTA's hidden units, then the LSTM cell (gate order i, f, g, o); rows(r) -> PnRow
template <class Rows>
__device__ void lstm_step(const float* U, const __half* sWhh, int nrows, int H, int u0, int nhl, Rows rows) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int pi = warp; pi < nrows * nhl; pi += TD_NW) {
        const int b = pi / nhl, u = pi - b * nhl;
        const PnRow row = rows(b);
        const int tok = row.tok;
        if (tok < 0) continue;
        const float* hb = row.h;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = lane * 2; k < H; k += 64) {
            const float2 hv = *reinterpret_cast<const float2*>(hb + k);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 w = __half22float2(*reinterpret_cast<const __half2*>(sWhh + size_t(u * 4 + q) * H + k));
                acc[q] = fmaf(w.x, hv.x, acc[q]);
                acc[q] = fmaf(w.y, hv.y, acc[q]);
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] = warp_sum(acc[q]);
        if (lane == 0) {
            const int unit = u0 + u;
            const float* Ur = U + size_t(tok) * 4 * H + unit;
            const float gi = sigmoidf_(Ur[0] + acc[0]);
            const float gf = sigmoidf_(Ur[H] + acc[1]);
            const float gg = tanhf(Ur[2 * H] + acc[2]);
            const float go = sigmoidf_(Ur[3 * H] + acc[3]);
            const float cn = gf * row.c[unit] + gi * gg;
            row.c_out[unit] = cn;
            row.h_out[unit] = go * tanhf(cn);
        }
    }
}

// p = W_pd h_next for this CTA's joint rows; rows(r) -> PnRow (h_out: the new h, c_out unused; tok < 0 skips), p(r) -> the
// row's out_PN [J]
template <class Rows, class POut>
__device__ void proj_step(const __half* sWpd, int nrows, int H, int j0, int njl, Rows rows, POut p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int pi = warp; pi < nrows * njl; pi += TD_NW) {
        const int b = pi / njl, j = pi - b * njl;
        const PnRow row = rows(b);
        if (row.tok < 0) continue;
        const float* hb = row.h_out;
        float acc = 0.f;
        for (int k = lane * 2; k < H; k += 64) {
            const float2 hv = *reinterpret_cast<const float2*>(hb + k);
            const float2 w = __half22float2(*reinterpret_cast<const __half2*>(sWpd + size_t(j) * H + k));
            acc = fmaf(w.x, hv.x, acc);
            acc = fmaf(w.y, hv.y, acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) p(b)[j0 + j] = acc;
    }
}

// The greedy search's rows: utterance b steps from (h, c) when it emitted st_tok[b] >= 0; the new h goes to h_next
struct GreedyRows {
    const TdArgs* a; const int* st_tok;
    __device__ PnRow operator()(int b) const {
        const size_t o = size_t(b) * a->H;
        return PnRow{st_tok[b], a->h + o, a->c + o, a->hn + o, a->c + o};
    }
};

__device__ void lstm_update(const TdArgs& a, const __half* sWhh, const int* st_tok, int u0, int nhl) {
    lstm_step(a.U, sWhh, a.B, a.H, u0, nhl, GreedyRows{&a, st_tok});
}

// p = W_pd h_next for this CTA's joint rows, and h <- h_next for its hidden units
__device__ void proj_update(const TdArgs& a, const __half* sWpd, const int* st_tok, int j0, int njl, int u0, int nhl) {
    const int H = a.H;
    proj_step(sWpd, a.B, H, j0, njl, GreedyRows{&a, st_tok}, [&](int b) { return a.p + size_t(b) * a.J; });
    for (int i = threadIdx.x; i < a.B * nhl; i += TD_THREADS) {
        const int b = i / nhl, u = i - b * nhl;
        if (st_tok[b] < 0) continue;
        const size_t o = size_t(b) * H + u0 + u;
        a.h[o] = a.hn[o];
    }
}

struct JointRow { const float* tn; const float* p; };   // tn null: the row is not live

// The CTA's logits slice sLg[r * nv + v] = W_out[v0 + v] . GELU(tn_b + p_b) for the rows b = rb0 + r < B of a TD_RB chunk;
// rows(b) -> JointRow.  Every thread of the CTA calls it; it ends with the slice in shared memory.
template <class Rows>
__device__ void joint_logits(const __half* sWout, float* sZ, float* sLg, int B, int J, int nv, int nvl, int rb0, Rows rows) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < TD_RB * J; i += TD_THREADS) {
        const int r = i / J, k = i - r * J, b = rb0 + r;
        if (b >= B) continue;
        const JointRow row = rows(b);
        if (row.tn) sZ[i] = gelu_erf_f(row.tn[k] + row.p[k]);
    }
    __syncthreads();
    for (int pi = warp; pi < TD_RB * nvl; pi += TD_NW) {
        const int r = pi / nvl, v = pi - r * nvl, b = rb0 + r;
        if (b >= B || !rows(b).tn) continue;
        float acc = 0.f;
        for (int k = lane * 2; k < J; k += 64) {
            const float2 z = *reinterpret_cast<const float2*>(sZ + r * J + k);
            const float2 w = __half22float2(*reinterpret_cast<const __half2*>(sWout + size_t(v) * J + k));
            acc = fmaf(w.x, z.x, acc);
            acc = fmaf(w.y, z.y, acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) sLg[r * nv + v] = acc;
    }
    __syncthreads();
}

// One warp: (max, first arg-max, sum exp(x - max)) of a row's logits slice x[0, nvl) at vocabulary offset v0
__device__ void slice_lse(const float* x, int nvl, int v0, float& m, int& am, float& s) {
    const int lane = threadIdx.x & 31;
    m = -INFINITY;
    am = td::NO_ARG;
    for (int v = lane; v < nvl; v += 32) {
        if (td::argmax_before(x[v], v0 + v, m, am)) { m = x[v]; am = v0 + v; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
        const int a2 = __shfl_xor_sync(0xffffffffu, am, o);
        if (td::argmax_before(m2, a2, m, am)) { m = m2; am = a2; }
    }
    s = 0.f;
    for (int v = lane; v < nvl; v += 32) s += expf(x[v] - m);
    s = warp_sum(s);
}

// One warp folds the G partials (max, arg-max, sum) of row b in a fixed order; every lane gets the result
__device__ void merge_lse(const float* pmax, const int* parg, const float* psum, int G, int B, int b, float& m, int& am,
                          float& s) {
    const int lane = threadIdx.x & 31;
    m = -INFINITY; s = 0.f;
    am = td::NO_ARG;
    for (int gg = lane; gg < G; gg += 32)
        td::lse_merge(m, am, s, pmax[size_t(gg) * B + b], parg[size_t(gg) * B + b], psum[size_t(gg) * B + b]);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float m2 = __shfl_down_sync(0xffffffffu, m, o);
        const int a2 = __shfl_down_sync(0xffffffffu, am, o);
        const float s2 = __shfl_down_sync(0xffffffffu, s, o);
        if ((lane & (2 * o - 1)) == 0) td::lse_merge(m, am, s, m2, a2, s2);
    }
    m = __shfl_sync(0xffffffffu, m, 0);
    am = __shfl_sync(0xffffffffu, am, 0);
    s = __shfl_sync(0xffffffffu, s, 0);
}

// the CTA's fp16 weight slices: W_out rows [v0, v0 + nvl), the four gate rows of hidden units [u0, u0 + nhl) (unit-major),
// W_pd rows [j0, j0 + njl)
__device__ void load_slices(const __half* Wout, const __half* Whh, const __half* Wpd, __half* sWout, __half* sWhh,
                            __half* sWpd, int H, int J, int v0, int nvl, int u0, int nhl, int j0, int njl) {
    const int tid = threadIdx.x;
    for (int i = tid; i < nvl * J; i += TD_THREADS) sWout[i] = Wout[size_t(v0) * J + i];
    for (int i = tid; i < 4 * nhl * H; i += TD_THREADS) {
        const int r = i / H, k = i - r * H, u = r >> 2, q = r & 3;
        sWhh[i] = Whh[size_t(q * H + u0 + u) * H + k];
    }
    for (int i = tid; i < njl * H; i += TD_THREADS) sWpd[i] = Wpd[size_t(j0) * H + i];
}

__global__ void __launch_bounds__(TD_THREADS, 1) transducer_greedy_kernel(TdArgs a) {
    cg::grid_group grid = cg::this_grid();
    extern __shared__ __align__(16) unsigned char smem[];
    const int G = gridDim.x, g = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int B = a.B, T = a.T, H = a.H, J = a.J, V = a.V;
    const TdSmem L(a.nv, a.nh, a.nj, H, J, B);
    __half* sWout = reinterpret_cast<__half*>(smem + L.wout);
    __half* sWhh = reinterpret_cast<__half*>(smem + L.whh);
    __half* sWpd = reinterpret_cast<__half*>(smem + L.wpd);
    float* sZ = reinterpret_cast<float*>(smem + L.z);
    float* sLg = reinterpret_cast<float*>(smem + L.lg);
    int* st_t = reinterpret_cast<int*>(smem + L.st);
    int* st_cnt = st_t + B;
    int* st_n = st_cnt + B;
    int* st_tok = st_n + B;
    float* st_sum = reinterpret_cast<float*>(st_tok + B);

    const int v0 = min(g * a.nv, V), nvl = min(v0 + a.nv, V) - v0;
    const int u0 = min(g * a.nh, H), nhl = min(u0 + a.nh, H) - u0;
    const int j0 = min(g * a.nj, J), njl = min(j0 + a.nj, J) - j0;

    load_slices(a.Wout, a.Whh, a.Wpd, sWout, sWhh, sWpd, H, J, v0, nvl, u0, nhl, j0, njl);
    for (int b = tid; b < B; b += TD_THREADS) {
        st_t[b] = 0; st_cnt[b] = 0; st_n[b] = 0; st_sum[b] = 0.f;
        st_tok[b] = a.start ? a.blank : -1;   // the start state is PN(blank) from a zero LSTM state
    }
    __syncthreads();
    int rounds = 0, barriers = 0;
    if (a.start) {
        lstm_update(a, sWhh, st_tok, u0, nhl);
        grid.sync();
        proj_update(a, sWpd, st_tok, j0, njl, u0, nhl);
        grid.sync();
        barriers += 2;
    }

    for (;;) {
        int live = 0;
        for (int b = tid; b < B; b += TD_THREADS) live |= st_t[b] < T;
        if (!__syncthreads_or(live)) break;
        const size_t pbuf = size_t(rounds & 1) * G * B;
        // ---- phase A: logits slice and partial log-sum-exp per live row
        for (int rb0 = 0; rb0 < B; rb0 += TD_RB) {
            joint_logits(sWout, sZ, sLg, B, J, a.nv, nvl, rb0, [&](int b) {
                return st_t[b] < T ? JointRow{a.tn + (size_t(b) * T + st_t[b]) * J, a.p + size_t(b) * J}
                                   : JointRow{nullptr, nullptr};
            });
            for (int r = warp; r < TD_RB; r += TD_NW) {
                const int b = rb0 + r;
                if (b >= B || st_t[b] >= T) continue;
                float m, s;
                int am;
                slice_lse(sLg + r * a.nv, nvl, v0, m, am, s);
                if (lane == 0) {
                    a.pmax[pbuf + size_t(g) * B + b] = m;
                    a.parg[pbuf + size_t(g) * B + b] = am;
                    a.psum[pbuf + size_t(g) * B + b] = s;
                }
            }
            __syncthreads();
        }
        grid.sync();
        ++barriers;
        // ---- phase B: every CTA takes the same decision per row from the G partials
        for (int b = warp; b < B; b += TD_NW) {
            if (st_t[b] >= T) {
                if (lane == 0) st_tok[b] = -1;
                continue;
            }
            float m, s;
            int am;
            merge_lse(a.pmax + pbuf, a.parg + pbuf, a.psum + pbuf, G, B, b, m, am, s);
            if (lane == 0) {
                const int tok = td::decision(m, am, V);   // a valid index even for a row of NaN logits
                const float lp = -logf(s);   // log_softmax at the arg-max: x_max - (x_max + log sum exp(x - x_max))
                if (tok != a.blank) {
                    if (g == 0) {
                        a.tokens[size_t(b) * a.tok_stride + st_n[b]] = tok;
                        if (a.frames) a.frames[size_t(b) * a.tok_stride + st_n[b]] = st_t[b];
                    }
                    st_n[b] += 1;
                    st_sum[b] += lp;
                    st_tok[b] = tok;
                    if (++st_cnt[b] > a.maxsym) { st_t[b] += 1; st_cnt[b] = 0; }
                } else {
                    st_tok[b] = -1;
                    st_t[b] += 1;
                    st_cnt[b] = 0;
                }
            }
        }
        ++rounds;
        int emit = 0;
        __syncthreads();
        for (int b = tid; b < B; b += TD_THREADS) emit |= st_tok[b] >= 0;
        if (__syncthreads_or(emit)) {
            lstm_update(a, sWhh, st_tok, u0, nhl);
            grid.sync();
            proj_update(a, sWpd, st_tok, j0, njl, u0, nhl);
            grid.sync();
            barriers += 2;
        }
    }
    if (g == 0) {
        for (int b = tid; b < B; b += TD_THREADS) {
            a.ntok[b] = st_n[b];
            a.lsum[b] = st_sum[b];
        }
        if (tid == 0 && a.stats) { a.stats[0] = rounds; a.stats[1] = barriers; }
    }
}

// ------------------------------------------------------------------------------------------------ beam search
// A hypothesis.  tok >= 0: a non-blank child not popped yet; its prediction is node's chain + tok and it needs a PN step
// on (tok, the (h, c) of slot), slot -1 being the zero state.  tok < 0: node is its whole prediction and slot holds the
// PN output and (h, c) of its last token (a popped hypothesis, or a blank child sharing its parent's step).
struct TbHyp { float score; int len, node, tok, slot; };

// Per-utterance bookkeeping, owned by CTA b % G
struct TbUtt {
    TbHyp cur;                 // the popped hypothesis of the round (node materialised, slot = its PN output)
    int t, nproc, nbeam, pf;   // frame, list sizes, pops in the frame
    int hyp, nnode, pops, pn_steps, cursor, done;
    int live[SBK_TRANSDUCER_BEAM_MAX];   // the slots of the hypotheses the frame started with
};

struct TbArgs {
    const float* U; const __half* Whh; const __half* Wpd; const __half* Wout;
    const float* tn; int B, T, V, H, J, blank, K, nbest, cap;
    float state_beam, expand_beam;
    int nv, nh, nj;
    int NS, NP, NN, R;            // slots, list entries and nodes per utterance; trace record stride
    float* slots;                 // [B][NS][2H + J]: h, c, out_PN
    const float* zero;            // [H] zeros: the start state
    float* pmax; int* parg; float* psum;   // [G][B]
    float* ptv; int* pti;         // [G][B][K]: the CTA's top-K logits of its vocabulary slice, and their token ids
    TbHyp* proc; TbHyp* beam;     // [B][NP], [B][K]
    int2* nodes;                  // [B][NN]: (token, parent node)
    TbUtt* utt;                   // [B]
    int4* rowd;                   // [B]: the round's row (PN token or -1, input slot, output slot, frame; T: done)
    int* out_tokens; int* out_lens; float* out_scores; int* trace; int* stats;
};

// the key of the reference's max / sort: score / len(prediction) in fp32
__device__ __forceinline__ float tb_key(const TbHyp& h) { return __fdiv_rn(h.score, float(h.len)); }

// One warp: the first of hyps[0, n) with the largest key (len 0: removed); every lane gets its index (-1: none)
__device__ int tb_argmax_key(const TbHyp* hyps, int n) {
    const int lane = threadIdx.x & 31;
    float bk = -INFINITY;
    int bi = INT_MAX;
    for (int i = lane; i < n; i += 32) {
        const TbHyp h = hyps[i];
        if (h.len <= 0) continue;
        const float k = tb_key(h);
        if (bi == INT_MAX || k > bk) { bk = k; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float k2 = __shfl_xor_sync(0xffffffffu, bk, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        if (i2 != INT_MAX && (bi == INT_MAX || k2 > bk || (k2 == bk && i2 < bi))) { bk = k2; bi = i2; }
    }
    return bi == INT_MAX ? -1 : bi;
}

// Pop hypothesis i of utterance b's list (lane 0): materialise its node, give it a new slot when it needs a PN step, and
// publish the row of the next round.  Returns false at the pop cap.
__device__ bool tb_pop(const TbArgs& a, int b, TbUtt& u, int i) {
    TbHyp* proc = a.proc + size_t(b) * a.NP;
    if (u.pf == a.cap || i < 0) return false;
    TbHyp h = proc[i];
    proc[i].len = 0;
    u.pf += 1; u.pops += 1; u.hyp = i;
    int4 row;
    if (h.tok >= 0) {
        int s = u.cursor;   // the next slot no hypothesis of the frame's start refers to
        for (bool used = true; used;) {
            used = false;
            for (int k = 0; k < a.K; ++k) used |= u.live[k] == s;
            s += used ? 1 : 0;
        }
        u.cursor = s + 1;
        a.nodes[size_t(b) * a.NN + u.nnode] = make_int2(h.tok, h.node);
        row = make_int4(h.tok, h.slot, s, u.t);
        h.node = u.nnode++;
        h.slot = s;
        u.pn_steps += 1;
    } else {
        row = make_int4(-1, -1, h.slot, u.t);
    }
    h.tok = -1;
    u.cur = h;
    a.rowd[b] = row;
    return true;
}

// Start a frame (lane 0): the list is the previous frame's beam, or the start hypothesis
__device__ void tb_start_frame(const TbArgs& a, int b, TbUtt& u) {
    TbHyp* proc = a.proc + size_t(b) * a.NP;
    const TbHyp* beam = a.beam + size_t(b) * a.K;
    if (u.t == 0) {
        proc[0] = TbHyp{0.f, 1, -1, a.blank, -1};
        u.nproc = 1;
    } else {
        for (int k = 0; k < u.nbeam; ++k) proc[k] = beam[k];
        u.nproc = u.nbeam;
    }
    for (int k = 0; k < a.K; ++k) u.live[k] = k < u.nproc ? proc[k].slot : -1;
    u.nbeam = 0; u.pf = 0; u.cursor = 0;
}

// The n-best of the last frame's beam, by key (stable), without the leading blank (one warp)
__device__ void tb_finish(const TbArgs& a, int b, const TbUtt& u) {
    const int lane = threadIdx.x & 31;
    const TbHyp* beam = a.beam + size_t(b) * a.K;
    const long long stride = (long long)a.T * a.cap;
    if (lane < u.nbeam) {
        const TbHyp h = beam[lane];
        const float k = tb_key(h);
        int rank = 0;
        for (int j = 0; j < u.nbeam; ++j) {
            const float kj = tb_key(beam[j]);
            rank += (kj > k || (kj == k && j < lane)) ? 1 : 0;
        }
        if (rank < a.nbest) {
            const size_t o = size_t(b) * a.nbest + rank;
            a.out_scores[o] = k;
            a.out_lens[o] = h.len - 1;
            int n = h.node;
            for (int pos = h.len - 2; pos >= 0; --pos) {
                const int2 nd = a.nodes[size_t(b) * a.NN + n];
                a.out_tokens[o * stride + pos] = nd.x;
                n = nd.y;
            }
        }
    }
    for (int r = u.nbeam + lane; r < a.nbest; r += 32) a.out_lens[size_t(b) * a.nbest + r] = -1;
}

// One warp: the round's decision for utterance b from the G partials -- top-K and log-softmax, children, then the next
// pop (or the frame's end: the beam is full, or its best raw score is state_beam above the best of the list)
__device__ void tb_bookkeep(const TbArgs& a, int b) {
    const int lane = threadIdx.x & 31, G = gridDim.x, K = a.K;
    TbUtt& u = a.utt[b];
    float m, s;
    int am;
    merge_lse(a.pmax, a.parg, a.psum, G, a.B, b, m, am, s);
    const float lse = logf(s);
    // top-K: merge the G sorted partial lists, (value desc, token asc); lane l follows lists l, l + 32, ...
    int head[TB_MAX_G / 32];
#pragma unroll
    for (int q = 0; q < TB_MAX_G / 32; ++q) head[q] = 0;
    float myx = 0.f;
    int mytok = 0;
    for (int k = 0; k < K; ++k) {
        float bx = -INFINITY;
        int bt = td::NO_ARG, bq = -1;
#pragma unroll
        for (int q = 0; q < TB_MAX_G / 32; ++q) {
            const int gg = lane + 32 * q;
            if (gg >= G || head[q] >= K) continue;
            const size_t o = (size_t(gg) * a.B + b) * K + head[q];
            const int t = a.pti[o];
            if (t == td::NO_ARG) continue;
            const float x = a.ptv[o];
            if (td::argmax_before(x, t, bx, bt)) { bx = x; bt = t; bq = q; }
        }
        int src = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float x2 = __shfl_xor_sync(0xffffffffu, bx, o);
            const int t2 = __shfl_xor_sync(0xffffffffu, bt, o);
            const int s2 = __shfl_xor_sync(0xffffffffu, src, o);
            if (td::argmax_before(x2, t2, bx, bt)) { bx = x2; bt = t2; src = s2; }
        }
        if (lane == src) {
#pragma unroll
            for (int q = 0; q < TB_MAX_G / 32; ++q) head[q] += q == bq ? 1 : 0;
        }
        if (lane == k) { myx = bx; mytok = bt; }
    }
    // log_softmax at the K tokens: x - max - log sum exp(x - max)
    const float lp = __fsub_rn(__fsub_rn(myx, m), lse);
    const int tok0 = __shfl_sync(0xffffffffu, mytok, 0);
    const float best = tok0 != a.blank ? __shfl_sync(0xffffffffu, lp, 0) : __shfl_sync(0xffffffffu, lp, 1);
    const TbHyp cur = u.cur;
    const bool in = lane < K;
    const bool is_blank = in && mytok == a.blank;
    const bool keep = in && !is_blank && lp >= __fsub_rn(best, a.expand_beam);
    const unsigned kmask = __ballot_sync(0xffffffffu, keep), bmask = __ballot_sync(0xffffffffu, is_blank);
    const float score = __fadd_rn(cur.score, lp);
    const int nproc = u.nproc, nbeam = u.nbeam;
    if (keep)
        a.proc[size_t(b) * a.NP + nproc + __popc(kmask & ((1u << lane) - 1u))] = TbHyp{score, cur.len + 1, cur.node, mytok,
                                                                                      cur.slot};
    if (is_blank) a.beam[size_t(b) * K + nbeam] = TbHyp{score, cur.len, cur.node, -1, cur.slot};
    int* rec = nullptr;
    if (a.trace) {
        rec = a.trace + (size_t(b) * a.T * a.cap + (u.pops - 1)) * a.R;
        if (in) { rec[6 + lane] = mytok; rec[6 + K + lane] = __float_as_int(lp); }
        if (lane == 0) {
            rec[0] = b; rec[1] = u.t; rec[2] = u.hyp; rec[3] = 0; rec[4] = int(kmask | bmask);
            rec[5] = __float_as_int(cur.score);
        }
    }
    __syncwarp();
    if (lane == 0) { u.nproc = nproc + __popc(kmask); u.nbeam = nbeam + (bmask ? 1 : 0); }
    __syncwarp();
    // the next pop
    for (;;) {
        int ended = 0, ia = -1;
        if (u.nbeam >= K) {
            ended = 2;
        } else {
            ia = tb_argmax_key(a.proc + size_t(b) * a.NP, u.nproc);
            if (u.nbeam > 0) {
                const int ib = tb_argmax_key(a.beam + size_t(b) * K, u.nbeam);
                if (a.beam[size_t(b) * K + ib].score >= __fadd_rn(a.state_beam, a.proc[size_t(b) * a.NP + ia].score))
                    ended = 1;
            }
        }
        bool capped = false;
        if (lane == 0 && !ended) capped = !tb_pop(a, b, u, ia);
        capped = __shfl_sync(0xffffffffu, capped, 0);
        if (capped) {
            if (lane == 0) {
                a.out_lens[size_t(b) * a.nbest] = -2 - u.t;
                for (int r = 1; r < a.nbest; ++r) a.out_lens[size_t(b) * a.nbest + r] = -1;
                u.done = 1;
                a.rowd[b] = make_int4(-1, -1, -1, a.T);
            }
            break;
        }
        if (!ended) break;
        if (lane == 0) {
            if (rec) rec[3] = ended;   // 1: the state_beam test, 2: the beam is full
            u.t += 1;
        }
        __syncwarp();
        if (u.t == a.T) {
            tb_finish(a, b, u);
            if (lane == 0) { u.done = 1; a.rowd[b] = make_int4(-1, -1, -1, a.T); }
            break;
        }
        if (lane == 0) tb_start_frame(a, b, u);
        __syncwarp();
    }
    __syncwarp();
}

// Per round: the PN step of the rows that need one (LSTM, grid barrier, projection, grid barrier), the joint and the CTA's
// logits slice with its partial log-sum-exp and top-K (grid barrier), then each utterance's bookkeeping by its owner CTA
// b % G (grid barrier).  One row per live utterance per round.
__global__ void __launch_bounds__(TD_THREADS, 1) transducer_beam_kernel(TbArgs a) {
    cg::grid_group grid = cg::this_grid();
    extern __shared__ __align__(16) unsigned char smem[];
    const int G = gridDim.x, g = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int B = a.B, T = a.T, H = a.H, J = a.J, V = a.V, K = a.K, SW = 2 * H + J;
    const TdSmem L(a.nv, a.nh, a.nj, H, J, B);
    __half* sWout = reinterpret_cast<__half*>(smem + L.wout);
    __half* sWhh = reinterpret_cast<__half*>(smem + L.whh);
    __half* sWpd = reinterpret_cast<__half*>(smem + L.wpd);
    float* sZ = reinterpret_cast<float*>(smem + L.z);
    float* sLg = reinterpret_cast<float*>(smem + L.lg);
    int4* st = reinterpret_cast<int4*>(smem + L.st);   // the rows of the round

    const int v0 = min(g * a.nv, V), nvl = min(v0 + a.nv, V) - v0;
    const int u0 = min(g * a.nh, H), nhl = min(u0 + a.nh, H) - u0;
    const int j0 = min(g * a.nj, J), njl = min(j0 + a.nj, J) - j0;
    load_slices(a.Wout, a.Whh, a.Wpd, sWout, sWhh, sWpd, H, J, v0, nvl, u0, nhl, j0, njl);
    if (warp == 0) {
        for (int b = g; b < B; b += G) {
            if (lane == 0) {
                TbUtt& u = a.utt[b];
                u.t = 0; u.nbeam = 0; u.nnode = 0; u.pops = 0; u.pn_steps = 0; u.done = 0;
                tb_start_frame(a, b, u);
                tb_pop(a, b, u, 0);
            }
        }
    }
    grid.sync();
    int rounds = 0, barriers = 1;
    auto slot = [&](int b, int s) { return a.slots + (size_t(b) * a.NS + s) * SW; };
    for (;;) {
        int live = 0, step = 0;
        for (int b = tid; b < B; b += TD_THREADS) {
            const int4 r = a.rowd[b];
            st[b] = r;
            live |= r.w < T;
            step |= r.w < T && r.x >= 0;
        }
        if (!__syncthreads_or(live)) break;
        if (__syncthreads_or(step)) {
            auto rows = [&](int b) {
                const int4 r = st[b];
                if (r.w >= T || r.x < 0) return PnRow{-1, nullptr, nullptr, nullptr, nullptr};
                const float* in = r.y < 0 ? nullptr : slot(b, r.y);
                float* out = slot(b, r.z);
                return PnRow{r.x, in ? in : a.zero, in ? in + H : a.zero, out, out + H};
            };
            lstm_step(a.U, sWhh, B, H, u0, nhl, rows);
            grid.sync();
            proj_step(sWpd, B, H, j0, njl, rows, [&](int b) { return slot(b, st[b].z) + 2 * H; });
            grid.sync();
            barriers += 2;
        }
        // ---- the joint, the logits slice, its partial log-sum-exp and top-K
        for (int rb0 = 0; rb0 < B; rb0 += TD_RB) {
            joint_logits(sWout, sZ, sLg, B, J, a.nv, nvl, rb0, [&](int b) {
                const int4 r = st[b];
                return r.w < T ? JointRow{a.tn + (size_t(b) * T + r.w) * J, slot(b, r.z) + 2 * H}
                               : JointRow{nullptr, nullptr};
            });
            for (int r = warp; r < TD_RB; r += TD_NW) {
                const int b = rb0 + r;
                if (b >= B || st[b].w >= T) continue;
                const float* x = sLg + r * a.nv;
                float m, s;
                int am;
                slice_lse(x, nvl, v0, m, am, s);
                const size_t o = size_t(g) * B + b;
                if (lane == 0) { a.pmax[o] = m; a.parg[o] = am; a.psum[o] = s; }
                // the slice's top-K in (value desc, token asc) order: each entry's rank is its count of predecessors
                for (int v = lane; v < nvl; v += 32) {
                    int rank = 0;
                    for (int w = 0; w < nvl; ++w) rank += td::argmax_before(x[w], v0 + w, x[v], v0 + v) ? 1 : 0;
                    if (rank < K) { a.ptv[o * K + rank] = x[v]; a.pti[o * K + rank] = v0 + v; }
                }
                for (int k = nvl + lane; k < K; k += 32) a.pti[o * K + k] = td::NO_ARG;
            }
            __syncthreads();
        }
        grid.sync();
        // ---- bookkeeping of the utterances this CTA owns
        if (warp == 0)
            for (int b = g; b < B; b += G)
                if (st[b].w < T) tb_bookkeep(a, b);
        ++rounds;
        grid.sync();
        barriers += 2;
    }
    if (g == 0 && tid == 0 && a.stats) {
        int pops = 0, steps = 0;
        for (int b = 0; b < B; ++b) { pops += a.utt[b].pops; steps += a.utt[b].pn_steps; }
        a.stats[0] = rounds; a.stats[1] = pops; a.stats[2] = steps; a.stats[3] = barriers;
    }
}

// U[v, r] = sum_e W_ih[r, e] E[v, e] + b_ih[r] + b_hh[r]  (fp32, 16 x 16 tiles; create time only)
__global__ void transducer_input_table_kernel(const float* E, const float* Wih, const float* bih, const float* bhh, float* U,
                                              int V, int R, int K) {
    __shared__ float sE[16][17], sW[16][17];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int v = blockIdx.y * 16 + ty, r = blockIdx.x * 16 + tx;
    float acc = 0.f;
    for (int k0 = 0; k0 < K; k0 += 16) {
        sE[ty][tx] = (v < V && k0 + tx < K) ? E[size_t(v) * K + k0 + tx] : 0.f;
        const int rw = blockIdx.x * 16 + ty;
        sW[ty][tx] = (rw < R && k0 + tx < K) ? Wih[size_t(rw) * K + k0 + tx] : 0.f;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) acc = fmaf(sE[ty][k], sW[tx][k], acc);
        __syncthreads();
    }
    if (v < V && r < R) U[size_t(v) * R + r] = acc + bih[r] + bhh[r];
}

const sbk_tensor* find_tensor(const sbk_tensor* w, int n, const char* name) {
    for (int i = 0; i < n; ++i)
        if (w[i].name && strcmp(w[i].name, name) == 0) return &w[i];
    return nullptr;
}

int upload_f16(const float* host, size_t n, __half** out) {
    std::vector<__half> tmp(n);
    for (size_t i = 0; i < n; ++i) tmp[i] = __float2half_rn(host[i]);
    SBK_CUDA_CHECK(cudaMalloc(out, n * sizeof(__half)));
    SBK_CUDA_CHECK(cudaMemcpy(*out, tmp.data(), n * sizeof(__half), cudaMemcpyHostToDevice));
    return SBK_OK;
}

void free_model(sbk_transducer* m) {
    if (!m) return;
    cudaFree(m->U); cudaFree(m->Whh); cudaFree(m->Wpd); cudaFree(m->Wout);
    delete m;
}

// The kernel's dynamic shared-memory limit is set to the device's opt-in maximum, the same value for every handle and
// call, so concurrent creates never lower it under another handle's needs; occupancy is checked at the largest batch.
int td_prepare_kernel(size_t smem_at_max_b, int smem_max) {
    SBK_CUDA_CHECK(cudaFuncSetAttribute(transducer_greedy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
    int occ = 0;
    SBK_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, transducer_greedy_kernel, TD_THREADS, smem_at_max_b));
    SBK_REQUIRE(occ >= 1, "transducer: the search kernel does not fit on an SM (%zu bytes of shared memory)", smem_at_max_b);
    SBK_CUDA_CHECK(cudaFuncSetAttribute(transducer_beam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
    SBK_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, transducer_beam_kernel, TD_THREADS, smem_at_max_b));
    SBK_REQUIRE(occ >= 1, "transducer: the beam search kernel does not fit on an SM (%zu bytes of shared memory)",
                smem_at_max_b);
    return SBK_OK;
}

}  // namespace

}  // namespace sbk

extern "C" {

int sbk_transducer_create(const sbk_transducer_config* cfg, const sbk_tensor* w, int n, sbk_transducer** out) {
    using namespace sbk;
    SBK_REQUIRE(cfg && w && out, "transducer: null pointer");
    *out = nullptr;
    const int V = cfg->vocab, E = cfg->emb_dim, H = cfg->hidden, J = cfg->joint;
    SBK_REQUIRE(V >= 2 && V <= TD_MAX_V, "transducer: vocabulary size %d outside [2, %d]", V, TD_MAX_V);
    SBK_REQUIRE(E >= 1, "transducer: embedding size %d", E);
    SBK_REQUIRE(H >= 64 && H <= TD_MAX_HJ && H % 64 == 0, "transducer: LSTM hidden size %d is not a multiple of 64 in [64, %d]",
                H, TD_MAX_HJ);
    SBK_REQUIRE(J >= 64 && J <= TD_MAX_HJ && J % 64 == 0, "transducer: joint size %d is not a multiple of 64 in [64, %d]", J,
                TD_MAX_HJ);
    struct Want { const char* name; int64_t numel; } want[] = {
        {"emb.weight", int64_t(V) * E}, {"lstm.weight_ih", int64_t(4) * H * E}, {"lstm.weight_hh", int64_t(4) * H * H},
        {"lstm.bias_ih", int64_t(4) * H}, {"lstm.bias_hh", int64_t(4) * H}, {"proj_dec.weight", int64_t(J) * H},
        {"out.weight", int64_t(V) * J}};
    const sbk_tensor* t[7];
    for (int i = 0; i < 7; ++i) {
        t[i] = find_tensor(w, n, want[i].name);
        SBK_REQUIRE(t[i] && t[i]->data, "transducer: weight %s missing", want[i].name);
        SBK_REQUIRE(t[i]->numel == want[i].numel, "transducer: weight %s has %lld elements, expected %lld", want[i].name,
                    (long long)t[i]->numel, (long long)want[i].numel);
    }
    int dev = 0, sms = 0, smem_max = 0;
    SBK_CUDA_CHECK(cudaGetDevice(&dev));
    SBK_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    SBK_CUDA_CHECK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const int G = sms;
    const int nv = (V + G - 1) / G, nh = (H + G - 1) / G, nj = (J + G - 1) / G;
    const TdSmem L(nv, nh, nj, H, J, TD_MAX_B);
    SBK_REQUIRE(L.total <= size_t(smem_max),
                "transducer: the fp16 weight slices need %zu bytes of shared memory per SM over %d SMs, above the %d available",
                L.total, G, smem_max);
    const int prc = td_prepare_kernel(L.total, smem_max);
    if (prc) return prc;
    sbk_transducer* m = new sbk_transducer();
    m->V = V; m->E = E; m->H = H; m->J = J; m->G = G; m->nv = nv; m->nh = nh; m->nj = nj; m->device = dev;
    int rc = upload_f16(t[2]->data, size_t(4) * H * H, &m->Whh);
    if (!rc) rc = upload_f16(t[5]->data, size_t(J) * H, &m->Wpd);
    if (!rc) rc = upload_f16(t[6]->data, size_t(V) * J, &m->Wout);
    if (rc) { free_model(m); return rc; }
    float *dE = nullptr, *dW = nullptr, *db = nullptr;
    cudaError_t e = cudaMalloc(&m->U, size_t(V) * 4 * H * 4);
    if (e == cudaSuccess) e = cudaMalloc(&dE, size_t(V) * E * 4);
    if (e == cudaSuccess) e = cudaMalloc(&dW, size_t(4) * H * E * 4);
    if (e == cudaSuccess) e = cudaMalloc(&db, size_t(8) * H * 4);
    if (e == cudaSuccess) e = cudaMemcpy(dE, t[0]->data, size_t(V) * E * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dW, t[1]->data, size_t(4) * H * E * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(db, t[3]->data, size_t(4) * H * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(db + 4 * H, t[4]->data, size_t(4) * H * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        dim3 grid((4 * H + 15) / 16, (V + 15) / 16), block(16, 16);
        transducer_input_table_kernel<<<grid, block>>>(dE, dW, db, db + 4 * H, m->U, V, 4 * H, E);
        count_launch();
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaFree(dE); cudaFree(dW); cudaFree(db);
    if (e != cudaSuccess) {
        free_model(m);
        SBK_CUDA_CHECK(e);
    }
    *out = m;
    return SBK_OK;
}

void sbk_transducer_destroy(sbk_transducer* m) { sbk::free_model(m); }

int sbk_transducer_info(const sbk_transducer* m, int* ctas, int* smem_bytes_at_b1) {
    using namespace sbk;
    SBK_REQUIRE(m && ctas && smem_bytes_at_b1, "transducer: null pointer");
    *ctas = m->G;
    *smem_bytes_at_b1 = int(TdSmem(m->nv, m->nh, m->nj, m->H, m->J, 1).total);
    return SBK_OK;
}

int sbk_transducer_greedy(sbk_transducer* m, const float* tn_dev, int B, int T, int blank, int max_symbols_per_step,
                          int start_from_blank, float* h_dev, float* c_dev, float* out_pn_dev, int* tokens_dev,
                          int* frames_dev, int* n_tokens_dev, float* logp_sum_dev, int* stats_dev, void* stream) {
    using namespace sbk;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(m && tn_dev && h_dev && c_dev && out_pn_dev && tokens_dev && n_tokens_dev && logp_sum_dev,
                "transducer: null pointer");
    SBK_REQUIRE(B >= 1 && B <= TD_MAX_B, "transducer: batch size %d outside [1, %d]", B, TD_MAX_B);
    SBK_REQUIRE(T >= 1, "transducer: %d frames", T);
    SBK_REQUIRE(blank >= 0 && blank < m->V, "transducer: blank index %d outside [0, %d)", blank, m->V);
    SBK_REQUIRE(max_symbols_per_step >= 0, "transducer: max_symbols_per_step %d < 0", max_symbols_per_step);
    int dev = 0;
    SBK_CUDA_CHECK(cudaGetDevice(&dev));
    SBK_REQUIRE(dev == m->device, "transducer: handle made on device %d, called on device %d", m->device, dev);
    const size_t smem = TdSmem(m->nv, m->nh, m->nj, m->H, m->J, B).total;   // <= the size checked at create time
    // partials [2][G][B] (max, arg-max, sum) and h_next [B, H]
    const size_t np = size_t(2) * m->G * B;
    char* ws = nullptr;
    const size_t ws_bytes = np * 12 + size_t(B) * m->H * 4;
    SBK_CUDA_CHECK(cudaMallocAsync(&ws, ws_bytes, st));
    if (start_from_blank) {
        cudaError_t e = cudaMemsetAsync(h_dev, 0, size_t(B) * m->H * 4, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(c_dev, 0, size_t(B) * m->H * 4, st);
        if (e != cudaSuccess) { cudaFreeAsync(ws, st); SBK_CUDA_CHECK(e); }
    }
    TdArgs a;
    a.U = m->U; a.Whh = m->Whh; a.Wpd = m->Wpd; a.Wout = m->Wout;
    a.tn = tn_dev; a.B = B; a.T = T; a.V = m->V; a.H = m->H; a.J = m->J; a.blank = blank; a.maxsym = max_symbols_per_step;
    a.start = start_from_blank ? 1 : 0;
    a.h = h_dev; a.c = c_dev; a.p = out_pn_dev;
    a.pmax = reinterpret_cast<float*>(ws); a.parg = reinterpret_cast<int*>(ws + np * 4);
    a.psum = reinterpret_cast<float*>(ws + np * 8); a.hn = reinterpret_cast<float*>(ws + np * 12);
    a.tokens = tokens_dev; a.frames = frames_dev; a.tok_stride = (long long)T * (max_symbols_per_step + 1); a.ntok = n_tokens_dev;
    a.lsum = logp_sum_dev; a.stats = stats_dev;
    a.nv = m->nv; a.nh = m->nh; a.nj = m->nj;
    void* args[] = {&a};
    cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(transducer_greedy_kernel), dim3(m->G),
                                                dim3(TD_THREADS), args, smem, st);
    count_launch();
    cudaFreeAsync(ws, st);
    SBK_CUDA_CHECK(e);
    SBK_CUDA_CHECK(cudaGetLastError());
    return SBK_OK;
}

int sbk_transducer_beam(sbk_transducer* m, const float* tn_dev, int B, int T, int blank, int beam_size, int nbest,
                        float state_beam, float expand_beam, int* out_tokens_dev, int* out_lens_dev, float* out_scores_dev,
                        int* trace_dev, int* stats_dev, void* stream) {
    using namespace sbk;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SBK_REQUIRE(m && tn_dev && out_tokens_dev && out_lens_dev && out_scores_dev, "transducer beam: null pointer");
    SBK_REQUIRE(B >= 1 && B <= TD_MAX_B, "transducer beam: batch size %d outside [1, %d]", B, TD_MAX_B);
    SBK_REQUIRE(T >= 1, "transducer beam: %d frames", T);
    SBK_REQUIRE(blank >= 0 && blank < m->V, "transducer beam: blank index %d outside [0, %d)", blank, m->V);
    SBK_REQUIRE(beam_size >= 2 && beam_size <= SBK_TRANSDUCER_BEAM_MAX, "transducer beam: beam_size %d outside [2, %d]",
                beam_size, SBK_TRANSDUCER_BEAM_MAX);
    SBK_REQUIRE(beam_size <= m->V, "transducer beam: beam_size %d above the vocabulary size %d", beam_size, m->V);
    SBK_REQUIRE(nbest >= 1 && nbest <= beam_size, "transducer beam: nbest %d outside [1, beam_size %d]", nbest, beam_size);
    SBK_REQUIRE(m->G <= TB_MAX_G, "transducer beam: %d CTAs, the top-K merge follows at most %d", m->G, TB_MAX_G);
    int dev = 0;
    SBK_CUDA_CHECK(cudaGetDevice(&dev));
    SBK_REQUIRE(dev == m->device, "transducer beam: handle made on device %d, called on device %d", m->device, dev);
    const int K = beam_size, cap = SBK_TRANSDUCER_BEAM_POP_CAP(beam_size);
    TbArgs a;
    a.U = m->U; a.Whh = m->Whh; a.Wpd = m->Wpd; a.Wout = m->Wout;
    a.tn = tn_dev; a.B = B; a.T = T; a.V = m->V; a.H = m->H; a.J = m->J; a.blank = blank; a.K = K; a.nbest = nbest;
    a.cap = cap; a.state_beam = state_beam; a.expand_beam = expand_beam;
    a.nv = m->nv; a.nh = m->nh; a.nj = m->nj;
    // per utterance: a slot per hypothesis of the frame's start (at most K, the previous beam) and per pop; the list holds
    // the frame's start and at most K children per pop (all K are tokens when blank is not in the pop's top K), with at
    // most cap pops per frame; a node per pop
    a.NS = K + cap; a.NP = K + cap * K; a.NN = T * cap + 1; a.R = 6 + 2 * K;
    const size_t G = m->G, slot_f = size_t(B) * a.NS * (2 * m->H + m->J), part = G * B;
    const size_t off_zero = slot_f * 4, off_p = align16(off_zero + size_t(m->H) * 4);
    const size_t off_top = align16(off_p + part * 12), off_proc = align16(off_top + part * K * 8);
    const size_t off_beam = align16(off_proc + size_t(B) * a.NP * sizeof(TbHyp));
    const size_t off_nodes = align16(off_beam + size_t(B) * K * sizeof(TbHyp));
    const size_t off_utt = align16(off_nodes + size_t(B) * a.NN * 8);
    const size_t off_row = align16(off_utt + size_t(B) * sizeof(TbUtt));
    const size_t ws_bytes = off_row + size_t(B) * 16;
    char* ws = nullptr;
    SBK_CUDA_CHECK(cudaMallocAsync(&ws, ws_bytes, st));
    a.slots = reinterpret_cast<float*>(ws); a.zero = reinterpret_cast<float*>(ws + off_zero);
    a.pmax = reinterpret_cast<float*>(ws + off_p); a.parg = reinterpret_cast<int*>(ws + off_p + part * 4);
    a.psum = reinterpret_cast<float*>(ws + off_p + part * 8);
    a.ptv = reinterpret_cast<float*>(ws + off_top); a.pti = reinterpret_cast<int*>(ws + off_top + part * K * 4);
    a.proc = reinterpret_cast<TbHyp*>(ws + off_proc); a.beam = reinterpret_cast<TbHyp*>(ws + off_beam);
    a.nodes = reinterpret_cast<int2*>(ws + off_nodes); a.utt = reinterpret_cast<TbUtt*>(ws + off_utt);
    a.rowd = reinterpret_cast<int4*>(ws + off_row);
    a.out_tokens = out_tokens_dev; a.out_lens = out_lens_dev; a.out_scores = out_scores_dev; a.trace = trace_dev;
    a.stats = stats_dev;
    cudaError_t e = cudaMemsetAsync(ws + off_zero, 0, size_t(m->H) * 4, st);
    if (e == cudaSuccess && trace_dev) e = cudaMemsetAsync(trace_dev, 0xff, size_t(B) * T * cap * a.R * 4, st);
    if (e == cudaSuccess) {
        const size_t smem = TdSmem(m->nv, m->nh, m->nj, m->H, m->J, B).total;   // <= the size checked at create time
        void* args[] = {&a};
        e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(transducer_beam_kernel), dim3(m->G), dim3(TD_THREADS), args,
                                        smem, st);
        count_launch();
    }
    cudaFreeAsync(ws, st);
    SBK_CUDA_CHECK(e);
    SBK_CUDA_CHECK(cudaGetLastError());
    return SBK_OK;
}

}  // extern "C"
