// CTC prefix scorer for joint CTC/attention beam search (full-vocabulary scoring), sm_90a.
//
// Reference: speechbrain/decoders/ctc.py:46-295 (CTCPrefixScore.__init__/forward_step/permute_mem) driven by
// CTCScorer (decoders/scorer.py:183-249) as a *full* scorer of ScorerBuilder.score (:1221-1268), ctc_window_size = 0.
//
// The reference materialises the forward variables r (T, 2, n_bh, V) for EVERY candidate token at every step (1.3 GB
// at B=32, beam 4) and then gathers the `beam` survivors (permute_mem).  The score it returns, though, only needs
//   psi(h, c) = logsumexp_t( phi_h[t-1] + x[t, c] )        phi_h = the PARENT's forward variables (Alg.2-10/13),
// i.e. a log-semiring product [n_bh, T] x [T, V] per utterance.  Here it is evaluated in the linear domain: the
// posteriors are exponentiated once per utterance (xlin = exp(x), next to x), each hypothesis' phi is shifted by its
// own maximum and exponentiated once per step into shared memory, and thread (utterance, token) accumulates
// sum_t A_h[t] * xlin[t, c] for all the `beam` hypotheses of its utterance at once -- no transcendental in the inner
// loop, xlin read once per utterance per step (coalesced over the token axis) instead of once per hypothesis.  A sum
// that underflows (every term more than ~e^-69 below the row maximum) is redone for that one (hypothesis, token) in
// the log domain, so the result never depends on the fp32 exponent range.  Nothing of r is stored; after the beam
// kernel has picked the survivors, `ctc_update` runs the recurrence for just those n_bh (parent, token) pairs and
// writes their forward variables (T x 2 per hypothesis) for the next step.
//
// State per hypothesis row (ping-pong by step parity):  rsum[t] = logsumexp(r_nb[t], r_b[t]),  rb[t] = r_b[t],
// psi_prev = psi of the prefix itself.
#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

namespace {

constexpr float CTC_NEG = -1e20f;  // CTCPrefixScore.minus_inf (ctc.py:54)

// Frame of the eos column (Alg.2-3): the reference indexes r_sum with last_frame_index = enc_len - 1 as a Python index, so
// enc_len = 0 reads the last frame T - 1 (never the element before the hypothesis' row).
__device__ __forceinline__ int ctc_eos_frame(int enc_len, int T) { return enc_len > 0 ? enc_len - 1 : T - 1; }

// log(exp(a) + exp(b))
__device__ __forceinline__ float logaddexp_acc(float a, float b) {
    const float m = fmaxf(a, b);
    return m + log1pf(expf(-fabsf(a - b)));
}

// In place: x[b, t, :] = log_softmax(x[b, t, :]); frames t >= enc_len[b]: minus_inf everywhere, 0 at index 0
// (ctc.py:59-62 hard-codes channel 0 there); xb[b, t] = x[b, t, blank].
__global__ void __launch_bounds__(256)
ctc_logsoftmax_mask_kernel(float* __restrict__ x, float* __restrict__ xlin, float* __restrict__ xb,
                           const int* __restrict__ enc_len, int T, int V, int blank) {
    __shared__ float s_red[8];
    const int row = blockIdx.x, b = row / T, t = row - b * T, tid = threadIdx.x;
    float* xr = x + static_cast<size_t>(row) * V;
    float* xl = xlin + static_cast<size_t>(row) * V;
    if (t >= enc_len[b]) {
        for (int j = tid; j < V; j += 256) { xr[j] = (j == 0) ? 0.0f : CTC_NEG; xl[j] = (j == 0) ? 1.0f : 0.0f; }
        if (tid == 0) xb[row] = (blank == 0) ? 0.0f : CTC_NEG;
        return;
    }
    float mx = -INFINITY;
    for (int j = tid; j < V; j += 256) mx = fmaxf(mx, xr[j]);
    mx = warp_max(mx);
    if ((tid & 31) == 0) s_red[tid >> 5] = mx;
    __syncthreads();
    mx = s_red[0];
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w]);
    __syncthreads();
    float sm = 0.0f;
    for (int j = tid; j < V; j += 256) sm += expf(xr[j] - mx);
    sm = warp_sum(sm);
    if ((tid & 31) == 0) s_red[tid >> 5] = sm;
    __syncthreads();
    float tot = 0.0f;
    for (int w = 0; w < 8; ++w) tot += s_red[w];
    const float lse = mx + logf(tot);
    for (int j = tid; j < V; j += 256) {
        const float v = xr[j] - lse;
        xr[j] = v;
        xl[j] = expf(v);
        if (j == blank) xb[row] = v;
    }
}

// The score kernel's operand of one hypothesis for the step that extends it: A[var][t] = exp(phi_var[t-1] - M_var) for the
// frames t >= t_lo of the sum (Alg.2-13), phi_0 = logsumexp(r_nb, r_b), phi_1 = r_b (Alg.2-10), M_var the maximum exponent; at
// step 0 the seed psi_init = x[0, c] (Alg.2-6) is the extra term A[.][0] = exp(-M) with M >= 0.  Written by the kernel that
// produces the hypothesis' forward variables (ctc_init / ctc_update: one CTA per hypothesis, off the search step's critical
// path), chunk-major per group of R hypotheses: tab[group][var][t / 4][h][t % 4], tabM[group][var][h] -- the score kernel
// pulls a group's table with one bulk copy (built inside the score kernel it was 45 % of that kernel, 20 x per utterance).
__device__ __forceinline__ void ctc_write_tables(const float* s_rsum, const float* s_rb, int T, int t_lo, float* tab, float* tabM,
                                                 int R, int row, float* s_red /*[8]*/) {
    const int Tp = (T + 3) & ~3, NC = Tp >> 2, g = row / R, h = row - g * R;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    float* tg = tab + static_cast<size_t>(g) * 2 * NC * R * 4;
    for (int var = 0; var < 2; ++var) {
        const float* phi = var ? s_rb : s_rsum;
        float mx = t_lo == 0 ? 0.0f : -INFINITY;
        for (int t = max(t_lo, 1) + threadIdx.x; t < T; t += blockDim.x) mx = fmaxf(mx, phi[t - 1]);
        mx = warp_max(mx);
        __syncthreads();
        if (lane == 0) s_red[warp] = mx;
        __syncthreads();
        float M = s_red[0];
        for (int w = 1; w < nw; ++w) M = fmaxf(M, s_red[w]);
        if (threadIdx.x == 0) tabM[static_cast<size_t>(g) * 2 * R + var * R + h] = M;
        for (int t = threadIdx.x; t < Tp; t += blockDim.x) {
            float v = 0.0f;
            if (t < T && t >= t_lo) v = t == 0 ? __expf(-M) : __expf(phi[t - 1] - M);
            tg[((static_cast<size_t>(var) * NC + (t >> 2)) * R + h) * 4 + (t & 3)] = v;
        }
    }
}

// states = None (ctc.py:112-126): r_nb = minus_inf, r_b[t] = cumsum_t x[t, blank]; psi_prev = 0.
__global__ void ctc_init_kernel(const float* __restrict__ xb, int T, int beam, float* __restrict__ rsum,
                                float* __restrict__ rb, float* __restrict__ psi_prev, float* __restrict__ tab,
                                float* __restrict__ tabM, int R) {
    extern __shared__ float s_cum[];   // [T] r_b, [T] rsum
    __shared__ float s_red[8];
    float* s_rs = s_cum + T;
    const int row = blockIdx.x, b = row / beam;
    if (threadIdx.x == 0) {
        float acc = 0.0f;
        for (int t = 0; t < T; ++t) { acc += xb[static_cast<size_t>(b) * T + t]; s_cum[t] = acc; }
        psi_prev[row] = 0.0f;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float rs = logaddexp_acc(CTC_NEG, s_cum[t]);
        rb[static_cast<size_t>(row) * T + t] = s_cum[t];
        rsum[static_cast<size_t>(row) * T + t] = rs;
        s_rs[t] = rs;
    }
    __syncthreads();
    ctc_write_tables(s_rs, s_cum, T, 0, tab, tabM, R, row, s_red);
}

// The step index comes from DEVICE memory (the beam search's per-row step counters) so that one captured CUDA graph of a
// whole search step can be replayed for every step; the ping-pong halves of the state follow the step's parity.
struct CtcArgs {
    const float* x; const float* xb;         // [B, T, V], [B, T]
    const float* xlin;                       // exp(x)
    float* rsum_base; float* rb_base;        // [2][n_bh, T]: half (step & 1) holds the prefixes being extended
    float* psi_base;                         // [2][n_bh]
    const int* enc_len;                      // [B]
    const int* hist_tok; const int* hist_pred;  // beam history [steps, n_bh]
    const int* step_ptr; int step_adj;       // step = step_ptr[row] + step_adj (the update runs after the counters advanced)
    int n_bh, bos, T, V, beam, blank, eos;
    float weight; float* out; int accumulate;   // score kernel: out[n_bh, V] (+)= weight * (psi - psi_prev)
    float* tab; float* tabM; int R;            // score-kernel operand tables (ctc_write_tables)
};

// forward_step (ctc.py:80-249), candidates = None, for the R hypotheses blockIdx.y * R .. + R of one utterance (R divides
// the beam width) and 128 tokens.  Shared memory: A[2][R][Tp] -- variant 0 from rsum (Alg.2-10, c != last token), variant 1
// from r_b (c == last token); A[.][h][t] = exp(phi_h[t-1] - M_h) for t >= max(step, 1), and at step 0 the seed
// psi_init = x[0, c] (Alg.2-6) is the extra term A[.][h][0] = exp(-M_h) of the same sum.
// One CTA = CTC_TOK = 256 tokens x the R hypotheses of an utterance; every thread accumulates CTC_TPT tokens (c, c + 128) for
// all R hypotheses, so one 16-byte broadcast read of A feeds 4 * CTC_TPT FMAs.  The CTA's [T x 256] panel of exp(x) is
// STREAMED through a shared-memory ring by bulk copies (one 1 KB row segment per copy, CTC_STAGE_ROWS rows per stage,
// CTC_STAGES stages in flight, the first ones issued at kernel entry); the A tables arrive by ONE bulk copy from where
// ctc_init / ctc_update left them.
// History of this kernel: thread per (hypothesis, token) log-domain recurrence (L2-bound: x re-read per hypothesis, one ex2
// per term) -> linear domain; the prologue that built the operand tables (two passes with integer divisions over 2 R T
// elements, redone by all 20 CTAs of an utterance) then dominated, so the tables moved to the kernels that produce the
// forward variables.
// Every token uses the `rsum` table in the main loop; the one token per hypothesis that equals its last token (Alg.2-10:
// phi = r_b instead) is recomputed from the second table by one warp of CTA column 0.
constexpr int CTC_THREADS = 128;
constexpr int CTC_TPT = 2;
constexpr int CTC_TOK = CTC_THREADS * CTC_TPT;
constexpr int CTC_STAGE_ROWS = 16;
constexpr int CTC_STAGES = 3;
constexpr int CTC_RING_FLOATS = CTC_STAGES * CTC_STAGE_ROWS * CTC_TOK;

// The same sum in the log domain, for a (hypothesis, token) whose linear-domain sum left the fp32 range (rare; keeps the
// result range-independent): Alg.2-6 / 2-13 with an online log-sum-exp.
__device__ __noinline__ float ctc_psi_logdomain(const CtcArgs& a, int b, int c, int step, const float* phi_row) {
    const int T = a.T, V = a.V;
    const float* xg = a.x + static_cast<size_t>(b) * T * V + c;
    float pm, ps = 1.0f;
    int start;
    if (step == 0) { pm = xg[0]; start = 1; } else { pm = CTC_NEG; start = step; }
    for (int t = start; t < T; ++t) {
        const float term = phi_row[t - 1] + xg[static_cast<size_t>(t) * V];
        if (term > pm) { ps = ps * __expf(pm - term) + 1.0f; pm = term; }
        else ps += __expf(term - pm);
    }
    return pm + __logf(ps);
}
// psi -> weighted score -> out (the last-token path)
__device__ __forceinline__ void ctc_emit(const CtcArgs& a, int row, int b, int c, int step, float acc, float M, const float* phi_row,
                                         const float* rsum_row, float psi_prev) {
    float psi;
    if (c == a.blank && a.eos != a.blank) psi = CTC_NEG;
    else if (c == a.eos) psi = rsum_row[ctc_eos_frame(a.enc_len[b], a.T)];   // Alg.2-3
    else if (acc > 1e-30f) psi = M + __logf(acc);
    else psi = ctc_psi_logdomain(a, b, c, step, phi_row);
    const float sc = a.weight * (psi - psi_prev);
    float* o = a.out + static_cast<size_t>(row) * a.V + c;
    *o = a.accumulate ? *o + sc : sc;
}

template <int R>
__global__ void __launch_bounds__(CTC_THREADS) ctc_score_kernel(const CtcArgs a) {
    extern __shared__ __align__(16) float smem[];
    __shared__ float s_M[2][R];
    __shared__ int s_last[R];
    __shared__ uint64_t s_full[CTC_STAGES];
    __shared__ uint64_t s_tabbar;
    constexpr int NT = CTC_THREADS;
    const int T = a.T, V = a.V, Tp = (T + 3) & ~3, NC = Tp >> 2;
    // A tables, chunk-major: s_A[var][chunk][h] is the float4 of frames 4*chunk .. +3 of hypothesis h
    float4* s_A = reinterpret_cast<float4*>(smem);
    float* s_ring = smem + 2 * R * Tp;   // [CTC_STAGES][CTC_STAGE_ROWS][CTC_TOK]
    const int row0 = blockIdx.y * R, b = row0 / a.beam;
    const int step = a.step_ptr[row0] + a.step_adj;
    const size_t half = static_cast<size_t>(step & 1);
    const float* rsum_in = a.rsum_base + half * a.n_bh * T;
    const float* rb_in = a.rb_base + half * a.n_bh * T;
    const float* psi_prev = a.psi_base + half * a.n_bh;
    const int t_lo = step == 0 ? 0 : step;   // first term of the sum
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int c_base = blockIdx.x * CTC_TOK;
    const int r0 = t_lo & ~3;                                        // first frame streamed (chunk-aligned)
    const int n_st = (T - r0 + CTC_STAGE_ROWS - 1) / CTC_STAGE_ROWS;  // stages of CTC_STAGE_ROWS frames
    const bool bulk = (V & 3) == 0;                                   // 16-byte aligned row segments
    const float* xu = a.xlin + static_cast<size_t>(b) * T * V;
    const uint32_t seg_bytes = static_cast<uint32_t>(min(CTC_TOK, V - c_base)) * 4u;
    auto issue_stage = [&](int i) {   // thread 0: frames r0 + 16 i .. of this CTA's token columns -> ring slot i % CTC_STAGES
        const int s = i % CTC_STAGES, t_begin = r0 + i * CTC_STAGE_ROWS;
        const int rows = min(CTC_STAGE_ROWS, T - t_begin);
        mbar_arrive_expect_tx(&s_full[s], seg_bytes * static_cast<uint32_t>(rows));
        for (int r = 0; r < rows; ++r)
            bulk_load_1d(s_ring + (static_cast<size_t>(s) * CTC_STAGE_ROWS + r) * CTC_TOK,
                         xu + static_cast<size_t>(t_begin + r) * V + c_base, seg_bytes, &s_full[s]);
    };
    // the group's operand tables (written by ctc_init / ctc_update): one bulk copy
    const uint32_t tab_bytes = static_cast<uint32_t>(2 * NC * R) * 16u;
    if (tid == 0) {
        for (int s = 0; s < CTC_STAGES; ++s) mbar_init(&s_full[s], 1);
        mbar_init(&s_tabbar, 1);
        mbar_fence_init();
        mbar_arrive_expect_tx(&s_tabbar, tab_bytes);
        bulk_load_1d(smem, a.tab + static_cast<size_t>(blockIdx.y) * 2 * NC * R * 4, tab_bytes, &s_tabbar);
        if (bulk)
            for (int i = 0; i < CTC_STAGES && i < n_st; ++i) issue_stage(i);
    }
    if (tid < 2 * R) s_M[tid / R][tid % R] = a.tabM[static_cast<size_t>(blockIdx.y) * 2 * R + tid];
    if (tid < R) s_last[tid] = step == 0 ? a.bos : a.hist_tok[static_cast<size_t>(step - 1) * a.n_bh + row0 + tid];
    __syncthreads();
    for (uint32_t spins = 0; !mbar_try_wait(&s_tabbar, 0); ++spins)
        if (spins > (1u << 26)) __trap();
    const int tx = tid;
    const int c0 = c_base + tx;
    float acc[CTC_TPT][R];
#pragma unroll
    for (int q = 0; q < CTC_TPT; ++q)
#pragma unroll
        for (int h = 0; h < R; ++h) acc[q][h] = 0.0f;
    auto fma_chunk = [&](int k, const float (&xv)[CTC_TPT][4]) {
        const float4* ak = s_A + static_cast<size_t>(k) * R;
#pragma unroll
        for (int h = 0; h < R; ++h) {
            const float4 av = ak[h];
#pragma unroll
            for (int q = 0; q < CTC_TPT; ++q) {
                acc[q][h] = fmaf(av.x, xv[q][0], acc[q][h]); acc[q][h] = fmaf(av.y, xv[q][1], acc[q][h]);
                acc[q][h] = fmaf(av.z, xv[q][2], acc[q][h]); acc[q][h] = fmaf(av.w, xv[q][3], acc[q][h]);
            }
        }
    };
    if (bulk) {
        for (int i = 0; i < n_st; ++i) {
            const int s = i % CTC_STAGES;
            for (uint32_t spins = 0; !mbar_try_wait(&s_full[s], (i / CTC_STAGES) & 1); ++spins)
                if (spins > (1u << 26)) __trap();   // a protocol bug must fail the test, never hang the GPU
            const float* slot = s_ring + static_cast<size_t>(s) * CTC_STAGE_ROWS * CTC_TOK;
#pragma unroll
            for (int j = 0; j < CTC_STAGE_ROWS / 4; ++j) {
                const int t = r0 + i * CTC_STAGE_ROWS + 4 * j;
                if (t < T) {
                    float xv[CTC_TPT][4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const bool in = t + u < T;   // (frames past T were not copied: whatever the slot holds must not be used)
#pragma unroll
                        for (int q = 0; q < CTC_TPT; ++q) xv[q][u] = in ? slot[(4 * j + u) * CTC_TOK + tx + q * CTC_THREADS] : 0.0f;
                    }
                    fma_chunk(t >> 2, xv);
                }
            }
            __syncthreads();   // every thread is done with slot s
            if (tid == 0 && i + CTC_STAGES < n_st) issue_stage(i + CTC_STAGES);
        }
    } else {   // row segments not 16-byte aligned (V % 4 != 0): per-thread loads
        int cc[CTC_TPT];   // columns past V read column V - 1 (their sums are never written)
#pragma unroll
        for (int q = 0; q < CTC_TPT; ++q) cc[q] = min(c0 + q * CTC_THREADS, V - 1);
        for (int k = t_lo >> 2; k < NC; ++k) {
            const int t = k << 2;
            float xv[CTC_TPT][4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const bool in = t + u < T;
#pragma unroll
                for (int q = 0; q < CTC_TPT; ++q) xv[q][u] = in ? __ldg(xu + static_cast<size_t>(t + u) * V + cc[q]) : 0.0f;
            }
            fma_chunk(k, xv);
        }
    }
    // scores: with an LM in front the output is accumulated -- the 2 R old values are requested together (as 2 R
    // load-then-store pairs in program order they were 2 R dependent memory round trips)
    float old[CTC_TPT][R];
#pragma unroll
    for (int q = 0; q < CTC_TPT; ++q) {
        const int c = c0 + q * CTC_THREADS;
#pragma unroll
        for (int h = 0; h < R; ++h)
            old[q][h] = (a.accumulate && c < V) ? __ldcg(a.out + static_cast<size_t>(row0 + h) * V + c) : 0.0f;
    }
    float eos_psi[R], pprev[R];
    const int t_eos = ctc_eos_frame(a.enc_len[b], T);
#pragma unroll
    for (int h = 0; h < R; ++h) {
        eos_psi[h] = rsum_in[static_cast<size_t>(row0 + h) * T + t_eos];   // Alg.2-3
        pprev[h] = psi_prev[row0 + h];
    }
#pragma unroll
    for (int q = 0; q < CTC_TPT; ++q) {
        const int c = c0 + q * CTC_THREADS;
        if (c >= V) continue;
#pragma unroll
        for (int h = 0; h < R; ++h) {
            if (c == s_last[h]) continue;  // phi = r_b for this one: below
            const int row = row0 + h;
            float psi;
            if (c == a.blank && a.eos != a.blank) psi = CTC_NEG;
            else if (c == a.eos) psi = eos_psi[h];
            else if (acc[q][h] > 1e-30f) psi = s_M[0][h] + __logf(acc[q][h]);
            else psi = ctc_psi_logdomain(a, b, c, step, rsum_in + static_cast<size_t>(row) * T);
            a.out[static_cast<size_t>(row) * V + c] = old[q][h] + a.weight * (psi - pprev[h]);
        }
    }
    if (blockIdx.x == 0) {
        // the hypothesis' own last token (Alg.2-10: phi = r_b): one warp per hypothesis, lanes over the chunks
        for (int h = warp; h < R; h += NT / 32) {
            const int row = row0 + h, c = s_last[h];
            if (c < 0 || c >= V) continue;
            const float* xu = a.xlin + static_cast<size_t>(b) * T * V + c;
            float v = 0.0f;
            for (int k = (t_lo >> 2) + lane; k < NC; k += 32) {
                const float4 av = s_A[(static_cast<size_t>(NC) + k) * R + h];
                const int t = k << 2;
                v = fmaf(av.x, xu[static_cast<size_t>(t) * V], v);
                if (t + 1 < T) v = fmaf(av.y, xu[static_cast<size_t>(t + 1) * V], v);
                if (t + 2 < T) v = fmaf(av.z, xu[static_cast<size_t>(t + 2) * V], v);
                if (t + 3 < T) v = fmaf(av.w, xu[static_cast<size_t>(t + 3) * V], v);
            }
            v = warp_sum(v);
            if (lane == 0)
                ctc_emit(a, row, b, c, step, v, s_M[1][h], rb_in + static_cast<size_t>(row) * T, rsum_in + static_cast<size_t>(row) * T,
                         psi_prev[row]);
        }
    }
}

// permute_mem (ctc.py:251-295) without the (T, 2, n_bh, V) tensor: re-run the recurrence for the chosen (parent, token)
// of every new hypothesis and keep its forward variables.
__global__ void __launch_bounds__(128) ctc_update_kernel(const CtcArgs a) {
    extern __shared__ float smem[];
    const int T = a.T, V = a.V;
    float* s_phi = smem;
    float* s_xn = smem + T;
    float* s_xb = smem + 2 * T;
    float* s_nb = smem + 3 * T;
    float* s_bl = smem + 4 * T;
    const int row = blockIdx.x, b = row / a.beam;
    const int step = a.step_ptr[row] + a.step_adj;   // the step whose survivors are being updated
    if (step < 0) return;                            // enqueued at the head of every search step: nothing to do before the first
    const size_t half = static_cast<size_t>(step & 1), other = half ^ 1;
    const float* rsum_in = a.rsum_base + half * a.n_bh * T;
    const float* rb_in = a.rb_base + half * a.n_bh * T;
    float* rsum_out = a.rsum_base + other * a.n_bh * T;
    float* rb_out = a.rb_base + other * a.n_bh * T;
    float* psi_out = a.psi_base + other * a.n_bh;
    const size_t h = static_cast<size_t>(step) * a.n_bh + row;
    const int tok = a.hist_tok[h], prow = a.hist_pred[h];
    const int last_char = step == 0 ? a.bos : a.hist_tok[static_cast<size_t>(step - 1) * a.n_bh + prow];
    const float* phi = (tok == last_char) ? rb_in : rsum_in;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        s_phi[t] = phi[static_cast<size_t>(prow) * T + t];
        s_xn[t] = a.x[(static_cast<size_t>(b) * T + t) * V + tok];
        s_xb[t] = a.xb[static_cast<size_t>(b) * T + t];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float r_nb, r_b = CTC_NEG;
        int start;
        if (step == 0) { r_nb = s_xn[0]; start = 1; }
        else { r_nb = CTC_NEG; start = step; }
        for (int t = 0; t < start - 1 && t < T; ++t) { s_nb[t] = CTC_NEG; s_bl[t] = CTC_NEG; }
        if (start - 1 < T) { s_nb[start - 1] = r_nb; s_bl[start - 1] = CTC_NEG; }
        float pm = r_nb, ps = 1.0f;
        for (int t = start; t < T; ++t) {
            const float ph = s_phi[t - 1], xn = s_xn[t];
            const float nb = logaddexp_acc(r_nb, ph) + xn;
            const float bl = logaddexp_acc(r_nb, r_b) + s_xb[t];
            const float term = ph + xn;
            if (term > pm) { ps = ps * expf(pm - term) + 1.0f; pm = term; }
            else ps += expf(term - pm);
            r_nb = nb; r_b = bl;
            s_nb[t] = nb; s_bl[t] = bl;
        }
        float psi = pm + logf(ps);
        if (tok == a.eos) psi = rsum_in[static_cast<size_t>(prow) * T + ctc_eos_frame(a.enc_len[b], T)];
        if (tok == a.blank && a.eos != a.blank) psi = CTC_NEG;
        psi_out[row] = psi;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float rs = logaddexp_acc(s_nb[t], s_bl[t]);
        rb_out[static_cast<size_t>(row) * T + t] = s_bl[t];
        rsum_out[static_cast<size_t>(row) * T + t] = rs;
        s_nb[t] = rs;   // (each thread rewrites only the entries it has just read)
    }
    __syncthreads();
    // the operand tables of the step that will extend this hypothesis (step + 1: its sums start at frame step + 1)
    __shared__ float s_red[8];
    ctc_write_tables(s_nb, s_bl, T, step + 1, a.tab, a.tabM, a.R, row, s_red);
}

}  // namespace

// --------------------------------------------------------------------------- CTC greedy (EncoderASR, decoders/ctc.py:335-378)
// One CTA per frame: optional in-place log_softmax of the row (what the recipe's `log_softmax` module does after ctc_lin) and
// its arg-max (first index on ties, like torch.max).
__global__ void __launch_bounds__(256)
rows_logsoftmax_argmax_kernel(float* __restrict__ x, int V, int do_logsoftmax, int* __restrict__ idx) {
    __shared__ float s_val[8];
    __shared__ int s_idx[8];
    const int row = blockIdx.x, tid = threadIdx.x;
    float* xr = x + static_cast<size_t>(row) * V;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = tid; j < V; j += 256) {
        const float v = xr[j];
        if (argmax_takes(v, j, best, bi)) { best = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if ((tid & 31) == 0) { s_val[tid >> 5] = best; s_idx[tid >> 5] = bi; }
    __syncthreads();
    best = s_val[0]; bi = s_idx[0];
    for (int w = 1; w < 8; ++w)
        if (argmax_takes(s_val[w], s_idx[w], best, bi)) { best = s_val[w]; bi = s_idx[w]; }
    if (idx != nullptr && tid == 0) idx[row] = bi;
    if (!do_logsoftmax) return;
    __syncthreads();
    float sm = 0.0f;
    for (int j = tid; j < V; j += 256) sm += expf(xr[j] - best);
    sm = warp_sum(sm);
    if ((tid & 31) == 0) s_val[tid >> 5] = sm;
    __syncthreads();
    float tot = 0.0f;
    for (int w = 0; w < 8; ++w) tot += s_val[w];
    const float lse = best + logf(tot);
    for (int j = tid; j < V; j += 256) xr[j] -= lse;
}

int rows_logsoftmax_argmax(float* x, int rows, int V, bool do_logsoftmax, int* idx, cudaStream_t stream) {
    if (rows == 0) return SBK_OK;
    rows_logsoftmax_argmax_kernel<<<rows, 256, 0, stream>>>(x, V, do_logsoftmax ? 1 : 0, idx);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// hypotheses per score CTA: the widest compiled group that divides the beam and whose operand tables fit shared memory next to
// the streaming ring
static int ctc_group_width(int beam, int T) {
    const int Tp = (T + 3) & ~3;
    const int fit = (200 * 1024 - CTC_RING_FLOATS * 4) / (2 * Tp * 4);
    static const int widths[] = {16, 12, 11, 10, 8, 6, 5, 4, 3, 2, 1};
    for (int w : widths) if (beam % w == 0 && w <= fit) return w;
    return 1;
}
int ctc_prefix_group_width(int beam, int T) { return ctc_group_width(beam, T); }

int ctc_prefix_reset(float* x, float* xlin, float* xb, const int* enc_len, int B, int T, int V, int blank, int beam, float* rsum,
                     float* rb, float* psi_prev, float* tab, float* tabM, cudaStream_t stream) {
    SBK_REQUIRE(T >= 1 && T * 5 * 4 <= 200 * 1024, "ctc scorer: T=%d out of range", T);
    // ctc_init (2 T floats) and ctc_update (5 T floats) exceed the default 48 KB of dynamic shared memory from T = 6145 and
    // T = 2458 on; the reset runs before either is launched (the update is enqueued ahead of the score kernel in a step)
    static bool attr = false;
    if (!attr) {
        SBK_CUDA_CHECK(cudaFuncSetAttribute(ctc_init_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        SBK_CUDA_CHECK(cudaFuncSetAttribute(ctc_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr = true;
    }
    ctc_logsoftmax_mask_kernel<<<B * T, 256, 0, stream>>>(x, xlin, xb, enc_len, T, V, blank);
    SBK_LAUNCH_CHECK();
    ctc_init_kernel<<<B * beam, 128, 2 * T * 4, stream>>>(xb, T, beam, rsum, rb, psi_prev, tab, tabM, ctc_group_width(beam, T));
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

static CtcArgs make_args(const CtcStep& p, int step_adj) {
    CtcArgs a;
    a.x = p.x; a.xlin = p.xlin; a.xb = p.xb; a.rsum_base = p.rsum_base; a.rb_base = p.rb_base; a.psi_base = p.psi_base; a.enc_len = p.enc_len;
    a.hist_tok = p.hist_tok; a.hist_pred = p.hist_pred; a.step_ptr = p.step_ptr; a.step_adj = step_adj;
    a.n_bh = p.n_bh; a.bos = p.bos; a.T = p.T; a.V = p.V;
    a.beam = p.beam; a.blank = p.blank; a.eos = p.eos; a.weight = p.weight; a.out = p.out; a.accumulate = p.accumulate;
    a.tab = p.tab; a.tabM = p.tabM; a.R = ctc_group_width(p.beam, p.T);
    return a;
}

template <int R>
static int launch_score(const CtcArgs& a, cudaStream_t stream) {
    static bool attr = false;
    if (!attr) {
        SBK_CUDA_CHECK(cudaFuncSetAttribute(ctc_score_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr = true;
    }
    const int Tp = (a.T + 3) & ~3;
    ctc_score_kernel<R><<<dim3(ceil_div(a.V, CTC_TOK), a.n_bh / R), CTC_THREADS, ((size_t)2 * R * Tp + CTC_RING_FLOATS) * 4, stream>>>(a);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int ctc_prefix_score(const CtcStep& p, cudaStream_t stream) {
    const CtcArgs a = make_args(p, 0);   // runs before the beam kernel advances the step counters
    const int R = a.R;
    switch (R) {
        case 16: return launch_score<16>(a, stream);
        case 12: return launch_score<12>(a, stream);
        case 11: return launch_score<11>(a, stream);
        case 10: return launch_score<10>(a, stream);
        case 8: return launch_score<8>(a, stream);
        case 6: return launch_score<6>(a, stream);
        case 5: return launch_score<5>(a, stream);
        case 4: return launch_score<4>(a, stream);
        case 3: return launch_score<3>(a, stream);
        case 2: return launch_score<2>(a, stream);
        default: return launch_score<1>(a, stream);
    }
}

int ctc_prefix_update(const CtcStep& p, cudaStream_t stream) {
    const CtcArgs a = make_args(p, -1);  // runs after it (at the head of the next search step)
    ctc_update_kernel<<<p.n_bh, 128, 5 * p.T * 4, stream>>>(a);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // namespace sbk
