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

// gates = U[tok] + W_hh h for this CTA's hidden units, then the LSTM cell (gate order i, f, g, o); rows with tok < 0 skip
__device__ void lstm_update(const TdArgs& a, const __half* sWhh, const int* st_tok, int u0, int nhl) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, H = a.H;
    for (int pi = warp; pi < a.B * nhl; pi += TD_NW) {
        const int b = pi / nhl, u = pi - b * nhl;
        const int tok = st_tok[b];
        if (tok < 0) continue;
        const float* hb = a.h + size_t(b) * H;
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
            const float* Ur = a.U + size_t(tok) * 4 * H + unit;
            const float gi = sigmoidf_(Ur[0] + acc[0]);
            const float gf = sigmoidf_(Ur[H] + acc[1]);
            const float gg = tanhf(Ur[2 * H] + acc[2]);
            const float go = sigmoidf_(Ur[3 * H] + acc[3]);
            const size_t o = size_t(b) * H + unit;
            const float cn = gf * a.c[o] + gi * gg;
            a.c[o] = cn;
            a.hn[o] = go * tanhf(cn);
        }
    }
}

// p = W_pd h_next for this CTA's joint rows, and h <- h_next for its hidden units
__device__ void proj_update(const TdArgs& a, const __half* sWpd, const int* st_tok, int j0, int njl, int u0, int nhl) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, H = a.H;
    for (int pi = warp; pi < a.B * njl; pi += TD_NW) {
        const int b = pi / njl, j = pi - b * njl;
        if (st_tok[b] < 0) continue;
        const float* hb = a.hn + size_t(b) * H;
        float acc = 0.f;
        for (int k = lane * 2; k < H; k += 64) {
            const float2 hv = *reinterpret_cast<const float2*>(hb + k);
            const float2 w = __half22float2(*reinterpret_cast<const __half2*>(sWpd + size_t(j) * H + k));
            acc = fmaf(w.x, hv.x, acc);
            acc = fmaf(w.y, hv.y, acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) a.p[size_t(b) * a.J + j0 + j] = acc;
    }
    for (int i = threadIdx.x; i < a.B * nhl; i += TD_THREADS) {
        const int b = i / nhl, u = i - b * nhl;
        if (st_tok[b] < 0) continue;
        const size_t o = size_t(b) * H + u0 + u;
        a.h[o] = a.hn[o];
    }
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

    for (int i = tid; i < nvl * J; i += TD_THREADS) sWout[i] = a.Wout[size_t(v0) * J + i];
    for (int i = tid; i < 4 * nhl * H; i += TD_THREADS) {
        const int r = i / H, k = i - r * H, u = r >> 2, q = r & 3;
        sWhh[i] = a.Whh[size_t(q * H + u0 + u) * H + k];
    }
    for (int i = tid; i < njl * H; i += TD_THREADS) sWpd[i] = a.Wpd[size_t(j0) * H + i];
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
            for (int i = tid; i < TD_RB * J; i += TD_THREADS) {
                const int r = i / J, k = i - r * J, b = rb0 + r;
                if (b < B && st_t[b] < T)
                    sZ[i] = gelu_erf_f(a.tn[(size_t(b) * T + st_t[b]) * J + k] + a.p[size_t(b) * J + k]);
            }
            __syncthreads();
            for (int pi = warp; pi < TD_RB * nvl; pi += TD_NW) {
                const int r = pi / nvl, v = pi - r * nvl, b = rb0 + r;
                if (b >= B || st_t[b] >= T) continue;
                float acc = 0.f;
                for (int k = lane * 2; k < J; k += 64) {
                    const float2 z = *reinterpret_cast<const float2*>(sZ + r * J + k);
                    const float2 w = __half22float2(*reinterpret_cast<const __half2*>(sWout + size_t(v) * J + k));
                    acc = fmaf(w.x, z.x, acc);
                    acc = fmaf(w.y, z.y, acc);
                }
                acc = warp_sum(acc);
                if (lane == 0) sLg[r * a.nv + v] = acc;
            }
            __syncthreads();
            for (int r = warp; r < TD_RB; r += TD_NW) {
                const int b = rb0 + r;
                if (b >= B || st_t[b] >= T) continue;
                float m = -INFINITY;
                int am = td::NO_ARG;
                for (int v = lane; v < nvl; v += 32) {
                    const float x = sLg[r * a.nv + v];
                    if (td::argmax_before(x, v0 + v, m, am)) { m = x; am = v0 + v; }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
                    const int a2 = __shfl_xor_sync(0xffffffffu, am, o);
                    if (td::argmax_before(m2, a2, m, am)) { m = m2; am = a2; }
                }
                float s = 0.f;
                for (int v = lane; v < nvl; v += 32) s += expf(sLg[r * a.nv + v] - m);
                s = warp_sum(s);
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
            float m = -INFINITY, s = 0.f;
            int am = td::NO_ARG;
            for (int gg = lane; gg < G; gg += 32)
                td::lse_merge(m, am, s, a.pmax[pbuf + size_t(gg) * B + b], a.parg[pbuf + size_t(gg) * B + b],
                          a.psum[pbuf + size_t(gg) * B + b]);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float m2 = __shfl_down_sync(0xffffffffu, m, o);
                const int a2 = __shfl_down_sync(0xffffffffu, am, o);
                const float s2 = __shfl_down_sync(0xffffffffu, s, o);
                if ((lane & (2 * o - 1)) == 0) td::lse_merge(m, am, s, m2, a2, s2);
            }
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

}  // extern "C"
