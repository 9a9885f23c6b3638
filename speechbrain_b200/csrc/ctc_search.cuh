// Pieces shared by the two CTC beam searches without a language model (ctc_beam.cu, ctc_prefix_beam.cu): polynomial
// string hashes modulo 2^61 - 1, np.logaddexp's float32 formula, the block-wide ordered compaction, arg-max and max, the
// prune and stable ranking of the merged beams (radix_select of common.cuh), the host input checks and the token-count
// pre-pass that sizes their workspaces.
#pragma once
#include <vector>

#include "common.cuh"
#include "../../include/sbk.h"

namespace sbk {
namespace {

constexpr int CB_THREADS = 512;
constexpr int CB_NW = CB_THREADS / 32;
constexpr int CB_MAX_BEAM = 256;
constexpr int CB_MAX_VOCAB = 8192;
constexpr uint64_t HP = (1ull << 61) - 1;
constexpr uint64_t HBASE = SBK_CTC_HASH_BASE;

__device__ __forceinline__ uint64_t hmul(uint64_t a, uint64_t b) {   // a * b mod 2^61 - 1, a, b < 2^61 - 1
    const uint64_t lo = a * b, hi = __umul64hi(a, b);
    uint64_t r = (lo & HP) + ((lo >> 61) | (hi << 3));
    r = (r & HP) + (r >> 61);
    return r >= HP ? r - HP : r;
}
__device__ __forceinline__ uint64_t hadd(uint64_t a, uint64_t b) {
    const uint64_t r = a + b;
    return r >= HP ? r - HP : r;
}

// np.logaddexp for float32 (npy_logaddexpf)
__device__ __forceinline__ float logaddexp_np(float x, float y) {
    if (x == y) return __fadd_rn(x, 0.693147180559945309417232121458176568f);
    const float tmp = __fsub_rn(x, y);
    if (tmp > 0.0f) return __fadd_rn(x, log1pf(expf(-tmp)));
    if (tmp <= 0.0f) return __fadd_rn(y, log1pf(expf(tmp)));
    return tmp;
}

// Ordered compaction: the rank of this thread's flag among the set flags of lower threads; *total = set flags in the block.
// Every thread of a CB_THREADS block must call it; it synchronises the block twice.
__device__ __forceinline__ int block_rank(bool flag, int* s_w, int* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_w[w] = __popc(m);
    __syncthreads();
    int off = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < CB_NW; ++i) {
        const int v = s_w[i];
        off += i < w ? v : 0;
        tot += v;
    }
    __syncthreads();
    *total = tot;
    return off + __popc(m & ((1u << lane) - 1u));
}

// arg-max of a row, first index on ties (np.argmax)
__device__ __forceinline__ int block_argmax(const float* col, int V, float* s_f, int* s_i) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = threadIdx.x; j < V; j += blockDim.x) {
        const float v = col[j];
        if (argmax_takes(v, j, best, bi)) { best = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_f[threadIdx.x >> 5] = best; s_i[threadIdx.x >> 5] = bi; }
    __syncthreads();
    best = s_f[0]; bi = s_i[0];
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w)
        if (argmax_takes(s_f[w], s_i[w], best, bi)) { best = s_f[w]; bi = s_i[w]; }
    __syncthreads();
    return bi;
}

template <typename T>
__device__ __forceinline__ T block_max(T v, T* s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    T r = s_red[0];
    for (int i = 1; i < static_cast<int>(blockDim.x >> 5); ++i) r = fmax(r, s_red[i]);
    __syncthreads();
    return r;
}

// The beam prune and sort_beams of both searches (decoders/ctc.py:811-824) over the U merged beams: the beams whose
// score_of(u) >= max + beam_thr, and of those the `beam` best -- a radix select of the beam-th largest key, the ties at
// it kept by position -- ranked by (score desc, position asc), heapq.nlargest's stable order.  lmax: the max of this
// thread's scores (u = tid, tid + CB_THREADS, ...); key: U keys of workspace.  Leaves the kept positions in rank order in
// s_pos and returns their count.  Every thread of the CB_THREADS block calls it.
template <typename Score, typename Key, typename ScoreOf>
__device__ __forceinline__ int prune_and_rank(int U, int beam, Score lmax, Score beam_thr, ScoreOf score_of, Key* key, int* s_w,
                                              int* s_pos) {
    __shared__ Score s_red[CB_NW];
    __shared__ int s_kept[CB_MAX_BEAM];
    __shared__ Key s_kkey[CB_MAX_BEAM];
    const int tid = threadIdx.x;
    const Score thr = block_max(lmax, s_red) + beam_thr;
    int ns = 0;
    for (int u = tid; u < U; u += CB_THREADS) {
        const Score s = score_of(u);
        const bool ok = s >= thr;
        key[u] = ok ? score_key(s) : Key(0);   // no NaN passes: key 0 marks the pruned beams
        ns += ok ? 1 : 0;
    }
    ns = __reduce_add_sync(0xffffffffu, ns);
    if ((tid & 31) == 0) s_w[tid >> 5] = ns;
    __syncthreads();
    ns = 0;
    for (int i = 0; i < CB_NW; ++i) ns += s_w[i];
    __syncthreads();
    const bool select = ns > beam;
    KthKey<Key> kth = {0, 0};
    if (select) kth = radix_select<Key>(U, beam, [&](int u) { return key[u]; });
    int nk = 0, neq = 0;
    for (int base = 0; base < U; base += CB_THREADS) {
        const int u = base + tid;
        const Key k = u < U ? key[u] : Key(0);
        const bool eq = select && k != 0 && k == kth.key;
        int tot_eq;
        const int r_eq = block_rank(eq, s_w, &tot_eq);
        const bool keep = k != 0 && (!select || k > kth.key || (eq && neq + r_eq < kth.ties));
        int tot;
        const int r = block_rank(keep, s_w, &tot);
        if (keep) { s_kept[nk + r] = u; s_kkey[nk + r] = k; }
        nk += tot;
        neq += tot_eq;
    }
    __syncthreads();
    if (tid < nk) {
        const Key k = s_kkey[tid];
        int rk = 0;
        for (int j = 0; j < nk; ++j) {
            const Key kj = s_kkey[j];
            rk += (kj > k || (kj == k && j < tid)) ? 1 : 0;
        }
        s_pos[rk] = s_kept[tid];
    }
    __syncthreads();
    return nk;
}

// Host checks of both searches' inputs (who: the message prefix); synchronises the stream to read the lengths.
template <typename Params>
int ctc_check(const char* who, const float* lp, const int* lens, int B, int T, int V, int nv, const Params* p, cudaStream_t st) {
    SBK_REQUIRE(lp && lens && p, "%s: null pointer", who);
    SBK_REQUIRE(B >= 1 && T >= 1 && V >= 1, "%s: bad sizes B=%d T=%d V=%d", who, B, T, V);
    SBK_REQUIRE(V <= CB_MAX_VOCAB, "%s: V=%d above the supported %d", who, V, CB_MAX_VOCAB);
    SBK_REQUIRE(nv >= 1 && nv <= V, "%s: n_vocab=%d outside [1, V=%d]", who, nv, V);
    SBK_REQUIRE(p->beam_size >= 1 && p->beam_size <= CB_MAX_BEAM, "%s: beam_size=%d outside [1, %d]", who, p->beam_size,
                CB_MAX_BEAM);
    SBK_REQUIRE(p->blank >= 0 && p->blank < V, "%s: blank index %d outside [0, %d)", who, p->blank, V);
    std::vector<int> len(B);
    SBK_CUDA_CHECK(cudaMemcpyAsync(len.data(), lens, B * 4, cudaMemcpyDeviceToHost, st));
    SBK_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int v : len) SBK_REQUIRE(v >= 0 && v <= T, "%s: length %d outside [0, %d]", who, v, T);
    return SBK_OK;
}

// Pre-pass: the largest candidate-token count of any processed frame (sizes the candidate workspace).
__global__ void __launch_bounds__(256) ctc_beam_count_kernel(const float* __restrict__ lp, const int* __restrict__ lens, int T, int V,
                                                             int nv, int blank, float tok_thr, float skip_thr, int* max_count) {
    __shared__ float s_f[8];
    __shared__ int s_i[8];
    const int row = blockIdx.x, b = row / T, f = row - b * T;
    if (f >= lens[b]) return;
    const float* col = lp + static_cast<size_t>(row) * V;
    if (col[blank] > skip_thr) return;
    const int am = block_argmax(col, V, s_f, s_i);
    int cnt = 0;
    for (int j = threadIdx.x; j < nv; j += blockDim.x) cnt += (col[j] > tok_thr || j == am) ? 1 : 0;
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0) s_i[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < 8; ++w) tot += s_i[w];
        atomicMax(max_count, tot);
    }
}

__host__ __device__ inline size_t cb_align(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

// The largest count over the processed frames of {t < nv : lp[t] > tok_thr} + the arg-max (synchronises the stream).
int ctc_max_tokens(const float* lp, const int* lens, int B, int T, int V, int nv, int blank, float tok_thr, float skip_thr,
                   cudaStream_t st, int* out) {
    int* d = nullptr;
    SBK_CUDA_CHECK(cudaMallocAsync(&d, sizeof(int), st));
    SBK_CUDA_CHECK(cudaMemsetAsync(d, 0, sizeof(int), st));
    ctc_beam_count_kernel<<<B * T, 256, 0, st>>>(lp, lens, T, V, nv, blank, tok_thr, skip_thr, d);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d, sizeof(int), cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(d, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    SBK_CUDA_CHECK(e);
    return SBK_OK;
}

}  // namespace
}  // namespace sbk
