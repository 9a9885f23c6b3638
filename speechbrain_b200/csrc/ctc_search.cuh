// Pieces shared by the two CTC beam searches without a language model (ctc_beam.cu, ctc_prefix_beam.cu): polynomial
// string hashes modulo 2^61 - 1, np.logaddexp's float32 formula, the block-wide ordered compaction and arg-max, and the
// token-count pre-pass that sizes their workspaces.
#pragma once
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
