// KV-cached Transformer decoder step + greedy bookkeeping for S2STransformer{Greedy,Beam}Searcher.
//
// The reference (decoders/seq2seq.py:360-367,1929-1934 -> TransformerASR.decode
// lobes/models/transformer/TransformerASR.py:426-473 -> Transformer.py:751-834,915-963) re-embeds and
// re-runs all decoder layers over the WHOLE prefix every step and re-projects the encoder memory to K/V in
// every layer every step. Here: cross-attention K/V are projected once per utterance (one wgmma GEMM
// over all layers), self-attention K/V are appended to a cache, and one step touches only the newest token.
// Numerically the step computes exactly the reference's last-position output.
//
// All step kernels read the current step index from device memory so that a single captured CUDA graph
// can be replayed for every step.
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

__device__ __forceinline__ void mma16816_d(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Programmatic dependent launch (common.cuh): every decode-step kernel lets its successor start launching immediately
// and waits for its predecessor's memory only right before it touches activations, so launch latency and the
// weight prefetch of kernel N+1 overlap the tail of kernel N.
static bool g_use_pdl = true;
void set_pdl(bool on) { g_use_pdl = on; }

template <typename... KArgs, typename... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    return launch_pdl(kern, grid, block, smem, st, g_use_pdl, args...);
}

// --------------------------------------------------------------------------- skinny GEMM (weight streaming)
// y[n_rows, N] = epi( A[n_rows, K] x W[N, K]^T (fp16) + bias ).  n_rows is the number of live hypotheses
// (32..320): the cost is streaming W once plus a chain of dependent L2 round trips, so one CTA owns 8 output
// columns x 32 rows, its 8 warps split K, and every warp issues all the loads of a chunk of UNR k-steps
// before the first mma.  A is either fp16 in global memory, or (LN variant) LayerNorm(x fp32) computed by the
// CTA itself into shared memory -- this fuses the decoder's pre-norms (Transformer.py:788-827) into the
// projection that consumes them.  Deterministic in-CTA split-K reduction through shared memory.
constexpr int SK_WARPS = 8;

// UNR: k-steps whose loads are issued back to back; NT: 8-column tiles per CTA; VPL: LayerNorm-fused variant
// when > 0, with K == 128 * VPL (each lane holds VPL float4 of each of its 4 rows).
template <int UNR, int NT, int VPL>
__global__ void __launch_bounds__(SK_WARPS * 32, (VPL <= 4 ? 2 : 1)) skinny_gemm_kernel(const SkinnyArgs a) {
    constexpr bool LN = VPL > 0;
    constexpr int MT = 2;  // 16-row mma tiles per CTA
    constexpr int SK_ROWS = 16 * MT;
    __shared__ float red[SK_WARPS][SK_ROWS][8 * NT + 1];
    extern __shared__ __align__(16) __half a_sm[];  // LN: [32][K + 8]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int n0 = blockIdx.x * 8 * NT;
    const int row0 = blockIdx.y * SK_ROWS;
    const int rows = min(SK_ROWS, a.n_rows - row0);
    const int k_per_warp = ((a.K / 16 + SK_WARPS - 1) / SK_WARPS) * 16;
    const int k_begin = warp * k_per_warp, k_end = min(a.K, k_begin + k_per_warp);
    pdl_trigger();

    float acc[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0f;
    const __half* wrow[NT];
#pragma unroll
    for (int j = 0; j < NT; ++j)
        wrow[j] = a.W + static_cast<size_t>(min(n0 + 8 * j + g, a.N - 1)) * a.ldw + 2 * c;  // clamp: N tail discarded
    // weights do not depend on the previous kernel: fetch the first chunk before waiting on it
    uint32_t bf[UNR][NT][2];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
        const int k = k_begin + 16 * u;
        const bool ok = k < k_end;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            bf[u][j][0] = ok ? __ldg(reinterpret_cast<const uint32_t*>(wrow[j] + k)) : 0u;
            bf[u][j][1] = ok ? __ldg(reinterpret_cast<const uint32_t*>(wrow[j] + k + 8)) : 0u;
        }
    }
    pdl_wait();

    const int astr = LN ? a.K + 8 : a.lda;
    const __half* abase = LN ? a_sm : a.A;
    if constexpr (LN) {
        // LayerNorm of this CTA's 32 rows: warp w owns rows w, w+8, w+16, w+24; all 4*VPL loads are issued before
        // the first reduction (fp32 statistics, two-pass), result fp16 in shared memory.
        float4 v[4][VPL];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float* xr = a.X + static_cast<size_t>(min(row0 + warp + 8 * r, a.n_rows - 1)) * a.K;
#pragma unroll
            for (int i = 0; i < VPL; ++i) v[r][i] = *reinterpret_cast<const float4*>(xr + 4 * (lane + 32 * i));
        }
        float4 gm[VPL], bt[VPL];
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
            gm[i] = __ldg(reinterpret_cast<const float4*>(a.ln_g + 4 * (lane + 32 * i)));
            bt[i] = __ldg(reinterpret_cast<const float4*>(a.ln_b + 4 * (lane + 32 * i)));
        }
        float s[4], q[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            s[r] = 0.0f;
#pragma unroll
            for (int i = 0; i < VPL; ++i) s[r] += (v[r][i].x + v[r][i].y) + (v[r][i].z + v[r][i].w);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int r = 0; r < 4; ++r) s[r] += __shfl_xor_sync(0xffffffffu, s[r], o);
        const float inv_k = 1.0f / static_cast<float>(a.K);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            s[r] *= inv_k;  // mean
            q[r] = 0.0f;
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                v[r][i].x -= s[r]; v[r][i].y -= s[r]; v[r][i].z -= s[r]; v[r][i].w -= s[r];
                q[r] += (v[r][i].x * v[r][i].x + v[r][i].y * v[r][i].y) + (v[r][i].z * v[r][i].z + v[r][i].w * v[r][i].w);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int r = 0; r < 4; ++r) q[r] += __shfl_xor_sync(0xffffffffu, q[r], o);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float rstd = rsqrtf(q[r] * inv_k + a.ln_eps);
            __half* dst = a_sm + (warp + 8 * r) * astr;
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                __half2 h0 = floats2half2_sat(v[r][i].x * rstd * gm[i].x + bt[i].x, v[r][i].y * rstd * gm[i].y + bt[i].y);
                __half2 h1 = floats2half2_sat(v[r][i].z * rstd * gm[i].z + bt[i].z, v[r][i].w * rstd * gm[i].w + bt[i].w);
                uint2 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0);
                u.y = *reinterpret_cast<uint32_t*>(&h1);
                *reinterpret_cast<uint2*>(dst + 4 * (lane + 32 * i)) = u;
            }
        }
        __syncthreads();
    }
    const __half* arow[2 * MT];
#pragma unroll
    for (int i = 0; i < 2 * MT; ++i) {
        const int rr = LN ? (i * 8 + g) : min(row0 + i * 8 + g, a.n_rows - 1);
        arow[i] = abase + static_cast<size_t>(rr) * astr + 2 * c;
    }
    for (int k0 = k_begin; k0 < k_end; k0 += 16 * UNR) {
        uint32_t af[UNR][MT][4];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int k = k0 + 16 * u;
            const bool ok = k < k_end;
            if (k0 != k_begin) {
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    bf[u][j][0] = ok ? __ldg(reinterpret_cast<const uint32_t*>(wrow[j] + k)) : 0u;
                    bf[u][j][1] = ok ? __ldg(reinterpret_cast<const uint32_t*>(wrow[j] + k + 8)) : 0u;
                }
            }
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                af[u][mt][0] = ok ? *reinterpret_cast<const uint32_t*>(arow[2 * mt] + k) : 0u;
                af[u][mt][1] = ok ? *reinterpret_cast<const uint32_t*>(arow[2 * mt + 1] + k) : 0u;
                af[u][mt][2] = ok ? *reinterpret_cast<const uint32_t*>(arow[2 * mt] + k + 8) : 0u;
                af[u][mt][3] = ok ? *reinterpret_cast<const uint32_t*>(arow[2 * mt + 1] + k + 8) : 0u;
            }
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u)
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) mma16816_d(acc[mt][j], af[u][mt], bf[u][j][0], bf[u][j][1]);
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            red[warp][mt * 16 + g][8 * j + 2 * c] = acc[mt][j][0];
            red[warp][mt * 16 + g][8 * j + 2 * c + 1] = acc[mt][j][1];
            red[warp][mt * 16 + g + 8][8 * j + 2 * c] = acc[mt][j][2];
            red[warp][mt * 16 + g + 8][8 * j + 2 * c + 1] = acc[mt][j][3];
        }
    __syncthreads();
    const int step = a.step_ptr ? *a.step_ptr : 0;
#pragma unroll
    for (int it = 0; it < NT * MT / 2; ++it) {
        const int idx = threadIdx.x + it * SK_WARPS * 32;  // (16*MT) rows x (8*NT) columns
        const int r = idx / (8 * NT), j = idx - r * (8 * NT);
        const int col = n0 + j;
        const int row = row0 + r;
        if (r < rows && col < a.N) {
            float v = 0.0f;
#pragma unroll
            for (int w = 0; w < SK_WARPS; ++w) v += red[w][r][j];
            if (a.bias) v += __ldg(a.bias + col);
            switch (a.epi) {
                case SK_F16: reinterpret_cast<__half*>(a.out)[static_cast<size_t>(row) * a.ldo + col] = float2half_sat(v); break;
                case SK_F16_RELU:
                    reinterpret_cast<__half*>(a.out)[static_cast<size_t>(row) * a.ldo + col] = float2half_sat(fmaxf(v, 0.0f));
                    break;
                case SK_F16_GELU:
                    reinterpret_cast<__half*>(a.out)[static_cast<size_t>(row) * a.ldo + col] = float2half_sat(gelu_erf_f(v));
                    break;
                case SK_F16_SILU:
                    reinterpret_cast<__half*>(a.out)[static_cast<size_t>(row) * a.ldo + col] = float2half_sat(silu_f(v));
                    break;
                case SK_F32: reinterpret_cast<float*>(a.out)[static_cast<size_t>(row) * a.ldo + col] = v; break;
                case SK_RESID: reinterpret_cast<float*>(a.out)[static_cast<size_t>(row) * a.ldo + col] += v; break;
                case SK_QKV_CACHE: {
                    if (col < a.d) {
                        reinterpret_cast<__half*>(a.out)[static_cast<size_t>(row) * a.ldo + col] = float2half_sat(v * a.q_scale);
                    } else if (col < 2 * a.d) {
                        a.kcache[(static_cast<size_t>(row) * a.S_max + step) * a.d + (col - a.d)] = float2half_sat(v);
                    } else {
                        a.vcache[(static_cast<size_t>(row) * a.S_max + step) * a.d + (col - 2 * a.d)] = float2half_sat(v);
                    }
                    break;
                }
            }
        }
    }
}

int skinny_gemm(const SkinnyArgs& a, cudaStream_t stream) {
    SBK_REQUIRE(a.K % 16 == 0 && a.lda % 2 == 0 && a.ldw % 2 == 0, "skinny_gemm: K %% 16 required (K=%d)", a.K);
    if (a.n_rows == 0) return SBK_OK;
    cudaError_t e;
    const int ry = ceil_div(a.n_rows, 32);
    if (a.X != nullptr) {
        const size_t smem = static_cast<size_t>(32) * (a.K + 8) * 2;
        dim3 grid(ceil_div(a.N, 16), ry);
        static bool attr_done = false;  // static + dynamic shared memory exceeds the 48 KB default
        if (!attr_done) {
            cudaFuncSetAttribute(skinny_gemm_kernel<4, 2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
            cudaFuncSetAttribute(skinny_gemm_kernel<2, 2, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
            cudaFuncSetAttribute(skinny_gemm_kernel<4, 2, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
            cudaFuncSetAttribute(skinny_gemm_kernel<8, 2, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
            attr_done = true;
        }
        if (a.K == 512) e = launch_k(skinny_gemm_kernel<4, 2, 4>, grid, dim3(SK_WARPS * 32), smem, stream, a);
        else if (a.K == 256) e = launch_k(skinny_gemm_kernel<2, 2, 2>, grid, dim3(SK_WARPS * 32), smem, stream, a);
        else if (a.K == 768) e = launch_k(skinny_gemm_kernel<4, 2, 6>, grid, dim3(SK_WARPS * 32), smem, stream, a);
        else if (a.K == 1024) e = launch_k(skinny_gemm_kernel<8, 2, 8>, grid, dim3(SK_WARPS * 32), smem, stream, a);
        else {
            set_error("skinny_gemm(LN): d_model=%d not built (256/512/768/1024)", a.K);
            return SBK_ERR_UNSUPPORTED;
        }
    } else if (a.K <= 1024 && a.N >= 1024) {
        e = launch_k(skinny_gemm_kernel<4, 2, 0>, dim3(ceil_div(a.N, 16), ry), dim3(SK_WARPS * 32), 0, stream, a);
    } else if (a.K <= 1024) {
        e = launch_k(skinny_gemm_kernel<4, 1, 0>, dim3(ceil_div(a.N, 8), ry), dim3(SK_WARPS * 32), 0, stream, a);
    } else {
        e = launch_k(skinny_gemm_kernel<8, 1, 0>, dim3(ceil_div(a.N, 8), ry), dim3(SK_WARPS * 32), 0, stream, a);
    }
    SBK_CUDA_CHECK(e);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// --------------------------------------------------------------------------- decode-time attention (1 query / row)
// One CTA per (row, head), 4 warps split the keys (flash-decoding style).  Within a warp, lane group g = lane / 8 owns
// keys c0 + g + 4 i (i < 8) of a 32-key chunk and lane % 8 owns 8 of the 64 head dims, for BOTH q.k and p.V: every
// 16-byte load instruction of the warp covers 4 whole 128-byte key rows (4 cache lines -- a lane-per-key layout costs
// 32 L1 tag lookups per instruction and bounded the kernel), q.k partials are reduced over the 8 lanes of a group with
// 3 shuffles, and the probabilities stay in registers for p.V.  The 4 warps' (max, sum, out) triples are merged
// through shared memory.
// Self-attention: keys = cache positions [0, step]; cross-attention: keys = encoder frames [0, enc_len[utt]).
// (nn.MultiheadAttention semantics, scale 1/sqrt(d_h) already folded into q.)  head_dim DH == 64, 80 (the d_model 640
// recipes' 8 heads of 80) or 128 (the Transformer recipes' 4 heads of 128): a lane then owns dims [8 (lane % 8), +8) of
// each 64-dim slice, NV = 2 16-byte vectors per key; at 80 the second slice is 16 dims wide, held by lanes 0 and 1 of each
// group (the other lanes' second vector is zero and never stored).
constexpr int DA_WARPS = 4;
constexpr int DA_CHUNK = 32;  // keys a warp handles per round (8 per lane group)
constexpr int DA_KPG = DA_CHUNK / 4;

template <int DH>
__global__ void __launch_bounds__(DA_WARPS * 32, DH == 64 ? 4 : 2) dec_attention_kernel(const DecAttnArgs a) {
    static_assert(DH % 8 == 0 && DH <= 128, "dec_attention_kernel: 16-byte vectors, at most two 64-dim slices");
    constexpr int NV = (DH + 63) / 64;
    __shared__ float part_o[DA_WARPS][DH];
    __shared__ float part_m[DA_WARPS], part_l[DA_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // heads on the fast grid axis: the 8 CTAs that share an utterance's K/V rows (2 KB per frame, 128 B per head) are
    // co-scheduled, so each DRAM page / L2 line set is consumed while it is open
    const int r = blockIdx.y, h = blockIdx.x;
    const int blk = r / a.rows_per_block;
    // cross-attention reads only ckv16 and enc_len before pdl_wait() (see common.cuh): enc_len and the first chunk's K/V
    // loads are issued before it.  Self-attention waits first: its keys are this step's cache writes and its length is
    // the step counter.
    const bool xatt = a.n_keys_ptr == nullptr && a.lineage == nullptr && a.tok_cache == nullptr;
    pdl_trigger();
    if (!xatt) pdl_wait();
    int n_keys;
    if (a.n_keys_ptr) n_keys = *a.n_keys_ptr + 1;
    else n_keys = a.enc_len ? min(a.enc_len[blk], a.n_keys_fixed) : a.n_keys_fixed;
    const int per = (n_keys + DA_WARPS - 1) / DA_WARPS;
    const int kb = warp * per, ke = min(n_keys, kb + per);
    const int gq = lane >> 3, dl = (lane & 7) * 8;
    auto owns = [&](int v) { return DH % 64 == 0 || 64 * v + dl < DH; };  // this lane holds dims 64 v + dl .. + 8
    const int hs = a.head_stride > 0 ? a.head_stride : DH;
    const __half* kbase = a.kbase + static_cast<size_t>(blk) * a.row_stride + static_cast<size_t>(h) * hs + dl;
    const __half* vbase = a.vbase + static_cast<size_t>(blk) * a.row_stride + static_cast<size_t>(h) * hs + dl;
    // beam search: position j of hypothesis r lives in the cache row of the ancestor that wrote it
    const int* lin = nullptr;
    if (a.lineage) lin = a.lineage + static_cast<size_t>((n_keys - 1) & 1) * gridDim.y * a.lin_stride + static_cast<size_t>(r) * a.lin_stride;
    const int* tokc = a.tok_cache;  // TransformerLM.make_masks: keys whose token id is pad_idx (0) are masked
    // every load of the chunk at c0: 8 keys x (16 B of K + 16 B of V) per lane
    uint4 kv[DA_KPG][NV], vv[DA_KPG][NV];
    bool live[DA_KPG];
    auto load_chunk = [&](int c0) {
#pragma unroll
        for (int i = 0; i < DA_KPG; ++i) {
            const int j = c0 + gq + 4 * i;
            live[i] = j < ke;
            if (live[i]) {
                ptrdiff_t off = static_cast<ptrdiff_t>(j) * a.key_stride;
                int src_row = r;
                if (lin) { src_row = lin[j]; off += (static_cast<ptrdiff_t>(src_row) - r) * static_cast<ptrdiff_t>(a.row_stride); }
#pragma unroll
                for (int v = 0; v < NV; ++v) {
                    kv[i][v] = owns(v) ? *reinterpret_cast<const uint4*>(kbase + off + 64 * v) : make_uint4(0u, 0u, 0u, 0u);
                    vv[i][v] = owns(v) ? *reinterpret_cast<const uint4*>(vbase + off + 64 * v) : make_uint4(0u, 0u, 0u, 0u);
                }
                if (tokc) live[i] = tokc[static_cast<size_t>(src_row) * a.lin_stride + j] != a.pad_tok;
            } else {
#pragma unroll
                for (int v = 0; v < NV; ++v) {
                    kv[i][v] = make_uint4(0u, 0u, 0u, 0u);
                    vv[i][v] = make_uint4(0u, 0u, 0u, 0u);
                }
            }
        }
    };
    if (xatt) {
        load_chunk(kb);
        pdl_wait();
    }
    // this lane's 8 dims of the query
    float qf[8 * NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) {
        const uint4 qv = owns(v) ? *reinterpret_cast<const uint4*>(a.q + static_cast<size_t>(r) * a.ldq + h * DH + 64 * v + dl)
                                 : make_uint4(0u, 0u, 0u, 0u);
        const __half2* q2 = reinterpret_cast<const __half2*>(&qv);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const float2 f = __half22float2(q2[u]);
            qf[8 * v + 2 * u] = f.x; qf[8 * v + 2 * u + 1] = f.y;
        }
    }
    float m_run = -INFINITY, l_run = 0.0f;
    float o[8 * NV];
#pragma unroll
    for (int e = 0; e < 8 * NV; ++e) o[e] = 0.0f;
    for (int c0 = kb; c0 < ke; c0 += DA_CHUNK) {
        if (!xatt || c0 != kb) load_chunk(c0);  // issue every load of this chunk up front
        // ---- scores: 8-dim partial dot per lane, summed over the 8 lanes of the key's group
        float sc[DA_KPG];
        float cm = -INFINITY;
#pragma unroll
        for (int i = 0; i < DA_KPG; ++i) {
            float dot = 0.0f;
#pragma unroll
            for (int v = 0; v < NV; ++v) {
                const __half2* k2 = reinterpret_cast<const __half2*>(&kv[i][v]);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float2 kf = __half22float2(k2[u]);
                    dot = fmaf(kf.x, qf[8 * v + 2 * u], dot);
                    dot = fmaf(kf.y, qf[8 * v + 2 * u + 1], dot);
                }
            }
            dot += __shfl_xor_sync(0xffffffffu, dot, 1);
            dot += __shfl_xor_sync(0xffffffffu, dot, 2);
            dot += __shfl_xor_sync(0xffffffffu, dot, 4);
            sc[i] = live[i] ? dot : -INFINITY;
            cm = fmaxf(cm, sc[i]);
        }
        cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 8));
        cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 16));
        const float m_new = fmaxf(m_run, cm);
        const float alpha = (m_run == -INFINITY) ? 0.0f : __expf(m_run - m_new);
        // ---- p.V with the probabilities still in registers
        float psum = 0.0f;
#pragma unroll
        for (int e = 0; e < 8 * NV; ++e) o[e] *= alpha;
#pragma unroll
        for (int i = 0; i < DA_KPG; ++i) {
            const float p = (sc[i] == -INFINITY) ? 0.0f : __expf(sc[i] - m_new);
            psum += p;
#pragma unroll
            for (int v = 0; v < NV; ++v) {
                const __half2* v2 = reinterpret_cast<const __half2*>(&vv[i][v]);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float2 vf = __half22float2(v2[u]);
                    o[8 * v + 2 * u] = fmaf(p, vf.x, o[8 * v + 2 * u]);
                    o[8 * v + 2 * u + 1] = fmaf(p, vf.y, o[8 * v + 2 * u + 1]);
                }
            }
        }
        psum += __shfl_xor_sync(0xffffffffu, psum, 8);
        psum += __shfl_xor_sync(0xffffffffu, psum, 16);
        l_run = l_run * alpha + psum;
        m_run = m_new;
    }
#pragma unroll
    for (int e = 0; e < 8 * NV; ++e) {
        o[e] += __shfl_xor_sync(0xffffffffu, o[e], 8);
        o[e] += __shfl_xor_sync(0xffffffffu, o[e], 16);
    }
    if (lane < 8) {
#pragma unroll
        for (int e = 0; e < 8 * NV; ++e)
            if (owns(e >> 3)) part_o[warp][64 * (e >> 3) + dl + (e & 7)] = o[e];
    }
    if (lane == 0) { part_m[warp] = m_run; part_l[warp] = l_run; }
    __syncthreads();
    if (threadIdx.x < DH) {
        float M = part_m[0];
#pragma unroll
        for (int w = 1; w < DA_WARPS; ++w) M = fmaxf(M, part_m[w]);
        float num = 0.0f, den = 0.0f;
#pragma unroll
        for (int w = 0; w < DA_WARPS; ++w) {
            const float sc = part_m[w] == -INFINITY ? 0.0f : __expf(part_m[w] - M);
            num += part_o[w][threadIdx.x] * sc;
            den += part_l[w] * sc;
        }
        a.out[static_cast<size_t>(r) * a.ldo + h * DH + threadIdx.x] = float2half_sat(num / den);
    }
}

// Generic head_dim (<= 64, multiple of 4) variant of dec_attention_kernel: conformer_small's decoder has 4 heads of 36
// (conformer_small.yaml).  One CTA (128 threads) per (row, head): thread-per-key scores into shared memory, block softmax,
// then thread-per-dim p.V.  Small models only: no attempt at bandwidth efficiency.
constexpr int DG_MAXKEYS = 2560;
__global__ void __launch_bounds__(128) dec_attention_generic_kernel(const DecAttnArgs a) {
    __shared__ float s_q[64];
    __shared__ float s_p[DG_MAXKEYS];
    __shared__ float s_red[4];
    const int r = blockIdx.y, h = blockIdx.x, dh = a.dh, tid = threadIdx.x;
    const int blk = r / a.rows_per_block;
    pdl_trigger();
    pdl_wait();
    int n_keys;
    if (a.n_keys_ptr) n_keys = *a.n_keys_ptr + 1;
    else n_keys = a.enc_len ? min(a.enc_len[blk], a.n_keys_fixed) : a.n_keys_fixed;
    const int hs = a.head_stride > 0 ? a.head_stride : dh;
    const __half* kbase = a.kbase + static_cast<size_t>(blk) * a.row_stride + static_cast<size_t>(h) * hs;
    const __half* vbase = a.vbase + static_cast<size_t>(blk) * a.row_stride + static_cast<size_t>(h) * hs;
    const int* lin = nullptr;
    if (a.lineage) lin = a.lineage + static_cast<size_t>((n_keys - 1) & 1) * gridDim.y * a.lin_stride + static_cast<size_t>(r) * a.lin_stride;
    if (tid < dh) s_q[tid] = __half2float(a.q[static_cast<size_t>(r) * a.ldq + h * dh + tid]);
    __syncthreads();
    float mx = -INFINITY;
    for (int j = tid; j < n_keys; j += 128) {
        ptrdiff_t off = static_cast<ptrdiff_t>(j) * a.key_stride;
        int src_row = r;
        if (lin) { src_row = lin[j]; off += (static_cast<ptrdiff_t>(src_row) - r) * static_cast<ptrdiff_t>(a.row_stride); }
        float dot = 0.0f;
        for (int e = 0; e < dh; e += 4) {
            const uint2 kv = *reinterpret_cast<const uint2*>(kbase + off + e);
            const __half2* k2 = reinterpret_cast<const __half2*>(&kv);
            const float2 f0 = __half22float2(k2[0]), f1 = __half22float2(k2[1]);
            dot = fmaf(f0.x, s_q[e], dot); dot = fmaf(f0.y, s_q[e + 1], dot);
            dot = fmaf(f1.x, s_q[e + 2], dot); dot = fmaf(f1.y, s_q[e + 3], dot);
        }
        if (a.tok_cache && a.tok_cache[static_cast<size_t>(src_row) * a.lin_stride + j] == a.pad_tok) dot = -INFINITY;
        s_p[j] = dot;
        mx = fmaxf(mx, dot);
    }
    mx = warp_max(mx);
    if ((tid & 31) == 0) s_red[tid >> 5] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(s_red[0], s_red[1]), fmaxf(s_red[2], s_red[3]));
    __syncthreads();
    float sum = 0.0f;
    for (int j = tid; j < n_keys; j += 128) {
        const float p = s_p[j] == -INFINITY ? 0.0f : __expf(s_p[j] - mx);
        s_p[j] = p;
        sum += p;
    }
    sum = warp_sum(sum);
    if ((tid & 31) == 0) s_red[tid >> 5] = sum;
    __syncthreads();
    const float den = (s_red[0] + s_red[1]) + (s_red[2] + s_red[3]);
    if (tid < dh) {
        float o = 0.0f;
        for (int j = 0; j < n_keys; ++j) {
            ptrdiff_t off = static_cast<ptrdiff_t>(j) * a.key_stride;
            if (lin) off += (static_cast<ptrdiff_t>(lin[j]) - r) * static_cast<ptrdiff_t>(a.row_stride);
            o = fmaf(s_p[j], __half2float(vbase[off + tid]), o);
        }
        a.out[static_cast<size_t>(r) * a.ldo + h * dh + tid] = float2half_sat(o / den);
    }
}

int dec_attention(const DecAttnArgs& a, int n_rows, int max_keys, cudaStream_t stream) {
    if (a.dh != 64 && a.dh != 80 && a.dh != 128) {
        SBK_REQUIRE(a.dh >= 4 && a.dh <= 64 && a.dh % 4 == 0 && a.key_stride % 4 == 0 && a.row_stride % 4 == 0,
                    "dec_attention: head_dim=%d not built (128, 80, 64, or a multiple of 4 below 64)", a.dh);
        SBK_REQUIRE(max_keys <= DG_MAXKEYS, "dec_attention: %d keys exceed the generic kernel's limit %d", max_keys, DG_MAXKEYS);
        if (n_rows == 0) return SBK_OK;
        DecAttnArgs g = a;
        g.n_keys_fixed = max_keys;
        SBK_CUDA_CHECK(launch_k(dec_attention_generic_kernel, dim3(a.H, n_rows), dim3(128), 0, stream, g));
        SBK_LAUNCH_CHECK();
        return SBK_OK;
    }

    if (n_rows == 0) return SBK_OK;
    DecAttnArgs b = a;
    b.n_keys_fixed = max_keys;
    if (a.dh == 128 || a.dh == 80) {
        SBK_REQUIRE(a.key_stride % 8 == 0 && a.row_stride % 8 == 0 && a.ldq % 8 == 0 && (a.dh == 128 || a.head_stride % 8 == 0),
                    "dec_attention: head_dim %d needs 16-byte aligned key rows", a.dh);
        SBK_CUDA_CHECK(launch_k(a.dh == 128 ? dec_attention_kernel<128> : dec_attention_kernel<80>, dim3(a.H, n_rows),
                                dim3(DA_WARPS * 32), 0, stream, b));
    } else {
        SBK_CUDA_CHECK(launch_k(dec_attention_kernel<64>, dim3(a.H, n_rows), dim3(DA_WARPS * 32), 0, stream, b));
    }
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// --------------------------------------------------------------------------- folded cross-attention (1 row / utterance)
// Every head's keys and values are linear in the same encoder states e: k_t = W_k,h e_t + b_k,h, v_t = W_v,h e_t + b_v,h.
// So q_h . k_t = (W_k,h^T q_h) . e_t + q_h . b_k,h, whose last term is the same for every key and cancels in the softmax,
// and sum_t p_t v_t = W_v,h (sum_t p_t e_t) + b_v,h since the p_t sum to 1.  The step's query projection writes the folded
// queries q'_h = W_k,h^T q_h, this kernel the context vectors sum_t p_t e_t, and the output projection applies
// W_o[:, h] W_v,h to them (asr_weights.cu packs both).  A layer then reads e (2 D bytes per frame) instead of its K and V
// (4 D bytes per frame).
// One CTA per utterance, warp w of 8 owning dims [w D / 8, (w + 1) D / 8) of e.  Blocks of XF_FRAMES frames stream through a
// cp.async ring; per block each warp computes the H heads' partial scores over its dims (mma m16n8k16, the heads padded to
// 16 rows), the 8 partials are summed through shared memory in a fixed order, every warp runs the same online softmax and
// accumulates P e over its own dims.  Results depend on the utterance alone.
constexpr int XF_WARPS = 8;
constexpr int XF_FRAMES = 32;
constexpr int XF_STAGES = 3;
constexpr int XF_RED = XF_FRAMES + 8;  // row stride of the partial scores: at most 2-way bank conflicts
template <int D>
constexpr size_t xf_smem_bytes() {  // frame rows padded by 16 bytes: the 8 rows of an ldmatrix tile hit distinct banks
    return (size_t)XF_STAGES * XF_FRAMES * (D + 8) * 2 + (size_t)XF_WARPS * 8 * XF_RED * 4;
}

template <int D>
__global__ void __launch_bounds__(XF_WARPS * 32, 2) dec_xatt_fold_kernel(const XattFoldArgs a) {
    constexpr int SROW = D + 8, KW = D / XF_WARPS, NKS = KW / 16, NNT = KW / 8, NJ = XF_FRAMES / 8;
    constexpr int CHUNKS = XF_FRAMES * D / 8;  // 16-byte pieces of one block
    static_assert(CHUNKS % (XF_WARPS * 32) == 0 && NKS % 2 == 0 && NNT % 2 == 0, "dec_xatt_fold_kernel: tile shape");
    extern __shared__ __align__(16) uint8_t xf_sm[];
    __half* ring = reinterpret_cast<__half*>(xf_sm);
    float* red = reinterpret_cast<float*>(xf_sm + (size_t)XF_STAGES * XF_FRAMES * SROW * 2);  // [warp][head][frame]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int utt = blockIdx.x;
    // enc16 and enc_len come from kernels that never trigger early (see common.cuh): the first blocks' loads are issued
    // before pdl_wait().  The successor is only triggered after the main loop: its CTAs would otherwise sit on the SMs
    // waiting, holding the shared memory this kernel's second CTA per SM needs.
    const int n_keys = min(a.enc_len[utt], a.T);
    const int n_blk = ceil_div(n_keys, XF_FRAMES);
    const __half* e = a.e + static_cast<size_t>(utt) * a.T * D;
    auto load_block = [&](int blk) {  // frames past n_keys are zero-filled: their p is 0, and 0 * garbage could be NaN
        if (blk < n_blk) {
            __half* dst = ring + static_cast<size_t>(blk % XF_STAGES) * XF_FRAMES * SROW;
#pragma unroll
            for (int i = 0; i < CHUNKS / (XF_WARPS * 32); ++i) {
                const int idx = threadIdx.x + i * XF_WARPS * 32;
                const int f = idx / (D / 8), v8 = idx % (D / 8);
                const int t = blk * XF_FRAMES + f;
                const __half* src = e + static_cast<size_t>(t < n_keys ? t : 0) * D + v8 * 8;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst + f * SROW + v8 * 8)),
                             "l"(src), "r"(t < n_keys ? 16 : 0));
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
#pragma unroll
    for (int s = 0; s < XF_STAGES - 1; ++s) load_block(s);
    pdl_wait();
    // A fragments of this warp's dims of q'_h, h = g (rows g + 8 and heads >= H are zero)
    uint32_t qa[NKS][2];
    const __half* qrow = a.q + static_cast<size_t>(utt) * a.ldq + static_cast<size_t>(g) * D + warp * KW + 2 * c;
#pragma unroll
    for (int ks = 0; ks < NKS; ++ks) {
        qa[ks][0] = g < a.H ? *reinterpret_cast<const uint32_t*>(qrow + 16 * ks) : 0u;
        qa[ks][1] = g < a.H ? *reinterpret_cast<const uint32_t*>(qrow + 16 * ks + 8) : 0u;
    }
    float acc[NNT][4];
#pragma unroll
    for (int nt = 0; nt < NNT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;
    float m_run = -INFINITY, l_run = 0.0f;
    for (int blk = 0; blk < n_blk; ++blk) {
        asm volatile("cp.async.wait_group %0;" ::"n"(XF_STAGES - 2) : "memory");
        __syncthreads();  // block blk landed for every thread; everyone is done with the stage and `red` reused below
        load_block(blk + XF_STAGES - 1);
        const __half* st = ring + static_cast<size_t>(blk % XF_STAGES) * XF_FRAMES * SROW + warp * KW;
        // ---- partial scores over this warp's dims: frames 8 j .. 8 j + 7 per n8 tile, two k16 steps per ldmatrix.x4
        float sp[NJ][4];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            sp[j][0] = sp[j][1] = sp[j][2] = sp[j][3] = 0.0f;
#pragma unroll
            for (int ks = 0; ks < NKS; ks += 2) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(b0, b1, b2, b3, st + (8 * j + (lane & 7)) * SROW + 16 * ks + 8 * (lane >> 3));
                const uint32_t a0[4] = {qa[ks][0], 0u, qa[ks][1], 0u};
                const uint32_t a1[4] = {qa[ks + 1][0], 0u, qa[ks + 1][1], 0u};
                mma16816_d(sp[j], a0, b0, b1);
                mma16816_d(sp[j], a1, b2, b3);
            }
            *reinterpret_cast<float2*>(red + (warp * 8 + g) * XF_RED + 8 * j + 2 * c) = make_float2(sp[j][0], sp[j][1]);
        }
        __syncthreads();
        // ---- full scores of head g at this lane's frames 8 j + 2 c (+1), online softmax (same in every warp)
        float s[NJ][2];
        float cm = -INFINITY;
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                float v = 0.0f;
#pragma unroll
                for (int w = 0; w < XF_WARPS; ++w) v += red[(w * 8 + g) * XF_RED + 8 * j + 2 * c + u];
                s[j][u] = blk * XF_FRAMES + 8 * j + 2 * c + u < n_keys ? v : -INFINITY;
                cm = fmaxf(cm, s[j][u]);
            }
        cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 1));
        cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 2));
        const float m_new = fmaxf(m_run, cm);  // finite: every block processed has a visible key
        const float alpha = m_run == -INFINITY ? 0.0f : __expf(m_run - m_new);
        float psum = 0.0f;
        uint32_t pa[NJ / 2][4];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const float p0 = __expf(s[j][0] - m_new), p1 = __expf(s[j][1] - m_new);
            psum += p0 + p1;
            const __half2 h = floats2half2_sat(p0, p1);
            pa[j / 2][(j & 1) * 2] = *reinterpret_cast<const uint32_t*>(&h);  // a0: frames 16 ks + 2c, a2: + 8
            pa[j / 2][(j & 1) * 2 + 1] = 0u;                                  // rows g + 8
        }
        psum += __shfl_xor_sync(0xffffffffu, psum, 1);
        psum += __shfl_xor_sync(0xffffffffu, psum, 2);
        l_run = l_run * alpha + psum;
        m_run = m_new;
        // ---- context += P e over this warp's dims (B fragments of e[frame][dim] via ldmatrix.trans)
#pragma unroll
        for (int nt = 0; nt < NNT; ++nt) { acc[nt][0] *= alpha; acc[nt][1] *= alpha; }
#pragma unroll
        for (int ks = 0; ks < NJ / 2; ++ks)
#pragma unroll
            for (int nt = 0; nt < NNT; nt += 2) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_trans(b0, b1, b2, b3, st + (16 * ks + (lane & 15)) * SROW + 8 * nt + 8 * (lane >> 4));
                mma16816_d(acc[nt], pa[ks], b0, b1);
                mma16816_d(acc[nt + 1], pa[ks], b2, b3);
            }
    }
    pdl_trigger();
    if (g < a.H) {  // no visible key: 0 / 0 = NaN, like the unfolded path
        __half* o = a.out + static_cast<size_t>(utt) * a.ldo + static_cast<size_t>(g) * D + warp * KW + 2 * c;
#pragma unroll
        for (int nt = 0; nt < NNT; ++nt)
            *reinterpret_cast<__half2*>(o + 8 * nt) = floats2half2_sat(acc[nt][0] / l_run, acc[nt][1] / l_run);
    }
}

int dec_xatt_fold(const XattFoldArgs& a, int n_utt, cudaStream_t stream) {
    SBK_REQUIRE((a.D == 512 && a.H >= 1 && a.H <= 8) || (a.D == 256 && a.H >= 1 && a.H <= 4),
                "dec_xatt_fold: D=%d with %d heads not built (512 with <= 8, 256 with <= 4)", a.D, a.H);
    SBK_REQUIRE(a.ldq % 8 == 0 && a.ldo % 2 == 0 && a.ldq >= a.H * a.D && a.ldo >= a.H * a.D && a.T >= 1 &&
                    (reinterpret_cast<uintptr_t>(a.q) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.e) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(a.out) & 3) == 0,
                "dec_xatt_fold: bad strides or alignment");
    if (n_utt == 0) return SBK_OK;
    static bool attr_done = false;  // above the 48 KB default
    if (!attr_done) {
        SBK_CUDA_CHECK(cudaFuncSetAttribute(dec_xatt_fold_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)xf_smem_bytes<512>()));
        SBK_CUDA_CHECK(cudaFuncSetAttribute(dec_xatt_fold_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)xf_smem_bytes<256>()));
        attr_done = true;
    }
    if (a.D == 512)
        SBK_CUDA_CHECK(launch_k(dec_xatt_fold_kernel<512>, dim3(n_utt), dim3(XF_WARPS * 32), xf_smem_bytes<512>(), stream, a));
    else
        SBK_CUDA_CHECK(launch_k(dec_xatt_fold_kernel<256>, dim3(n_utt), dim3(XF_WARPS * 32), xf_smem_bytes<256>(), stream, a));
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}


// --------------------------------------------------------------------------- greedy step bookkeeping
// decoders/seq2seq.py:226-257: argmax, fp32 log_softmax, has_ended |= (tok == eos); ended rows get
// log_probs = -inf (=> prediction eos, score 0 after :259-263) and keep feeding eos.
// One CTA per row. Writes tokens[r][step+1], pred[r][step], score[r][step], optional log-prob row, then the
// NEXT step's decoder input x[r] = emb[tok] * sqrt(d) + pe[step+1] (Transformer.py:966-995, :252-303) and
// advances this row's step counter (every kernel of the next step reads step[0] after this kernel is done).
__global__ void __launch_bounds__(256)
greedy_select_kernel(const float* __restrict__ logits, int V, int* __restrict__ step_arr, int eos, int* tokens,
                     int tok_stride, int* has_ended, int* ended_count, int* pred, float* score, int out_stride,
                     float* log_probs /* [n, L, V] or null */, int L, const float* __restrict__ emb,
                     const float* __restrict__ pe, int d, float sqrt_d, float* __restrict__ x_next) {
    __shared__ float s_val[8];
    __shared__ int s_idx[8];
    __shared__ float s_sum[8];
    pdl_trigger();
    pdl_wait();
    const int r = blockIdx.x, step = step_arr[r];
    const float* lg = logits + static_cast<size_t>(r) * V;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        const float v = lg[i];
        if (argmax_takes(v, i, best, bi)) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_val[threadIdx.x >> 5] = best; s_idx[threadIdx.x >> 5] = bi; }
    __syncthreads();
    best = s_val[0]; bi = s_idx[0];
    for (int w = 1; w < 8; ++w)
        if (argmax_takes(s_val[w], s_idx[w], best, bi)) { best = s_val[w]; bi = s_idx[w]; }
    float sum = 0.0f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) sum += expf(lg[i] - best);
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = 0.0f;
    for (int w = 0; w < 8; ++w) sum += s_sum[w];
    const float lse = best + logf(sum);
    const int was_ended = has_ended[r];
    const int ended = was_ended | (bi == eos ? 1 : 0);
    if (log_probs) {
        float* lp = log_probs + (static_cast<size_t>(r) * L + step) * V;
        for (int i = threadIdx.x; i < V; i += blockDim.x) lp[i] = ended ? -INFINITY : lg[i] - lse;
    }
    const int tok = ended ? eos : bi;
    __syncthreads();  // everyone has read has_ended[r] / step_arr[r] before thread 0 updates them
    if (threadIdx.x == 0) {
        tokens[static_cast<size_t>(r) * tok_stride + step + 1] = tok;
        pred[static_cast<size_t>(r) * out_stride + step] = tok;
        score[static_cast<size_t>(r) * out_stride + step] = ended ? 0.0f : best - lse;
        if (ended && !was_ended) {
            has_ended[r] = 1;
            atomicAdd(ended_count, 1);
        }
        step_arr[r] = step + 1;
    }
    const float* e = emb + static_cast<size_t>(tok) * d;
    const float* p = pe + static_cast<size_t>(step + 1) * d;
    for (int i = threadIdx.x; i < d; i += blockDim.x) x_next[static_cast<size_t>(r) * d + i] = e[i] * sqrt_d + p[i];
}

// tokens[r][0] = bos, step[r] = 0, x[r] = emb[bos] * sqrt(d) + pe[0]
__global__ void greedy_reset_kernel(int* tokens, int tok_stride, int bos, int* step_arr, int* has_ended,
                                    int* ended_count, const float* __restrict__ emb, const float* __restrict__ pe, int d,
                                    float sqrt_d, float* __restrict__ x) {
    const int r = blockIdx.x;
    if (threadIdx.x == 0) {
        tokens[static_cast<size_t>(r) * tok_stride] = bos;
        has_ended[r] = 0;
        step_arr[r] = 0;
        if (r == 0) *ended_count = 0;
    }
    const float* e = emb + static_cast<size_t>(bos) * d;
    for (int i = threadIdx.x; i < d; i += blockDim.x) x[static_cast<size_t>(r) * d + i] = e[i] * sqrt_d + pe[i];
}

int greedy_reset(int* tokens, int tok_stride, int n_rows, int bos, int* step_arr, int* has_ended, int* ended_count,
                 const float* emb, const float* pe, int d, float* x, cudaStream_t stream) {
    if (n_rows == 0) return SBK_OK;
    greedy_reset_kernel<<<n_rows, 128, 0, stream>>>(tokens, tok_stride, bos, step_arr, has_ended, ended_count, emb, pe, d,
                                                   sqrtf(static_cast<float>(d)), x);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int greedy_select(const float* logits, int n_rows, int V, int* step_arr, int eos, int* tokens, int tok_stride,
                  int* has_ended, int* ended_count, int* pred, float* score, int out_stride, float* log_probs, int L,
                  const float* emb, const float* pe, int d, float* x_next, cudaStream_t stream) {
    if (n_rows == 0) return SBK_OK;
    SBK_CUDA_CHECK(launch_k(greedy_select_kernel, dim3(n_rows), dim3(256), 0, stream, logits, V, step_arr, eos, tokens,
                            tok_stride, has_ended, ended_count, pred, score, out_stride, log_probs, L, emb, pe, d,
                            sqrtf(static_cast<float>(d)), x_next));
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}


// --------------------------------------------------------------------------- post-norm helpers (TransformerLM)
// x = LayerNorm(x) in place (fp32) + fp16 copy for the next projection: the post-norm residual stream of
// TransformerEncoderLayer(normalize_before=False) (Transformer.py:466-481). One warp per row.  Rows lie `pitch` apart; the
// statistics are over the first D channels, and channels D .. pitch - 1 are written as zero (a padded LM's residual stream).
__global__ void __launch_bounds__(256)
layernorm_dual_kernel(float* __restrict__ x, __half* __restrict__ x16, const float* __restrict__ gamma,
                      const float* __restrict__ beta, int M, int D, int pitch, float eps, int write_f32) {
    pdl_trigger();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31;
    float* xr = x + static_cast<size_t>(row) * pitch;
    float s = 0.0f;
    for (int j = lane; j < D; j += 32) s += xr[j];
    const float mean = warp_sum(s) / D;
    float q = 0.0f;
    for (int j = lane; j < D; j += 32) {
        const float d0 = xr[j] - mean;
        q += d0 * d0;
    }
    const float rstd = rsqrtf(warp_sum(q) / D + eps);
    for (int j = lane; j < pitch; j += 32) {
        const float y = j < D ? (xr[j] - mean) * rstd * __ldg(gamma + j) + __ldg(beta + j) : 0.0f;
        if (write_f32) xr[j] = y;
        x16[static_cast<size_t>(row) * pitch + j] = float2half_sat(y);
    }
}

// Same, the row held in registers (NV float4 per lane, D = 128 * NV): one read of x instead of three dependent passes --
// this kernel sits 26 times on the critical path of every TransformerLM scorer step.
template <int NV>
__global__ void __launch_bounds__(128)
layernorm_dual_reg_kernel(float* __restrict__ x, __half* __restrict__ x16, const float* __restrict__ gamma,
                          const float* __restrict__ beta, int M, float eps, int write_f32) {
    pdl_trigger();
    pdl_wait();
    constexpr int D = NV * 128;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31;
    float4* xr = reinterpret_cast<float4*>(x + static_cast<size_t>(row) * D);
    float4 v[NV];
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < NV; ++i) { v[i] = xr[i * 32 + lane]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
    const float mean = warp_sum(s) / D;
    float q = 0.0f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
        q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
    const float rstd = rsqrtf(warp_sum(q) / D + eps);
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
    uint2* o16 = reinterpret_cast<uint2*>(x16 + static_cast<size_t>(row) * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const float4 g = __ldg(g4 + i * 32 + lane), bb = __ldg(b4 + i * 32 + lane);
        float4 y;
        y.x = v[i].x * rstd * g.x + bb.x; y.y = v[i].y * rstd * g.y + bb.y;
        y.z = v[i].z * rstd * g.z + bb.z; y.w = v[i].w * rstd * g.w + bb.w;
        if (write_f32) xr[i * 32 + lane] = y;
        const __half2 h0 = floats2half2_sat(y.x, y.y), h1 = floats2half2_sat(y.z, y.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&h0); pk.y = *reinterpret_cast<const uint32_t*>(&h1);
        o16[i * 32 + lane] = pk;
    }
}

int layernorm_dual(float* x, __half* x16, const float* gamma, const float* beta, int M, int D, int pitch, float eps,
                   bool write_f32, cudaStream_t stream) {
    SBK_REQUIRE(D >= 1 && pitch >= D, "layernorm_dual: D=%d, pitch=%d", D, pitch);
    if (M == 0) return SBK_OK;
    const int wf = write_f32 ? 1 : 0;
    const dim3 grid(ceil_div(M, 4)), block(128);
    switch (D % 128 == 0 && pitch == D ? D / 128 : 0) {
        case 2: SBK_CUDA_CHECK(launch_k(layernorm_dual_reg_kernel<2>, grid, block, 0, stream, x, x16, gamma, beta, M, eps, wf)); break;
        case 4: SBK_CUDA_CHECK(launch_k(layernorm_dual_reg_kernel<4>, grid, block, 0, stream, x, x16, gamma, beta, M, eps, wf)); break;
        case 6: SBK_CUDA_CHECK(launch_k(layernorm_dual_reg_kernel<6>, grid, block, 0, stream, x, x16, gamma, beta, M, eps, wf)); break;
        case 8: SBK_CUDA_CHECK(launch_k(layernorm_dual_reg_kernel<8>, grid, block, 0, stream, x, x16, gamma, beta, M, eps, wf)); break;
        default:
            SBK_CUDA_CHECK(launch_k(layernorm_dual_kernel, dim3(ceil_div(M, 8)), dim3(256), 0, stream, x, x16, gamma, beta, M, D,
                                    pitch, eps, wf));
    }
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// out[r][j] = weight * log_softmax(logits[r] / temperature)[j]   (TransformerLMScorer.score scorer.py:532-543 times
// ScorerBuilder's weight :1252).  One CTA per row.
__global__ void __launch_bounds__(256)
weighted_log_softmax_kernel(const float* __restrict__ logits, float* __restrict__ out, int V, float inv_temp, float weight) {
    __shared__ float s_red[8];
    pdl_trigger();
    pdl_wait();
    const int r = blockIdx.x, tid = threadIdx.x;
    const float* lg = logits + static_cast<size_t>(r) * V;
    float mx = -INFINITY;
    for (int j = tid; j < V; j += 256) mx = fmaxf(mx, lg[j] * inv_temp);
    mx = warp_max(mx);
    if ((tid & 31) == 0) s_red[tid >> 5] = mx;
    __syncthreads();
    mx = s_red[0];
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w]);
    __syncthreads();
    float sm = 0.0f;
    for (int j = tid; j < V; j += 256) sm += expf(lg[j] * inv_temp - mx);
    sm = warp_sum(sm);
    if ((tid & 31) == 0) s_red[tid >> 5] = sm;
    __syncthreads();
    float tot = 0.0f;
    for (int w = 0; w < 8; ++w) tot += s_red[w];
    const float lse = mx + logf(tot);
    for (int j = tid; j < V; j += 256) out[static_cast<size_t>(r) * V + j] = weight * (lg[j] * inv_temp - lse);
}

int weighted_log_softmax(const float* logits, float* out, int rows, int V, float temperature, float weight,
                         cudaStream_t stream) {
    if (rows == 0) return SBK_OK;
    SBK_CUDA_CHECK(launch_k(weighted_log_softmax_kernel, dim3(rows), dim3(256), 0, stream, logits, out, V, 1.0f / temperature,
                            weight));
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// --------------------------------------------------------------------------- beam search step
// decoders/seq2seq.py search_step (:1478-1598) for one utterance per CTA, scorer-less path:
//   log_probs = log_softmax(logits / temperature)                                   (:1929-1934)
//   eos -> minus_inf while step < min_decode_steps (:978-996); eos threshold (:998-1017, :851-867)
//   scores = (sequence_scores + log_probs) / (step + 1) if length_normalization      (:1229-1234)
//   top-`beam` over beam * V candidates, tokens = cand % V, predecessors = cand // V (:1237-1257)
//   sequence_scores of beams that emitted eos -> -inf                                (:1586)
// plus: the per-step history the host needs to replay hypothesis bookkeeping, the KV-cache lineage of the new
// beams, their next decoder input (embedding + positional encoding) and the per-utterance finished counters.
constexpr int BS_MAXB = 16;
constexpr int BS_THREADS = 256;

struct BeamArgs {
    const float* logits; int V; int beam; int n_bh; int S_max;
    float* seq_scores;            // [2][n_bh] ping-pong by step parity
    int* lineage;                 // [2][n_bh][S_max] ping-pong by step parity
    int* step_arr;                // [n_bh]
    int* finished;                // [B] eos hypotheses seen so far (capped at beam)
    int* n_full;                  // number of utterances whose beam is full
    int* hist_tok; int* hist_pred; float* hist_score; float* hist_lp;  // [max_steps][n_bh]
    float inv_temp, eos_threshold, minus_inf;
    int min_steps, eos, use_eos_threshold, length_norm;
    const float* emb; const float* pe; int d; float sqrt_d; float* x_next;
    // optional shallow-fusion scorer (TransformerLMScorer): pre-weighted scores added to the (masked) log-probs,
    // and the LM's own next input (embedding + PE in fp32 and fp16) and token cache (pad-mask on id 0)
    const float* add_scores;
    const float* add_row;   // [n_bh] per-hypothesis score added to every token (CoverageScorer), or null
    float attn_weight; int blank; float add_const;
    const float* lm_emb; const float* lm_pe; int lm_d; float lm_scale; float* lm_x_next; __half* lm_x16_next; int* tok_cache;
    float* scr_val; int* scr_idx; float* scr_lse;   // beam_rows_kernel -> beam_merge_kernel
};

// Two kernels.  beam_rows_kernel, one CTA per hypothesis row (B * beam CTAs instead of B): the row's log-sum-exp, masked eos
// log-prob and its own top-`beam` candidates under the final score -- the utterance's top-`beam` of beam * V is a subset
// of the union of the rows' top-`beam`.  Both kernels rank candidates in argmax_takes's order: NaN first whatever its sign,
// then score descending, then candidate index ascending; every candidate counts, -inf ones included, so that an utterance
// with fewer than `beam` finite candidates takes real (token, row) pairs as torch.topk does.  beam_merge_kernel, one
// CTA per utterance: ranks the beam * beam survivors, then does the bookkeeping.  Scratch: [n_bh][BS_MAXB] scores,
// [n_bh][BS_MAXB] candidate indices (k * V + token), [n_bh] log-sum-exp.
__global__ void __launch_bounds__(BS_THREADS) beam_rows_kernel(const BeamArgs a) {
    __shared__ float s_red[BS_THREADS / 32];
    __shared__ int s_redi[BS_THREADS / 32];
    __shared__ float s_lse, s_eos;
    __shared__ float s_val[BS_THREADS][BS_MAXB + 1];
    __shared__ int s_idx[BS_THREADS][BS_MAXB + 1];
    __shared__ int s_redx[BS_THREADS / 32];
    pdl_trigger();
    pdl_wait();
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int beam = a.beam, V = a.V;
    const int k = row % beam;
    const int step = a.step_arr[row];
    const float seq = a.seq_scores[static_cast<size_t>(step & 1) * a.n_bh + row];
    const float* lg = a.logits + static_cast<size_t>(row) * V;
    const float* add = a.add_scores ? a.add_scores + static_cast<size_t>(row) * V : nullptr;
    const float add_row = a.add_row ? a.add_row[row] : 0.0f;
    // ---- phase 1: log-sum-exp of logits / T and the (masked) eos log-prob
    {
        float mx = -INFINITY;
        for (int j = tid; j < V; j += BS_THREADS) mx = fmaxf(mx, lg[j] * a.inv_temp);
        mx = warp_max(mx);
        if (lane == 0) s_red[warp] = mx;
        __syncthreads();
        mx = s_red[0];
        for (int w = 1; w < BS_THREADS / 32; ++w) mx = fmaxf(mx, s_red[w]);
        __syncthreads();
        float sm = 0.0f, mx_noeos = -INFINITY;
        for (int j = tid; j < V; j += BS_THREADS) {
            const float v = lg[j] * a.inv_temp;
            sm += expf(v - mx);
            if (j != a.eos) mx_noeos = fmaxf(mx_noeos, v);
        }
        sm = warp_sum(sm);
        mx_noeos = warp_max(mx_noeos);
        if (lane == 0) { s_red[warp] = sm; s_redi[warp] = __float_as_int(mx_noeos); }
        __syncthreads();
        if (tid == 0) {
            float tot = 0.0f, mne = -INFINITY;
            for (int w = 0; w < BS_THREADS / 32; ++w) { tot += s_red[w]; mne = fmaxf(mne, __int_as_float(s_redi[w])); }
            const float lse = mx + logf(tot);
            float eos_lp = a.attn_weight * (lg[a.eos] * a.inv_temp - lse);
            if (step < a.min_steps) eos_lp = a.minus_inf;
            if (a.use_eos_threshold) {
                const float max_lp = fmaxf(a.attn_weight * (mne - lse), eos_lp);
                if (!(eos_lp > a.eos_threshold * max_lp)) eos_lp = a.minus_inf;
            }
            if (add) eos_lp += add[a.eos];  // ScorerBuilder.score
            eos_lp += a.add_const + add_row;
            s_lse = lse;
            s_eos = eos_lp;
            a.scr_lse[row] = lse;
        }
        __syncthreads();
    }
    // ---- phase 2: every thread keeps its own sorted top-`beam` of the candidates it scans
    float bv[BS_MAXB];
    int bi[BS_MAXB];
#pragma unroll
    for (int i = 0; i < BS_MAXB; ++i) { bv[i] = -INFINITY; bi[i] = 0x7fffffff; }
    const float inv_len = a.length_norm ? 1.0f / static_cast<float>(step + 1) : 1.0f;
    const float lse = s_lse, eos_lp = s_eos;
    for (int j = tid; j < V; j += BS_THREADS) {
        float lp;
        if (j == a.eos) lp = eos_lp;
        else {
            lp = a.attn_weight * (lg[j] * a.inv_temp - lse);
            if (j == a.blank) lp = a.minus_inf;
            if (add) lp += add[j];
            lp += a.add_const;
            if (a.add_row) lp += add_row;
        }
        const float sc = (seq + lp) * inv_len;
        int ix = k * V + j;
        if (argmax_takes(sc, ix, bv[BS_MAXB - 1], bi[BS_MAXB - 1])) {  // insert (list in candidate order; first `beam` matter)
            float v = sc;
#pragma unroll
            for (int i = 0; i < BS_MAXB; ++i) {
                if (argmax_takes(v, ix, bv[i], bi[i])) {
                    const float tv = bv[i]; const int ti = bi[i];
                    bv[i] = v; bi[i] = ix;
                    v = tv; ix = ti;
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < BS_MAXB; ++i) { s_val[tid][i] = bv[i]; s_idx[tid][i] = bi[i]; }
    s_val[tid][BS_MAXB] = -INFINITY;
    s_idx[tid][BS_MAXB] = 0x7fffffff;
    __syncthreads();
    // ---- phase 3: merge -- `beam` rounds of a block-wide arg-max over the heads of the per-thread lists
    int head = 0;
    for (int r = 0; r < beam; ++r) {
        float v = s_val[tid][head];
        int ix = s_idx[tid][head];
        int who = tid;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, v, o);
            const int oi = __shfl_xor_sync(0xffffffffu, ix, o);
            const int ow = __shfl_xor_sync(0xffffffffu, who, o);
            if (argmax_takes(ov, oi, v, ix) || (oi == ix && ow < who)) { v = ov; ix = oi; who = ow; }
        }
        if (lane == 0) { s_red[warp] = v; s_redi[warp] = who; s_redx[warp] = ix; }
        __syncthreads();
        if (tid == 0) {
            float best = s_red[0];
            int bw = s_redi[0], bx = s_redx[0];
            for (int w = 1; w < BS_THREADS / 32; ++w)
                if (argmax_takes(s_red[w], s_redx[w], best, bx)) { best = s_red[w]; bw = s_redi[w]; bx = s_redx[w]; }
            s_redi[0] = bw;
            a.scr_val[row * BS_MAXB + r] = best;
            a.scr_idx[row * BS_MAXB + r] = bx;
        }
        __syncthreads();
        if (tid == s_redi[0]) ++head;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(BS_THREADS) beam_merge_kernel(const BeamArgs a) {
    __shared__ float s_v[BS_MAXB * BS_MAXB];
    __shared__ int s_i[BS_MAXB * BS_MAXB];
    __shared__ int s_wtok[BS_MAXB], s_wpred[BS_MAXB];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, tid = threadIdx.x;
    const int beam = a.beam, V = a.V;
    const int row0 = b * beam;
    const int step = a.step_arr[row0];
    float* seq_out = a.seq_scores + static_cast<size_t>((step + 1) & 1) * a.n_bh;
    const int n = beam * beam;
    float v = -INFINITY;
    int ix = 0x7fffffff;
    if (tid < n) {
        const int r = tid / beam, q = tid - r * beam;
        v = a.scr_val[(row0 + r) * BS_MAXB + q];
        ix = a.scr_idx[(row0 + r) * BS_MAXB + q];
        s_v[tid] = v; s_i[tid] = ix;
    }
    __syncthreads();
    if (tid < n) {
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const float ov = s_v[j];
            const int oi = s_i[j];
            rank += (argmax_takes(ov, oi, v, ix) || (oi == ix && j < tid)) ? 1 : 0;
        }
        if (rank < beam) {
            int kk = 0, tok = 0;
            if (ix != 0x7fffffff) { kk = ix / V; tok = ix - kk * V; }
            const int row = row0 + rank, prow = row0 + kk;
            const float raw_lp = a.attn_weight * (a.logits[static_cast<size_t>(prow) * V + tok] * a.inv_temp - a.scr_lse[prow]);
            const size_t h = static_cast<size_t>(step) * a.n_bh + row;
            a.hist_tok[h] = tok; a.hist_pred[h] = prow; a.hist_score[h] = v; a.hist_lp[h] = raw_lp;
            float ns = a.length_norm ? v * static_cast<float>(step + 1) : v;
            if (tok == a.eos) ns = -INFINITY;
            seq_out[row] = ns;
            s_wtok[rank] = tok; s_wpred[rank] = prow;
        }
    }
    __syncthreads();
    // ---- finished counters, lineage of the new beams, next decoder inputs, step counters
    if (tid == 0) {
        int n_eos = 0;
        for (int k = 0; k < beam; ++k) n_eos += (s_wtok[k] == a.eos) ? 1 : 0;
        const int before = a.finished[b];
        const int after = min(beam, before + n_eos);
        a.finished[b] = after;
        if (before < beam && after >= beam) atomicAdd(a.n_full, 1);
    }
    const int* lin_in = a.lineage + static_cast<size_t>(step & 1) * a.n_bh * a.S_max;
    int* lin_out = a.lineage + static_cast<size_t>((step + 1) & 1) * a.n_bh * a.S_max;
    for (int i = tid; i < beam * (step + 2); i += BS_THREADS) {
        const int k = i / (step + 2), p = i - k * (step + 2);
        const int row = row0 + k, prow = s_wpred[k];
        int src;
        if (p < step) src = lin_in[static_cast<size_t>(prow) * a.S_max + p];
        else if (p == step) src = prow;   // this step's K/V were written at the predecessor's physical row
        else src = row;                   // next step writes at the new row itself
        lin_out[static_cast<size_t>(row) * a.S_max + p] = src;
    }
    for (int i = tid; i < beam * a.d; i += BS_THREADS) {
        const int k = i / a.d, c = i - k * a.d;
        a.x_next[static_cast<size_t>(row0 + k) * a.d + c] =
            a.emb[static_cast<size_t>(s_wtok[k]) * a.d + c] * a.sqrt_d + a.pe[static_cast<size_t>(step + 1) * a.d + c];
    }
    if (a.lm_emb) {
        for (int i = tid; i < beam * a.lm_d; i += BS_THREADS) {
            const int k = i / a.lm_d, c = i - k * a.lm_d;
            const float v2 = a.lm_emb[static_cast<size_t>(s_wtok[k]) * a.lm_d + c] * a.lm_scale +
                             a.lm_pe[static_cast<size_t>(step + 1) * a.lm_d + c];
            a.lm_x_next[static_cast<size_t>(row0 + k) * a.lm_d + c] = v2;
            a.lm_x16_next[static_cast<size_t>(row0 + k) * a.lm_d + c] = float2half_sat(v2);
        }
        if (tid < beam) a.tok_cache[static_cast<size_t>(row0 + tid) * a.S_max + step + 1] = s_wtok[tid];
    }
    __syncthreads();
    if (tid < beam) a.step_arr[row0 + tid] = step + 1;
}



// --------------------------------------------------------------------------- CoverageScorer (decoders/scorer.py:788-955)
// For the Transformer decoder `attn` is the LAST decoder layer's head-averaged cross-attention distribution of every
// prefix position (Transformer.py:915-963 multihead_attns[-1]); coverage = its sum over the positions, the score
// -(sum_t max(coverage_t, threshold) - T * threshold) / time_step is the same for every token of a hypothesis.
// One CTA per hypothesis row: recompute this step's last-layer attention from the query the layer loop left in q
// (pre-scaled) and the layer's cached keys, add it to the coverage inherited from the row's predecessor (ping-pong by
// step parity, like the CTC state), write the row's score.
struct CoverageArgs {
    const __half* q; int ldq;             // last layer's cross-attention queries [rows, d]
    const __half* kbase; size_t utt_stride; int key_stride; int head_stride;  // key (utt, h, t) at kbase + utt * utt_stride + h * head_stride + t * key_stride
    const int* enc_len; int rows_per_utt; int T; int H;
    float* cov_base;                      // [2][rows][T]
    const int* hist_pred; const int* step_ptr; int n_bh;
    float threshold, weight; float* out;  // out[row] = weight * score
};

__global__ void __launch_bounds__(256) coverage_score_kernel(const CoverageArgs a) {
    extern __shared__ float cv_smem[];  // [T] probabilities of the current head, [T] head average
    float* s_p = cv_smem;
    float* s_avg = cv_smem + a.T;
    __shared__ float s_q[64];
    __shared__ float s_red[8];
    pdl_trigger();
    pdl_wait();
    const int r = blockIdx.x, tid = threadIdx.x, T = a.T;
    const int utt = r / a.rows_per_utt;
    const int n_keys = min(a.enc_len[utt], T);
    const int step = a.step_ptr[r];
    // no visible key: the reference's attention row is NaN (nn.MultiheadAttention), and so are the coverage and the score
    for (int t = tid; t < T; t += 256) s_avg[t] = n_keys > 0 ? 0.0f : NAN;
    for (int h = 0; h < a.H; ++h) {
        __syncthreads();
        if (tid < 64) s_q[tid] = __half2float(a.q[static_cast<size_t>(r) * a.ldq + h * 64 + tid]);
        __syncthreads();
        float mx = -INFINITY;
        for (int t = tid; t < n_keys; t += 256) {
            const __half* kp = a.kbase + static_cast<size_t>(utt) * a.utt_stride + static_cast<size_t>(t) * a.key_stride +
                               static_cast<size_t>(h) * a.head_stride;
            float dot = 0.0f;
#pragma unroll
            for (int e = 0; e < 64; e += 8) {
                const uint4 kv = *reinterpret_cast<const uint4*>(kp + e);
                const __half2* k2 = reinterpret_cast<const __half2*>(&kv);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float2 f = __half22float2(k2[u]);
                    dot = fmaf(f.x, s_q[e + 2 * u], dot);
                    dot = fmaf(f.y, s_q[e + 2 * u + 1], dot);
                }
            }
            s_p[t] = dot;
            mx = fmaxf(mx, dot);
        }
        mx = warp_max(mx);
        if ((tid & 31) == 0) s_red[tid >> 5] = mx;
        __syncthreads();
        mx = s_red[0];
        for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w]);
        __syncthreads();
        float sm = 0.0f;
        for (int t = tid; t < n_keys; t += 256) {
            const float p = __expf(s_p[t] - mx);
            s_p[t] = p;
            sm += p;
        }
        sm = warp_sum(sm);
        if ((tid & 31) == 0) s_red[tid >> 5] = sm;
        __syncthreads();
        float tot = 0.0f;
        for (int w = 0; w < 8; ++w) tot += s_red[w];
        const float inv = 1.0f / (tot * static_cast<float>(a.H));
        for (int t = tid; t < n_keys; t += 256) s_avg[t] += s_p[t] * inv;
    }
    __syncthreads();
    // coverage of the prefix = coverage of the predecessor's prefix + this position's attention
    const float* cov_in = a.cov_base + static_cast<size_t>(step & 1) * a.n_bh * T;
    float* cov_out = a.cov_base + static_cast<size_t>((step + 1) & 1) * a.n_bh * T;
    const int prow = step == 0 ? r : a.hist_pred[static_cast<size_t>(step - 1) * a.n_bh + r];
    float pen = 0.0f;
    for (int t = tid; t < T; t += 256) {
        const float c = (step == 0 ? 0.0f : cov_in[static_cast<size_t>(prow) * T + t]) + s_avg[t];
        cov_out[static_cast<size_t>(r) * T + t] = c;
        pen += c < a.threshold ? a.threshold : c;   // torch.max: a NaN coverage stays NaN
    }
    pen = warp_sum(pen);
    if ((tid & 31) == 0) s_red[tid >> 5] = pen;
    __syncthreads();
    if (tid == 0) {
        float p = 0.0f;
        for (int w = 0; w < 8; ++w) p += s_red[w];
        p -= static_cast<float>(T) * a.threshold;
        a.out[r] = a.weight * (-p / static_cast<float>(step + 1));
    }
}

int coverage_score(const CoverageStep& p, cudaStream_t stream) {
    SBK_REQUIRE(p.T >= 1 && p.T * 8 <= 96 * 1024, "coverage scorer: T=%d out of range", p.T);
    CoverageArgs a;
    a.q = p.q; a.ldq = p.ldq; a.kbase = p.kbase; a.utt_stride = p.utt_stride; a.key_stride = p.key_stride; a.enc_len = p.enc_len;
    a.head_stride = p.head_stride > 0 ? p.head_stride : 64;
    a.rows_per_utt = p.rows_per_utt; a.T = p.T; a.H = p.H; a.cov_base = p.cov_base; a.hist_pred = p.hist_pred;
    a.step_ptr = p.step_ptr; a.n_bh = p.n_bh; a.threshold = p.threshold; a.weight = p.weight; a.out = p.out;
    static bool attr = false;
    if (!attr) {
        SBK_CUDA_CHECK(cudaFuncSetAttribute(coverage_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr = true;
    }
    SBK_CUDA_CHECK(launch_k(coverage_score_kernel, dim3(p.n_bh), dim3(256), static_cast<size_t>(p.T) * 8, stream, a));
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// --------------------------------------------------------------------------- beam step for wide beams (16 < beam <= 128)
// Same contract as beam_step_kernel; the per-thread sorted lists of that kernel (beam registers per thread) do not scale to
// the recipes' test_beam_size = 66 (conformer_large.yaml:132), so the top-`beam` of the beam * V candidates is found by an
// exact radix select: 4 passes of 8 bits over an order-preserving integer image of the score find the beam-th largest value,
// one more pass collects everything above it plus the lowest-index ties, a bitonic sort orders the <= 128 survivors by
// (score descending, candidate index ascending) -- the order the small-beam kernel produces.
constexpr int BL_MAXB = 128;
constexpr int BL_TIECAP = 1024;

// larger score <-> larger key, -inf the smallest; every NaN, whatever its sign, maps to the largest key (argmax_takes's order)
__device__ __forceinline__ uint32_t score_key(float v) {
    if (isnan(v)) return 0xFFFFFFFFu;
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(BS_THREADS) beam_step_large_kernel(const BeamArgs a) {
    __shared__ float s_red[BS_THREADS / 32];
    __shared__ int s_redi[BS_THREADS / 32];
    __shared__ float s_lse[BL_MAXB], s_eos[BL_MAXB], s_seq[BL_MAXB];
    __shared__ int s_hist[256];
    __shared__ uint32_t s_prefix;
    __shared__ int s_remaining, s_nsel, s_ntie;
    __shared__ float s_selv[BL_MAXB];
    __shared__ int s_seli[BL_MAXB];
    __shared__ int s_tie[BL_TIECAP];
    __shared__ int s_wtok[BL_MAXB], s_wpred[BL_MAXB];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int beam = a.beam, V = a.V;
    const int row0 = b * beam;
    const int step = a.step_arr[row0];
    const float* seq_in = a.seq_scores + static_cast<size_t>(step & 1) * a.n_bh;
    float* seq_out = a.seq_scores + static_cast<size_t>((step + 1) & 1) * a.n_bh;
    // ---- phase 1: per beam row log-sum-exp of logits / T and the (masked) eos log-prob (one warp per row)
    for (int k = warp; k < beam; k += BS_THREADS / 32) {
        const float* lg = a.logits + static_cast<size_t>(row0 + k) * V;
        float mx = -INFINITY;
        for (int j = lane; j < V; j += 32) mx = fmaxf(mx, lg[j] * a.inv_temp);
        mx = warp_max(mx);
        float sm = 0.0f, mne = -INFINITY;
        for (int j = lane; j < V; j += 32) {
            const float v = lg[j] * a.inv_temp;
            sm += expf(v - mx);
            if (j != a.eos) mne = fmaxf(mne, v);
        }
        sm = warp_sum(sm);
        mne = warp_max(mne);
        if (lane == 0) {
            const float lse = mx + logf(sm);
            float eos_lp = a.attn_weight * (lg[a.eos] * a.inv_temp - lse);
            if (step < a.min_steps) eos_lp = a.minus_inf;
            if (a.use_eos_threshold) {
                const float max_lp = fmaxf(a.attn_weight * (mne - lse), eos_lp);
                if (!(eos_lp > a.eos_threshold * max_lp)) eos_lp = a.minus_inf;
            }
            if (a.add_scores) eos_lp += a.add_scores[static_cast<size_t>(row0 + k) * V + a.eos];
            eos_lp += a.add_const;
            if (a.add_row) eos_lp += a.add_row[row0 + k];
            s_lse[k] = lse;
            s_eos[k] = eos_lp;
            s_seq[k] = seq_in[row0 + k];
        }
    }
    if (tid == 0) { s_prefix = 0u; s_remaining = beam; s_nsel = 0; s_ntie = 0; }
    __syncthreads();
    const float inv_len = a.length_norm ? 1.0f / static_cast<float>(step + 1) : 1.0f;
    const int n_cand = beam * V;
    auto cand_score = [&](int cidx) -> float {
        const int k = cidx / V, j = cidx - k * V;
        float lp = (j == a.eos) ? s_eos[k]
                                : a.attn_weight * (a.logits[static_cast<size_t>(row0 + k) * V + j] * a.inv_temp - s_lse[k]);
        if (j == a.blank) lp = a.minus_inf;
        if (a.add_scores && j != a.eos) lp += a.add_scores[static_cast<size_t>(row0 + k) * V + j];
        if (j != a.eos) lp += a.add_const;
        if (a.add_row && j != a.eos) lp += a.add_row[row0 + k];
        return (s_seq[k] + lp) * inv_len;
    };
    // ---- phase 2: radix select of the beam-th largest key
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        s_hist[tid] = 0;
        __syncthreads();
        const uint32_t prefix = s_prefix;
        const uint32_t himask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
        for (int cidx = tid; cidx < n_cand; cidx += BS_THREADS) {
            const uint32_t key = score_key(cand_score(cidx));
            if ((key & himask) == (prefix & himask)) atomicAdd(&s_hist[(key >> shift) & 255u], 1);
        }
        __syncthreads();
        if (tid == 0) {
            int need = s_remaining, acc = 0, bin = 255;
            for (; bin > 0; --bin) {
                if (acc + s_hist[bin] >= need) break;
                acc += s_hist[bin];
            }
            s_prefix = prefix | (static_cast<uint32_t>(bin) << shift);
            s_remaining = need - acc;  // how many of the candidates inside this bin are still wanted
        }
        __syncthreads();
    }
    // ---- phase 3: collect keys above the threshold, and the ties
    const uint32_t thr = s_prefix;
    for (int cidx = tid; cidx < n_cand; cidx += BS_THREADS) {
        const float sc = cand_score(cidx);
        const uint32_t key = score_key(sc);
        if (key > thr) {
            const int p = atomicAdd(&s_nsel, 1);
            if (p < BL_MAXB) { s_selv[p] = sc; s_seli[p] = cidx; }
        } else if (key == thr) {
            const int p = atomicAdd(&s_ntie, 1);
            if (p < BL_TIECAP) s_tie[p] = cidx;
        }
    }
    __syncthreads();
    // the lowest-index `remaining` ties complete the selection.  Past BL_TIECAP ties (a row of equal logits gives V of them)
    // the buffer keeps the first to arrive, which the scan order makes the lowest-index ones unless a warp lags four
    // passes behind the others; test_gpu_beam_step.py checks a flat row at V = 5000.
    {
        const int nsel = min(s_nsel, BL_MAXB), ntie = min(s_ntie, BL_TIECAP), want = min(s_remaining, beam - nsel);
        const float tv = [&] { const uint32_t k = thr; const uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k; return __uint_as_float(u); }();
        for (int r = 0; r < want; ++r) {
            int best = 0x7fffffff, bp = -1;
            for (int i = tid; i < ntie; i += BS_THREADS)
                if (s_tie[i] < best) { best = s_tie[i]; bp = i; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const int ob = __shfl_xor_sync(0xffffffffu, best, o), op = __shfl_xor_sync(0xffffffffu, bp, o);
                if (ob < best) { best = ob; bp = op; }
            }
            if (lane == 0) { s_redi[warp] = best; s_red[warp] = __int_as_float(bp); }
            __syncthreads();
            if (tid == 0) {
                int bb = s_redi[0], pp = __float_as_int(s_red[0]);
                for (int w = 1; w < BS_THREADS / 32; ++w)
                    if (s_redi[w] < bb) { bb = s_redi[w]; pp = __float_as_int(s_red[w]); }
                if (pp >= 0) { s_selv[nsel + r] = tv; s_seli[nsel + r] = bb; s_tie[pp] = 0x7fffffff; }
                else { s_selv[nsel + r] = -INFINITY; s_seli[nsel + r] = 0x7fffffff; }
            }
            __syncthreads();
        }
        for (int i = nsel + want + tid; i < BL_MAXB; i += BS_THREADS) { s_selv[i] = -INFINITY; s_seli[i] = 0x7fffffff; }
        __syncthreads();
    }
    // ---- bitonic sort of the 128 slots: score descending, candidate index ascending
    for (int k2 = 2; k2 <= BL_MAXB; k2 <<= 1) {
        for (int j2 = k2 >> 1; j2 > 0; j2 >>= 1) {
            if (tid < BL_MAXB) {
                const int ixj = tid ^ j2;
                if (ixj > tid) {
                    const float v0 = s_selv[tid], v1 = s_selv[ixj];
                    const int i0 = s_seli[tid], i1 = s_seli[ixj];
                    const bool first_after = argmax_takes(v1, i1, v0, i0);  // element at tid should come after ixj
                    const bool up = (tid & k2) == 0;
                    if (first_after == up) { s_selv[tid] = v1; s_selv[ixj] = v0; s_seli[tid] = i1; s_seli[ixj] = i0; }
                }
            }
            __syncthreads();
        }
    }
    // ---- winners (thread k handles new beam k)
    if (tid < beam) {
        const int k = tid;
        const int cand = s_seli[k];
        const float sc = s_selv[k];
        int kk = 0, tok = 0;
        if (cand != 0x7fffffff) { kk = cand / V; tok = cand - kk * V; }
        const int row = row0 + k, prow = row0 + kk;
        const float raw_lp = a.attn_weight * (a.logits[static_cast<size_t>(prow) * V + tok] * a.inv_temp - s_lse[kk]);
        const size_t h = static_cast<size_t>(step) * a.n_bh + row;
        a.hist_tok[h] = tok; a.hist_pred[h] = prow; a.hist_score[h] = sc; a.hist_lp[h] = raw_lp;
        float ns = a.length_norm ? sc * static_cast<float>(step + 1) : sc;
        if (tok == a.eos) ns = -INFINITY;
        seq_out[row] = ns;
        s_wtok[k] = tok; s_wpred[k] = prow;
    }
    __syncthreads();
    // ---- phase 4: finished counters, lineage of the new beams, next decoder inputs, step counters (as beam_step_kernel)
    if (tid == 0) {
        int n_eos = 0;
        for (int k = 0; k < beam; ++k) n_eos += (s_wtok[k] == a.eos) ? 1 : 0;
        const int before = a.finished[b];
        const int after = min(beam, before + n_eos);
        a.finished[b] = after;
        if (before < beam && after >= beam) atomicAdd(a.n_full, 1);
    }
    const int* lin_in = a.lineage + static_cast<size_t>(step & 1) * a.n_bh * a.S_max;
    int* lin_out = a.lineage + static_cast<size_t>((step + 1) & 1) * a.n_bh * a.S_max;
    for (int i = tid; i < beam * (step + 2); i += BS_THREADS) {
        const int k = i / (step + 2), p = i - k * (step + 2);
        const int row = row0 + k, prow = s_wpred[k];
        int src;
        if (p < step) src = lin_in[static_cast<size_t>(prow) * a.S_max + p];
        else if (p == step) src = prow;
        else src = row;
        lin_out[static_cast<size_t>(row) * a.S_max + p] = src;
    }
    for (int i = tid; i < beam * a.d; i += BS_THREADS) {
        const int k = i / a.d, c = i - k * a.d;
        a.x_next[static_cast<size_t>(row0 + k) * a.d + c] =
            a.emb[static_cast<size_t>(s_wtok[k]) * a.d + c] * a.sqrt_d + a.pe[static_cast<size_t>(step + 1) * a.d + c];
    }
    if (a.lm_emb) {
        for (int i = tid; i < beam * a.lm_d; i += BS_THREADS) {
            const int k = i / a.lm_d, c = i - k * a.lm_d;
            const float v = a.lm_emb[static_cast<size_t>(s_wtok[k]) * a.lm_d + c] * a.lm_scale +
                            a.lm_pe[static_cast<size_t>(step + 1) * a.lm_d + c];
            a.lm_x_next[static_cast<size_t>(row0 + k) * a.lm_d + c] = v;
            a.lm_x16_next[static_cast<size_t>(row0 + k) * a.lm_d + c] = float2half_sat(v);
        }
        if (tid < beam) a.tok_cache[static_cast<size_t>(row0 + tid) * a.S_max + step + 1] = s_wtok[tid];
    }
    __syncthreads();
    if (tid < beam) a.step_arr[row0 + tid] = step + 1;
}

// step = 0 state: x = emb[bos] * sqrt(d) + pe[0] (the LM's: lm_emb[bos] * lm_scale + lm_pe[0]); beam 0 alive (score 0),
// others -inf; identity lineage.
__global__ void beam_reset_kernel(int n_bh, int beam, int S_max, int bos, int* step_arr, float* seq_scores, int* lineage,
                                  int* finished, int* n_full, const float* __restrict__ emb, const float* __restrict__ pe,
                                  int d, float sqrt_d, float* __restrict__ x, const float* __restrict__ lm_emb,
                                  const float* __restrict__ lm_pe, int lm_d, float lm_scale, float* __restrict__ lm_x,
                                  __half* __restrict__ lm_x16, int* __restrict__ tok_cache) {
    const int r = blockIdx.x;
    if (threadIdx.x == 0) {
        step_arr[r] = 0;
        seq_scores[r] = (r % beam == 0) ? 0.0f : -INFINITY;
        seq_scores[n_bh + r] = -INFINITY;
        lineage[static_cast<size_t>(r) * S_max] = r;
        if (r % beam == 0) finished[r / beam] = 0;
        if (r == 0) *n_full = 0;
    }
    const float* e = emb + static_cast<size_t>(bos) * d;
    for (int i = threadIdx.x; i < d; i += blockDim.x) x[static_cast<size_t>(r) * d + i] = e[i] * sqrt_d + pe[i];
    if (lm_emb) {
        for (int i = threadIdx.x; i < lm_d; i += blockDim.x) {
            const float v = lm_emb[static_cast<size_t>(bos) * lm_d + i] * lm_scale + lm_pe[i];
            lm_x[static_cast<size_t>(r) * lm_d + i] = v;
            lm_x16[static_cast<size_t>(r) * lm_d + i] = float2half_sat(v);
        }
        if (threadIdx.x == 0) tok_cache[static_cast<size_t>(r) * S_max] = bos;
    }
}

int beam_reset(int n_bh, int beam, int S_max, int bos, int* step_arr, float* seq_scores, int* lineage, int* finished,
               int* n_full, const float* emb, const float* pe, int d, float* x, const BeamLm* lm, cudaStream_t stream) {
    beam_reset_kernel<<<n_bh, 128, 0, stream>>>(n_bh, beam, S_max, bos, step_arr, seq_scores, lineage, finished, n_full, emb,
                                                pe, d, sqrtf(static_cast<float>(d)), x, lm ? lm->emb : nullptr,
                                                lm ? lm->pe : nullptr, lm ? lm->d : 0, lm ? lm->scale : 0.f,
                                                lm ? lm->x : nullptr, lm ? lm->x16 : nullptr, lm ? lm->tok_cache : nullptr);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int beam_step(const BeamStepArgs& p, int B, cudaStream_t stream) {
    SBK_REQUIRE(p.beam >= 1 && p.beam <= BL_MAXB, "beam_step: beam_size=%d not in [1, %d]", p.beam, BL_MAXB);
    SBK_REQUIRE(p.beam <= p.V, "beam_step: beam_size=%d exceeds the vocabulary (%d)", p.beam, p.V);
    SBK_REQUIRE(p.path >= 0 && p.path <= 2, "beam_step: path %d (0 by width, 1 rows + merge, 2 radix select)", p.path);
    SBK_REQUIRE(p.path != 1 || p.beam <= BS_MAXB, "beam_step: the rows + merge kernels take beam_size <= %d, not %d", BS_MAXB,
                p.beam);
    BeamArgs a;
    a.logits = p.logits; a.V = p.V; a.beam = p.beam; a.n_bh = B * p.beam; a.S_max = p.S_max;
    a.seq_scores = p.seq_scores; a.lineage = p.lineage; a.step_arr = p.step_arr; a.finished = p.finished; a.n_full = p.n_full;
    a.hist_tok = p.hist_tok; a.hist_pred = p.hist_pred; a.hist_score = p.hist_score; a.hist_lp = p.hist_lp;
    a.inv_temp = 1.0f / p.temperature; a.eos_threshold = p.eos_threshold; a.minus_inf = p.minus_inf;
    a.min_steps = p.min_steps; a.eos = p.eos; a.use_eos_threshold = p.use_eos_threshold; a.length_norm = p.length_norm;
    a.emb = p.emb; a.pe = p.pe; a.d = p.d; a.sqrt_d = sqrtf(static_cast<float>(p.d)); a.x_next = p.x_next;
    a.add_scores = p.add_scores; a.add_row = p.add_row; a.attn_weight = p.attn_weight; a.blank = p.blank; a.add_const = p.add_const;
    a.lm_emb = p.lm.emb; a.lm_pe = p.lm.pe; a.lm_d = p.lm.d; a.lm_scale = p.lm.scale;
    a.lm_x_next = p.lm.x; a.lm_x16_next = p.lm.x16; a.tok_cache = p.lm.tok_cache;
    a.scr_val = nullptr; a.scr_idx = nullptr; a.scr_lse = nullptr;
    if (p.path == 2 || (p.path == 0 && p.beam > BS_MAXB))
        SBK_CUDA_CHECK(launch_k(beam_step_large_kernel, dim3(B), dim3(BS_THREADS), 0, stream, a));
    else {
        SBK_REQUIRE(p.scratch != nullptr, "beam_step: no scratch buffer");
        a.scr_val = p.scratch; a.scr_idx = reinterpret_cast<int*>(p.scratch + (size_t)a.n_bh * BS_MAXB);
        a.scr_lse = p.scratch + (size_t)2 * a.n_bh * BS_MAXB;
        SBK_CUDA_CHECK(launch_k(beam_rows_kernel, dim3(a.n_bh), dim3(BS_THREADS), 0, stream, a));
        SBK_CUDA_CHECK(launch_k(beam_merge_kernel, dim3(B), dim3(BS_THREADS), 0, stream, a));
    }
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // namespace sbk
