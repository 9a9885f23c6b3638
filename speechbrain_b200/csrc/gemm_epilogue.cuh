// Fused GEMM epilogue of the 128 x BN wgmma kernel (gemm_tc.cu): applied to 32 consecutive fp32 accumulator columns of one
// output row, read from the staged accumulator tile (gemm_mainloop.cuh).  The wide kernel (gemm_tc2.cu) has its own,
// working on the accumulator fragments in registers.
#pragma once
#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

// Apply the epilogue to 32 consecutive accumulator columns of one row.
// `pre`: bias (and, for EPI_RESID, residual) values of this full, in-range chunk were fetched by the caller before the
// accumulator was ready (the latency-bound decode-step GEMMs hide two L2 round trips that way).  The bias is a weight
// and may be fetched before pdl_wait(); the residual is the previous kernel's output and only after it.
struct EpiPrefetch {
    float4 bias[8];
    float4 res[8];
    bool on = false;
};
__device__ __forceinline__ void epilogue_prefetch_bias(const GemmEpilogue& e, EpiPrefetch& p, int row, int col0, int M, int N) {
    p.on = row < M && col0 + 32 <= N;
    if (!p.on) return;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        p.bias[j] = e.bias != nullptr ? __ldg(reinterpret_cast<const float4*>(e.bias + col0) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
}
__device__ __forceinline__ void epilogue_prefetch_resid(const GemmEpilogue& e, EpiPrefetch& p, int row, int col0) {
    if (p.on && e.mode == EPI_RESID) {
        const float4* r = reinterpret_cast<const float4*>(e.resid + static_cast<size_t>(row) * e.ldo + col0);
#pragma unroll
        for (int j = 0; j < 8; ++j) p.res[j] = __ldcg(r + j);
    }
}

__device__ __forceinline__ void epilogue_chunk(const GemmEpilogue& e, const uint32_t (&acc)[32], int row, int col0,
                                               int M, int N, const EpiPrefetch& pre) {
    if (row >= M || col0 >= N) return;
    const bool full = (col0 + 32 <= N);
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(acc[j]);
    if (pre.on) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const float4 b = pre.bias[j >> 2];
            v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
        }
    } else if (e.bias != nullptr) {
        if (full) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + col0 + j));
                v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (col0 + j < N) v[j] += __ldg(e.bias + col0 + j);
        }
    }
    switch (e.mode) {
        case EPI_F16: {
            if (e.act == ACT_SILU) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = silu_f(v[j]);
            } else if (e.act == ACT_GELU) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = gelu_erf_f(v[j]);
            } else if (e.act == ACT_RELU) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
            }
            __half* o = reinterpret_cast<__half*>(e.out) + static_cast<size_t>(row) * e.ldo + col0;
            if (full) {
#pragma unroll
                for (int j = 0; j < 32; j += 8) {
                    __half2 h0 = floats2half2_sat(v[j], v[j + 1]), h1 = floats2half2_sat(v[j + 2], v[j + 3]);
                    __half2 h2 = floats2half2_sat(v[j + 4], v[j + 5]), h3 = floats2half2_sat(v[j + 6], v[j + 7]);
                    uint4 u;
                    u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                    u.z = *reinterpret_cast<uint32_t*>(&h2); u.w = *reinterpret_cast<uint32_t*>(&h3);
                    *reinterpret_cast<uint4*>(o + j) = u;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (col0 + j < N) o[j] = float2half_sat(v[j]);
            }
            break;
        }
        case EPI_F32: {
            float* o = reinterpret_cast<float*>(e.out) + static_cast<size_t>(row) * e.ldo + col0;
            if (full) {
#pragma unroll
                for (int j = 0; j < 32; j += 4)
                    *reinterpret_cast<float4*>(o + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (col0 + j < N) o[j] = v[j];
            }
            break;
        }
        case EPI_RESID: {  // out = resid + alpha * (acc + bias); masked rows contribute 0
            float alpha = e.alpha;
            if (e.row_lens != nullptr) {
                const int b = row / e.T, t = row - b * e.T;
                if (t >= e.row_lens[b]) alpha = 0.0f;
            }
            const float* r = e.resid + static_cast<size_t>(row) * e.ldo + col0;
            float* o = reinterpret_cast<float*>(e.out) + static_cast<size_t>(row) * e.ldo + col0;
            if (full) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const float4 x = pre.on ? pre.res[j >> 2] : *reinterpret_cast<const float4*>(r + j);
                    *reinterpret_cast<float4*>(o + j) = make_float4(fmaf(alpha, v[j], x.x), fmaf(alpha, v[j + 1], x.y),
                                                                    fmaf(alpha, v[j + 2], x.z), fmaf(alpha, v[j + 3], x.w));
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (col0 + j < N) o[j] = fmaf(alpha, v[j], r[j]);
            }
            break;
        }
        case EPI_QKV_CACHE: {  // qkv_d % 32 == 0, N == 3 * qkv_d: a 32-column chunk lies in exactly one of q / k / v
            const int sect = col0 / e.qkv_d, c = col0 - sect * e.qkv_d;
            __half* o;
            if (sect == 0) o = reinterpret_cast<__half*>(e.out) + static_cast<size_t>(row) * e.ldo + c;
            else o = (sect == 1 ? e.kcache : e.vcache) +
                     (static_cast<size_t>(row) * e.S_max + __ldg(e.step_ptr + row)) * e.qkv_d + c;
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
                __half2 h0 = floats2half2_sat(v[j], v[j + 1]), h1 = floats2half2_sat(v[j + 2], v[j + 3]);
                __half2 h2 = floats2half2_sat(v[j + 4], v[j + 5]), h3 = floats2half2_sat(v[j + 6], v[j + 7]);
                uint4 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                u.z = *reinterpret_cast<uint32_t*>(&h2); u.w = *reinterpret_cast<uint32_t*>(&h3);
                *reinterpret_cast<uint4*>(o + j) = u;
            }
            break;
        }
        case EPI_GLU: {  // weight rows pre-interleaved [16 values | 16 gates] per 32 columns
            float* o = reinterpret_cast<float*>(e.out) + static_cast<size_t>(row) * e.ldo + (col0 >> 1);
#pragma unroll
            for (int j = 0; j < 16; j += 4)
                *reinterpret_cast<float4*>(o + j) =
                    make_float4(v[j] * sigmoid_f(v[j + 16]), v[j + 1] * sigmoid_f(v[j + 17]),
                                v[j + 2] * sigmoid_f(v[j + 18]), v[j + 3] * sigmoid_f(v[j + 19]));
            break;
        }
        case EPI_ROPE: {  // columns = per-head [q(dh) | k(dh) | v(dh)], dh % 32 == 0
            const int dh = e.head_dim;
            const int within = col0 % (3 * dh);
            const int sect = within / dh;  // 0 q, 1 k, 2 v
            if (sect < 2) {
                const int t = row % e.T;
                const int p0 = (within - sect * dh) >> 1;
                const float* cs = e.rope_cos + static_cast<size_t>(t) * (dh >> 1) + p0;
                const float* sn = e.rope_sin + static_cast<size_t>(t) * (dh >> 1) + p0;
                const float sc = sect == 0 ? e.alpha : 1.0f;
#pragma unroll
                for (int j = 0; j < 32; j += 2) {
                    const float c = __ldg(cs + (j >> 1)), s = __ldg(sn + (j >> 1));
                    const float x0 = v[j], x1 = v[j + 1];
                    v[j] = (x0 * c - x1 * s) * sc;
                    v[j + 1] = (x1 * c + x0 * s) * sc;
                }
            }
            __half* o = reinterpret_cast<__half*>(e.out) + static_cast<size_t>(row) * e.ldo + col0;
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
                __half2 h0 = floats2half2_sat(v[j], v[j + 1]), h1 = floats2half2_sat(v[j + 2], v[j + 3]);
                __half2 h2 = floats2half2_sat(v[j + 4], v[j + 5]), h3 = floats2half2_sat(v[j + 6], v[j + 7]);
                uint4 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                u.z = *reinterpret_cast<uint32_t*>(&h2); u.w = *reinterpret_cast<uint32_t*>(&h3);
                *reinterpret_cast<uint4*>(o + j) = u;
            }
            break;
        }
    }
}

}  // namespace sbk
