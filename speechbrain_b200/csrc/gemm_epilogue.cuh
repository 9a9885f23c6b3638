// Fused GEMM epilogues shared by the wgmma kernels: applied to 32 consecutive fp32 accumulator columns of one output row,
// read from the staged accumulator tile (gemm_mainloop.cuh).
#pragma once
#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

// Apply the epilogue to 32 consecutive accumulator columns of one row.
// `pre`: bias (and, for EPI_RESID, residual) values of this full, in-range chunk were fetched by the caller before the
// accumulator was ready (the latency-bound decode-step GEMMs hide two L2 round trips that way).
struct EpiPrefetch {
    float4 bias[8];
    float4 res[8];
    bool on = false;
};
__device__ __forceinline__ void epilogue_prefetch(const GemmEpilogue& e, EpiPrefetch& p, int row, int col0, int M, int N) {
    p.on = row < M && col0 + 32 <= N;
    if (!p.on) return;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        p.bias[j] = e.bias != nullptr ? __ldg(reinterpret_cast<const float4*>(e.bias + col0) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (e.mode == EPI_RESID) {
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


// ---------------------------------------------------------------------------------------------------------
// Warp-cooperative, COALESCED variant (used by the wide-tile kernel; needs N % 32 == 0 columns per chunk).
// With one row x 32 columns per lane, storing that directly makes every warp-wide store touch
// 32 different 128-byte lines (the epilogue, not the MMA, would bound the GEMM).  Here the chunk is staged
// through a per-warp shared-memory tile (row pitch 144 B, conflict-free for 16-byte accesses) and written back
// with each instruction covering whole row segments (4 rows x 128 B or 8 rows x 64 B).
constexpr int EPI_STG_PITCH = 144;                 // bytes per staged row (32 fp32 + 16 B pad)
constexpr int EPI_STG_BYTES = 32 * EPI_STG_PITCH;  // per warp

// staging pitch per mode: 32 fp32 (+16 B pad) for fp32 outputs, 64 B of payload (+16 B pad) for fp16 / GLU outputs
template <int MODE>
__host__ __device__ constexpr int epi_stg_pitch() { return (MODE == EPI_F32 || MODE == EPI_RESID || MODE == EPI_ROPE) ? EPI_STG_PITCH : 80; }

// EPI_RESID: out aliases resid (x += ...).  The 8 residual loads of a chunk are issued through this helper one chunk AHEAD
// of the epilogue math (the first one before the accumulator is even complete), so their L2/HBM round trip hides behind
// the main loop / the previous chunk instead of being eaten once per chunk (a long-scoreboard stall in every chunk
// of the N=512 GEMMs otherwise); they must also precede the first store or the compiler serialises load i after store i-1.
__device__ __forceinline__ void epilogue_resid_prefetch(const GemmEpilogue& e, float4 (&res)[8], int row_base, int col0, int M,
                                                        int lane) {
    const int seg = lane & 7, rsub = lane >> 3;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = row_base + i * 4 + rsub;
        res[i] = row < M ? __ldcg(reinterpret_cast<const float4*>(e.resid + static_cast<size_t>(row) * e.ldo + col0 + seg * 4))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// EPI_ROPE: the rotation is applied in the write-back phase, where 4 lanes cover 32 consecutive columns of a row (8 rows
// per instruction): each lane needs 4 cos + 4 sin of its row -- one 16-byte load each, 64 contiguous bytes per row.  (With
// one row per lane, every table load touched 32 different lines and the L1 tag stage, not the tensor
// pipe, bounded the QKV GEMM: tensor pipe 18 %, issue slots 12 % busy.)  The 8 loads of a chunk are fetched one chunk
// ahead: with ~200 KB of the SM carved out as shared memory the tables do not survive in L1.
__device__ __forceinline__ void epilogue_rope_prefetch(const GemmEpilogue& e, float4 (&rc)[4], float4 (&rs)[4], int row_base,
                                                       int col0, int lane) {
    const int dh = e.head_dim;
    const int within = col0 % (3 * dh);
    const int sect = within / dh;  // 0 q, 1 k, 2 v
    if (sect < 2) {
        const int p = ((within - sect * dh) >> 1) + (lane & 3) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int t = (row_base + i * 8 + (lane >> 2)) % e.T;
            rc[i] = __ldg(reinterpret_cast<const float4*>(e.rope_cos + static_cast<size_t>(t) * (dh >> 1) + p));
            rs[i] = __ldg(reinterpret_cast<const float4*>(e.rope_sin + static_cast<size_t>(t) * (dh >> 1) + p));
        }
    }
}

template <int MODE, int ACT, int PITCH = EPI_STG_PITCH>
// sbias: this chunk's 32 bias values in shared memory (staged once per tile by the caller), or null -> read e.bias
__device__ __forceinline__ void epilogue_chunk_coalesced(const GemmEpilogue& e, const uint32_t (&acc)[32], uint8_t* stg,
                                                         int row_base, int col0, int M, int lane, float4 (&res)[8],
                                                         int next_col0, float4 (&rc)[4], float4 (&rs)[4],
                                                         const float* sbias = nullptr) {
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(acc[j]);
    if (sbias != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const float4 b = *reinterpret_cast<const float4*>(sbias + j);   // same address in every lane: broadcast
            v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
        }
    } else if (e.bias != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + col0 + j));
            v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
        }
    }
    const int my_row = row_base + lane;
    const uint32_t stg_s = smem_u32(stg);
    const uint32_t my = stg_s + lane * PITCH;
    constexpr int out_bytes_per_row = (MODE == EPI_F32 || MODE == EPI_RESID) ? 128 : 64;  // 32 fp32 | 32 fp16 / 16 fp32
    {
        if constexpr (MODE == EPI_F32 || MODE == EPI_RESID || MODE == EPI_ROPE) {  // staged as fp32
            if constexpr (MODE == EPI_RESID) {
                float alpha = e.alpha;
                if (e.row_lens != nullptr && my_row < M) {
                    const int b = my_row / e.T, t = my_row - b * e.T;
                    if (t >= e.row_lens[b]) alpha = 0.0f;
                }
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] *= alpha;
            }
#pragma unroll
            for (int j = 0; j < 32; j += 4)
                sts128(my + j * 4, f4_as_u4(make_float4(v[j], v[j + 1], v[j + 2], v[j + 3])));
        } else if constexpr (MODE == EPI_GLU) {
            if constexpr (ACT == ACT_SILU_FAST) {
#pragma unroll
                for (int j = 0; j < 16; j += 4)
                    sts128(my + j * 4, f4_as_u4(make_float4(v[j] * sigmoid_fast(v[j + 16]), v[j + 1] * sigmoid_fast(v[j + 17]),
                                                            v[j + 2] * sigmoid_fast(v[j + 18]), v[j + 3] * sigmoid_fast(v[j + 19]))));
            } else {
#pragma unroll
                for (int j = 0; j < 16; j += 4)
                    sts128(my + j * 4, f4_as_u4(make_float4(v[j] * sigmoid_f(v[j + 16]), v[j + 1] * sigmoid_f(v[j + 17]),
                                                            v[j + 2] * sigmoid_f(v[j + 18]), v[j + 3] * sigmoid_f(v[j + 19]))));
            }
        } else {  // EPI_F16 -> 32 halfs
            if constexpr (ACT == ACT_SILU) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = silu_f(v[j]);
            } else if constexpr (ACT == ACT_SILU_FAST) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = silu_fast(v[j]);
            } else if constexpr (ACT == ACT_GELU) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = gelu_erf_f(v[j]);
            }
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
                __half2 h0 = floats2half2_sat(v[j], v[j + 1]), h1 = floats2half2_sat(v[j + 2], v[j + 3]);
                __half2 h2 = floats2half2_sat(v[j + 4], v[j + 5]), h3 = floats2half2_sat(v[j + 6], v[j + 7]);
                uint4 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                u.z = *reinterpret_cast<uint32_t*>(&h2); u.w = *reinterpret_cast<uint32_t*>(&h3);
                sts128(my + j * 2, u);
            }
        }
    }
    __syncwarp();
    if constexpr (out_bytes_per_row == 128) {
        const int seg = lane & 7, rsub = lane >> 3;  // 8 lanes x 16 B per row, 4 rows per instruction
        float* outp = reinterpret_cast<float*>(e.out);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = i * 4 + rsub;
            const int row = row_base + r;
            if (row < M) {
                float4 val = u4_as_f4(lds128(stg_s + r * PITCH + seg * 16));
                if constexpr (MODE == EPI_RESID) {
                    val.x += res[i].x; val.y += res[i].y; val.z += res[i].z; val.w += res[i].w;
                }
                *reinterpret_cast<float4*>(outp + static_cast<size_t>(row) * e.ldo + col0 + seg * 4) = val;
            }
        }
        if constexpr (MODE == EPI_RESID)
            if (next_col0 >= 0) epilogue_resid_prefetch(e, res, row_base, next_col0, M, lane);
    } else if constexpr (MODE == EPI_ROPE) {
        const int seg = lane & 3, rsub = lane >> 2;  // 4 lanes x 8 columns (4 rotation pairs) per row, 8 rows per instruction
        const int dh = e.head_dim;
        const int sect = (col0 % (3 * dh)) / dh;     // 0 q (rotated, scaled), 1 k (rotated), 2 v
        const float sc = sect == 0 ? e.alpha : 1.0f;
        __half* outp = reinterpret_cast<__half*>(e.out);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = i * 8 + rsub;
            const int row = row_base + r;
            float4 x0 = u4_as_f4(lds128(stg_s + r * PITCH + seg * 32));
            float4 x1 = u4_as_f4(lds128(stg_s + r * PITCH + seg * 32 + 16));
            if (sect < 2) {
                const float4 c = rc[i], s4 = rs[i];
                const float a0 = (x0.x * c.x - x0.y * s4.x) * sc, a1 = (x0.y * c.x + x0.x * s4.x) * sc;
                const float a2 = (x0.z * c.y - x0.w * s4.y) * sc, a3 = (x0.w * c.y + x0.z * s4.y) * sc;
                const float b0 = (x1.x * c.z - x1.y * s4.z) * sc, b1 = (x1.y * c.z + x1.x * s4.z) * sc;
                const float b2 = (x1.z * c.w - x1.w * s4.w) * sc, b3 = (x1.w * c.w + x1.z * s4.w) * sc;
                x0 = make_float4(a0, a1, a2, a3);
                x1 = make_float4(b0, b1, b2, b3);
            }
            if (row < M) {
                __half2 h0 = floats2half2_sat(x0.x, x0.y), h1 = floats2half2_sat(x0.z, x0.w);
                __half2 h2 = floats2half2_sat(x1.x, x1.y), h3 = floats2half2_sat(x1.z, x1.w);
                uint4 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                u.z = *reinterpret_cast<uint32_t*>(&h2); u.w = *reinterpret_cast<uint32_t*>(&h3);
                *reinterpret_cast<uint4*>(outp + static_cast<size_t>(row) * e.ldo + col0 + seg * 8) = u;
            }
        }
        if (next_col0 >= 0) epilogue_rope_prefetch(e, rc, rs, row_base, next_col0, lane);
    } else {
        const int seg = lane & 3, rsub = lane >> 2;  // 4 lanes x 16 B per row, 8 rows per instruction
        uint8_t* outp = reinterpret_cast<uint8_t*>(e.out);
        // byte offset of this chunk inside a row: fp16 -> col0 * 2 ; GLU fp32 (16 columns) -> (col0 / 2) * 4
        const size_t row_pitch = MODE == EPI_GLU ? static_cast<size_t>(e.ldo) * 4 : static_cast<size_t>(e.ldo) * 2;
        const size_t col_off = static_cast<size_t>(col0) * 2;
        if (MODE == EPI_F16 && e.kv_heads > 0) {
            // cross-attention K/V scatter: column c of the [K (d) | V (d)] row goes to part[c / d][utt][head][t][64], so
            // that the decode-step attention streams one contiguous T x 128 B block per (utterance, head)
            const int d = e.kv_heads * 64;
            const int part = col0 / d, cc = col0 - part * d, head = cc >> 6, dcol = cc & 63;
            __half* pbase = reinterpret_cast<__half*>(e.out) + static_cast<size_t>(part) * e.kv_part_stride;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = i * 8 + rsub;
                const int row = row_base + r;
                if (row < M) {
                    const int b = row / e.T, t = row - b * e.T;
                    __half* dst = pbase + ((static_cast<size_t>(b) * e.kv_heads + head) * e.T + t) * 64 + dcol + seg * 8;
                    *reinterpret_cast<uint4*>(dst) = lds128(stg_s + r * PITCH + seg * 16);
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = i * 8 + rsub;
                const int row = row_base + r;
                if (row < M)
                    *reinterpret_cast<uint4*>(outp + static_cast<size_t>(row) * row_pitch + col_off + seg * 16) =
                        lds128(stg_s + r * PITCH + seg * 16);
            }
        }
    }
    __syncwarp();  // staging tile is reused by the next chunk
}

}  // namespace sbk
