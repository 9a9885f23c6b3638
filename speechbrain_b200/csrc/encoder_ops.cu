// Non-GEMM pieces of the Conformer encoder layer:
//   * row LayerNorm fp32 -> fp16 (GEMM A operand) or fp32 in place        (nn.LayerNorm call sites in
//     Conformer.py:425-445 ffn LN, :146-157 conv LN, nnet/normalization.py:242 norm1/norm2, final norm :700)
//   * depthwise Conv1d(k=31) + bias + LayerNorm + Swish                   (Conformer.py:136-157,318-325)
//   * self-attention, flash style on mma.sync tensor cores, RoPE or Transformer-XL relative
//     position bias                                                       (nnet/attention.py:555-742, :1284-1399)
#include <algorithm>

#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

// --------------------------------------------------------------------------- LayerNorm
// One warp per row, two-pass statistics in registers. D <= 32 * LN_MAX_PER_LANE.
// PDL (decode step, launched with programmatic stream serialisation): gamma / beta are fetched before pdl_wait(), x after.
constexpr int LN_MAX_PER_LANE = 32;

template <bool OUT_HALF, bool PDL>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float* __restrict__ x, void* __restrict__ out, const float* __restrict__ gamma,
                      const float* __restrict__ beta, int M, int D, float eps, int act_silu) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int nv = D >> 2;  // float4 vectors per row (D % 4 == 0)
    float4 gp[PDL ? LN_MAX_PER_LANE / 4 : 1], bp[PDL ? LN_MAX_PER_LANE / 4 : 1];
    if constexpr (PDL) {
#pragma unroll
        for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
            const int vi = lane + i * 32;
            if (vi < nv && row < M) {
                gp[i] = __ldg(reinterpret_cast<const float4*>(gamma + vi * 4));
                bp[i] = __ldg(reinterpret_cast<const float4*>(beta + vi * 4));
            }
        }
        pdl_trigger();
        pdl_wait();
    }
    if (row >= M) return;
    const float* xr = x + static_cast<size_t>(row) * D;
    float v[LN_MAX_PER_LANE];
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < nv) {
            const float4 t = *reinterpret_cast<const float4*>(xr + vi * 4);
            v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
            s += (t.x + t.y) + (t.z + t.w);
        } else {
            v[4 * i] = v[4 * i + 1] = v[4 * i + 2] = v[4 * i + 3] = 0.0f;
        }
    }
    const float mean = warp_sum(s) / D;
    float q = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < nv) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float d = v[4 * i + j] - mean;
                q += d * d;
            }
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / D + eps);
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < nv) {
            const float4 g = PDL ? gp[PDL ? i : 0] : __ldg(reinterpret_cast<const float4*>(gamma + vi * 4));
            const float4 b = PDL ? bp[PDL ? i : 0] : __ldg(reinterpret_cast<const float4*>(beta + vi * 4));
            float y0 = (v[4 * i] - mean) * rstd * g.x + b.x;
            float y1 = (v[4 * i + 1] - mean) * rstd * g.y + b.y;
            float y2 = (v[4 * i + 2] - mean) * rstd * g.z + b.z;
            float y3 = (v[4 * i + 3] - mean) * rstd * g.w + b.w;
            if (act_silu) { y0 = silu_f(y0); y1 = silu_f(y1); y2 = silu_f(y2); y3 = silu_f(y3); }
            if constexpr (OUT_HALF) {
                __half2 h0 = floats2half2_sat(y0, y1), h1 = floats2half2_sat(y2, y3);
                uint2 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0);
                u.y = *reinterpret_cast<uint32_t*>(&h1);
                *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out) + static_cast<size_t>(row) * D + vi * 4) = u;
            } else {
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + static_cast<size_t>(row) * D + vi * 4) =
                    make_float4(y0, y1, y2, y3);
            }
        }
    }
}

int layernorm_rows(const float* x, void* out, bool out_half, const float* gamma, const float* beta, int M, int D,
                   float eps, bool act_silu, cudaStream_t stream, bool pdl) {
    SBK_REQUIRE(D % 4 == 0 && D <= 32 * LN_MAX_PER_LANE, "layernorm_rows: D=%d unsupported", D);
    if (M == 0) return SBK_OK;
    const int rows_per_cta = 8;
    const dim3 grid(ceil_div(M, rows_per_cta)), block(rows_per_cta * 32);
    if (pdl) {
        SBK_REQUIRE(out_half, "layernorm_rows: the PDL variant writes fp16");
        SBK_CUDA_CHECK(launch_pdl(layernorm_rows_kernel<true, true>, grid, block, 0, stream, true, x, out, gamma, beta, M, D,
                                  eps, static_cast<int>(act_silu)));
    } else if (out_half) {
        layernorm_rows_kernel<true, false><<<grid, block, 0, stream>>>(x, out, gamma, beta, M, D, eps, act_silu);
    } else {
        layernorm_rows_kernel<false, false><<<grid, block, 0, stream>>>(x, out, gamma, beta, M, D, eps, act_silu);
    }
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}


// Two chained LayerNorms over the same row in one pass: y = LN_a(x) (fp32, optional store) and z = LN_b(y) (fp16 GEMM operand
// or fp32).  The Conformer layer ends with norm2 and the next layer starts with the LayerNorm of its first feed-forward
// module (Conformer.py:498 -> :479), the last layer's norm2 is followed by the encoder's final norm (:700): fusing the pair
// saves one launch and one 16 MB read of x per layer.  One warp per row, the row (D <= 1024) lives in registers.
template <bool OUT_HALF>
__global__ void __launch_bounds__(256)
layernorm2_rows_kernel(const float* __restrict__ x, float* __restrict__ y_out, void* __restrict__ z_out,
                       const float* __restrict__ ga, const float* __restrict__ ba, float eps_a,
                       const float* __restrict__ gb, const float* __restrict__ bb, float eps_b, int M, int D) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31;
    const float* xr = x + static_cast<size_t>(row) * D;
    float v[LN_MAX_PER_LANE];
    const int nv = D >> 2;
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (vi < nv) t = *reinterpret_cast<const float4*>(xr + vi * 4);
        v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
        s += (t.x + t.y) + (t.z + t.w);
    }
    float mean = warp_sum(s) / D;
    float q = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i)
        if (lane + i * 32 < nv) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { const float d = v[4 * i + j] - mean; q += d * d; }
        }
    float rstd = rsqrtf(warp_sum(q) / D + eps_a);
    s = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < nv) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(ga + vi * 4));
            const float4 b = __ldg(reinterpret_cast<const float4*>(ba + vi * 4));
            v[4 * i] = (v[4 * i] - mean) * rstd * g.x + b.x;
            v[4 * i + 1] = (v[4 * i + 1] - mean) * rstd * g.y + b.y;
            v[4 * i + 2] = (v[4 * i + 2] - mean) * rstd * g.z + b.z;
            v[4 * i + 3] = (v[4 * i + 3] - mean) * rstd * g.w + b.w;
            if (y_out != nullptr)
                *reinterpret_cast<float4*>(y_out + static_cast<size_t>(row) * D + vi * 4) =
                    make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
            s += (v[4 * i] + v[4 * i + 1]) + (v[4 * i + 2] + v[4 * i + 3]);
        }
    }
    mean = warp_sum(s) / D;
    q = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i)
        if (lane + i * 32 < nv) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { const float d = v[4 * i + j] - mean; q += d * d; }
        }
    rstd = rsqrtf(warp_sum(q) / D + eps_b);
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < nv) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(gb + vi * 4));
            const float4 b = __ldg(reinterpret_cast<const float4*>(bb + vi * 4));
            const float z0 = (v[4 * i] - mean) * rstd * g.x + b.x, z1 = (v[4 * i + 1] - mean) * rstd * g.y + b.y;
            const float z2 = (v[4 * i + 2] - mean) * rstd * g.z + b.z, z3 = (v[4 * i + 3] - mean) * rstd * g.w + b.w;
            if constexpr (OUT_HALF) {
                __half2 h0 = floats2half2_sat(z0, z1), h1 = floats2half2_sat(z2, z3);
                uint2 u;
                u.x = *reinterpret_cast<uint32_t*>(&h0);
                u.y = *reinterpret_cast<uint32_t*>(&h1);
                *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(z_out) + static_cast<size_t>(row) * D + vi * 4) = u;
            } else {
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(z_out) + static_cast<size_t>(row) * D + vi * 4) =
                    make_float4(z0, z1, z2, z3);
            }
        }
    }
}

int layernorm2_rows(const float* x, float* y_out, void* z_out, bool z_half, const float* ga, const float* ba, float eps_a,
                    const float* gb, const float* bb, float eps_b, int M, int D, cudaStream_t stream) {
    SBK_REQUIRE(D % 4 == 0 && D <= 32 * LN_MAX_PER_LANE, "layernorm2_rows: D=%d unsupported", D);
    if (M == 0) return SBK_OK;
    const int rows_per_cta = 8;
    if (z_half)
        layernorm2_rows_kernel<true><<<ceil_div(M, rows_per_cta), rows_per_cta * 32, 0, stream>>>(x, y_out, z_out, ga, ba, eps_a,
                                                                                                 gb, bb, eps_b, M, D);
    else
        layernorm2_rows_kernel<false><<<ceil_div(M, rows_per_cta), rows_per_cta * 32, 0, stream>>>(x, y_out, z_out, ga, ba, eps_a,
                                                                                                  gb, bb, eps_b, M, D);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// fp32 -> fp16 cast (used for goldens-driven tests and the decoder memory)
__global__ void cast_f32_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, size_t n) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x)
        out[i] = float2half_sat(in[i]);
}
int cast_f32_f16(const float* in, __half* out, size_t n, cudaStream_t stream) {
    if (n == 0) return SBK_OK;
    const int blocks = static_cast<int>(std::min<size_t>((n + 255) / 256, SBK_NUM_SMS * 16));
    cast_f32_f16_kernel<<<blocks, 256, 0, stream>>>(in, out, n);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// --------------------------------------------------------------------------- depthwise conv + LN + Swish
// glu [B*T, D] fp32 (GLU output) -> out [B*T, D] fp16 = Swish(LN(dwconv(glu) + bias)).  The tap weights arrive TAP-MAJOR
// ([K, D], repacked from the reference's (D, 1, K) at load time): thread = channel, so the 31 weight loads of a thread are
// coalesced across the warp (the channel-major layout made every load touch 32 cache lines).
// Zero padding at utterance edges only: padded frames inside T are real inputs (Conformer.py:318-325
// runs the conv before masking). One CTA per (utterance, tile of DW_TT frames); the (DW_TT + K - 1) x D
// input slab is staged in shared memory once.
constexpr int DW_TT = 16;

// KT > 0: compile-time kernel size (taps held in registers); KT == 0: runtime K.  MAXC: channels per thread (D <= 256 * MAXC)
// CHUNKED: Dynamic Chunk Convolution (Conformer.py:190-313): for every output frame the inputs beyond the end of its own
// chunk of `chunk` frames count as zero (the past, other chunks included, is visible as usual).
template <int KT, int MAXC, bool CHUNKED = false>
__global__ void __launch_bounds__(256, 2)
dwconv_ln_swish_kernel(const float* __restrict__ glu, int T, int D, int K, const float* __restrict__ wdw /*[K,D] tap-major*/,
                       const float* __restrict__ bdw, const float* __restrict__ gamma, const float* __restrict__ beta,
                       float eps, __half* __restrict__ out, int chunk) {
    extern __shared__ __align__(128) float dw_smem[];
    __shared__ uint64_t bar;
    const int halo = (K - 1) / 2;
    const int rows_in = DW_TT + K - 1;
    float* slab = dw_smem;   // [rows_in][D]; rows [0, DW_TT) are re-used for the conv outputs after the tap loop
    const int b = blockIdx.y, t0 = blockIdx.x * DW_TT;
    const float* src = glu + static_cast<size_t>(b) * T * D;
    // valid input rows [r_lo, r_hi) of the slab are contiguous in global memory: stage them with bulk TMA copies
    const int r_lo = max(0, halo - t0), r_hi = min(rows_in, T + halo - t0);
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t row_bytes = static_cast<uint32_t>(D) * 4;
        mbar_arrive_expect_tx(&bar, row_bytes * static_cast<uint32_t>(r_hi - r_lo));
        // the valid rows are contiguous on both sides: a few large bulk copies instead of one 2 KB copy per row (whose
        // serial issue by this one thread was a visible part of the CTA's life)
        for (int r = r_lo; r < r_hi; r += 8) {
            const int nr = min(8, r_hi - r);
            bulk_load_1d(slab + r * D, src + static_cast<size_t>(t0 - halo + r) * D, row_bytes * nr, &bar);
        }
    }
    // zero rows outside the utterance (Conv1d zero padding)
    for (int i = threadIdx.x; i < (r_lo + rows_in - r_hi) * D; i += blockDim.x) {
        int r = i / D;
        const int ch = i - r * D;
        if (r >= r_lo) r += r_hi - r_lo;
        slab[r * D + ch] = 0.0f;
    }
    // tap weights and biases of this thread's channels: fetched while the slab is still in flight
    float wreg[KT > 0 ? MAXC : 1][KT > 0 ? KT : 1];
    float breg[MAXC];
#pragma unroll
    for (int cc = 0; cc < MAXC; ++cc) {
        const int ch = threadIdx.x + cc * 256;
        breg[cc] = 0.0f;
        if (ch < D) {
            breg[cc] = __ldg(bdw + ch);
            if constexpr (KT > 0) {
#pragma unroll
                for (int k = 0; k < KT; ++k) wreg[cc][k] = __ldg(wdw + static_cast<size_t>(k) * D + ch);  // coalesced over channels
            }
        }
    }
    mbar_wait(&bar, 0);
    __syncthreads();
    float acc[MAXC][DW_TT];
#pragma unroll
    for (int cc = 0; cc < MAXC; ++cc) {
        const int ch = threadIdx.x + cc * 256;
        if (ch < D) {
            const float bz = breg[cc];
#pragma unroll
            for (int i = 0; i < DW_TT; ++i) acc[cc][i] = bz;
            const float* w = wdw + ch;  // tap k at w[k * D]
            if constexpr (KT > 0) {
                int lim[CHUNKED ? DW_TT : 1];  // slab row of the first frame past output i's chunk
                if constexpr (CHUNKED) {
#pragma unroll
                    for (int i = 0; i < DW_TT; ++i) lim[i] = ((t0 + i) / chunk + 1) * chunk - t0 + halo;
                }
#pragma unroll
                for (int r = 0; r < DW_TT + KT - 1; ++r) {
                    const float xv = slab[r * D + ch];
#pragma unroll
                    for (int i = 0; i < DW_TT; ++i)
                        if (r - i >= 0 && r - i < KT) {
                            if constexpr (CHUNKED) acc[cc][i] = fmaf(r < lim[i] ? xv : 0.0f, wreg[cc][r - i], acc[cc][i]);
                            else acc[cc][i] = fmaf(xv, wreg[cc][r - i], acc[cc][i]);
                        }
                }
            } else {
                for (int r = 0; r < rows_in; ++r) {
                    const float xv = slab[r * D + ch];
#pragma unroll
                    for (int i = 0; i < DW_TT; ++i) {
                        const int k = r - i;
                        if (k >= 0 && k < K && (!CHUNKED || r < ((t0 + i) / chunk + 1) * chunk - t0 + halo))
                            acc[cc][i] = fmaf(xv, __ldg(w + static_cast<size_t>(k) * D), acc[cc][i]);
                    }
                }
            }
        }
    }
    __syncthreads();  // every thread is done reading the slab: rows [0, DW_TT) now hold the conv outputs
#pragma unroll
    for (int cc = 0; cc < MAXC; ++cc) {
        const int ch = threadIdx.x + cc * 256;
        if (ch < D) {
#pragma unroll
            for (int i = 0; i < DW_TT; ++i) slab[i * D + ch] = acc[cc][i];
        }
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int MAXP = MAXC * 4;  // channel pairs per lane (D <= 256 * MAXC): LayerNorm scale / shift held in registers
    float2 g2[MAXP], b2[MAXP];
#pragma unroll
    for (int p = 0; p < MAXP; ++p) {
        const int j = 2 * lane + 64 * p;
        if (j < D) {
            g2[p] = __ldg(reinterpret_cast<const float2*>(gamma + j));
            b2[p] = __ldg(reinterpret_cast<const float2*>(beta + j));
        }
    }
    for (int i = warp; i < DW_TT; i += (blockDim.x >> 5)) {
        const int t = t0 + i;
        if (t >= T) continue;
        const float* c = slab + i * D;
        float s = 0.0f;
        for (int j = lane; j < D; j += 32) s += c[j];
        const float mean = warp_sum(s) / D;
        float q = 0.0f;
        for (int j = lane; j < D; j += 32) {
            const float d = c[j] - mean;
            q += d * d;
        }
        const float rstd = rsqrtf(warp_sum(q) / D + eps);
        __half* o = out + (static_cast<size_t>(b) * T + t) * D;
#pragma unroll
        for (int p = 0; p < MAXP; ++p) {
            const int j = 2 * lane + 64 * p;
            if (j < D) {
                const float2 cv = *reinterpret_cast<const float2*>(c + j);
                const float y0 = silu_f((cv.x - mean) * rstd * g2[p].x + b2[p].x);
                const float y1 = silu_f((cv.y - mean) * rstd * g2[p].y + b2[p].y);
                *reinterpret_cast<__half2*>(o + j) = floats2half2_sat(y0, y1);
            }
        }
    }
}

int dwconv_ln_swish(const float* glu, int B, int T, int D, int K, const float* wdw, const float* bdw,
                    const float* gamma, const float* beta, float eps, __half* out, cudaStream_t stream, int chunk) {
    SBK_REQUIRE(D % 4 == 0 && D <= 1024 && (K & 1) == 1, "dwconv_ln_swish: D %% 4, D <= 1024 and odd K required (D=%d K=%d)", D, K);
    SBK_REQUIRE((reinterpret_cast<uintptr_t>(glu) & 15) == 0, "dwconv_ln_swish: input must be 16-byte aligned");
    const size_t smem = static_cast<size_t>(DW_TT + K - 1) * D * sizeof(float);
    SBK_REQUIRE(smem <= 200 * 1024, "dwconv_ln_swish: tile too large for shared memory (D=%d K=%d)", D, K);
    auto kern = dwconv_ln_swish_kernel<0, 4>;
    if (chunk > 0) {
        kern = dwconv_ln_swish_kernel<0, 4, true>;
        if (K == 31) kern = D <= 256 ? dwconv_ln_swish_kernel<31, 1, true> : D <= 512 ? dwconv_ln_swish_kernel<31, 2, true>
                                                                                        : dwconv_ln_swish_kernel<31, 4, true>;
    } else if (K == 31) {
        kern = D <= 256 ? dwconv_ln_swish_kernel<31, 1> : D <= 512 ? dwconv_ln_swish_kernel<31, 2> : dwconv_ln_swish_kernel<31, 4>;
    }
    SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(ceil_div(T, DW_TT), B), 256, smem, stream>>>(glu, T, D, K, wdw, bdw, gamma, beta, eps, out, chunk);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// =========================================================================== self-attention
// Flash-style attention for the Conformer encoder on mma.sync.m16n8k16 (fp16 operands, fp32
// accumulate, fp32 online softmax).  One CTA = (utterance b, head h, 64 query rows), 4 warps x 16 rows.
//
//  RoPE  (nnet/attention.py:1284-1399): q,k arrive already rotated (and q pre-scaled by 1/sqrt(d_model))
//        from the QKV GEMM epilogue; scores = q.k ; keys >= len_b are masked (masks_union :1402-1440).
//  RelPos(nnet/attention.py:555-742):   scores = (q+u)s.k + (q+v)s.p_{|i-j|}.  The reference builds a
//        (2T-1)-row table and rel_shifts it (:537-553); row r of the table depends only on |r| (RelPosEncXL
//        :360-408 uses +sin for both halves), so BD[i,j] = (q_i+v).P[|i-j|] with P = linear_pos(pe[0..T-1]).
//        Per key block each warp computes the 16 x 80 band G = Qv.Pband^T on tensor cores, parks it in
//        shared memory and re-reads it diagonally shifted.
//  Padded *query* rows are computed like any other row (the reference does; they leak into valid frames
//  through the depthwise conv), only padded *keys* are masked.
constexpr int ATT_BQ = 64;
constexpr int ATT_BK = 64;

__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t& r0, uint32_t& r1, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    __half2 h = floats2half2_sat(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

template <int DH, int DHP, bool RELPOS>  // DHP = DH rounded up to a multiple of 16 (zero-padded in shared memory)
__global__ void __launch_bounds__(128)
encoder_attention_kernel(const __half* __restrict__ qkv, int ld, int T, const int* __restrict__ lens,
                         const float* __restrict__ pos_u, const float* __restrict__ pos_v,
                         const __half* __restrict__ P, int ldp, float scale, __half* __restrict__ out, int ldo,
                         int chunk, int left_chunks) {
    constexpr int STR = DHP + 8;  // padded row stride (halfs): conflict-free fragment loads
    constexpr int KS = DHP / 16;
    constexpr int GW = 80;        // relpos band width (16 + 64 - 1 rounded to 8)
    constexpr int VPR = DH / 4;   // 8-byte vectors per row (DH % 4 == 0)
    extern __shared__ __align__(16) uint8_t att_smem[];
    __half* Qs = reinterpret_cast<__half*>(att_smem);  // [64][STR]   (RELPOS: Qu)
    __half* Ks = Qs + ATT_BQ * STR;                    // [64][STR]
    __half* Vs = Ks + ATT_BK * STR;                    // [64][STR]
    __half* Qv = Vs + ATT_BK * STR;                    // RELPOS: [64][STR]
    __half* Ps = Qv + ATT_BQ * STR;                    // RELPOS: [T][STR]
    float* Gs = reinterpret_cast<float*>(Ps + (RELPOS ? T : 0) * STR);  // RELPOS: [4 warps][16][GW+1]
    // head dims that are whole 16-byte vectors: K/V blocks are double-buffered with cp.async (block jb+1 streams in while
    // block jb is multiplied); the second buffer pair sits behind everything else
    constexpr bool ASYNC = (DH % 8 == 0) && (DHP == DH);
    __half* KV1 = reinterpret_cast<__half*>(Gs + (RELPOS ? 4 * 16 * (GW + 1) : 0));  // [2][64][STR] when ASYNC

    const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * ATT_BQ;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int len = lens ? min(lens[b], T) : T;
    const __half* base = qkv + static_cast<size_t>(b) * T * ld + h * 3 * DH;

    if constexpr (DHP != DH) {  // zero the padding columns once (they take part in the k-loop / PV n-tiles)
        constexpr int PADC = DHP - DH;
        const int n_rows_pad = 4 * ATT_BQ + (RELPOS ? T : 0);
        for (int i = threadIdx.x; i < n_rows_pad * PADC; i += blockDim.x) {
            const int r = i / PADC, cc = i - r * PADC;
            Qs[r * STR + DH + cc] = __float2half(0.0f);  // Qs, Ks, Vs, Qv, Ps are contiguous with the same stride
        }
    }
    // ---- stage Q (and RELPOS: Qu/Qv, P_h)
    for (int i = threadIdx.x; i < ATT_BQ * VPR; i += blockDim.x) {
        const int r = i / VPR, v4 = i - r * VPR;
        uint2 val = make_uint2(0, 0);
        if (i0 + r < T) val = *reinterpret_cast<const uint2*>(base + static_cast<size_t>(i0 + r) * ld + v4 * 4);
        if constexpr (RELPOS) {
            const __half* hv = reinterpret_cast<const __half*>(&val);
            __half qu[4], qv[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float q = __half2float(hv[e]);
                qu[e] = float2half_sat((q + __ldg(pos_u + h * DH + v4 * 4 + e)) * scale);
                qv[e] = float2half_sat((q + __ldg(pos_v + h * DH + v4 * 4 + e)) * scale);
            }
            *reinterpret_cast<uint2*>(Qs + r * STR + v4 * 4) = *reinterpret_cast<uint2*>(qu);
            *reinterpret_cast<uint2*>(Qv + r * STR + v4 * 4) = *reinterpret_cast<uint2*>(qv);
        } else {
            *reinterpret_cast<uint2*>(Qs + r * STR + v4 * 4) = val;
        }
    }
    if constexpr (RELPOS) {
        for (int i = threadIdx.x; i < T * VPR; i += blockDim.x) {
            const int r = i / VPR, v4 = i - r * VPR;
            *reinterpret_cast<uint2*>(Ps + r * STR + v4 * 4) =
                *reinterpret_cast<const uint2*>(P + static_cast<size_t>(r) * ldp + h * DH + v4 * 4);
        }
    }
    __syncthreads();

    uint32_t qa[KS][4];
    uint32_t qva[RELPOS ? KS : 1][4];
    {
        const __half* q0 = Qs + (warp * 16 + g) * STR + 2 * c;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            qa[ks][0] = *reinterpret_cast<const uint32_t*>(q0 + ks * 16);
            qa[ks][1] = *reinterpret_cast<const uint32_t*>(q0 + 8 * STR + ks * 16);
            qa[ks][2] = *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 8);
            qa[ks][3] = *reinterpret_cast<const uint32_t*>(q0 + 8 * STR + ks * 16 + 8);
        }
        if constexpr (RELPOS) {
            const __half* v0 = Qv + (warp * 16 + g) * STR + 2 * c;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                qva[ks][0] = *reinterpret_cast<const uint32_t*>(v0 + ks * 16);
                qva[ks][1] = *reinterpret_cast<const uint32_t*>(v0 + 8 * STR + ks * 16);
                qva[ks][2] = *reinterpret_cast<const uint32_t*>(v0 + ks * 16 + 8);
                qva[ks][3] = *reinterpret_cast<const uint32_t*>(v0 + 8 * STR + ks * 16 + 8);
            }
        }
    }

    float o[DHP / 8][4];
#pragma unroll
    for (int i = 0; i < DHP / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.0f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};
    const float LOG2E = 1.4426950408889634f;
    // Dynamic-chunk (streaming-equivalent) attention, TransformerASR.py:46-105: query i of chunk c = i / chunk sees keys
    // [max(0, (c - left_chunks) * chunk), min(len, (c + 1) * chunk)); left_chunks < 0 = unlimited past.  chunk == 0: off.
    int blk_begin = 0, n_blk = (len + ATT_BK - 1) / ATT_BK;
    int klo[2] = {0, 0}, khi[2] = {len, len};  // key window of this thread's two query rows (g and g + 8 of the warp's 16)
    if (chunk > 0) {
        const int i_last = min(i0 + ATT_BQ, T) - 1;
        const int hi_last = min(len, (i_last / chunk + 1) * chunk);
        n_blk = (hi_last + ATT_BK - 1) / ATT_BK;
        if (left_chunks >= 0) blk_begin = max(0, (i0 / chunk - left_chunks) * chunk) / ATT_BK;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int i = min(i0 + warp * 16 + g + 8 * r, T - 1);
            khi[r] = min(len, (i / chunk + 1) * chunk);
            klo[r] = left_chunks >= 0 ? max(0, (i / chunk - left_chunks) * chunk) : 0;
        }
    }

    auto stage_async = [&](int jb, __half* kd, __half* vd) {  // 16-byte cp.async, rows >= T zero-filled
        const int j0 = jb * ATT_BK;
        constexpr int V8 = DH / 8;
        for (int i = threadIdx.x; i < ATT_BK * V8; i += blockDim.x) {
            const int r = i / V8, v8 = i - r * V8;
            const bool ok = j0 + r < T;
            const __half* rowp = base + static_cast<size_t>(ok ? j0 + r : 0) * ld + v8 * 8;
            const uint32_t nbytes = ok ? 16u : 0u;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(kd + r * STR + v8 * 8)),
                         "l"(rowp + DH), "r"(nbytes) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(vd + r * STR + v8 * 8)),
                         "l"(rowp + 2 * DH), "r"(nbytes) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if constexpr (ASYNC) {
        if (n_blk > blk_begin) stage_async(blk_begin, Ks, Vs);
    }

    for (int jb = blk_begin; jb < n_blk; ++jb) {
        const int j0 = jb * ATT_BK;
        const __half* Kc = Ks;
        const __half* Vc = Vs;
        if constexpr (ASYNC) {
            if ((jb - blk_begin) & 1) { Kc = KV1; Vc = KV1 + ATT_BK * STR; }
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();  // block jb has landed for everyone; block jb-1 (the other buffer) is fully consumed
            if (jb + 1 < n_blk) {
                if ((jb - blk_begin) & 1) stage_async(jb + 1, Ks, Vs);
                else stage_async(jb + 1, KV1, KV1 + ATT_BK * STR);
            }
        } else {
            __syncthreads();  // previous block's K/V fully consumed
            for (int i = threadIdx.x; i < ATT_BK * VPR; i += blockDim.x) {
                const int r = i / VPR, v4 = i - r * VPR;
                uint2 kv = make_uint2(0, 0), vv = make_uint2(0, 0);
                if (j0 + r < T) {
                    const __half* rowp = base + static_cast<size_t>(j0 + r) * ld + v4 * 4;
                    kv = *reinterpret_cast<const uint2*>(rowp + DH);
                    vv = *reinterpret_cast<const uint2*>(rowp + 2 * DH);
                }
                *reinterpret_cast<uint2*>(Ks + r * STR + v4 * 4) = kv;
                *reinterpret_cast<uint2*>(Vs + r * STR + v4 * 4) = vv;
            }
            __syncthreads();
        }

        float s[ATT_BK / 8][4];
#pragma unroll
        for (int nt = 0; nt < ATT_BK / 8; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.0f;
            // B fragments of K[key][dim] for two k16 steps per ldmatrix.x4 (lanes 8m..8m+7 address matrix m = dims 8m..)
            const __half* kp = Kc + (nt * 8 + (lane & 7)) * STR + (lane >> 3) * 8;
#pragma unroll
            for (int ks = 0; ks + 1 < KS; ks += 2) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(b0, b1, b2, b3, kp + ks * 16);
                mma16816(s[nt], qa[ks], b0, b1);
                mma16816(s[nt], qa[ks + 1], b2, b3);
            }
            if constexpr (KS & 1) {
                uint32_t b0, b1;
                ldmatrix_x2(b0, b1, Kc + (nt * 8 + (lane & 7)) * STR + ((lane >> 3) & 1) * 8 + (KS - 1) * 16);
                mma16816(s[nt], qa[KS - 1], b0, b1);
            }
        }
        if constexpr (RELPOS) {
            // band G[li][rr] = Qv[li] . P[|rmin + rr|], rr in [0, 80): rmin = iw - j0 - 63
            float* Gw = Gs + warp * 16 * (GW + 1);
            const int rmin = (i0 + warp * 16) - j0 - (ATT_BK - 1);
#pragma unroll 1
            for (int nt = 0; nt < GW / 8; ++nt) {
                float gacc[4] = {0.f, 0.f, 0.f, 0.f};
                int pr = rmin + nt * 8 + g;
                pr = pr < 0 ? -pr : pr;
                pr = min(pr, T - 1);  // columns outside the band that are never read back
                const __half* pp = Ps + pr * STR + 2 * c;
#pragma unroll
                for (int ks = 0; ks < KS; ++ks)
                    mma16816(gacc, qva[ks], *reinterpret_cast<const uint32_t*>(pp + ks * 16),
                             *reinterpret_cast<const uint32_t*>(pp + ks * 16 + 8));
                const int col = nt * 8 + 2 * c;
                Gw[g * (GW + 1) + col] = gacc[0];
                Gw[g * (GW + 1) + col + 1] = gacc[1];
                Gw[(g + 8) * (GW + 1) + col] = gacc[2];
                Gw[(g + 8) * (GW + 1) + col + 1] = gacc[3];
            }
            __syncwarp();
#pragma unroll
            for (int nt = 0; nt < ATT_BK / 8; ++nt) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int li = g + (e >> 1) * 8, lj = nt * 8 + 2 * c + (e & 1);
                    s[nt][e] += Gw[li * (GW + 1) + (li - lj + ATT_BK - 1)];
                }
            }
            __syncwarp();
        }
        // ---- key padding mask + online softmax (rows g and g+8 of this warp's 16)
        float mx[2] = {-INFINITY, -INFINITY};
        if (chunk > 0) {  // chunked attention: every block can hold keys outside a row's window
#pragma unroll
            for (int nt = 0; nt < ATT_BK / 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int j = j0 + nt * 8 + 2 * c + (e & 1);
                    if (j < klo[e >> 1] || j >= khi[e >> 1]) s[nt][e] = -INFINITY;
                }
        } else if (j0 + ATT_BK > len) {  // only the last key block holds masked keys
#pragma unroll
            for (int nt = 0; nt < ATT_BK / 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (j0 + nt * 8 + 2 * c + (e & 1) >= len) s[nt][e] = -INFINITY;
        }
#pragma unroll
        for (int nt = 0; nt < ATT_BK / 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            // (a row can meet a fully masked block before its first visible key when chunk windows differ inside the tile)
            alpha[r] = m_new == -INFINITY ? 1.0f : ex2_ftz((m_run[r] - m_new) * LOG2E);
            m_run[r] = m_new;
        }
        float rs[2] = {0.0f, 0.0f};
        uint32_t pa[ATT_BK / 16][4];
#pragma unroll
        for (int nt = 0; nt < ATT_BK / 8; ++nt) {
            const float ms0 = m_run[0] == -INFINITY ? 0.0f : m_run[0] * LOG2E, ms1 = m_run[1] == -INFINITY ? 0.0f : m_run[1] * LOG2E;
            const float p0 = ex2_ftz(fmaf(s[nt][0], LOG2E, -ms0)), p1 = ex2_ftz(fmaf(s[nt][1], LOG2E, -ms0));
            const float p2 = ex2_ftz(fmaf(s[nt][2], LOG2E, -ms1)), p3 = ex2_ftz(fmaf(s[nt][3], LOG2E, -ms1));
            rs[0] += p0 + p1;
            rs[1] += p2 + p3;
            pa[nt >> 1][(nt & 1) * 2 + 0] = pack_half2(p0, p1);
            pa[nt >> 1][(nt & 1) * 2 + 1] = pack_half2(p2, p3);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_run[r] = l_run[r] * alpha[r] + rs[r];
        }
#pragma unroll
        for (int nt = 0; nt < DHP / 8; ++nt) {
            o[nt][0] *= alpha[0]; o[nt][1] *= alpha[0];
            o[nt][2] *= alpha[1]; o[nt][3] *= alpha[1];
        }
        // ---- O += P V : B fragments of V[key][dim] via ldmatrix.trans
#pragma unroll
        for (int kk = 0; kk < ATT_BK / 16; ++kk) {
#pragma unroll
            for (int nt = 0; nt + 1 < DHP / 8; nt += 2) {  // two 8-wide dim tiles per ldmatrix.x4.trans
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_trans(b0, b1, b2, b3, Vc + (kk * 16 + (lane & 15)) * STR + nt * 8 + (lane >> 4) * 8);
                mma16816(o[nt], pa[kk], b0, b1);
                mma16816(o[nt + 1], pa[kk], b2, b3);
            }
            if constexpr ((DHP / 8) & 1) {
                uint32_t b0, b1;
                ldmatrix_x2_trans(b0, b1, Vc + (kk * 16 + (lane & 15)) * STR + (DHP / 8 - 1) * 8);
                mma16816(o[DHP / 8 - 1], pa[kk], b0, b1);
            }
        }
    }
    // ---- normalise and store
    const int r0 = i0 + warp * 16 + g, r1 = r0 + 8;
    // (l == 0: a padded query row whose whole window is padding -- only possible with chunked attention; emit zeros)
    const float inv0 = l_run[0] > 0.0f ? 1.0f / l_run[0] : 0.0f, inv1 = l_run[1] > 0.0f ? 1.0f / l_run[1] : 0.0f;
    __half* ob = out + static_cast<size_t>(b) * T * ldo + h * DH;
#pragma unroll
    for (int nt = 0; nt < DHP / 8; ++nt) {
        const int col = nt * 8 + 2 * c;
        if (col >= DH) continue;  // zero-padding columns
        if (r0 < T) *reinterpret_cast<uint32_t*>(ob + static_cast<size_t>(r0) * ldo + col) = pack_half2(o[nt][0] * inv0, o[nt][1] * inv0);
        if (r1 < T) *reinterpret_cast<uint32_t*>(ob + static_cast<size_t>(r1) * ldo + col) = pack_half2(o[nt][2] * inv1, o[nt][3] * inv1);
    }
}

template <int DH, int DHP>
static int launch_encoder_attention(const __half* qkv, int ld, int B, int T, int H, const int* lens, bool relpos,
                                    const float* pos_u, const float* pos_v, const __half* P, int ldp, float scale,
                                    __half* out, int ldo, int chunk, int left_chunks, cudaStream_t stream) {
    constexpr int STR = DHP + 8;
    dim3 grid(ceil_div(T, ATT_BQ), H, B);
    if (!relpos) {
        const size_t smem = 4ull * ATT_BQ * STR * 2 + 2ull * ATT_BK * STR * 2;  // + second K/V buffer pair
        auto kern = encoder_attention_kernel<DH, DHP, false>;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, 128, smem, stream>>>(qkv, ld, T, lens, nullptr, nullptr, nullptr, 0, scale, out, ldo, chunk, left_chunks);
    } else {
        SBK_REQUIRE(ldp % 4 == 0, "encoder_attention: bad ldp");
        const size_t smem = 4ull * ATT_BQ * STR * 2 + static_cast<size_t>(T) * STR * 2 + 4ull * 16 * 81 * 4 +
                            2ull * ATT_BK * STR * 2;
        SBK_REQUIRE(smem <= 220 * 1024, "encoder_attention(RelPos): T=%d too long for the shared-memory table", T);
        auto kern = encoder_attention_kernel<DH, DHP, true>;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, 128, smem, stream>>>(qkv, ld, T, lens, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks);
    }
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// qkv [B*T, ld] fp16 with per-head [q | k | v] blocks of head_dim; out [B*T, ldo] fp16.
int encoder_attention(const __half* qkv, int ld, int B, int T, int H, int head_dim, const int* lens, bool relpos,
                      const float* pos_u, const float* pos_v, const __half* P, int ldp, float scale, __half* out,
                      int ldo, cudaStream_t stream, int chunk, int left_chunks) {
    SBK_REQUIRE(chunk >= 0, "encoder_attention: chunk size must be >= 0");
    SBK_REQUIRE(ld % 4 == 0 && ldo % 2 == 0, "encoder_attention: bad leading dims");
    if (head_dim % 8 == 0)  // cp.async 16-byte K/V staging
        SBK_REQUIRE(ld % 8 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "encoder_attention: qkv must be 16-byte aligned");
    if (head_dim == 64)
        return launch_encoder_attention<64, 64>(qkv, ld, B, T, H, lens, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks, stream);
    if (head_dim == 36)  // conformer_small: 144 / 4 heads, zero-padded to 48 for the k16 steps
        return launch_encoder_attention<36, 48>(qkv, ld, B, T, H, lens, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks, stream);
    if (head_dim == 32)
        return launch_encoder_attention<32, 32>(qkv, ld, B, T, H, lens, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks, stream);
    set_error("encoder_attention: head_dim=%d not built (64, 36, 32)", head_dim);
    return SBK_ERR_UNSUPPORTED;
}

// =========================================================================== TransformerLM causal self-attention
// Whole-sequence attention of TransformerLM.forward (TransformerLM.py:127-169: nn.MultiheadAttention under make_masks'
// look-ahead mask and key-padding mask on pad_idx).  qkv [n*s, 3d] fp16 with columns [q | k | v] (nn.MultiheadAttention's
// in_proj order, heads of 64 side by side, q pre-scaled by 1/sqrt(64)) -> out [n*s, d] fp16.
// One CTA = (64 query rows, head, sequence), 4 warps x 16 rows, mma.sync m16n8k16 with an fp32 online softmax like
// encoder_attention_kernel.  Query block qb reads key blocks 0..qb only: blocks above the diagonal are never loaded.
// Masked: keys j > i (diagonal block only) and keys whose token id is pad_tok -- the rule the KV-cached step applies
// through tok_cache / pad_tok (dec_attention_kernel).  A query whose visible keys are all padding (a sequence that starts
// with the pad id) has an empty softmax and yields NaN, as in the reference and the step path.
constexpr int LMA_B = 64;

__global__ void __launch_bounds__(128)
lm_causal_attention_kernel(const __half* __restrict__ qkv, int s, int d, const int* __restrict__ tokens, int pad_tok,
                           __half* __restrict__ out) {
    constexpr int DH = 64, STR = DH + 8, KS = DH / 16;
    __shared__ __align__(16) __half Qs[LMA_B * STR];
    __shared__ __align__(16) __half KVs[2][2][LMA_B * STR];  // [buffer][K | V]
    __shared__ bool s_masked[2][LMA_B];                       // [buffer][key]: pad token or past the sequence
    const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z, i0 = qb * LMA_B;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int ld = 3 * d;
    const __half* base = qkv + static_cast<size_t>(b) * s * ld + h * DH;
    const int* tok = tokens + static_cast<size_t>(b) * s;

    auto cp16 = [](__half* dst, const __half* src, bool ok) {  // rows past the sequence are zero-filled
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 16u : 0u)
                     : "memory");
    };
    auto stage = [&](int jb, int buf) {  // key block jb -> buffer buf (one cp.async group)
        const int j0 = jb * LMA_B;
        for (int i = threadIdx.x; i < LMA_B * (DH / 8); i += blockDim.x) {
            const int r = i / (DH / 8), v8 = i - r * (DH / 8);
            const bool ok = j0 + r < s;
            const __half* rowp = base + static_cast<size_t>(ok ? j0 + r : 0) * ld + v8 * 8;
            cp16(KVs[buf][0] + r * STR + v8 * 8, rowp + d, ok);
            cp16(KVs[buf][1] + r * STR + v8 * 8, rowp + 2 * d, ok);
        }
        if (threadIdx.x < LMA_B) {
            const int j = j0 + threadIdx.x;
            s_masked[buf][threadIdx.x] = j >= s || tok[j] == pad_tok;
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    for (int i = threadIdx.x; i < LMA_B * (DH / 8); i += blockDim.x) {  // Q rides in key block 0's group
        const int r = i / (DH / 8), v8 = i - r * (DH / 8);
        const bool ok = i0 + r < s;
        cp16(Qs + r * STR + v8 * 8, base + static_cast<size_t>(ok ? i0 + r : 0) * ld + v8 * 8, ok);
    }
    stage(0, 0);

    uint32_t qa[KS][4];
    float o[DH / 8][4];
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.0f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};
    const float LOG2E = 1.4426950408889634f;
    const int qi[2] = {i0 + warp * 16 + g, i0 + warp * 16 + g + 8};  // this thread's two query rows

    for (int jb = 0; jb <= qb; ++jb) {
        const int buf = jb & 1, j0 = jb * LMA_B;
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();  // block jb has landed for everyone; block jb-1 (the other buffer) is fully consumed
        if (jb + 1 <= qb) stage(jb + 1, buf ^ 1);
        if (jb == 0) {
            const __half* q0 = Qs + (warp * 16 + g) * STR + 2 * c;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                qa[ks][0] = *reinterpret_cast<const uint32_t*>(q0 + ks * 16);
                qa[ks][1] = *reinterpret_cast<const uint32_t*>(q0 + 8 * STR + ks * 16);
                qa[ks][2] = *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 8);
                qa[ks][3] = *reinterpret_cast<const uint32_t*>(q0 + 8 * STR + ks * 16 + 8);
            }
        }
        const __half* Kc = KVs[buf][0];
        const __half* Vc = KVs[buf][1];
        float sc[LMA_B / 8][4];
#pragma unroll
        for (int nt = 0; nt < LMA_B / 8; ++nt) {
            sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.0f;
            const __half* kp = Kc + (nt * 8 + (lane & 7)) * STR + (lane >> 3) * 8;
#pragma unroll
            for (int ks = 0; ks < KS; ks += 2) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(b0, b1, b2, b3, kp + ks * 16);
                mma16816(sc[nt], qa[ks], b0, b1);
                mma16816(sc[nt], qa[ks + 1], b2, b3);
            }
        }
        // ---- key-padding and (diagonal block) look-ahead mask, then the online softmax of rows g and g + 8
        const bool diag = jb == qb;
#pragma unroll
        for (int nt = 0; nt < LMA_B / 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int lj = nt * 8 + 2 * c + (e & 1);
                if (s_masked[buf][lj] || (diag && j0 + lj > qi[e >> 1])) sc[nt][e] = -INFINITY;
            }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < LMA_B / 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], sc[nt][e]);
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            // (a block whose keys are all padding leaves a row with no visible key so far)
            alpha[r] = m_new == -INFINITY ? 1.0f : ex2_ftz((m_run[r] - m_new) * LOG2E);
            m_run[r] = m_new;
        }
        float rs[2] = {0.0f, 0.0f};
        uint32_t pa[LMA_B / 16][4];
        const float ms0 = m_run[0] == -INFINITY ? 0.0f : m_run[0] * LOG2E, ms1 = m_run[1] == -INFINITY ? 0.0f : m_run[1] * LOG2E;
#pragma unroll
        for (int nt = 0; nt < LMA_B / 8; ++nt) {
            const float p0 = ex2_ftz(fmaf(sc[nt][0], LOG2E, -ms0)), p1 = ex2_ftz(fmaf(sc[nt][1], LOG2E, -ms0));
            const float p2 = ex2_ftz(fmaf(sc[nt][2], LOG2E, -ms1)), p3 = ex2_ftz(fmaf(sc[nt][3], LOG2E, -ms1));
            rs[0] += p0 + p1;
            rs[1] += p2 + p3;
            pa[nt >> 1][(nt & 1) * 2 + 0] = pack_half2(p0, p1);
            pa[nt >> 1][(nt & 1) * 2 + 1] = pack_half2(p2, p3);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_run[r] = l_run[r] * alpha[r] + rs[r];
        }
#pragma unroll
        for (int nt = 0; nt < DH / 8; ++nt) {
            o[nt][0] *= alpha[0]; o[nt][1] *= alpha[0];
            o[nt][2] *= alpha[1]; o[nt][3] *= alpha[1];
        }
        // ---- O += P V : B fragments of V[key][dim] via ldmatrix.trans
#pragma unroll
        for (int kk = 0; kk < LMA_B / 16; ++kk) {
#pragma unroll
            for (int nt = 0; nt < DH / 8; nt += 2) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_trans(b0, b1, b2, b3, Vc + (kk * 16 + (lane & 15)) * STR + nt * 8 + (lane >> 4) * 8);
                mma16816(o[nt], pa[kk], b0, b1);
                mma16816(o[nt + 1], pa[kk], b2, b3);
            }
        }
    }
    // ---- normalise and store (l == 0 only for a row without any visible key: 0 * inf = NaN, see above)
    const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
    __half* ob = out + static_cast<size_t>(b) * s * d + h * DH;
#pragma unroll
    for (int nt = 0; nt < DH / 8; ++nt) {
        const int col = nt * 8 + 2 * c;
        if (qi[0] < s) *reinterpret_cast<uint32_t*>(ob + static_cast<size_t>(qi[0]) * d + col) = pack_half2(o[nt][0] * inv0, o[nt][1] * inv0);
        if (qi[1] < s) *reinterpret_cast<uint32_t*>(ob + static_cast<size_t>(qi[1]) * d + col) = pack_half2(o[nt][2] * inv1, o[nt][3] * inv1);
    }
}

int lm_causal_attention(const __half* qkv, int n, int s, int d, int H, const int* tokens, int pad_tok, __half* out,
                        cudaStream_t stream) {
    SBK_REQUIRE(d == H * 64 && d % 8 == 0, "lm_causal_attention: head_dim must be 64 (d=%d, H=%d)", d, H);
    SBK_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
                "lm_causal_attention: misaligned operands");
    if (n == 0 || s == 0) return SBK_OK;
    lm_causal_attention_kernel<<<dim3(ceil_div(s, LMA_B), H, n), 128, 0, stream>>>(qkv, s, d, tokens, pad_tok, out);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // namespace sbk
