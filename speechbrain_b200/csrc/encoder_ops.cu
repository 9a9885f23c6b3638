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
// DUAL: a second fp16 output out2 = LN(x; gamma2, beta2) from the same statistics (the Branchformer layer's two pre-norms
// norm_mhsa / norm_conv of the same x, Branchformer.py:204-221).
constexpr int LN_MAX_PER_LANE = 32;

// One warp's row of D values, float4 vi = lane + 32 i in v[4 i .. 4 i + 3] (zeros past the row).  The mean sums each float4
// as (x + y) + (z + w) and the variance adds the centred squares one by one: every LayerNorm kernel here keeps that order, so
// they agree bit for bit.
struct LnRow {
    float v[LN_MAX_PER_LANE];
    float mean, rstd;
    int lane, D, nv;  // nv: float4 vectors per row (D % 4 == 0)

    __device__ __forceinline__ LnRow(const float* xr, int lane_, int D_) : lane(lane_), D(D_), nv(D_ >> 2) {
#pragma unroll
        for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
            const int vi = lane + i * 32;
            float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
            if (vi < nv) t = *reinterpret_cast<const float4*>(xr + vi * 4);
            v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
        }
    }
    __device__ __forceinline__ void stats(float eps) {
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) s += (v[4 * i] + v[4 * i + 1]) + (v[4 * i + 2] + v[4 * i + 3]);
        mean = warp_sum(s) / D;
        float q = 0.0f;
#pragma unroll
        for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i)
            if (lane + i * 32 < nv) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float d = v[4 * i + j] - mean;
                    q += d * d;
                }
            }
        rstd = rsqrtf(warp_sum(q) / D + eps);
    }
    // float4 i of the row normalised with gamma / beta float4s g, b
    __device__ __forceinline__ float4 norm(int i, float4 g, float4 b) const {
        return make_float4((v[4 * i] - mean) * rstd * g.x + b.x, (v[4 * i + 1] - mean) * rstd * g.y + b.y,
                           (v[4 * i + 2] - mean) * rstd * g.z + b.z, (v[4 * i + 3] - mean) * rstd * g.w + b.w);
    }
    // y -> float4 vi of the row at out + off, fp16 or fp32
    template <bool OUT_HALF>
    __device__ __forceinline__ static void store(void* out, size_t off, int vi, float4 y) {
        if constexpr (OUT_HALF) {
            __half2 h0 = floats2half2_sat(y.x, y.y), h1 = floats2half2_sat(y.z, y.w);
            uint2 u;
            u.x = *reinterpret_cast<uint32_t*>(&h0);
            u.y = *reinterpret_cast<uint32_t*>(&h1);
            *reinterpret_cast<uint2*>(static_cast<__half*>(out) + off + vi * 4) = u;
        } else {
            *reinterpret_cast<float4*>(static_cast<float*>(out) + off + vi * 4) = y;
        }
    }
};

__device__ __forceinline__ float4 ldg4(const float* p, int vi) { return __ldg(reinterpret_cast<const float4*>(p + vi * 4)); }

template <bool OUT_HALF, bool PDL, bool DUAL = false>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float* __restrict__ x, void* __restrict__ out, const float* __restrict__ gamma,
                      const float* __restrict__ beta, int M, int D, float eps, __half* __restrict__ out2 = nullptr,
                      const float* __restrict__ gamma2 = nullptr, const float* __restrict__ beta2 = nullptr) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    float4 gp[PDL ? LN_MAX_PER_LANE / 4 : 1], bp[PDL ? LN_MAX_PER_LANE / 4 : 1];
    if constexpr (PDL) {
#pragma unroll
        for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
            const int vi = lane + i * 32;
            if (vi < D >> 2 && row < M) {
                gp[i] = ldg4(gamma, vi);
                bp[i] = ldg4(beta, vi);
            }
        }
        pdl_trigger();
        pdl_wait();
    }
    if (row >= M) return;
    const size_t off = static_cast<size_t>(row) * D;
    LnRow r(x + off, lane, D);
    r.stats(eps);
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < r.nv) {
            LnRow::store<OUT_HALF>(out, off, vi, r.norm(i, PDL ? gp[PDL ? i : 0] : ldg4(gamma, vi),
                                                            PDL ? bp[PDL ? i : 0] : ldg4(beta, vi)));
            if constexpr (DUAL) LnRow::store<true>(out2, off, vi, r.norm(i, ldg4(gamma2, vi), ldg4(beta2, vi)));
        }
    }
}

int layernorm_rows_dual(const float* x, __half* out, const float* gamma, const float* beta, __half* out2, const float* gamma2,
                        const float* beta2, int M, int D, float eps, cudaStream_t stream) {
    SBK_REQUIRE(D % 4 == 0 && D <= 32 * LN_MAX_PER_LANE, "layernorm_rows_dual: D=%d unsupported", D);
    if (M == 0) return SBK_OK;
    const int rows_per_cta = 8;
    layernorm_rows_kernel<true, false, true><<<ceil_div(M, rows_per_cta), rows_per_cta * 32, 0, stream>>>(
        x, out, gamma, beta, M, D, eps, out2, gamma2, beta2);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int layernorm_rows(const float* x, void* out, bool out_half, const float* gamma, const float* beta, int M, int D,
                   float eps, cudaStream_t stream, bool pdl) {
    SBK_REQUIRE(D % 4 == 0 && D <= 32 * LN_MAX_PER_LANE, "layernorm_rows: D=%d unsupported", D);
    if (M == 0) return SBK_OK;
    const int rows_per_cta = 8;
    const dim3 grid(ceil_div(M, rows_per_cta)), block(rows_per_cta * 32);
    if (pdl) {
        SBK_REQUIRE(out_half, "layernorm_rows: the PDL variant writes fp16");
        SBK_CUDA_CHECK(launch_pdl(layernorm_rows_kernel<true, true>, grid, block, 0, stream, true, x, out, gamma, beta, M, D,
                                  eps, static_cast<__half*>(nullptr), static_cast<const float*>(nullptr),
                                  static_cast<const float*>(nullptr)));
    } else if (out_half) {
        layernorm_rows_kernel<true, false><<<grid, block, 0, stream>>>(x, out, gamma, beta, M, D, eps);
    } else {
        layernorm_rows_kernel<false, false><<<grid, block, 0, stream>>>(x, out, gamma, beta, M, D, eps);
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
    const size_t off = static_cast<size_t>(row) * D;
    LnRow r(x + off, lane, D);
    r.stats(eps_a);
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < r.nv) {
            const float4 y = r.norm(i, ldg4(ga, vi), ldg4(ba, vi));
            if (y_out != nullptr) LnRow::store<false>(y_out, off, vi, y);
            r.v[4 * i] = y.x; r.v[4 * i + 1] = y.y; r.v[4 * i + 2] = y.z; r.v[4 * i + 3] = y.w;
        }
    }
    r.stats(eps_b);
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE / 4; ++i) {
        const int vi = lane + i * 32;
        if (vi < r.nv) LnRow::store<OUT_HALF>(z_out, off, vi, r.norm(i, ldg4(gb, vi), ldg4(bb, vi)));
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

// fp32 -> fp16 cast of `rows` rows of n values, row r read at in + r * ld_in and written packed at out + r * n (used for
// goldens-driven tests, the decoder memory and the CNN output, whole or a stream chunk's frames inside longer rows)
__global__ void cast_f32_f16_kernel(const float* __restrict__ in, size_t ld_in, __half* __restrict__ out, size_t n, int rows) {
    for (int r = blockIdx.y; r < rows; r += gridDim.y)
        for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
             i += static_cast<size_t>(gridDim.x) * blockDim.x)
            out[r * n + i] = float2half_sat(in[r * ld_in + i]);
}
int cast_f32_f16(const float* in, __half* out, size_t n, cudaStream_t stream, int rows, size_t ld_in) {
    if (n == 0 || rows == 0) return SBK_OK;
    const dim3 grid(static_cast<unsigned>(std::min<size_t>((n + 255) / 256, SBK_NUM_SMS * 16)), std::min(rows, 65535));
    cast_f32_f16_kernel<<<grid, 256, 0, stream>>>(in, ld_in, out, n, rows);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// --------------------------------------------------------------------------- depthwise conv + LN + Swish / GELU
// glu [B*T, D] fp32 (GLU output) -> out [B*T, D] fp16 = act(LN(dwconv(glu) + bias)), act the Conformer's activation: Swish,
// or the exact erf GELU of the recipes with conformer_activation=torch.nn.GELU.  The tap weights arrive TAP-MAJOR
// ([K, D], repacked from the reference's (D, 1, K) at load time): thread = channel, so the 31 weight loads of a thread are
// coalesced across the warp (the channel-major layout made every load touch 32 cache lines).
// Zero padding at utterance edges only: padded frames inside T are real inputs (Conformer.py:318-325
// runs the conv before masking). One CTA per (utterance, tile of DW_TT frames); the (DW_TT + K - 1) x D
// input slab is staged in shared memory once.
constexpr int DW_TT = 16;

template <bool GELU>
__device__ __forceinline__ float conv_act(float x) {
    if constexpr (GELU) return gelu_erf_f(x);
    else return silu_f(x);
}

// KT > 0: compile-time kernel size (taps held in registers); KT == 0: runtime K.  MAXC: channels per thread (D <= 256 * MAXC)
// CHUNKED: Dynamic Chunk Convolution (Conformer.py:190-313): for every output frame the inputs beyond the end of its own
// chunk of `chunk` frames count as zero (the past, other chunks included, is visible as usual).
// left: [B, (K-1)/2, D] inputs of the frames just before frame 0 (a stream's previous chunks), or null for zero padding.
// GELU: exact erf GELU after the LayerNorm instead of Swish.
template <int KT, int MAXC, bool CHUNKED = false, bool GELU = false>
__global__ void __launch_bounds__(256, 2)
dwconv_ln_act_kernel(const float* __restrict__ glu, int T, int D, int K, const float* __restrict__ wdw /*[K,D] tap-major*/,
                     const float* __restrict__ bdw, const float* __restrict__ gamma, const float* __restrict__ beta,
                     float eps, __half* __restrict__ out, int chunk, const float* __restrict__ left) {
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
    // zero rows outside the utterance (Conv1d zero padding); rows before frame 0 come from `left` when it is set
    for (int i = threadIdx.x; i < (r_lo + rows_in - r_hi) * D; i += blockDim.x) {
        int r = i / D;
        const int ch = i - r * D;
        if (r >= r_lo) r += r_hi - r_lo;
        slab[r * D + ch] = left && r < r_lo ? left[(static_cast<size_t>(b) * halo + t0 + r) * D + ch] : 0.0f;  // frame t0 - halo + r
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
                const float y0 = conv_act<GELU>((cv.x - mean) * rstd * g2[p].x + b2[p].x);
                const float y1 = conv_act<GELU>((cv.y - mean) * rstd * g2[p].y + b2[p].y);
                *reinterpret_cast<__half2*>(o + j) = floats2half2_sat(y0, y1);
            }
        }
    }
}

// The instantiation for (D, K, chunk): taps in registers at K = 31 with 1, 2 or 4 channels per thread (D <= 1024), else
// runtime K.  D = 768 takes the 4-channel form with its fourth channel slot idle.
template <bool GELU>
static auto dwconv_kernel_for(int D, int K, int chunk) {
    if (chunk > 0) {
        if (K != 31) return dwconv_ln_act_kernel<0, 4, true, GELU>;
        return D <= 256 ? dwconv_ln_act_kernel<31, 1, true, GELU> : D <= 512 ? dwconv_ln_act_kernel<31, 2, true, GELU>
                                                                             : dwconv_ln_act_kernel<31, 4, true, GELU>;
    }
    if (K != 31) return dwconv_ln_act_kernel<0, 4, false, GELU>;
    return D <= 256 ? dwconv_ln_act_kernel<31, 1, false, GELU> : D <= 512 ? dwconv_ln_act_kernel<31, 2, false, GELU>
                                                                          : dwconv_ln_act_kernel<31, 4, false, GELU>;
}

int dwconv_ln_act(const float* glu, int B, int T, int D, int K, const float* wdw, const float* bdw, const float* gamma,
                  const float* beta, float eps, __half* out, cudaStream_t stream, bool gelu, int chunk, const float* left) {
    SBK_REQUIRE(D % 4 == 0 && D <= 1024 && (K & 1) == 1, "dwconv_ln_act: D %% 4, D <= 1024 and odd K required (D=%d K=%d)", D, K);
    SBK_REQUIRE((reinterpret_cast<uintptr_t>(glu) & 15) == 0, "dwconv_ln_act: input must be 16-byte aligned");
    const size_t smem = static_cast<size_t>(DW_TT + K - 1) * D * sizeof(float);
    SBK_REQUIRE(smem <= 200 * 1024, "dwconv_ln_act: tile too large for shared memory (D=%d K=%d)", D, K);
    const auto kern = gelu ? dwconv_kernel_for<true>(D, K, chunk) : dwconv_kernel_for<false>(D, K, chunk);
    SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(ceil_div(T, DW_TT), B), 256, smem, stream>>>(glu, T, D, K, wdw, bdw, gamma, beta, eps, out, chunk, left);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// carry [B, halo, D] <- the last halo rows of [carry; glu [B, n, D]] (has_old == 0: the carry counts as zeros).  Thread =
// (utterance, channel); rows ascend, so row j is written only after row j + n, which it may read, has been read.
__global__ void dwconv_carry_kernel(const float* __restrict__ glu, int n, int D, int halo, int has_old, float* carry) {
    const int ch = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (ch >= D) return;
    float* cb = carry + static_cast<size_t>(b) * halo * D + ch;
    for (int j = 0; j < halo; ++j) {
        const int src = j + n - halo;  // row of the chunk, or (when < 0) of the old carry at j + n
        cb[static_cast<size_t>(j) * D] = src >= 0 ? glu[(static_cast<size_t>(b) * n + src) * D + ch]
                                                  : (has_old ? cb[static_cast<size_t>(j + n) * D] : 0.0f);
    }
}

int dwconv_carry(const float* glu, int B, int n, int D, int K, bool has_old, float* carry, cudaStream_t stream) {
    const int halo = (K - 1) / 2;
    if (halo == 0) return SBK_OK;
    dwconv_carry_kernel<<<dim3(ceil_div(D, 128), B), 128, 0, stream>>>(glu, n, D, halo, has_old ? 1 : 0, carry);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// (D, 1, K) reference taps -> tap-major [K, D] (the layout dwconv_ln_act reads)
void dwconv_repack_taps(const float* src, int D, int K, float* dst) {
    for (int ch = 0; ch < D; ++ch)
        for (int k = 0; k < K; ++k) dst[static_cast<size_t>(k) * D + ch] = src[static_cast<size_t>(ch) * K + k];
}

// --------------------------------------------------------------------------- CSGU (Branchformer convolution branch)
// ConvolutionalSpatialGatingUnit.forward (lobes/models/convolution.py:22-113) on u = GELU(pre_channel_proj(x)) [B*T, C] fp16:
//     a, b = u[:, :C/2], u[:, C/2:]          (x.chunk(2, dim=-1): the first half gates)
//     g    = a * (dwconv_K(LN(b)) + bias)     (gate activation Identity, no linear after the conv)
// The conv is speechbrain's Conv1d(padding="same"), padding_mode "reflect": (K-1)/2 frames on each side of the batch-padded
// length T, mirrored about frames 0 and T-1 (so T > (K-1)/2).  Padded frames inside T are real inputs: the reference never
// masks this branch (Branchformer.py:225).
//   pass 1: fp32 LayerNorm statistics (mean, rstd) of b for every row, padded rows included;
//   pass 2: one CTA per (CSGU_CC channels, CSGU_TT frames, utterance): the normalised halo'd b slab in shared memory (fp32),
//           31 taps per output in registers, then a * (conv + bias) -> g fp16.
// The taps arrive tap-major [CSGU_KMAX, C/2] with a kernel of K < CSGU_KMAX centred in zero rows, so every odd K <= 31
// runs the same fully unrolled loop.
constexpr int CSGU_KMAX = CSGU_TAP_ROWS, CSGU_HALO = (CSGU_KMAX - 1) / 2;
constexpr int CSGU_TT = 64, CSGU_CC = 64, CSGU_THREADS = 256;
constexpr int CSGU_FPT = CSGU_TT / (CSGU_THREADS / CSGU_CC);  // output frames per thread
constexpr int CSGU_ROWS = CSGU_TT + CSGU_KMAX - 1;

__global__ void __launch_bounds__(256)
csgu_stats_kernel(const __half* __restrict__ u, int M, int C, float eps, float2* __restrict__ stats) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31, C2 = C >> 1, nv = C2 >> 3;
    const uint4* src = reinterpret_cast<const uint4*>(u + static_cast<size_t>(row) * C + C2);
    float s = 0.0f;
    for (int j = lane; j < nv; j += 32) {
        const uint4 w = __ldg(src + j);
        const __half2* h = reinterpret_cast<const __half2*>(&w);
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 f = __half22float2(h[q]); s += f.x + f.y; }
    }
    const float mean = warp_sum(s) / C2;
    float v = 0.0f;  // second pass over the (L1-resident) row: exact two-pass variance, robust to large row means
    for (int j = lane; j < nv; j += 32) {
        const uint4 w = __ldg(src + j);
        const __half2* h = reinterpret_cast<const __half2*>(&w);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 f = __half22float2(h[q]);
            v += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
        }
    }
    const float rstd = rsqrtf(warp_sum(v) / C2 + eps);
    if (lane == 0) stats[row] = make_float2(mean, rstd);
}

__global__ void __launch_bounds__(CSGU_THREADS)
csgu_conv_gate_kernel(const __half* __restrict__ u, int T, int C, const float2* __restrict__ stats,
                      const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ taps,
                      const float* __restrict__ bias, __half* __restrict__ g) {
    __shared__ __align__(16) float slab[CSGU_ROWS][CSGU_CC];  // slab row r = frame t0 - CSGU_HALO + r; rows [0, TT) reused for the outputs
    const int C2 = C >> 1, c0 = blockIdx.x * CSGU_CC, t0 = blockIdx.y * CSGU_TT, b = blockIdx.z;
    const size_t row0 = static_cast<size_t>(b) * T;
    // normalised b slab: 8 channels (16 B) per load, reflect at the batch-padded edges
    for (int i = threadIdx.x; i < CSGU_ROWS * (CSGU_CC / 8); i += CSGU_THREADS) {
        const int r = i / (CSGU_CC / 8), j = (i % (CSGU_CC / 8)) * 8, ch = c0 + j;
        int t = t0 - CSGU_HALO + r;
        t = t < 0 ? -t : (t >= T ? 2 * (T - 1) - t : t);
        t = min(max(t, 0), T - 1);  // rows only a zero tap (K < 31) or an output frame >= T reads
        float y[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (ch < C2) {  // C/2 % 8 == 0: a vector lies entirely inside or outside the channels
            const float2 st = __ldg(stats + row0 + t);
            const uint4 w = __ldg(reinterpret_cast<const uint4*>(u + (row0 + t) * C + C2 + ch));
            const __half2* h = reinterpret_cast<const __half2*>(&w);
            const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + ch)), gb = __ldg(reinterpret_cast<const float4*>(gamma + ch + 4));
            const float4 ba = __ldg(reinterpret_cast<const float4*>(beta + ch)), bb = __ldg(reinterpret_cast<const float4*>(beta + ch + 4));
            const float gg[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
            const float bt[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 f = __half22float2(h[q]);
                y[2 * q] = (f.x - st.x) * st.y * gg[2 * q] + bt[2 * q];
                y[2 * q + 1] = (f.y - st.x) * st.y * gg[2 * q + 1] + bt[2 * q + 1];
            }
        }
        *reinterpret_cast<float4*>(&slab[r][j]) = make_float4(y[0], y[1], y[2], y[3]);
        *reinterpret_cast<float4*>(&slab[r][j + 4]) = make_float4(y[4], y[5], y[6], y[7]);
    }
    // this thread: channel c0 + cl, output frames f0 .. f0 + CSGU_FPT - 1 of the tile
    const int cl = threadIdx.x % CSGU_CC, f0 = (threadIdx.x / CSGU_CC) * CSGU_FPT, ch = c0 + cl;
    float w[CSGU_KMAX], acc[CSGU_FPT];
    const float bz = ch < C2 ? __ldg(bias + ch) : 0.0f;
#pragma unroll
    for (int k = 0; k < CSGU_KMAX; ++k) w[k] = ch < C2 ? __ldg(taps + static_cast<size_t>(k) * C2 + ch) : 0.0f;
#pragma unroll
    for (int i = 0; i < CSGU_FPT; ++i) acc[i] = bz;
    __syncthreads();
#pragma unroll
    for (int r = 0; r < CSGU_FPT + CSGU_KMAX - 1; ++r) {
        const float xv = slab[f0 + r][cl];
#pragma unroll
        for (int i = 0; i < CSGU_FPT; ++i)
            if (r - i >= 0 && r - i < CSGU_KMAX) acc[i] = fmaf(xv, w[r - i], acc[i]);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < CSGU_FPT; ++i) slab[f0 + i][cl] = acc[i];
    __syncthreads();
    // gate with a and store g: 8 channels per 16 B access
    for (int i = threadIdx.x; i < CSGU_TT * (CSGU_CC / 8); i += CSGU_THREADS) {
        const int r = i / (CSGU_CC / 8), j = (i % (CSGU_CC / 8)) * 8, t = t0 + r;
        if (t >= T || c0 + j >= C2) continue;
        const uint4 av = __ldg(reinterpret_cast<const uint4*>(u + (row0 + t) * C + c0 + j));
        const __half2* ah = reinterpret_cast<const __half2*>(&av);
        const float4 x0 = *reinterpret_cast<const float4*>(&slab[r][j]), x1 = *reinterpret_cast<const float4*>(&slab[r][j + 4]);
        const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
        uint4 o;
        uint32_t* op = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 af = __half22float2(ah[q]);
            __half2 hv = floats2half2_sat(af.x * xs[2 * q], af.y * xs[2 * q + 1]);
            op[q] = *reinterpret_cast<uint32_t*>(&hv);
        }
        *reinterpret_cast<uint4*>(g + (row0 + t) * C2 + c0 + j) = o;
    }
}

int csgu_forward(const __half* u, int B, int T, int C, const float* gamma, const float* beta, float eps, const float* taps,
                 const float* bias, int K, float2* stats, __half* g, cudaStream_t stream) {
    SBK_REQUIRE(C % 16 == 0, "csgu: csgu_linear_units=%d must be a multiple of 16 (C/2 %% 8 == 0)", C);
    SBK_REQUIRE((K & 1) == 1 && K <= CSGU_KMAX, "csgu: kernel_size=%d must be odd and <= %d", K, CSGU_KMAX);
    SBK_REQUIRE(T > (K - 1) / 2, "csgu: reflect padding needs T > (kernel_size - 1) / 2 (T=%d, kernel_size=%d)", T, K);
    SBK_REQUIRE(B <= 65535, "csgu: B=%d", B);
    SBK_REQUIRE(((reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(gamma) |
                  reinterpret_cast<uintptr_t>(beta)) & 15) == 0, "csgu: operands must be 16-byte aligned");
    const int M = B * T;
    if (M == 0) return SBK_OK;
    csgu_stats_kernel<<<ceil_div(M, 8), 256, 0, stream>>>(u, M, C, eps, stats);
    SBK_LAUNCH_CHECK();
    csgu_conv_gate_kernel<<<dim3(ceil_div(C / 2, CSGU_CC), ceil_div(T, CSGU_TT), B), CSGU_THREADS, 0, stream>>>(
        u, T, C, stats, gamma, beta, taps, bias, g);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// (C/2, 1, K) reference taps -> tap-major [CSGU_KMAX, C/2], K centred (the layout csgu_forward reads)
void csgu_repack_taps(const float* src, int C2, int K, float* dst) {
    const int off = CSGU_HALO - (K - 1) / 2;
    for (size_t i = 0; i < static_cast<size_t>(CSGU_KMAX) * C2; ++i) dst[i] = 0.0f;
    for (int ch = 0; ch < C2; ++ch)
        for (int k = 0; k < K; ++k) dst[static_cast<size_t>(k + off) * C2 + ch] = src[static_cast<size_t>(ch) * K + k];
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
//        shared memory and re-reads it diagonally shifted.  The four warps' bands of key block j0 read
//        P[min(|a + x|, T - 1)], x in [0, 128), a = i0 - j0 - 63.  That window moves down by 64 rows per key
//        block: a 192-row ring holds it, and each key block's 64 new rows stream in (cp.async) while the block
//        before it is multiplied, so shared memory does not grow with T.
//  Padded *query* rows are computed like any other row (the reference does; they leak into valid frames
//  through the depthwise conv), only padded *keys* are masked.
constexpr int ATT_BQ = 64;
constexpr int ATT_BK = 64;
constexpr int ATT_GW = 80;                      // relpos band width per warp (16 + 64 - 1 rounded to 8)
constexpr int ATT_PW = ATT_BQ - 16 + ATT_GW;    // relpos P window rows per key block: 4 warp bands, 16 rows apart
constexpr int ATT_PR = ATT_PW + ATT_BK;         // relpos P ring rows: one block's window + the next block's new rows

__device__ __forceinline__ float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// STREAM: one chunk of a stream (AttStream): T is the window [cached rows; chunk rows], the queries are its last sa.nq rows
// (from sa.q), keys / values come from the ring sa.kv, every key of the window is visible, and out holds the chunk's rows.
// Head dims that are whole 16-byte vectors stage K/V blocks with cp.async.  KV2: double-buffered (block jb+1 streams in while
// block jb is multiplied; the second buffer pair sits behind everything else); otherwise one buffer pair, refilled after
// the block has been multiplied.  RelPosMHAXL at head width 80 takes one pair: 97 KB of shared memory, two CTAs per SM,
// against 119 KB and one CTA with two (H100 80GB HBM3, 700 W: B = 32, 8 heads, T = 251 113 us against 158 us; T = 2500
// 5.56 ms against 7.92 ms).
template <int DH, int DHP, bool RELPOS>
__host__ __device__ constexpr bool att_kv2() { return (DH % 8 == 0) && (DHP == DH) && !(RELPOS && DH == 80); }

template <int DH, int DHP, bool RELPOS, bool STREAM = false>  // DHP = DH rounded up to a multiple of 16 (zero-padded in shared memory)
__global__ void __launch_bounds__(128)
encoder_attention_kernel(const __half* __restrict__ qkv, int ld, int T, const int* __restrict__ lens,
                         const float* __restrict__ pos_u, const float* __restrict__ pos_v,
                         const __half* __restrict__ P, int ldp, float scale, __half* __restrict__ out, int ldo,
                         int chunk, int left_chunks, AttStream sa) {
    constexpr int STR = DHP + 8;  // padded row stride (halfs): conflict-free fragment loads
    constexpr int KS = DHP / 16;
    constexpr int GW = ATT_GW;
    constexpr int VPR = DH / 4;   // 8-byte vectors per row (DH % 4 == 0)
    extern __shared__ __align__(16) uint8_t att_smem[];
    __half* Qs = reinterpret_cast<__half*>(att_smem);  // [64][STR]   (RELPOS: Qu)
    __half* Ks = Qs + ATT_BQ * STR;                    // [64][STR]
    __half* Vs = Ks + ATT_BK * STR;                    // [64][STR]
    __half* Qv = Vs + ATT_BK * STR;                    // RELPOS: [64][STR]
    __half* Ps = Qv + ATT_BQ * STR;                    // RELPOS: [ATT_PR][STR] ring of P rows (p_slot)
    float* Gs = reinterpret_cast<float*>(Ps + (RELPOS ? ATT_PR : 0) * STR);  // RELPOS: [4 warps][16][GW+1]
    constexpr bool ASYNC = (DH % 8 == 0) && (DHP == DH);
    constexpr bool KV2 = att_kv2<DH, DHP, RELPOS>();
    __half* KV1 = reinterpret_cast<__half*>(Gs + (RELPOS ? 4 * 16 * (GW + 1) : 0));  // [2][64][STR] when KV2

    const int q_off = STREAM ? T - sa.nq : 0;  // window row of the first query
    const int b = blockIdx.z, h = blockIdx.y, i0 = q_off + blockIdx.x * ATT_BQ;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int len = lens ? min(lens[b], T) : T;
    const __half* base = STREAM ? nullptr : qkv + static_cast<size_t>(b) * T * ld + h * 3 * DH;
    auto q_row = [&](int i) {
        if constexpr (STREAM) return sa.q + (static_cast<size_t>(b) * sa.nq + (i - q_off)) * sa.ldq + h * DH;
        else return base + static_cast<size_t>(i) * ld;
    };
    auto k_row = [&](int j) {  // the row's V follows its K at + DH
        if constexpr (STREAM) {
            const int slot = sa.start + j < sa.cap ? sa.start + j : sa.start + j - sa.cap;
            return sa.kv + (static_cast<size_t>(b) * sa.cap + slot) * sa.ldkv + h * 2 * DH;
        } else {
            return base + static_cast<size_t>(j) * ld + DH;
        }
    };

    if constexpr (DHP != DH) {  // zero the padding columns once (they take part in the k-loop / PV n-tiles)
        constexpr int PADC = DHP - DH;
        const int n_rows_pad = 4 * ATT_BQ + (RELPOS ? ATT_PR : 0);
        for (int i = threadIdx.x; i < n_rows_pad * PADC; i += blockDim.x) {
            const int r = i / PADC, cc = i - r * PADC;
            Qs[r * STR + DH + cc] = __float2half(0.0f);  // Qs, Ks, Vs, Qv, Ps are contiguous with the same stride
        }
    }
    // ---- stage Q (RELPOS: Qu/Qv)
    for (int i = threadIdx.x; i < ATT_BQ * VPR; i += blockDim.x) {
        const int r = i / VPR, v4 = i - r * VPR;
        uint2 val = make_uint2(0, 0);
        if (i0 + r < T) val = *reinterpret_cast<const uint2*>(q_row(i0 + r) + v4 * 4);
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

    // RELPOS: the band of key block jb reads P[min(|v|, T - 1)] for v = a + x, x in [0, ATT_PW), a = i0 - j0 - (ATT_BK - 1);
    // row v lives in ring slot v mod ATT_PR.  Block jb + 1's window is block jb's moved down by ATT_BK rows, so after the
    // first block only its ATT_BK new rows [a, a + ATT_BK) are staged.  They take the slots of rows
    // [a + ATT_PR, a + ATT_PR + ATT_BK), which lie above the window of the block before it (the one being multiplied while
    // they stream in).
    auto p_first = [&](int jb) { return i0 - jb * ATT_BK - (ATT_BK - 1); };
    auto p_slot = [](int v) {
        const int s = v % ATT_PR;
        return s < 0 ? s + ATT_PR : s;
    };
    auto p_src = [&](int v) { return P + static_cast<size_t>(min(v < 0 ? -v : v, T - 1)) * ldp + h * DH; };
    auto stage_async = [&](int jb, __half* kd, __half* vd) {  // 16-byte cp.async, rows >= T zero-filled
        const int j0 = jb * ATT_BK;
        constexpr int V8 = DH / 8;
        for (int i = threadIdx.x; i < ATT_BK * V8; i += blockDim.x) {
            const int r = i / V8, v8 = i - r * V8;
            const bool ok = j0 + r < T;
            const __half* rowp = k_row(ok ? j0 + r : 0) + v8 * 8;
            const uint32_t nbytes = ok ? 16u : 0u;
            cp_async16_zfill(smem_u32(kd + r * STR + v8 * 8), rowp, nbytes);
            cp_async16_zfill(smem_u32(vd + r * STR + v8 * 8), rowp + DH, nbytes);
        }
        if constexpr (RELPOS) {
            const int a = p_first(jb), n = jb == blk_begin ? ATT_PW : ATT_BK;
            for (int i = threadIdx.x; i < n * V8; i += blockDim.x) {
                const int x = i / V8, v8 = i - x * V8;
                cp_async16(smem_u32(Ps + p_slot(a + x) * STR + v8 * 8), p_src(a + x) + v8 * 8);
            }
        }
        cp_async_commit();
    };
    // RELPOS without 16-byte rows: only the P rows go through cp.async, in 8-byte pieces, one key block ahead
    auto stage_p8 = [&](int jb) {
        const int a = p_first(jb), n = jb == blk_begin ? ATT_PW : ATT_BK;
        for (int i = threadIdx.x; i < n * VPR; i += blockDim.x) {
            const int x = i / VPR, v4 = i - x * VPR;
            cp_async8(smem_u32(Ps + p_slot(a + x) * STR + v4 * 4), p_src(a + x) + v4 * 4);
        }
        cp_async_commit();
    };
    if (n_blk > blk_begin) {
        if constexpr (ASYNC) stage_async(blk_begin, Ks, Vs);
        else if constexpr (RELPOS) stage_p8(blk_begin);
    }

    for (int jb = blk_begin; jb < n_blk; ++jb) {
        const int j0 = jb * ATT_BK;
        const __half* Kc = Ks;
        const __half* Vc = Vs;
        if constexpr (KV2) {
            if ((jb - blk_begin) & 1) { Kc = KV1; Vc = KV1 + ATT_BK * STR; }
            cp_async_wait<0>();
            __syncthreads();  // block jb has landed for everyone; block jb-1 (the other buffer) is fully consumed
            if (jb + 1 < n_blk) {
                if ((jb - blk_begin) & 1) stage_async(jb + 1, Ks, Vs);
                else stage_async(jb + 1, KV1, KV1 + ATT_BK * STR);
            }
        } else if constexpr (ASYNC) {
            if (jb != blk_begin) {  // block jb-1 has been multiplied by every warp: refill the buffer pair with block jb
                __syncthreads();
                stage_async(jb, Ks, Vs);
            }
            cp_async_wait<0>();
            __syncthreads();  // block jb has landed for everyone
        } else {
            if constexpr (RELPOS) cp_async_wait<0>();
            __syncthreads();  // previous block's K/V fully consumed (RELPOS: block jb's P rows have landed for everyone)
            if constexpr (RELPOS) {
                if (jb + 1 < n_blk) stage_p8(jb + 1);
            }
            for (int i = threadIdx.x; i < ATT_BK * VPR; i += blockDim.x) {
                const int r = i / VPR, v4 = i - r * VPR;
                uint2 kv = make_uint2(0, 0), vv = make_uint2(0, 0);
                if (j0 + r < T) {
                    const __half* rowp = k_row(j0 + r) + v4 * 4;
                    kv = *reinterpret_cast<const uint2*>(rowp);
                    vv = *reinterpret_cast<const uint2*>(rowp + DH);
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
            // band G[li][rr] = Qv[li] . P[|rmin + rr|], rr in [0, 80): rmin = iw - j0 - 63 = a + warp * 16
            // (rows past T - 1 repeat row T - 1: columns outside the band that are never read back)
            float* Gw = Gs + warp * 16 * (GW + 1);
            const int rmin = p_first(jb) + warp * 16;
#pragma unroll 1
            for (int nt = 0; nt < GW / 8; ++nt) {
                float gacc[4] = {0.f, 0.f, 0.f, 0.f};
                const __half* pp = Ps + p_slot(rmin + nt * 8 + g) * STR + 2 * c;
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
    // output row of window row r (STREAM: the chunk's rows, [B * sa.nq, ldo])
    auto o_row = [&](int r) {
        const size_t row = STREAM ? static_cast<size_t>(b) * sa.nq + (r - q_off) : static_cast<size_t>(b) * T + r;
        return out + row * ldo + h * DH;
    };
#pragma unroll
    for (int nt = 0; nt < DHP / 8; ++nt) {
        const int col = nt * 8 + 2 * c;
        if (col >= DH) continue;  // zero-padding columns
        if (r0 < T) *reinterpret_cast<uint32_t*>(o_row(r0) + col) = pack_half2(o[nt][0] * inv0, o[nt][1] * inv0);
        if (r1 < T) *reinterpret_cast<uint32_t*>(o_row(r1) + col) = pack_half2(o[nt][2] * inv1, o[nt][3] * inv1);
    }
}

template <int DH, int DHP, bool STREAM = false>
static int launch_encoder_attention(const __half* qkv, int ld, int B, int T, int H, const int* lens, bool relpos,
                                    const float* pos_u, const float* pos_v, const __half* P, int ldp, float scale,
                                    __half* out, int ldo, int chunk, int left_chunks, cudaStream_t stream,
                                    const AttStream& sa = AttStream{}) {
    constexpr int STR = DHP + 8;
    dim3 grid(ceil_div(STREAM ? sa.nq : T, ATT_BQ), H, B);
    if (!relpos) {
        const size_t smem = 4ull * ATT_BQ * STR * 2 + 2ull * ATT_BK * STR * 2;  // + second K/V buffer pair
        auto kern = encoder_attention_kernel<DH, DHP, false, STREAM>;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, 128, smem, stream>>>(qkv, ld, T, lens, nullptr, nullptr, nullptr, 0, scale, out, ldo, chunk, left_chunks, sa);
    } else if constexpr (DH > 64 && DH != 80) {  // RelPosMHAXL is built for the recipes' head widths: up to 64, and 80
        set_error("encoder_attention: RelPosMHAXL with head_dim=%d not built", DH);
        return SBK_ERR_UNSUPPORTED;
    } else {
        constexpr bool ASYNC = (DH % 8 == 0) && (DHP == DH);  // as in the kernel
        if (ASYNC)
            SBK_REQUIRE(ldp % 8 == 0 && (reinterpret_cast<uintptr_t>(P) & 15) == 0, "encoder_attention: P must be 16-byte aligned");
        else
            SBK_REQUIRE(ldp % 4 == 0 && (reinterpret_cast<uintptr_t>(P) & 7) == 0, "encoder_attention: P must be 8-byte aligned");
        // independent of T: 101 KB at head_dim 64 and 97 KB at 80 (two CTAs per SM), 69 KB at 36 and 65 KB at 32 (three)
        const size_t smem = (4ull * ATT_BQ + ATT_PR) * STR * 2 + 4ull * 16 * (ATT_GW + 1) * 4 +
                            (att_kv2<DH, DHP, true>() ? 2ull * ATT_BK * STR * 2 : 0);
        auto kern = encoder_attention_kernel<DH, DHP, true, STREAM>;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, 128, smem, stream>>>(qkv, ld, T, lens, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks, sa);
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
    if (head_dim == 80)  // the d_model 640 conformer_large recipes (Libriheavy, People's Speech): 640 / 8 heads
        return launch_encoder_attention<80, 80>(qkv, ld, B, T, H, lens, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks, stream);
    if (head_dim == 128)  // the Transformer recipes' regularMHA (512 / 4 heads); no positional term
        return launch_encoder_attention<128, 128>(qkv, ld, B, T, H, lens, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, chunk, left_chunks, stream);
    set_error("encoder_attention: head_dim=%d not built (128, 80, 64, 36, 32)", head_dim);
    return SBK_ERR_UNSUPPORTED;
}

int encoder_attention_stream(const AttStream& sa, int B, int W, int H, int head_dim, bool relpos, const float* pos_u,
                             const float* pos_v, const __half* P, int ldp, float scale, __half* out, int ldo,
                             cudaStream_t stream) {
    SBK_REQUIRE(sa.nq >= 1 && sa.nq <= W && W <= sa.cap && sa.start >= 0 && sa.start < sa.cap,
                "encoder_attention_stream: bad window (%d queries, %d rows, ring of %d from %d)", sa.nq, W, sa.cap, sa.start);
    SBK_REQUIRE(sa.ldq % 8 == 0 && sa.ldkv % 8 == 0 && ldo % 2 == 0 && (reinterpret_cast<uintptr_t>(sa.q) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(sa.kv) & 15) == 0,
                "encoder_attention_stream: q / kv must be 16-byte aligned");
    if (head_dim == 64)
        return launch_encoder_attention<64, 64, true>(nullptr, 0, B, W, H, nullptr, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, 0, -1, stream, sa);
    if (head_dim == 36 && relpos)
        return launch_encoder_attention<36, 48, true>(nullptr, 0, B, W, H, nullptr, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, 0, -1, stream, sa);
    if (head_dim == 32)
        return launch_encoder_attention<32, 32, true>(nullptr, 0, B, W, H, nullptr, relpos, pos_u, pos_v, P, ldp, scale, out, ldo, 0, -1, stream, sa);
    set_error("encoder_attention_stream: head_dim=%d not built (64, 36 with RelPosMHAXL, 32)", head_dim);
    return SBK_ERR_UNSUPPORTED;
}

// One chunk's QKV projection qkv [B*n, 3d] fp32 (per-head [q | k | v] blocks) -> the attention's operands: q [B*n, d] fp16
// (RoPE: rotated and scaled by q_scale, as the full-sequence epilogue does; RelPos: as projected) and each row's [k | v]
// per head into the ring slot (slot0 + i) % cap of kv [B][cap][2d] fp16.  RoPE rotates q and k by the row's position in the
// stream: the angle pos * inv_freq is formed and reduced in double precision, so it stays exact however long the stream,
// and the scores, which depend on the position difference only, equal those of a window-local rotation.  Each cached key
// is rotated and rounded to fp16 once, like the full-sequence path's keys.
__global__ void stream_qkv_kernel(const float* __restrict__ qkv, int n, int H, int DH, const float* __restrict__ inv_freq,
                                  long long pos0, float q_scale, __half* __restrict__ q, __half* __restrict__ kv, int cap,
                                  int slot0) {
    const int half_dh = DH >> 1, d = H * DH;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // (pair, head) of row blockIdx.y
    if (idx >= H * half_dh) return;
    const int h = idx / half_dh, p = idx - h * half_dh, row = blockIdx.y, b = row / n, i = row - b * n;
    const float* src = qkv + static_cast<size_t>(row) * 3 * d + h * 3 * DH + 2 * p;
    float q0 = src[0], q1 = src[1], k0 = src[DH], k1 = src[DH + 1];
    if (inv_freq) {
        double sd, cd;
        sincos(static_cast<double>(pos0 + i) * static_cast<double>(inv_freq[p]), &sd, &cd);
        const float c = static_cast<float>(cd), s = static_cast<float>(sd);
        const float rq0 = (q0 * c - q1 * s) * q_scale, rq1 = (q1 * c + q0 * s) * q_scale;
        const float rk0 = k0 * c - k1 * s, rk1 = k1 * c + k0 * s;
        q0 = rq0; q1 = rq1; k0 = rk0; k1 = rk1;
    }
    *reinterpret_cast<__half2*>(q + static_cast<size_t>(row) * d + h * DH + 2 * p) = floats2half2_sat(q0, q1);
    const int slot = (slot0 + i) % cap;
    __half* dst = kv + (static_cast<size_t>(b) * cap + slot) * 2 * d + h * 2 * DH + 2 * p;
    *reinterpret_cast<__half2*>(dst) = floats2half2_sat(k0, k1);
    *reinterpret_cast<__half2*>(dst + DH) = floats2half2_sat(src[2 * DH], src[2 * DH + 1]);
}

int stream_qkv(const float* qkv, int B, int n, int H, int DH, const float* inv_freq, long long pos0, float q_scale,
               __half* q, __half* kv, int cap, int slot0, cudaStream_t stream) {
    SBK_REQUIRE(DH % 2 == 0 && n >= 1 && cap >= n && slot0 >= 0, "stream_qkv: bad shape");
    const int pairs = H * DH / 2;
    stream_qkv_kernel<<<dim3(ceil_div(pairs, 128), B * n), 128, 0, stream>>>(qkv, n, H, DH, inv_freq, pos0, q_scale, q, kv,
                                                                            cap, slot0);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

// =========================================================================== HyperMixing (HyperConformer token mixing)
// HyperMixing.forward (nnet/hypermixing.py:90-195, 249-372; tied=False, keep_output_size=False) on the norm1 output
// h16 [B*T, d] fp16, with M heads of e = d/M channels and a hypernetwork width of k = d_ffn/M per head:
//     xm = h16 * valid;  hin = xm + PE_hm[t]                       (the module's own sine table, HM_PE_ROWS rows)
//     per head m:  W1 = fc2_1(GELU(fc1_1(hin_m))), W2 = fc2_2(GELU(fc1_2(hin_m)))   [T, k], padded rows 0
//                  H_m = xm_m^T W1 [e, k] over every frame,  y_m = W2 GELU(H_m)^T [T, e]
//     x += LayerNorm_hm(y)   over the d channels of a frame (a padded frame has y = 0 and gets beta)
// W1 and W2 never go through global memory: each is regenerated from hin in shared memory where it is consumed.
//   hypermix_reduce:   one CTA per (HM_CHUNK frames, head, utterance).  Per 64-frame tile: w1_gen on tensor cores into
//                      shared memory, then H += xm^T W1 in registers.  Writes the chunk's fp32 partial H.
//   hypermix_finalize: per (head, utterance) the chunk partials summed in chunk order, G = GELU(H), stored fp16 as
//                      G * 2^-s with the power of two s that puts max |G| in [2^13, 2^14): H grows with the number of
//                      frames, and the scale keeps G finite and at full fp16 precision.  No atomics: chunks are aligned
//                      to frame 0 and chunks past an utterance's length are not read, so reruns are bit-identical and
//                      batch padding does not change an utterance's sums.
//   hypermix_expand:   one CTA per (TR frames, utterance) over all heads: w2_gen into shared memory, y = W2 G^T times 2^s
//                      in fp32 into a [TR, d] tile, then LayerNorm_hm of each frame and the residual add into x.
// 8 warps share every product; the 16 x 8 output tiles of an m16n8k16 product are dealt round-robin to the warps, with
// both operands K-contiguous in shared memory (ldmatrix without transposition).
constexpr int HM_WARPS = 8, HM_THREADS = 32 * HM_WARPS, HM_TILE = 64, HM_CHUNK = 256;

// acc[16 x 8] += A[16 rows, 0..K) . Bm[8 rows, 0..K)^T; row strides lda / ldb in halfs (multiples of 8), K % 16 == 0
__device__ __forceinline__ void hm_mma_tile(float (&acc)[4], const __half* A, int lda, const __half* Bm, int ldb, int K) {
    const int lane = threadIdx.x & 31;
    const __half* pa = A + (lane & 15) * lda + (lane >> 4) * 8;
    const __half* pb = Bm + (lane & 7) * ldb + ((lane >> 3) & 1) * 8;
    for (int k0 = 0; k0 < K; k0 += 16) {
        uint32_t a[4], b0, b1;
        ldmatrix_x4(a[0], a[1], a[2], a[3], pa + k0);
        ldmatrix_x2(b0, b1, pb + k0);
        mma16816(acc, a, b0, b1);
    }
}

// epi(r, n, C[r][n], C[r][n+1]) for every even n of C = A[R, K] . Bm[N, K]^T (R % 16 == 0, N % 8 == 0)
template <typename Epi>
__device__ __forceinline__ void hm_gemm(const __half* A, int lda, const __half* Bm, int ldb, int R, int N, int K, Epi epi) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int nt = N / 8, tiles = (R / 16) * nt;
    for (int t = warp; t < tiles; t += HM_WARPS) {
        const int r0 = (t / nt) * 16, n0 = (t % nt) * 8;
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        hm_mma_tile(acc, A + r0 * lda, lda, Bm + n0 * ldb, ldb, K);
        epi(r0 + g, n0 + 2 * c, acc[0], acc[1]);
        epi(r0 + g + 8, n0 + 2 * c, acc[2], acc[3]);
    }
}

// rows x cols fp16 matrix (row-major, contiguous) -> shared memory with row stride ld halfs; cols % 8 == 0
__device__ __forceinline__ void hm_copy_rows(__half* dst, int ld, const __half* __restrict__ src, int rows, int cols) {
    const int v = cols / 8;
    for (int i = threadIdx.x; i < rows * v; i += blockDim.x) {
        const int r = i / v, j = (i - r * v) * 8;
        *reinterpret_cast<uint4*>(dst + r * ld + j) = __ldg(reinterpret_cast<const uint4*>(src + static_cast<size_t>(r) * cols + j));
    }
}

// hin = xm + PE (fp16, [rows][ldh]) and, when xmT != null, xm transposed ([E][ldx]) for the frames t0 .. t0 + rows - 1 of
// the utterance at row0, channels ch0 .. ch0 + E - 1: xm = h16 for t < len, 0 otherwise; frames t >= T are 0 in both
template <int E>
__device__ __forceinline__ void hm_stage(const __half* __restrict__ h16, const float* __restrict__ pe, int d, int T, int len,
                                         size_t row0, int t0, int rows, int ch0, __half* hin, int ldh, __half* xmT, int ldx) {
    constexpr int V = E / 8;
    for (int i = threadIdx.x; i < rows * V; i += blockDim.x) {
        const int r = i / V, v = (i - r * V) * 8, t = t0 + r;
        uint4 raw = make_uint4(0u, 0u, 0u, 0u), hv = make_uint4(0u, 0u, 0u, 0u);
        if (t < len) raw = __ldg(reinterpret_cast<const uint4*>(h16 + (row0 + t) * d + ch0 + v));
        const __half* xh = reinterpret_cast<const __half*>(&raw);
        if (t < T) {
            const float4 p0 = __ldg(reinterpret_cast<const float4*>(pe + static_cast<size_t>(t) * d + ch0 + v));
            const float4 p1 = __ldg(reinterpret_cast<const float4*>(pe + static_cast<size_t>(t) * d + ch0 + v + 4));
            hv.x = pack_half2(__half2float(xh[0]) + p0.x, __half2float(xh[1]) + p0.y);
            hv.y = pack_half2(__half2float(xh[2]) + p0.z, __half2float(xh[3]) + p0.w);
            hv.z = pack_half2(__half2float(xh[4]) + p1.x, __half2float(xh[5]) + p1.y);
            hv.w = pack_half2(__half2float(xh[6]) + p1.z, __half2float(xh[7]) + p1.w);
        }
        *reinterpret_cast<uint4*>(hin + r * ldh + v) = hv;
        if (xmT != nullptr) {
#pragma unroll
            for (int j = 0; j < 8; ++j) xmT[(v + j) * ldx + r] = xh[j];
        }
    }
}

template <int E>
__global__ void __launch_bounds__(HM_THREADS)
hypermix_reduce_kernel(const __half* __restrict__ h16, int T, int d, int KH, const int* __restrict__ lens,
                       const float* __restrict__ pe, const __half* __restrict__ fc1w, const float* __restrict__ fc1b,
                       const __half* __restrict__ fc2w, const float* __restrict__ fc2b, float* __restrict__ part, int nchunk) {
    constexpr int LE = E + 8, LT = HM_TILE + 8;
    constexpr int MAXT = E / 4;  // 16 x 8 tiles of H per warp at k = 256: (E / 16) * (256 / 8) / HM_WARPS
    extern __shared__ __align__(16) uint8_t hm_smem[];
    __half* w1s = reinterpret_cast<__half*>(hm_smem);  // fc1 of head m [E][LE]
    __half* w2s = w1s + E * LE;                        // fc2 of head m [KH][LE]
    __half* hin = w2s + KH * LE;                       // [64][LE]
    __half* hid = hin + HM_TILE * LE;                  // GELU(fc1 hin) [64][LE]
    __half* xmT = hid + HM_TILE * LE;                  // xm^T [E][LT]
    __half* w1T = xmT + E * LT;                        // W1^T [KH][LT]
    const int chunk = blockIdx.x, m = blockIdx.y, b = blockIdx.z, M = gridDim.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int len = lens ? min(max(lens[b], 0), T) : T;
    const size_t row0 = static_cast<size_t>(b) * T;
    const float* b1 = fc1b + m * E;
    const float* b2 = fc2b + m * KH;
    hm_copy_rows(w1s, LE, fc1w + static_cast<size_t>(m) * E * E, E, E);
    hm_copy_rows(w2s, LE, fc2w + static_cast<size_t>(m) * KH * E, KH, E);
    const int nt = KH / 8, tiles = (E / 16) * nt;
    float acc[MAXT][4];
#pragma unroll
    for (int i = 0; i < MAXT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.0f;
    const int te = min(chunk * HM_CHUNK + HM_CHUNK, len);
    for (int t0 = chunk * HM_CHUNK; t0 < te; t0 += HM_TILE) {
        __syncthreads();  // the previous tile is consumed (first tile: the weights are staged)
        hm_stage<E>(h16, pe, d, T, len, row0, t0, HM_TILE, m * E, hin, LE, xmT, LT);
        __syncthreads();
        hm_gemm(hin, LE, w1s, LE, HM_TILE, E, E, [&](int r, int n, float v0, float v1) {
            *reinterpret_cast<uint32_t*>(hid + r * LE + n) =
                pack_half2(gelu_erf_f(v0 + __ldg(b1 + n)), gelu_erf_f(v1 + __ldg(b1 + n + 1)));
        });
        __syncthreads();
        hm_gemm(hid, LE, w2s, LE, HM_TILE, KH, E, [&](int r, int n, float v0, float v1) {
            const bool ok = t0 + r < len;  // padded frames: W1 row 0
            w1T[n * LT + r] = float2half_sat(ok ? v0 + __ldg(b2 + n) : 0.0f);
            w1T[(n + 1) * LT + r] = float2half_sat(ok ? v1 + __ldg(b2 + n + 1) : 0.0f);
        });
        __syncthreads();
#pragma unroll
        for (int i = 0; i < MAXT; ++i) {
            const int t = warp + HM_WARPS * i;
            if (t < tiles) hm_mma_tile(acc[i], xmT + (t / nt) * 16 * LT, LT, w1T + (t % nt) * 8 * LT, LT, HM_TILE);
        }
    }
    float* out = part + ((static_cast<size_t>(b) * M + m) * nchunk + chunk) * E * KH;
#pragma unroll
    for (int i = 0; i < MAXT; ++i) {
        const int t = warp + HM_WARPS * i;
        if (t >= tiles) continue;
        const int r = (t / nt) * 16 + g, n = (t % nt) * 8 + 2 * c;
        *reinterpret_cast<float2*>(out + static_cast<size_t>(r) * KH + n) = make_float2(acc[i][0], acc[i][1]);
        *reinterpret_cast<float2*>(out + static_cast<size_t>(r + 8) * KH + n) = make_float2(acc[i][2], acc[i][3]);
    }
}

__global__ void __launch_bounds__(256)
hypermix_finalize_kernel(float* __restrict__ part, int nchunk, int T, const int* __restrict__ lens, int EK,
                         __half* __restrict__ G, float* __restrict__ gscale) {
    __shared__ float red[8];
    const int m = blockIdx.x, b = blockIdx.y, M = gridDim.x;
    const int len = lens ? min(max(lens[b], 0), T) : T;
    const int nc = max(1, ceil_div(len, HM_CHUNK));  // chunks holding valid frames (chunk 0 is always written)
    float* p = part + (static_cast<size_t>(b) * M + m) * nchunk * EK;
    float mx = 0.0f;
    for (int i = threadIdx.x; i < EK; i += blockDim.x) {
        float s = p[i];
        for (int ch = 1; ch < nc; ++ch) s += p[static_cast<size_t>(ch) * EK + i];
        const float gv = gelu_erf_f(s);
        p[i] = gv;  // read back below by the same thread
        mx = fmaxf(mx, fabsf(gv));
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
    int ex = 0;
    frexpf(mx, &ex);  // mx < 2^ex
    const int s = mx > 0.0f ? ex - 14 : 0;
    const float down = ldexpf(1.0f, -s);
    __half* gp = G + (static_cast<size_t>(b) * M + m) * EK;
    for (int i = threadIdx.x; i < EK; i += blockDim.x) gp[i] = float2half_sat(p[i] * down);
    if (threadIdx.x == 0) gscale[b * M + m] = ldexpf(1.0f, s);
}

template <int E, int TR>
__global__ void __launch_bounds__(HM_THREADS)
hypermix_expand_kernel(const __half* __restrict__ h16, int T, int d, int KH, const int* __restrict__ lens,
                       const float* __restrict__ pe, const __half* __restrict__ fc1w, const float* __restrict__ fc1b,
                       const __half* __restrict__ fc2w, const float* __restrict__ fc2b, const __half* __restrict__ G,
                       const float* __restrict__ gscale, const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                       float eps, float* __restrict__ x) {
    constexpr int LE = E + 8;
    const int LK = KH + 8, LY = d + 4;
    extern __shared__ __align__(16) uint8_t hm_smem[];
    float* ys = reinterpret_cast<float*>(hm_smem);     // y of every head [TR][LY]
    __half* w1s = reinterpret_cast<__half*>(ys + TR * LY);  // [E][LE]
    __half* w2s = w1s + E * LE;                        // [KH][LE]
    __half* hin = w2s + KH * LE;                       // [TR][LE]
    __half* hid = hin + TR * LE;                       // [TR][LE]
    __half* w2t = hid + TR * LE;                       // W2 [TR][LK]
    __half* gs = w2t + TR * LK;                        // G * 2^-s [E][LK]
    const int t0 = blockIdx.x * TR, b = blockIdx.y, M = d / E;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int len = lens ? min(max(lens[b], 0), T) : T;
    const size_t row0 = static_cast<size_t>(b) * T;
    for (int m = 0; m < M; ++m) {
        const float* b1 = fc1b + m * E;
        const float* b2 = fc2b + m * KH;
        __syncthreads();  // the previous head's operands are consumed
        hm_copy_rows(w1s, LE, fc1w + static_cast<size_t>(m) * E * E, E, E);
        hm_copy_rows(w2s, LE, fc2w + static_cast<size_t>(m) * KH * E, KH, E);
        hm_copy_rows(gs, LK, G + (static_cast<size_t>(b) * M + m) * E * KH, E, KH);
        hm_stage<E>(h16, pe, d, T, len, row0, t0, TR, m * E, hin, LE, nullptr, 0);
        __syncthreads();
        hm_gemm(hin, LE, w1s, LE, TR, E, E, [&](int r, int n, float v0, float v1) {
            *reinterpret_cast<uint32_t*>(hid + r * LE + n) =
                pack_half2(gelu_erf_f(v0 + __ldg(b1 + n)), gelu_erf_f(v1 + __ldg(b1 + n + 1)));
        });
        __syncthreads();
        hm_gemm(hid, LE, w2s, LE, TR, KH, E, [&](int r, int n, float v0, float v1) {
            const bool ok = t0 + r < len;  // padded frames: W2 row 0
            *reinterpret_cast<uint32_t*>(w2t + r * LK + n) =
                pack_half2(ok ? v0 + __ldg(b2 + n) : 0.0f, ok ? v1 + __ldg(b2 + n + 1) : 0.0f);
        });
        __syncthreads();
        const float sc = __ldg(gscale + b * M + m);
        hm_gemm(w2t, LK, gs, LK, TR, E, KH, [&](int r, int n, float v0, float v1) {
            *reinterpret_cast<float2*>(ys + r * LY + m * E + n) = make_float2(v0 * sc, v1 * sc);
        });
    }
    __syncthreads();
    // LayerNorm_hm (fp32, two-pass) of each frame and x += it, for every frame < T (padded frames get + beta)
    for (int r = warp; r < TR; r += HM_WARPS) {
        const int t = t0 + r;
        if (t >= T) break;
        const float* yr = ys + r * LY;
        float s = 0.0f;
        for (int j = lane; j < d; j += 32) s += yr[j];
        const float mean = warp_sum(s) / d;
        float v = 0.0f;
        for (int j = lane; j < d; j += 32) v += (yr[j] - mean) * (yr[j] - mean);
        const float rstd = rsqrtf(warp_sum(v) / d + eps);
        float* xr = x + (row0 + t) * d;
        for (int j = lane; j < d; j += 32) xr[j] += (yr[j] - mean) * rstd * __ldg(ln_g + j) + __ldg(ln_b + j);
    }
}

size_t hypermix_part_floats(int B, int T, int d, int KH) {
    return static_cast<size_t>(B) * d * KH * ceil_div(std::max(T, 1), HM_CHUNK);
}

template <int E>
static size_t hm_reduce_smem(int KH) { return 2ull * (E * (E + 8) + KH * (E + 8) + 2 * HM_TILE * (E + 8) + (E + KH) * (HM_TILE + 8)); }
template <int E, int TR>
static size_t hm_expand_smem(int d, int KH) {
    return 4ull * TR * (d + 4) + 2ull * (E * (E + 8) + KH * (E + 8) + 2 * TR * (E + 8) + (TR + E) * (KH + 8));
}

template <int E>
static int launch_hypermix(const __half* h16, int B, int T, int d, int KH, const int* lens, const float* pe,
                           const HyperMixWeights& w, float* part, __half* G, float* gscale, float* x, cudaStream_t st) {
    constexpr int TR = E == 32 ? 64 : 32;
    const int M = d / E, nchunk = ceil_div(T, HM_CHUNK);
    const size_t sm_r = hm_reduce_smem<E>(KH), sm_e = hm_expand_smem<E, TR>(d, KH);
    SBK_REQUIRE(sm_e <= 227 * 1024, "hypermix: d_model=%d with k=%d needs %zu bytes of shared memory", d, KH, sm_e);
    auto kr = hypermix_reduce_kernel<E>;
    SBK_CUDA_CHECK(cudaFuncSetAttribute(kr, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_r));
    kr<<<dim3(nchunk, M, B), HM_THREADS, sm_r, st>>>(h16, T, d, KH, lens, pe, w.fc1w[0], w.fc1b[0], w.fc2w[0], w.fc2b[0], part,
                                                    nchunk);
    SBK_LAUNCH_CHECK();
    hypermix_finalize_kernel<<<dim3(M, B), 256, 0, st>>>(part, nchunk, T, lens, E * KH, G, gscale);
    SBK_LAUNCH_CHECK();
    auto ke = hypermix_expand_kernel<E, TR>;
    SBK_CUDA_CHECK(cudaFuncSetAttribute(ke, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_e));
    ke<<<dim3(ceil_div(T, TR), B), HM_THREADS, sm_e, st>>>(h16, T, d, KH, lens, pe, w.fc1w[1], w.fc1b[1], w.fc2w[1], w.fc2b[1],
                                                           G, gscale, w.ln_g, w.ln_b, 1e-5f, x);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int hypermix_forward(const __half* h16, int B, int T, int d, int M, int KH, const int* lens, const float* pe,
                     const HyperMixWeights& w, float* part, __half* G, float* gscale, float* x, cudaStream_t st) {
    SBK_REQUIRE(M > 0 && d % M == 0, "hypermix: d_model=%d, nhead=%d", d, M);
    const int E = d / M;
    SBK_REQUIRE(E == 32 || E == 64, "hypermix: head width d_model / nhead = %d not built (32, 64)", E);
    SBK_REQUIRE(KH > 0 && KH % 16 == 0 && KH <= 256, "hypermix: k = d_ffn / nhead = %d must be a multiple of 16 up to 256", KH);
    SBK_REQUIRE(T <= HM_PE_ROWS, "hypermix: %d frames exceed the HyperMixing positional table (%d)", T, HM_PE_ROWS);
    SBK_REQUIRE(B <= 65535, "hypermix: B=%d", B);
    if (B == 0 || T == 0) return SBK_OK;
    return E == 32 ? launch_hypermix<32>(h16, B, T, d, KH, lens, pe, w, part, G, gscale, x, st)
                   : launch_hypermix<64>(h16, B, T, d, KH, lens, pe, w, part, G, gscale, x, st);
}

// =========================================================================== TransformerLM causal self-attention
// Whole-sequence attention of TransformerLM.forward (TransformerLM.py:127-169: nn.MultiheadAttention under make_masks'
// look-ahead mask and key-padding mask on pad_idx).  qkv [n*s, 3d] fp16 with columns [q | k | v] (nn.MultiheadAttention's
// in_proj order, heads of DH side by side, q pre-scaled by 1/sqrt(true head width)) -> out [n*s, d] fp16.  DH = 64, or 32:
// the Switchboard LM's heads of 22 zero-padded to the 16-wide k-step of m16n8k16 (the padding adds zero to q.k and
// gives zero output columns).
// One CTA = (64 query rows, head, sequence), 4 warps x 16 rows, mma.sync m16n8k16 with an fp32 online softmax like
// encoder_attention_kernel.  Query block qb reads key blocks 0..qb only: blocks above the diagonal are never loaded.
// Masked: keys j > i (diagonal block only) and keys whose token id is pad_tok -- the rule the KV-cached step applies
// through tok_cache / pad_tok (dec_attention_kernel).  A query whose visible keys are all padding (a sequence that starts
// with the pad id) has an empty softmax and yields NaN, as in the reference and the step path.
constexpr int LMA_B = 64;

template <int DH>
__global__ void __launch_bounds__(128)
lm_causal_attention_kernel(const __half* __restrict__ qkv, int s, int d, const int* __restrict__ tokens, int pad_tok,
                           __half* __restrict__ out) {
    static_assert(DH % 32 == 0, "lm_causal_attention_kernel: K fragments are loaded 32 dims at a time");
    constexpr int STR = DH + 8, KS = DH / 16;  // row stride 16 B past a multiple of 64 B: ldmatrix rows hit distinct banks
    __shared__ __align__(16) __half Qs[LMA_B * STR];
    __shared__ __align__(16) __half KVs[2][2][LMA_B * STR];  // [buffer][K | V]
    __shared__ bool s_masked[2][LMA_B];                       // [buffer][key]: pad token or past the sequence
    const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z, i0 = qb * LMA_B;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const int ld = 3 * d;
    const __half* base = qkv + static_cast<size_t>(b) * s * ld + h * DH;
    const int* tok = tokens + static_cast<size_t>(b) * s;

    auto cp16 = [](__half* dst, const __half* src, bool ok) {  // rows past the sequence are zero-filled
        cp_async16_zfill(smem_u32(dst), src, ok ? 16u : 0u);
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
        cp_async_commit();
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
        cp_async_wait<0>();
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
    SBK_REQUIRE(H >= 1 && (d == H * 64 || d == H * 32), "lm_causal_attention: head_dim must be 64 or 32 (d=%d, H=%d)", d, H);
    SBK_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
                "lm_causal_attention: misaligned operands");
    if (n == 0 || s == 0) return SBK_OK;
    const dim3 grid(ceil_div(s, LMA_B), H, n);
    if (d == H * 64) lm_causal_attention_kernel<64><<<grid, 128, 0, stream>>>(qkv, s, d, tokens, pad_tok, out);
    else lm_causal_attention_kernel<32><<<grid, 128, 0, stream>>>(qkv, s, d, tokens, pad_tok, out);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // namespace sbk
