// ConvolutionFrontEnd: 2 x [reflect-pad + Conv2d(3x3, stride 2) + LayerNorm(F', C) + LeakyReLU], or the Transformer
// recipes' 3 blocks (5x5, 5x5, 1x1 with a residual 1x1).
//
// Replaces lobes/models/convolution.py:116-320 (ConvolutionFrontEnd / ConvBlock) with
// nnet/CNN.py:654-751 (Conv2d.forward, "same" reflect padding k//2 for stride > 1) and
// nnet/normalization.py:185-242 (LayerNorm over the last two dims), activation LeakyReLU(0.01).
//
// Layouts (channels-last, as the reference exposes them):
//   feats [B, T0, F0] fp32 -> act1 [B, T1, F1, C1] fp16 -> out [B, T2, F2*C2] fp16 (+ fp32)
//   T1 = (T0-1)/2+1, F1 = (F0-1)/2+1, likewise T2/F2.
// cnn_frontend_forward at the bottom makes every kernel choice from the weights' block count and channels.
//
// Each stage is written once and shared by the kernels that run it:
//   conv1 (C_in = 1, K x K taps, K = 3 or 5): conv1_stage_rows / conv1_taps / conv1_frame / conv1_centred_sq /
//     conv1_ln_pair.  A thread owns two channels of one frame in registers; conv1_warp_frame adds the warp-shuffle
//     LayerNorm statistics.  conv1_ln_kernel (3x3) and conv1k5_ln_kernel (5x5) write act1 with one warp per frame,
//     cnn_fused_kernel writes its frames into the conv2 patch in shared memory, conv1c256_ln_kernel reduces over 4 warps.
//   conv2 (64 input channels, K = 9 or 25 taps x 64) is an implicit GEMM on mma.sync.m16n8k16 (fp16 in, fp32 accumulate)
//     over a reflect-padded patch in shared memory (stage_patch, conv_tile_store); the 64 -> 32 conv2 of
//     conv2_ln_kernel and cnn_fused_kernel is conv2_gemm + conv2_ln_store; the per-frame LayerNorm statistics are
//     frame_ln_stats.  conv2c256_ln_kernel (256 -> 256) runs on wgmma.
#include <algorithm>

#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

__device__ __forceinline__ int reflect_idx(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }
__device__ __forceinline__ float leaky(float x) { return x > 0.0f ? x : 0.01f * x; }

// --------------------------------------------------------------------------- conv1 stage
// w1: [C1, K(kf), K(kt)] fp32 (reference weight (C1,1,kf,kt)), b1: [C1]; g/be: [F1, C1].  A thread owns channels c0, c0 + 1
// for all F1 feature rows of one frame, so the frame's outputs stay in registers and every store is a half2.

// in [K][F0 + K - 1] <- the K reflect-padded feature rows conv1 frame t1 reads; threads tid, tid + nthr, ...
template <int K>
__device__ __forceinline__ void conv1_stage_rows(float* in, const float* __restrict__ feats, int b, int t1, int T0, int F0,
                                                 int tid, int nthr) {
    const int FP = F0 + K - 1;
    for (int i = tid; i < K * FP; i += nthr) {
        const int kt = i / FP, fp = i - kt * FP;
        const int t = reflect_idx(2 * t1 + kt - K / 2, T0);
        const int f = reflect_idx(fp - K / 2, F0);
        in[i] = __ldg(feats + (static_cast<size_t>(b) * T0 + t) * F0 + f);
    }
}

template <int K>
struct Conv1Taps {
    float wa[K * K], wb[K * K], ba, bb;  // channels c0, c0 + 1
};
template <int K>
__device__ __forceinline__ Conv1Taps<K> conv1_taps(const float* __restrict__ w1, const float* __restrict__ b1, int c0) {
    Conv1Taps<K> w;
#pragma unroll
    for (int i = 0; i < K * K; ++i) { w.wa[i] = __ldg(w1 + c0 * K * K + i); w.wb[i] = __ldg(w1 + (c0 + 1) * K * K + i); }
    w.ba = __ldg(b1 + c0);
    w.bb = __ldg(b1 + c0 + 1);
    return w;
}

// The channel pair's conv outputs at f1 < F1 into va / vb (0 beyond); returns their sum
template <int K, int MAXF>
__device__ __forceinline__ float conv1_frame(const float* in, int F0, int F1, const Conv1Taps<K>& w, float (&va)[MAXF],
                                             float (&vb)[MAXF]) {
    const int FP = F0 + K - 1;
    float s = 0.0f;
#pragma unroll
    for (int f1 = 0; f1 < MAXF; ++f1) {
        va[f1] = 0.0f; vb[f1] = 0.0f;
        if (f1 < F1) {
            float a = w.ba, bq = w.bb;
#pragma unroll
            for (int kf = 0; kf < K; ++kf)
#pragma unroll
                for (int kt = 0; kt < K; ++kt) {
                    const float x = in[kt * FP + 2 * f1 + kf];
                    a = fmaf(w.wa[kf * K + kt], x, a);
                    bq = fmaf(w.wb[kf * K + kt], x, bq);
                }
            va[f1] = a; vb[f1] = bq;
            s += a + bq;
        }
    }
    return s;
}

template <int MAXF>
__device__ __forceinline__ float conv1_centred_sq(const float (&va)[MAXF], const float (&vb)[MAXF], int F1, float mean) {
    float q = 0.0f;
#pragma unroll
    for (int f1 = 0; f1 < MAXF; ++f1)
        if (f1 < F1) {
            const float da = va[f1] - mean, db = vb[f1] - mean;
            q += da * da + db * db;
        }
    return q;
}

// LayerNorm (gamma / beta at gi = f1 * C1 + c0) + LeakyReLU of the channel pair (va, vb), as fp16
__device__ __forceinline__ __half2 conv1_ln_pair(float va, float vb, float mean, float rstd, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, int gi) {
    const float2 g = __ldg(reinterpret_cast<const float2*>(gamma + gi));
    const float2 be = __ldg(reinterpret_cast<const float2*>(beta + gi));
    return floats2half2_sat(leaky((va - mean) * rstd * g.x + be.x), leaky((vb - mean) * rstd * g.y + be.y));
}

// One warp computes 64-channel conv1 frame t1 (lane l: channels 2l, 2l+1) and its LayerNorm statistics over (F1, 64) with
// warp shuffles only (no block barriers); in: this warp's [K][F0 + K - 1] staging rows.
template <int K, int MAXF>
__device__ __forceinline__ void conv1_warp_frame(float* in, const float* __restrict__ feats, int b, int t1, int T0, int F0,
                                                 int F1, const float* __restrict__ w1, const float* __restrict__ b1,
                                                 int lane, float (&va)[MAXF], float (&vb)[MAXF], float& mean, float& rstd) {
    conv1_stage_rows<K>(in, feats, b, t1, T0, F0, lane, 32);
    const Conv1Taps<K> w = conv1_taps<K>(w1, b1, 2 * lane);
    __syncwarp();
    const float n = static_cast<float>(F1 * 64);
    mean = warp_sum(conv1_frame<K>(in, F0, F1, w, va, vb)) / n;
    rstd = rsqrtf(warp_sum(conv1_centred_sq(va, vb, F1, mean)) / n + 1e-5f);
}

// One WARP per output frame (C1_WARPS frames per CTA) -> act1 [B, T1, F1, 64] fp16: every store is a 128-byte half2 row
// segment (instead of one 256-thread CTA per frame with three block barriers and 2-byte stores).
constexpr int C1_WARPS = 8;

template <int K, int MAXF>
__device__ __forceinline__ void conv1_warps_to_act1(float* smem, const float* __restrict__ feats, int T0, int F0, int T1,
                                                    int F1, const float* __restrict__ w1, const float* __restrict__ b1,
                                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                                    __half* __restrict__ out_h) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y, t1 = blockIdx.x * C1_WARPS + warp;
    if (t1 >= T1) return;
    float va[MAXF], vb[MAXF], mean, rstd;
    conv1_warp_frame<K>(smem + warp * K * (F0 + K - 1), feats, b, t1, T0, F0, F1, w1, b1, lane, va, vb, mean, rstd);
    const size_t obase = (static_cast<size_t>(b) * T1 + t1) * F1 * 64;
#pragma unroll
    for (int f1 = 0; f1 < MAXF; ++f1)
        if (f1 < F1) {
            const int gi = f1 * 64 + 2 * lane;
            *reinterpret_cast<__half2*>(out_h + obase + gi) = conv1_ln_pair(va[f1], vb[f1], mean, rstd, gamma, beta, gi);
        }
}

template <int C1, int MAXF>
__global__ void __launch_bounds__(C1_WARPS * 32)
conv1_ln_kernel(const float* __restrict__ feats, int T0, int F0, int T1, int F1, const float* __restrict__ w1,
                const float* __restrict__ b1, const float* __restrict__ gamma, const float* __restrict__ beta,
                __half* __restrict__ out_h) {
    static_assert(C1 == 64, "two channels per lane");
    extern __shared__ float c1_smem[];
    conv1_warps_to_act1<3, MAXF>(c1_smem, feats, T0, F0, T1, F1, w1, b1, gamma, beta, out_h);
}

// block 1 of the 3-block front-end: w1 [64, 5(kf), 5(kt)]
template <int MAXF>
__global__ void __launch_bounds__(C1_WARPS * 32)
conv1k5_ln_kernel(const float* __restrict__ feats, int T0, int F0, int T1, int F1, const float* __restrict__ w1,
                  const float* __restrict__ b1, const float* __restrict__ gamma, const float* __restrict__ beta,
                  __half* __restrict__ out_h) {
    extern __shared__ float c1_smem[];
    conv1_warps_to_act1<5, MAXF>(c1_smem, feats, T0, F0, T1, F1, w1, b1, gamma, beta, out_h);
}

// --------------------------------------------------------------------------- 64-channel conv2 stage (mma.sync)
constexpr int CELL = 72;       // padded channel stride (halfs) of one (t, f) cell of a 64-channel patch in smem

// patch [ROWS][F1 + K - 1][CELL] <- the reflect-padded act1 frames of the CTA's output frames from t0 (16-byte vectors)
template <int K, int ROWS>
__device__ __forceinline__ void stage_patch(__half* patch, const __half* __restrict__ act1, int b, int t0, int T1, int F1) {
    const int FPAD = F1 + K - 1;
    for (int i = threadIdx.x; i < ROWS * FPAD * 8; i += blockDim.x) {
        const int cell = i / 8, v8 = i - cell * 8;
        const int tr = cell / FPAD, fp = cell - tr * FPAD;
        int t = reflect_idx(2 * t0 + tr - K / 2, T1);
        t = min(max(t, 0), T1 - 1);  // tail tiles: keep loads in range (results discarded)
        const int f = reflect_idx(fp - K / 2, F1);
        *reinterpret_cast<uint4*>(patch + cell * CELL + v8 * 8) =
            *reinterpret_cast<const uint4*>(act1 + ((static_cast<size_t>(b) * T1 + t) * F1 + f) * 64 + v8 * 8);
    }
}

// acc + bias -> out [rows][LD] fp32 at the warp's rows r0, r1 = r0 + 8 (those < rows)
template <int NT, int LD>
__device__ __forceinline__ void conv_tile_store(const float (&acc)[NT][4], const float* __restrict__ bias, float* out, int r0,
                                                int r1, int rows, int c) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const int col = nt * 8 + 2 * c;
        const float bz0 = __ldg(bias + col), bz1 = __ldg(bias + col + 1);
        if (r0 < rows) { out[r0 * LD + col] = acc[nt][0] + bz0; out[r0 * LD + col + 1] = acc[nt][1] + bz1; }
        if (r1 < rows) { out[r1 * LD + col] = acc[nt][2] + bz0; out[r1 * LD + col + 1] = acc[nt][3] + bz1; }
    }
}

// LayerNorm statistics over the n = F2 * C values of one frame held in smem rows [F2][stride] (C channels each); one warp
template <int C>
__device__ __forceinline__ void frame_ln_stats(const float* src, int stride, int n, int lane, float& mean, float& rstd) {
    constexpr int LOG_C = C == 32 ? 5 : 6;
    static_assert(C == 1 << LOG_C, "32 or 64 channels per pixel");
    float s = 0.0f;
    for (int i = lane; i < n; i += 32) s += src[(i >> LOG_C) * stride + (i & (C - 1))];
    mean = warp_sum(s) / n;
    float q = 0.0f;
    for (int i = lane; i < n; i += 32) {
        const float d = src[(i >> LOG_C) * stride + (i & (C - 1))] - mean;
        q += d * d;
    }
    rstd = rsqrtf(warp_sum(q) / n + 1e-5f);
}

// conv2 64 -> 32: act1 [B, T1, F1, 64] fp16; w2p [32, 576] fp16 with k = (kf*3+kt)*64 + ch; out [B, T2, F2*32].
// A CTA computes C2_FRAMES output frames from a 9-frame patch; the weight matrix lives in shared memory too.
constexpr int C2_FRAMES = 4;   // output frames per CTA
constexpr int C2_PROWS = 2 * C2_FRAMES + 1;  // act1 frames of the patch
constexpr int C2_COUT = 32;
constexpr int C2_WROW = 9 * 64 + 8;  // padded weight row (halfs)
constexpr int C2_LD = C2_COUT + 1;   // fp32 row stride of cbuf

__device__ __forceinline__ void conv2_stage_weights(__half* wsm, const __half* __restrict__ w2p) {
    for (int i = threadIdx.x; i < C2_COUT * (9 * 64 / 8); i += blockDim.x) {
        const int o = i / (9 * 64 / 8), v8 = i - o * (9 * 64 / 8);
        *reinterpret_cast<uint4*>(wsm + o * C2_WROW + v8 * 8) =
            *reinterpret_cast<const uint4*>(w2p + static_cast<size_t>(o) * 9 * 64 + v8 * 8);
    }
}

// The implicit GEMM over patch [C2_PROWS][F1 + 2][CELL] and wsm [32][C2_WROW]: warp w computes GEMM rows 16 w .. 16 w + 15
// (row r = frame r / F2, pixel r % F2) and stores them + bias into cbuf [C2_FRAMES * F2][C2_LD].
__device__ __forceinline__ void conv2_gemm(const __half* patch, const __half* wsm, int F1, int F2, const float* __restrict__ b2,
                                           float* cbuf, int warp, int lane) {
    const int FPAD = F1 + 2, rows = C2_FRAMES * F2;
    const int g = lane >> 2, c = lane & 3;
    const int r0 = warp * 16 + g, r1 = r0 + 8;
    if (warp * 16 >= rows) return;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    const int rr0 = min(r0, rows - 1), rr1 = min(r1, rows - 1);
    const int fr0 = rr0 / F2, f20 = rr0 - fr0 * F2;
    const int fr1 = rr1 / F2, f21 = rr1 - fr1 * F2;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
        const int kf = tap / 3, kt = tap - kf * 3;
        const __half* a0p = patch + ((2 * fr0 + kt) * FPAD + 2 * f20 + kf) * CELL + 2 * c;
        const __half* a1p = patch + ((2 * fr1 + kt) * FPAD + 2 * f21 + kf) * CELL + 2 * c;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            uint32_t a[4];
            a[0] = *reinterpret_cast<const uint32_t*>(a0p + ks * 16);
            a[1] = *reinterpret_cast<const uint32_t*>(a1p + ks * 16);
            a[2] = *reinterpret_cast<const uint32_t*>(a0p + ks * 16 + 8);
            a[3] = *reinterpret_cast<const uint32_t*>(a1p + ks * 16 + 8);
            const int kk = tap * 64 + ks * 16 + 2 * c;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const __half* wp = wsm + (nt * 8 + g) * C2_WROW + kk;
                mma16816(acc[nt], a, *reinterpret_cast<const uint32_t*>(wp), *reinterpret_cast<const uint32_t*>(wp + 8));
            }
        }
    }
    conv_tile_store<4, C2_LD>(acc, b2, cbuf, r0, r1, rows, c);
}

// LayerNorm over (F2, 32) + LeakyReLU of output frame t0 + warp (one warp per frame) from cbuf -> out
__device__ __forceinline__ void conv2_ln_store(const float* cbuf, int b, int t0, int T2, int F2, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, __half* __restrict__ out_h,
                                               float* __restrict__ out_f, int warp, int lane) {
    if (warp >= C2_FRAMES) return;
    const int t = t0 + warp;
    if (t >= T2) return;
    const int n = F2 * C2_COUT;
    const float* src = cbuf + warp * F2 * C2_LD;
    float mean, rstd;
    frame_ln_stats<C2_COUT>(src, C2_LD, n, lane, mean, rstd);
    const size_t ob = (static_cast<size_t>(b) * T2 + t) * n;
    for (int i = lane; i < n; i += 32) {
        const float y = leaky((src[(i >> 5) * C2_LD + (i & 31)] - mean) * rstd * __ldg(gamma + i) + __ldg(beta + i));
        out_h[ob + i] = float2half_sat(y);
        if (out_f) out_f[ob + i] = y;
    }
}

// Requires F2 * C2_FRAMES <= 16 * n_warps (launch with ceil(F2*4/16) warps) and F2 * 32 <= 1024.
__global__ void __launch_bounds__(192)
conv2_ln_kernel(const __half* __restrict__ act1, int T1, int F1, int T2, int F2, const __half* __restrict__ w2p,
                const float* __restrict__ b2, const float* __restrict__ gamma, const float* __restrict__ beta,
                __half* __restrict__ out_h, float* __restrict__ out_f) {
    extern __shared__ __align__(16) uint8_t c2_smem[];
    __half* patch = reinterpret_cast<__half*>(c2_smem);                 // [C2_PROWS][F1 + 2][CELL]
    __half* wsm = patch + C2_PROWS * (F1 + 2) * CELL;                   // [32][C2_WROW]
    float* cbuf = reinterpret_cast<float*>(wsm + C2_COUT * C2_WROW);    // [C2_FRAMES * F2][C2_LD]
    const int b = blockIdx.y, t0 = blockIdx.x * C2_FRAMES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    stage_patch<3, C2_PROWS>(patch, act1, b, t0, T1, F1);
    conv2_stage_weights(wsm, w2p);
    __syncthreads();
    conv2_gemm(patch, wsm, F1, F2, b2, cbuf, warp, lane);
    __syncthreads();
    conv2_ln_store(cbuf, b, t0, T2, F2, gamma, beta, out_h, out_f, warp, lane);
}

// --------------------------------------------------------------------------- conv1 + conv2 fused
// The two-kernel version writes conv1's output (B x T1 x F1 x 64 fp16 = 82 MB per 32 x 10 s batch) to global memory and
// reads it back: conv2 is bound by those 82 MB of DRAM reads at low occupancy.
// Here one CTA produces C2_FRAMES output frames from the input features directly: its 9 warps each compute one conv1 frame
// (3x3 conv, LayerNorm over (F1, 64), LeakyReLU) with the frame held in registers, and write it -- fp16, reflect columns
// included -- straight into the shared-memory patch the implicit-GEMM conv2 reads.  Global traffic per batch: the 10 MB of
// features (re-read ~2.3x through L2) + the 10 MB output instead of 2 x 82 MB.  Same stage code as the two kernels, so the
// results are bit-identical to them.
constexpr int CF_WARPS = C2_PROWS;  // one per conv1 frame of the patch

template <int MAXF>
__global__ void __launch_bounds__(CF_WARPS * 32, 2)
cnn_fused_kernel(const float* __restrict__ feats, int T0, int F0, int T1, int F1, int T2, int F2, const float* __restrict__ w1,
                 const float* __restrict__ b1, const float* __restrict__ g1, const float* __restrict__ be1,
                 const __half* __restrict__ w2p, const float* __restrict__ b2, const float* __restrict__ g2,
                 const float* __restrict__ be2, __half* __restrict__ out_h, float* __restrict__ out_f) {
    extern __shared__ __align__(16) uint8_t c2_smem[];
    const int FPAD = F1 + 2;
    __half* patch = reinterpret_cast<__half*>(c2_smem);                 // [C2_PROWS][FPAD][CELL]
    __half* wsm = patch + C2_PROWS * FPAD * CELL;                       // [32][C2_WROW]
    float* cbuf = reinterpret_cast<float*>(wsm + C2_COUT * C2_WROW);    // [C2_FRAMES * F2][C2_LD]
    float* in_all = cbuf + C2_FRAMES * F2 * C2_LD;                      // [CF_WARPS][3][F0 + 2]
    const int b = blockIdx.y, t0 = blockIdx.x * C2_FRAMES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    conv2_stage_weights(wsm, w2p);  // independent of everything else: issued first
    // ---- stage 1: warp `warp` computes conv1 frame t1 = reflect(2 t0 + warp - 1) into patch row `warp`
    {
        int t1 = reflect_idx(2 * t0 + warp - 1, T1);
        t1 = min(max(t1, 0), T1 - 1);  // tail tiles: keep loads in range (results discarded)
        float va[MAXF], vb[MAXF], mean, rstd;
        conv1_warp_frame<3>(in_all + warp * 3 * (F0 + 2), feats, b, t1, T0, F0, F1, w1, b1, lane, va, vb, mean, rstd);
        const int c0 = 2 * lane;
        __half* prow = patch + static_cast<size_t>(warp) * FPAD * CELL;
#pragma unroll
        for (int f1 = 0; f1 < MAXF; ++f1)
            if (f1 < F1) {
                const __half2 y = conv1_ln_pair(va[f1], vb[f1], mean, rstd, g1, be1, f1 * 64 + c0);
                *reinterpret_cast<__half2*>(prow + (f1 + 1) * CELL + c0) = y;
                // reflect padding of the feature axis: column -1 mirrors f1 = 1, column F1 mirrors f1 = F1 - 2
                if (f1 == 1) *reinterpret_cast<__half2*>(prow + c0) = y;
                if (f1 == F1 - 2) *reinterpret_cast<__half2*>(prow + (F1 + 1) * CELL + c0) = y;
            }
    }
    __syncthreads();
    // ---- stage 2: conv2 as an implicit GEMM over the patch, then the per-frame LayerNorm
    conv2_gemm(patch, wsm, F1, F2, b2, cbuf, warp, lane);
    __syncthreads();
    conv2_ln_store(cbuf, b, t0, T2, F2, g2, be2, out_h, out_f, warp, lane);
}

// =========================================================================== 256-channel 2-block front-end (AISHELL-1)
// ConvolutionFrontEnd(num_blocks=2, out_channels=(256, 256)), otherwise the blocks above:
//   conv1 (1 -> 256): one CTA per output frame, LayerNorm over (F1, 256) with block reductions -> act1 [B, T1, F1, 256] fp16
//   conv2 (256 -> 256): implicit GEMM, M = B * T2 * F2 pixels, N = 256, K = 9 * 256 = 2304 (k = tap * 256 + ch), on wgmma.
// conv2's weights (1.18 MB) cannot stay in shared memory: they stream through a ring of 64-wide k-blocks, each one bulk
// copy of an image packed at load time in the 128B-swizzled layout wgmma reads.  The A rows are gathered from act1 by a
// producer warp with cp.async (TMA cannot reflect at the time and feature edges).  A CTA owns W2_BM = 128 GEMM rows =
// the 128 / F2 whole frames they hold (6 at 80 mels, 120 rows), so the epilogue normalises each frame from the fp32
// accumulator tile in shared memory: bias, LayerNorm over (F2, 256) and LeakyReLU, with no second pass over HBM.
constexpr int W1_THREADS = 128;            // conv1: two channels per thread
constexpr int W_C = 256;                   // channels of both blocks
constexpr int W2_BK = 64;                  // k-block: 64 input channels of one tap
constexpr int W2_KB = 9 * W_C / W2_BK;     // 36 k-blocks
constexpr int W2_BM = 128;                 // GEMM rows per CTA: two consumer warpgroups of 64
constexpr int W2_STAGES = 4;
constexpr int W2_LAG = 2;                  // k-blocks of A rows the producer keeps in flight before it marks one full
constexpr int W2_A_BYTES = W2_BM * W2_BK * 2;
constexpr int W2_B_BYTES = W_C * W2_BK * 2;
constexpr int W2_STAGE_BYTES = W2_A_BYTES + W2_B_BYTES;
constexpr int W2_BAR_OFFSET = W2_STAGES * W2_STAGE_BYTES;
constexpr int W2_SMEM = W2_BAR_OFFSET + 2 * W2_STAGES * 8 + 1024;  // + alignment slack
constexpr int W2_STG_PITCH = W_C * 4 + 16;  // fp32 accumulator row in the epilogue
constexpr int W2_CONSUMERS = 2 * 128;
constexpr int W2_THREADS = W2_CONSUMERS + 32;
static_assert(W2_STAGE_BYTES % 1024 == 0 && W2_BM * W2_STG_PITCH <= W2_BAR_OFFSET, "ring layout");
static_assert(W2_LAG <= W2_STAGES - 2, "the producer must mark stage kb full before it waits for stage kb + 2 to drain");

// w1: [256, 3(kf), 3(kt)] fp32, g/be: [F1, 256].  The conv1 stage above, with the LayerNorm sums reduced over 4 warps.
template <int MAXF>
__global__ void __launch_bounds__(W1_THREADS)
conv1c256_ln_kernel(const float* __restrict__ feats, int T0, int F0, int T1, int F1, const float* __restrict__ w1,
                    const float* __restrict__ b1, const float* __restrict__ gamma, const float* __restrict__ beta,
                    __half* __restrict__ out_h) {
    extern __shared__ float w1_in[];  // [3][F0 + 2] of the frame (reflect padded)
    __shared__ float red[2][W1_THREADS / 32];
    const int t1 = blockIdx.x, b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    conv1_stage_rows<3>(w1_in, feats, b, t1, T0, F0, threadIdx.x, W1_THREADS);
    const int c0 = 2 * threadIdx.x;
    const Conv1Taps<3> w = conv1_taps<3>(w1, b1, c0);
    __syncthreads();
    float va[MAXF], vb[MAXF];
    const float n = static_cast<float>(F1 * W_C);
    const float s = warp_sum(conv1_frame<3>(w1_in, F0, F1, w, va, vb));
    if (lane == 0) red[0][warp] = s;
    __syncthreads();
    const float mean = (red[0][0] + red[0][1] + red[0][2] + red[0][3]) / n;
    const float q = warp_sum(conv1_centred_sq(va, vb, F1, mean));
    if (lane == 0) red[1][warp] = q;
    __syncthreads();
    const float rstd = rsqrtf((red[1][0] + red[1][1] + red[1][2] + red[1][3]) / n + 1e-5f);
    const size_t obase = (static_cast<size_t>(b) * T1 + t1) * F1 * W_C;
#pragma unroll
    for (int f1 = 0; f1 < MAXF; ++f1)
        if (f1 < F1) {
            const int gi = f1 * W_C + c0;
            *reinterpret_cast<__half2*>(out_h + obase + gi) = conv1_ln_pair(va[f1], vb[f1], mean, rstd, gamma, beta, gi);
        }
}

// act1 [B, T1, F1, 256] fp16; w2s: W2_KB k-blocks of [256 out][64 k] fp16, each the 128B-swizzled image a stage holds
// (k = (kf * 3 + kt) * 256 + ch); frames = W2_BM / F2 output frames per CTA; out [B, T2, F2 * 256].
__global__ void __launch_bounds__(W2_THREADS, 1)
conv2c256_ln_kernel(const __half* __restrict__ act1, int T1, int F1, int T2, int F2, int frames,
                    const __half* __restrict__ w2s, const float* __restrict__ b2, const float* __restrict__ gamma,
                    const float* __restrict__ beta, __half* __restrict__ out_h, float* __restrict__ out_f) {
    extern __shared__ uint8_t w2_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(w2_smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + W2_BAR_OFFSET);
    uint64_t* empty_bar = full_bar + W2_STAGES;
    const int b = blockIdx.y, t0 = blockIdx.x * frames, rows = frames * F2;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < W2_STAGES; ++s) {
            mbar_init(&full_bar[s], 1 + 32);  // the weight copy's expect_tx arrive + one arrive per producer lane
            mbar_init(&empty_bar[s], 2);      // one arrive per consumer warpgroup
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (threadIdx.x >= W2_CONSUMERS) {
        // ---- producer warp: lane l gathers GEMM rows l, l + 32, l + 64, l + 96 (8 x 16-byte chunks each per k-block)
        int t2r[W2_BM / 32], f2r[W2_BM / 32];
#pragma unroll
        for (int j = 0; j < W2_BM / 32; ++j) {
            const int r = lane + 32 * j, fr = r / F2;
            t2r[j] = min(t0 + fr, T2 - 1);  // tail frames: keep loads in range (results discarded)
            f2r[j] = r - fr * F2;
        }
        const __half* act1_b = act1 + static_cast<size_t>(b) * T1 * F1 * W_C;
        for (int kb = 0; kb < W2_KB; ++kb) {
            const int s = kb % W2_STAGES;
            if (kb >= W2_STAGES) mbar_wait(&empty_bar[s], ((kb / W2_STAGES) & 1) ^ 1);
            uint8_t* stage = smem + s * W2_STAGE_BYTES;
            if (lane == 0) {
                mbar_arrive_expect_tx(&full_bar[s], W2_B_BYTES);
                bulk_load_1d(stage + W2_A_BYTES, w2s + static_cast<size_t>(kb) * W_C * W2_BK, W2_B_BYTES, &full_bar[s]);
            }
            const int tap = kb / (W_C / W2_BK), kf = tap / 3, kt = tap - 3 * kf;
            const int ch0 = (kb - tap * (W_C / W2_BK)) * W2_BK;
            const uint32_t a_base = smem_u32(stage);
#pragma unroll
            for (int j = 0; j < W2_BM / 32; ++j) {
                const int r = lane + 32 * j;
                if (r < rows) {  // rows past the last whole frame stay unwritten: their outputs are never read
                    const int t1 = reflect_idx(2 * t2r[j] + kt - 1, T1), f1 = reflect_idx(2 * f2r[j] + kf - 1, F1);
                    const __half* src = act1_b + (static_cast<size_t>(t1) * F1 + f1) * W_C + ch0;
                    const uint32_t dst = a_base + r * 128;
#pragma unroll
                    for (int c = 0; c < 8; ++c) cp_async16(dst + ((c ^ (r & 7)) << 4), src + c * 8);
                }
            }
            cp_async_commit();
            if (kb >= W2_LAG) {
                cp_async_wait<W2_LAG>();
                fence_proxy_async_smem();
                mbar_arrive(&full_bar[(kb - W2_LAG) % W2_STAGES]);
            }
        }
        cp_async_wait<0>();
        fence_proxy_async_smem();
        for (int kb = W2_KB - W2_LAG; kb < W2_KB; ++kb) mbar_arrive(&full_bar[kb % W2_STAGES]);
        return;
    }

    // ---- consumers: warpgroup g computes rows 64 g .. 64 g + 63 x all 256 columns (two n128 wgmma per k16 step)
    const int wg = threadIdx.x >> 7;
    float acc[2][64];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[i][j] = 0.0f;
    for (int kb = 0; kb < W2_KB; ++kb) {
        const int s = kb % W2_STAGES;
        mbar_wait(&full_bar[s], (kb / W2_STAGES) & 1);
        const uint32_t a_addr = smem_u32(smem + s * W2_STAGE_BYTES) + wg * 64 * 128;
        const uint32_t b_addr = smem_u32(smem + s * W2_STAGE_BYTES) + W2_A_BYTES;
        const uint64_t da = make_kmajor_sw128_desc(a_addr);
        const uint64_t db0 = make_kmajor_sw128_desc(b_addr), db1 = make_kmajor_sw128_desc(b_addr + 128 * 128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < W2_BK / 16; ++k) {  // +32 B per k16 step -> +2 in (addr >> 4)
            wgmma_f16<128>(acc[0], da + 2 * k, db0 + 2 * k, 1u);
            wgmma_f16<128>(acc[1], da + 2 * k, db1 + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(kb - 1) % W2_STAGES]);
    }
    wgmma_wait<0>();
    asm volatile("bar.sync 1, %0;" ::"n"(W2_CONSUMERS) : "memory");  // both warpgroups are done reading the ring
    {
        const int w = (threadIdx.x >> 5) & 3;
        uint8_t* base = smem + (wg * 64 + w * 16 + (lane >> 2)) * W2_STG_PITCH + (lane & 3) * 8;
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = i * 128 + j * 8 + 2 * (lane & 3);
                const float bz0 = __ldg(b2 + col), bz1 = __ldg(b2 + col + 1);
                *reinterpret_cast<float2*>(base + (i * 128 + j * 8) * 4) =
                    make_float2(acc[i][4 * j] + bz0, acc[i][4 * j + 1] + bz1);
                *reinterpret_cast<float2*>(base + 8 * W2_STG_PITCH + (i * 128 + j * 8) * 4) =
                    make_float2(acc[i][4 * j + 2] + bz0, acc[i][4 * j + 3] + bz1);
            }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(W2_CONSUMERS) : "memory");
    // LayerNorm over (F2, 256) per frame + LeakyReLU; one warp per frame, lane l owns columns 4 l .. 4 l + 3 and 128 + 4 l ..
    const int warp = threadIdx.x >> 5;
    const int n = F2 * W_C;
    const uint32_t stg = smem_u32(smem);
    for (int fr = warp; fr < frames; fr += W2_CONSUMERS / 32) {
        const int t = t0 + fr;
        if (t >= T2) break;
        const uint32_t fbase = stg + fr * F2 * W2_STG_PITCH + lane * 16;
        float s = 0.0f;
        for (int r = 0; r < F2; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float4 v = u4_as_f4(lds128(fbase + r * W2_STG_PITCH + h * 512));
                s += (v.x + v.y) + (v.z + v.w);
            }
        const float mean = warp_sum(s) / n;
        float q = 0.0f;
        for (int r = 0; r < F2; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float4 v = u4_as_f4(lds128(fbase + r * W2_STG_PITCH + h * 512));
                const float d0 = v.x - mean, d1 = v.y - mean, d2 = v.z - mean, d3 = v.w - mean;
                q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
            }
        const float rstd = rsqrtf(warp_sum(q) / n + 1e-5f);
        const size_t ob = (static_cast<size_t>(b) * T2 + t) * n;
        for (int r = 0; r < F2; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = r * W_C + h * 128 + 4 * lane;
                const float4 v = u4_as_f4(lds128(fbase + r * W2_STG_PITCH + h * 512));
                const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + i));
                const float4 be = __ldg(reinterpret_cast<const float4*>(beta + i));
                const float4 y = make_float4(leaky((v.x - mean) * rstd * g.x + be.x), leaky((v.y - mean) * rstd * g.y + be.y),
                                             leaky((v.z - mean) * rstd * g.z + be.z), leaky((v.w - mean) * rstd * g.w + be.w));
                const __half2 lo = floats2half2_sat(y.x, y.y), hi = floats2half2_sat(y.z, y.w);
                *reinterpret_cast<uint2*>(out_h + ob + i) =
                    make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
                if (out_f) *reinterpret_cast<float4*>(out_f + ob + i) = y;
            }
    }
}

// =========================================================================== 3-block front-end (Transformer recipes)
// ConvolutionFrontEnd(num_blocks=3, num_layers_per_block=1, out_channels=(64, 64, 64), kernel_sizes=(5, 5, 1),
// strides=(2, 2, 1), residuals=(False, False, True)):
//   block 1: reflect-pad 2 + Conv2d(5x5, 1 -> 64, stride 2) + LayerNorm(F1, 64) + LeakyReLU      -> act1 fp16
//            (conv1k5_ln_kernel, above)
//   block 2: reflect-pad 2 + Conv2d(5x5, 64 -> 64, stride 2) + LayerNorm(F2, 64) + LeakyReLU     -> y (fp32, in smem)
//   block 3: LeakyReLU(LayerNorm(Conv2d_1x1(y))) + LayerNorm(Conv2d_1x1 reduce_conv(y))          -> out [B, T2, F2*64]
// Blocks 2 and 3 are one kernel: block 3 is per-pixel work plus a per-frame LayerNorm, so it runs on block 2's
// LayerNorm output while that is still in shared memory, and only the 1280-wide row the input Linear reads is written.
constexpr int K5_C = 64;                   // channels of every block
constexpr int K5_FRAMES = 4;               // block-2 output frames per CTA
constexpr int K5_WARPS = 5;                // 16 GEMM rows per warp: K5_FRAMES * F2 <= 80
constexpr int K5_PROWS = 2 * K5_FRAMES + 3;  // act1 frames a CTA's patch holds
constexpr int K5_WROW = 5 * K5_C + 8;      // padded weight row (halfs) of one kf slice: k = kt * 64 + ch
constexpr int K5_YS = K5_C + 1;            // fp32 row stride of y
constexpr int K5_ZS = 2 * K5_C + 1;        // fp32 row stride of the two block-3 convolutions

// Bytes of the shared-memory region block 2 (patch + weight slice) and then block 3 (w3 + z) use.
__host__ __device__ __forceinline__ size_t k5_shared_region(int F1, int F2) {
    const size_t gemm = static_cast<size_t>(K5_PROWS) * (F1 + 4) * CELL * 2 + K5_C * K5_WROW * 2;
    const size_t blk3 = (2ull * K5_C * K5_YS + static_cast<size_t>(K5_FRAMES) * F2 * K5_ZS) * 4;
    return ((gemm > blk3 ? gemm : blk3) + 15) & ~size_t(15);
}

// blocks 2 + 3.  act1 [B, T1, F1, 64] fp16; w2p [64, 1600] fp16 with k = (kf * 5 + kt) * 64 + ch; w3 [128, 64] fp32 rows
// = [convs.conv_0 | reduce_conv.conv] output channels, b3 [128]; g2/be2, g3/be3, gr/ber: [F2, 64].
// Block 2 is an implicit GEMM (M = K5_FRAMES * F2 pixels, N = 64, K = 1600) on mma.sync.m16n8k16 with fp16 operands and
// fp32 accumulation; the weight slice of one kf (64 x 320) is staged per pass.  Block 3 runs in fp32.
__global__ void __launch_bounds__(K5_WARPS * 32)
cnn3_block23_kernel(const __half* __restrict__ act1, int T1, int F1, int T2, int F2, const __half* __restrict__ w2p,
                    const float* __restrict__ b2, const float* __restrict__ g2, const float* __restrict__ be2,
                    const float* __restrict__ w3, const float* __restrict__ b3, const float* __restrict__ g3,
                    const float* __restrict__ be3, const float* __restrict__ gr, const float* __restrict__ ber,
                    __half* __restrict__ out_h, float* __restrict__ out_f) {
    extern __shared__ __align__(16) uint8_t k5_smem[];
    const int FPAD = F1 + 4;
    __half* patch = reinterpret_cast<__half*>(k5_smem);              // [K5_PROWS][FPAD][CELL]
    __half* wsm = patch + K5_PROWS * FPAD * CELL;                     // [64][K5_WROW]
    // after block 2 the patch / weight region is free: block 3's weights and outputs reuse it
    float* w3s = reinterpret_cast<float*>(k5_smem);                   // [128][K5_YS]
    float* zs = w3s + 2 * K5_C * K5_YS;                               // [rows][K5_ZS]
    const int rows = K5_FRAMES * F2;
    float* ys = reinterpret_cast<float*>(k5_smem + k5_shared_region(F1, F2));  // [rows][K5_YS], behind both
    const int b = blockIdx.y, t0 = blockIdx.x * K5_FRAMES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    stage_patch<5, K5_PROWS>(patch, act1, b, t0, T1, F1);
    const int g = lane >> 2, c = lane & 3;
    const int r0 = warp * 16 + g, r1 = r0 + 8;
    const int rr0 = min(r0, rows - 1), rr1 = min(r1, rows - 1);
    const int fr0 = rr0 / F2, f20 = rr0 - fr0 * F2;
    const int fr1 = rr1 / F2, f21 = rr1 - fr1 * F2;
    const bool active = warp * 16 < rows;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.0f;
#pragma unroll 1
    for (int kf = 0; kf < 5; ++kf) {
        __syncthreads();  // the previous slice is consumed (kf == 0: nothing to wait for but the patch)
        for (int i = threadIdx.x; i < K5_C * (5 * K5_C / 8); i += blockDim.x) {
            const int o = i / (5 * K5_C / 8), v8 = i - o * (5 * K5_C / 8);
            *reinterpret_cast<uint4*>(wsm + o * K5_WROW + v8 * 8) =
                *reinterpret_cast<const uint4*>(w2p + static_cast<size_t>(o) * 25 * K5_C + kf * 5 * K5_C + v8 * 8);
        }
        __syncthreads();
        if (active) {
#pragma unroll  // a rolled kt loop inside the rolled kf loop kept one loop counter in local memory (8-byte spill)
            for (int kt = 0; kt < 5; ++kt) {
                const __half* a0p = patch + ((2 * fr0 + kt) * FPAD + 2 * f20 + kf) * CELL + 2 * c;
                const __half* a1p = patch + ((2 * fr1 + kt) * FPAD + 2 * f21 + kf) * CELL + 2 * c;
#pragma unroll
                for (int ks = 0; ks < K5_C / 16; ++ks) {
                    uint32_t a[4];
                    a[0] = *reinterpret_cast<const uint32_t*>(a0p + ks * 16);
                    a[1] = *reinterpret_cast<const uint32_t*>(a1p + ks * 16);
                    a[2] = *reinterpret_cast<const uint32_t*>(a0p + ks * 16 + 8);
                    a[3] = *reinterpret_cast<const uint32_t*>(a1p + ks * 16 + 8);
                    const int kk = kt * K5_C + ks * 16 + 2 * c;
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) {
                        const __half* wp = wsm + (nt * 8 + g) * K5_WROW + kk;
                        mma16816(acc[nt], a, *reinterpret_cast<const uint32_t*>(wp),
                                 *reinterpret_cast<const uint32_t*>(wp + 8));
                    }
                }
            }
        }
    }
    if (active) conv_tile_store<8, K5_YS>(acc, b2, ys, r0, r1, rows, c);
    __syncthreads();
    // block 2's LayerNorm + LeakyReLU in place (one warp per frame); block 3's weights into the freed region
    for (int i = threadIdx.x; i < 2 * K5_C * K5_C; i += blockDim.x) w3s[(i >> 6) * K5_YS + (i & 63)] = __ldg(w3 + i);
    const int n = F2 * K5_C;
    if (warp < K5_FRAMES) {
        float* src = ys + warp * F2 * K5_YS;
        float mean, rstd;
        frame_ln_stats<K5_C>(src, K5_YS, n, lane, mean, rstd);
        for (int i = lane; i < n; i += 32) {
            float& v = src[(i >> 6) * K5_YS + (i & 63)];
            v = leaky((v - mean) * rstd * __ldg(g2 + i) + __ldg(be2 + i));
        }
    }
    __syncthreads();
    // block 3's two 1x1 convolutions: z[r][0:64] = convs.conv_0(y[r]), z[r][64:128] = reduce_conv.conv(y[r])
    for (int i = threadIdx.x; i < rows * 2 * K5_C; i += blockDim.x) {
        const int r = i >> 7, o = i & 127;
        const float* yr = ys + r * K5_YS;
        const float* wr = w3s + o * K5_YS;
        float z = __ldg(b3 + o);
#pragma unroll 8
        for (int k = 0; k < K5_C; ++k) z = fmaf(wr[k], yr[k], z);
        zs[r * K5_ZS + o] = z;
    }
    __syncthreads();
    if (warp < K5_FRAMES) {
        const int t = t0 + warp;
        if (t < T2) {
            const float* src = zs + warp * F2 * K5_ZS;
            float ma, ra, mr, rr;
            frame_ln_stats<K5_C>(src, K5_ZS, n, lane, ma, ra);
            frame_ln_stats<K5_C>(src + K5_C, K5_ZS, n, lane, mr, rr);
            const size_t ob = (static_cast<size_t>(b) * T2 + t) * n;
            for (int i = lane; i < n; i += 32) {
                const float* zr = src + (i >> 6) * K5_ZS + (i & 63);
                const float y = leaky((zr[0] - ma) * ra * __ldg(g3 + i) + __ldg(be3 + i)) +
                                ((zr[K5_C] - mr) * rr * __ldg(gr + i) + __ldg(ber + i));
                out_h[ob + i] = float2half_sat(y);
                if (out_f) out_f[ob + i] = y;
            }
        }
    }
}

// =========================================================================== entry point
int cnn_frontend_forward(const float* feats, int B, int T0, int F0, const CnnWeights& w, __half* act1_h, __half* out_h,
                         float* out_f, cudaStream_t stream) {
    const int T1 = (T0 - 1) / 2 + 1, F1 = (F0 - 1) / 2 + 1;
    const int T2 = (T1 - 1) / 2 + 1, F2 = (F1 - 1) / 2 + 1;
    if (w.blocks == 3) {
        // the reference's reflect padding of 2 needs 3 rows / columns at both strided convolutions
        SBK_REQUIRE(T1 >= 3 && F1 >= 3, "cnn_frontend: the 5x5 reflect padding needs at least 5 frames and 5 features "
                    "(got %d frames, %d features)", T0, F0);
        SBK_REQUIRE(F1 <= 64 && K5_FRAMES * F2 <= 16 * K5_WARPS, "cnn_frontend: feature dim too large (F0=%d)", F0);
        conv1k5_ln_kernel<64><<<dim3(ceil_div(T1, C1_WARPS), B), C1_WARPS * 32, C1_WARPS * 5 * (F0 + 4) * sizeof(float),
                                stream>>>(feats, T0, F0, T1, F1, w.w1, w.b1, w.g1, w.be1, act1_h);
        SBK_LAUNCH_CHECK();
        const size_t smem = k5_shared_region(F1, F2) + static_cast<size_t>(K5_FRAMES) * F2 * K5_YS * 4;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(cnn3_block23_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        cnn3_block23_kernel<<<dim3(ceil_div(T2, K5_FRAMES), B), K5_WARPS * 32, smem, stream>>>(
            act1_h, T1, F1, T2, F2, w.w2, w.b2, w.g2, w.be2, w.w3, w.b3, w.g3, w.be3, w.gr, w.ber, out_h, out_f);
        SBK_LAUNCH_CHECK();
        return SBK_OK;
    }
    if (w.c1 == W_C && w.c2 == W_C) {
        // the reference's reflect padding of 1 needs 2 rows / columns at both strided convolutions
        SBK_REQUIRE(T0 >= 3 && F0 >= 3, "cnn_frontend: the 3x3 reflect padding needs at least 3 frames and 3 features "
                    "(got %d frames, %d features)", T0, F0);
        SBK_REQUIRE(F1 <= 40, "cnn_frontend: out_channels=(256, 256) is built for up to 80 features (F0=%d)", F0);
        conv1c256_ln_kernel<40><<<dim3(T1, B), W1_THREADS, 3 * (F0 + 2) * sizeof(float), stream>>>(
            feats, T0, F0, T1, F1, w.w1, w.b1, w.g1, w.be1, act1_h);
        SBK_LAUNCH_CHECK();
        const int frames = W2_BM / F2;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(conv2c256_ln_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W2_SMEM));
        conv2c256_ln_kernel<<<dim3(ceil_div(T2, frames), B), W2_THREADS, W2_SMEM, stream>>>(
            act1_h, T1, F1, T2, F2, frames, w.w2, w.b2, w.g2, w.be2, out_h, out_f);
        SBK_LAUNCH_CHECK();
        return SBK_OK;
    }
    SBK_REQUIRE(w.c1 == 64 && w.c2 == 32, "cnn_frontend: only out_channels=(64, 32) and (256, 256) are built (got %d, %d)",
                w.c1, w.c2);
    SBK_REQUIRE(T0 >= 2 && F0 >= 2, "cnn_frontend: input too small for reflect padding");
    SBK_REQUIRE(F1 <= 64 && F2 * C2_FRAMES <= 96, "cnn_frontend: feature dim too large (F0=%d)", F0);
    // patch + weights + cbuf, the shared memory of both (64, 32) conv2 kernels
    const size_t c2_smem = static_cast<size_t>(C2_PROWS) * (F1 + 2) * CELL * 2 + C2_COUT * C2_WROW * 2 +
                           static_cast<size_t>(C2_FRAMES) * F2 * C2_LD * 4;
    // the fused kernel (conv1 output never leaves the SM) for 3 <= F1 <= 40: it holds a conv1 frame in 40 registers per lane
    // and writes the reflect columns itself.  The two-kernel version otherwise (n_mels > 80, or n_mels <= 4).
    if (F1 <= 40 && F1 >= 3 && C2_FRAMES * F2 <= 16 * CF_WARPS) {
        const size_t smem = c2_smem + static_cast<size_t>(CF_WARPS) * 3 * (F0 + 2) * 4;
        SBK_CUDA_CHECK(cudaFuncSetAttribute(cnn_fused_kernel<40>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        cnn_fused_kernel<40><<<dim3(ceil_div(T2, C2_FRAMES), B), CF_WARPS * 32, smem, stream>>>(
            feats, T0, F0, T1, F1, T2, F2, w.w1, w.b1, w.g1, w.be1, w.w2, w.b2, w.g2, w.be2, out_h, out_f);
        SBK_LAUNCH_CHECK();
        return SBK_OK;
    }
    conv1_ln_kernel<64, 64><<<dim3(ceil_div(T1, C1_WARPS), B), C1_WARPS * 32, C1_WARPS * 3 * (F0 + 2) * sizeof(float),
                              stream>>>(feats, T0, F0, T1, F1, w.w1, w.b1, w.g1, w.be1, act1_h);
    SBK_LAUNCH_CHECK();
    SBK_CUDA_CHECK(cudaFuncSetAttribute(conv2_ln_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c2_smem));
    const int warps = std::max(C2_FRAMES, ceil_div(C2_FRAMES * F2, 16));
    conv2_ln_kernel<<<dim3(ceil_div(T2, C2_FRAMES), B), warps * 32, c2_smem, stream>>>(act1_h, T1, F1, T2, F2, w.w2, w.b2,
                                                                                        w.g2, w.be2, out_h, out_f);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // namespace sbk
