// Fused Fbank: framing + window + FFT + power + mel + dB in ONE kernel per tile of frames,
// followed by a tiny per-utterance top_db clip (+ optional fused global CMVN).
//
// Replaces (reference file:line, relative to speechbrain/):
//   processing/features.py:141-188  STFT.forward (torch.stft, center=True, zero pad, periodic hamming)
//   processing/features.py:341-378  spectral_magnitude (power spectrum)
//   processing/features.py:512-586  Filterbank.forward (triangular mel matmul)
//   processing/features.py:736-759  _amplitude_to_DB (10*log10(clamp), per-sequence top_db clip)
//   processing/features.py:1404-1455 InputNormalization.forward ("global" / "sentence", eval)
//
// Layout: wav [B, L] fp32 -> out [B, T_f, n_mels] fp32.  HBM-bound: 4*L + 4*T_f*n_mels bytes per utterance.
//
// Kernel 1 (fbank_tile_kernel): one CTA per (utterance, tile of FB_FRAMES frames).
//   * the zero-padded wav segment is staged into shared memory by TMA (2-D tensor map over
//     [B, L]; negative / past-the-end coordinates are zero-filled by the hardware, which is
//     exactly torch.stft's center=True constant padding) -- or by guarded loads if L % 4 != 0;
//   * two real frames are packed into one complex sequence; mixed-radix (8/4/2/5/3) Stockham
//     FFT in shared memory; the pair is separated with the conjugate-symmetry identity;
//   * sparse triangular mel (each filter touches a short band of bins), 10*log10, store, and a
//     block-reduced atomicMax of the per-utterance maximum (ordered-int encoding).
// Kernel 2 (fbank_finalize_kernel): x = max(x, max_b - top_db) [, (x - mean) / max(std, eps)].
#include <math.h>
#include <string.h>

#include <algorithm>

#include <vector>

#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

constexpr int FB_MAX_PASSES = 12;
constexpr int FB_THREADS = 256;
// frames per CTA (packed two per complex FFT): 8 frames = 42 KB of shared memory = 4-5 CTAs per SM hide the kernel's many
// short barrier-separated phases better than 16 frames = 80 KB = 2 CTAs per SM
constexpr int FB_FRAMES = 8;

struct FbankDev {
    int n_fft, hop, n_stft, n_mels, max_band;
    int n_pass;
    int radix[FB_MAX_PASSES];
    float amin, top_db;
    const float* window;    // [n_fft]
    const float2* twiddle;  // [n_fft] exp(-2*pi*i*k/n_fft)
    const int* band_start;  // [n_mels]
    const int* band_len;    // [n_mels]
    const float* band_w;    // [n_mels, max_band]
};

struct Fbank {
    FbankDev d;
    void* arena = nullptr;
};

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

template <int R>
__device__ __forceinline__ void dft_small(float2 (&v)[R], const float2* __restrict__ tw, int n_fft) {
    if constexpr (R == 2) {
        const float2 a = v[0], b = v[1];
        v[0] = make_float2(a.x + b.x, a.y + b.y);
        v[1] = make_float2(a.x - b.x, a.y - b.y);
    } else if constexpr (R == 4) {
        const float2 a = make_float2(v[0].x + v[2].x, v[0].y + v[2].y);
        const float2 b = make_float2(v[0].x - v[2].x, v[0].y - v[2].y);
        const float2 c = make_float2(v[1].x + v[3].x, v[1].y + v[3].y);
        const float2 d = make_float2(v[1].x - v[3].x, v[1].y - v[3].y);
        v[0] = make_float2(a.x + c.x, a.y + c.y);
        v[2] = make_float2(a.x - c.x, a.y - c.y);
        v[1] = make_float2(b.x + d.y, b.y - d.x);  // b - i*d
        v[3] = make_float2(b.x - d.y, b.y + d.x);  // b + i*d
    } else if constexpr (R == 8) {
        float2 e[4] = {v[0], v[2], v[4], v[6]};
        float2 o[4] = {v[1], v[3], v[5], v[7]};
        dft_small<4>(e, tw, n_fft);
        dft_small<4>(o, tw, n_fft);
        const float h = 0.70710678118654752f;
        const float2 o1 = make_float2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));   // * exp(-i*pi/4)
        const float2 o2 = make_float2(o[2].y, -o[2].x);                                // * (-i)
        const float2 o3 = make_float2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));  // * exp(-3i*pi/4)
        v[0] = make_float2(e[0].x + o[0].x, e[0].y + o[0].y);
        v[4] = make_float2(e[0].x - o[0].x, e[0].y - o[0].y);
        v[1] = make_float2(e[1].x + o1.x, e[1].y + o1.y);
        v[5] = make_float2(e[1].x - o1.x, e[1].y - o1.y);
        v[2] = make_float2(e[2].x + o2.x, e[2].y + o2.y);
        v[6] = make_float2(e[2].x - o2.x, e[2].y - o2.y);
        v[3] = make_float2(e[3].x + o3.x, e[3].y + o3.y);
        v[7] = make_float2(e[3].x - o3.x, e[3].y - o3.y);
    } else {  // generic O(R^2) DFT for odd radices (3, 5): W_R^m = twiddle[m * n_fft / R]
        float2 y[R];
        const int step = n_fft / R;
#pragma unroll
        for (int q = 0; q < R; ++q) {
            float2 acc = v[0];
#pragma unroll
            for (int r = 1; r < R; ++r) {
                const float2 w = tw[((r * q) % R) * step];
                const float2 p = cmul(v[r], w);
                acc.x += p.x;
                acc.y += p.y;
            }
            y[q] = acc;
        }
#pragma unroll
        for (int q = 0; q < R; ++q) v[q] = y[q];
    }
}

// One Stockham pass of radix R over `nfft_local` packed FFTs held in shared memory.
template <int R>
__device__ __forceinline__ void stockham_pass(const float2* __restrict__ src, float2* __restrict__ dst, int N, int Ns,
                                              int n_seq, const float2* __restrict__ tw) {
    const int per = N / R;
    const int tstep = N / (Ns * R);
    for (int idx = threadIdx.x; idx < n_seq * per; idx += blockDim.x) {
        const int s = idx / per, j = idx - s * per;
        const float2* x = src + s * N;
        float2* y = dst + s * N;
        const int k = j % Ns;
        float2 v[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            v[r] = x[j + r * per];
            if (r > 0 && k > 0) v[r] = cmul(v[r], tw[r * k * tstep]);
        }
        dft_small<R>(v, tw, N);
        const int j0 = (j - k) * R + k;
#pragma unroll
        for (int r = 0; r < R; ++r) y[j0 + r * Ns] = v[r];
    }
}

__global__ void __launch_bounds__(FB_THREADS)
fbank_tile_kernel(const __grid_constant__ CUtensorMap wav_map, const float* __restrict__ wav, int use_tma, int B, int L,
                  int T_f, const FbankDev p, float* __restrict__ out, int* __restrict__ utt_max) {
    extern __shared__ __align__(128) uint8_t fb_smem[];
    const int N = p.n_fft, hop = p.hop;
    const int n_seq = FB_FRAMES / 2;
    const int seg_len = (FB_FRAMES - 1) * hop + N;
    const int seg_pad = (seg_len + 255) & ~255;
    float* seg = reinterpret_cast<float*>(fb_smem);                           // [seg_pad]
    float2* buf0 = reinterpret_cast<float2*>(seg + seg_pad);                  // [n_seq, N]
    float2* buf1 = buf0 + n_seq * N;                                          // [n_seq, N]
    float2* tw = buf1 + n_seq * N;                                            // [N]
    __shared__ uint64_t bar;
    __shared__ float red[FB_THREADS / 32];

    const int b = blockIdx.y;
    const int f0 = blockIdx.x * FB_FRAMES;
    const int start = f0 * hop - N / 2;  // first sample of the segment (may be negative)

    if (use_tma) {
        if (threadIdx.x == 0) {
            mbar_init(&bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(&bar, seg_pad * 4);
            for (int c = 0; c < seg_pad; c += 256) tma_load_2d(seg + c, &wav_map, &bar, start + c, b);
        }
    } else {
        const float* w = wav + static_cast<size_t>(b) * L;
        for (int i = threadIdx.x; i < seg_len; i += blockDim.x) {
            const int s = start + i;
            seg[i] = (s >= 0 && s < L) ? __ldg(w + s) : 0.0f;
        }
    }
    for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = p.twiddle[i];
    if (use_tma) mbar_wait(&bar, 0);
    __syncthreads();

    // pack frame pairs: z[n] = w[n] * (x_{2s}[n] + i x_{2s+1}[n])
    for (int idx = threadIdx.x; idx < n_seq * N; idx += blockDim.x) {
        const int s = idx / N, n = idx - s * N;
        const float w = __ldg(p.window + n);
        buf0[idx] = make_float2(w * seg[(2 * s) * hop + n], w * seg[(2 * s + 1) * hop + n]);
    }
    __syncthreads();

    float2* src = buf0;
    float2* dst = buf1;
    int Ns = 1;
    for (int ps = 0; ps < p.n_pass; ++ps) {
        const int R = p.radix[ps];
        switch (R) {
            case 8: stockham_pass<8>(src, dst, N, Ns, n_seq, tw); break;
            case 4: stockham_pass<4>(src, dst, N, Ns, n_seq, tw); break;
            case 2: stockham_pass<2>(src, dst, N, Ns, n_seq, tw); break;
            case 5: stockham_pass<5>(src, dst, N, Ns, n_seq, tw); break;
            default: stockham_pass<3>(src, dst, N, Ns, n_seq, tw); break;
        }
        Ns *= R;
        __syncthreads();
        float2* t = src; src = dst; dst = t;
    }
    // src now holds Z = FFT(z). Separate the two real spectra and take |.|^2:
    //   Xa[k] = (Z[k] + conj(Z[N-k]))/2 ,  Xb[k] = (Z[k] - conj(Z[N-k]))/(2i)
    float* power = reinterpret_cast<float*>(dst);  // [FB_FRAMES, n_stft]  (n_stft <= N)
    const int n_stft = p.n_stft;
    for (int idx = threadIdx.x; idx < n_seq * n_stft; idx += blockDim.x) {
        const int s = idx / n_stft, k = idx - s * n_stft;
        const float2 zk = src[s * N + k];
        const float2 zn = src[s * N + ((N - k) % N)];
        const float ar = 0.5f * (zk.x + zn.x), ai = 0.5f * (zk.y - zn.y);
        const float br = 0.5f * (zk.y + zn.y), bi = -0.5f * (zk.x - zn.x);
        power[(2 * s) * n_stft + k] = ar * ar + ai * ai;
        power[(2 * s + 1) * n_stft + k] = br * br + bi * bi;
    }
    __syncthreads();

    float local_max = -INFINITY;
    const int n_mels = p.n_mels;
    for (int idx = threadIdx.x; idx < FB_FRAMES * n_mels; idx += blockDim.x) {
        const int f = idx / n_mels, m = idx - f * n_mels;
        const int t = f0 + f;
        if (t >= T_f) continue;
        const int ks = __ldg(p.band_start + m), kl = __ldg(p.band_len + m);
        const float* w = p.band_w + m * p.max_band;
        const float* pw = power + f * n_stft + ks;
        float acc = 0.0f;
        for (int k = 0; k < kl; ++k) acc = fmaf(pw[k], __ldg(w + k), acc);
        const float db = 10.0f * log10f(fmaxf(acc, p.amin));
        out[(static_cast<size_t>(b) * T_f + t) * n_mels + m] = db;
        local_max = fmaxf(local_max, db);
    }
    local_max = warp_max(local_max);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local_max;
    __syncthreads();
    if (threadIdx.x == 0) {
        float mx = red[0];
        for (int i = 1; i < FB_THREADS / 32; ++i) mx = fmaxf(mx, red[i]);
        atomicMax(utt_max + b, float_to_ordered(mx));
    }
}

__global__ void fbank_init_max_kernel(int* utt_max, int B) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) utt_max[i] = float_to_ordered(-INFINITY);
}

// x = max(x, max_b - top_db); optionally (x - mean[m]) / max(std[m], eps) (global CMVN).
__global__ void fbank_finalize_kernel(const float* in, float* out,  // in may alias out
                                      const int* __restrict__ utt_max, float top_db, int per_utt, int n_mels,
                                      const float* __restrict__ mean, const float* __restrict__ stdv, float eps,
                                      size_t total) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        float x = in[i];
        if (utt_max != nullptr) x = fmaxf(x, ordered_to_float(utt_max[i / per_utt]) - top_db);
        if (mean != nullptr) {
            const int m = static_cast<int>(i % n_mels);
            x = (x - __ldg(mean + m)) / fmaxf(__ldg(stdv + m), eps);
        }
        out[i] = x;
    }
}

// InputNormalization norm_type="sentence" (processing/features.py:1478-1486): masked per-utterance
// mean / std over time for each feature; every frame (padding included) is then normalised unless
// avoid_padding_norm. One CTA per utterance; thread (lane_t, m) strides over time.
__global__ void sentence_norm_kernel(const float* __restrict__ x, float* __restrict__ out,
                                     const float* __restrict__ rel_len, int T, int F, int std_norm,
                                     int avoid_padding_norm, float eps) {
    extern __shared__ float sn_smem[];  // [2 * F]
    float* s_mean = sn_smem;
    float* s_std = sn_smem + F;
    const int b = blockIdx.x;
    const float* xb = x + static_cast<size_t>(b) * T * F;
    float* ob = out + static_cast<size_t>(b) * T * F;
    // mask[t] = t < rel*T - 1e-6  (make_padding_mask :1605-1607)
    const float lim = rel_len ? rel_len[b] * static_cast<float>(T) - 1e-6f : static_cast<float>(T);
    int n_valid = 0;
    for (int t = 0; t < T; ++t) n_valid += (static_cast<float>(t) < lim) ? 1 : 0;
    const float n = static_cast<float>(n_valid);
    for (int m = threadIdx.x; m < F; m += blockDim.x) {
        float s = 0.0f;
        for (int t = 0; t < n_valid; ++t) s += xb[static_cast<size_t>(t) * F + m];
        const float mean = s / n;
        float v = 0.0f;
        if (std_norm) {
            for (int t = 0; t < n_valid; ++t) {
                const float dlt = xb[static_cast<size_t>(t) * F + m] - mean;
                v += dlt * dlt;
            }
            v = sqrtf(v / n);
        } else {
            v = 1.0f;
        }
        s_mean[m] = mean;
        s_std[m] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < T * F; i += blockDim.x) {
        const int t = i / F, m = i - t * F;
        float mean = s_mean[m], sd = s_std[m];
        if (avoid_padding_norm && t >= n_valid) { mean = 0.0f; sd = 1.0f; }
        ob[i] = (xb[i] - mean) / fmaxf(sd, eps);
    }
}

// ------------------------------------------------------------------ host side

static bool factorize(int n, int* radix, int* n_pass) {
    int np = 0;
    const int cand[5] = {8, 4, 2, 5, 3};
    for (int c = 0; c < 5; ++c)
        while (n % cand[c] == 0 && np < FB_MAX_PASSES) {
            radix[np++] = cand[c];
            n /= cand[c];
        }
    *n_pass = np;
    return n == 1;
}

int fbank_create(Fbank** out, int n_fft, int hop, int n_mels, const float* window_host,
                 const float* mel_matrix_host /* [n_stft, n_mels] */, float amin, float top_db) {
    SBK_REQUIRE(n_fft >= 16 && n_fft <= 2048 && hop > 0 && n_mels > 0, "fbank_create: bad sizes");
    Fbank* fb = new Fbank();
    FbankDev& d = fb->d;
    d.n_fft = n_fft; d.hop = hop; d.n_stft = n_fft / 2 + 1; d.n_mels = n_mels; d.amin = amin; d.top_db = top_db;
    if (!factorize(n_fft, d.radix, &d.n_pass)) {
        delete fb;
        set_error("fbank_create: n_fft=%d has a prime factor other than 2, 3, 5", n_fft);
        return SBK_ERR_UNSUPPORTED;
    }
    // sparse bands of the (dense) reference matrix
    std::vector<int> bs(n_mels), bl(n_mels);
    int max_band = 1;
    for (int m = 0; m < n_mels; ++m) {
        int lo = -1, hi = -1;
        for (int k = 0; k < d.n_stft; ++k)
            if (mel_matrix_host[k * n_mels + m] != 0.0f) { if (lo < 0) lo = k; hi = k; }
        bs[m] = lo < 0 ? 0 : lo;
        bl[m] = lo < 0 ? 0 : hi - lo + 1;
        if (bl[m] > max_band) max_band = bl[m];
    }
    d.max_band = max_band;
    std::vector<float> bw(static_cast<size_t>(n_mels) * max_band, 0.0f);
    for (int m = 0; m < n_mels; ++m)
        for (int k = 0; k < bl[m]; ++k) bw[m * max_band + k] = mel_matrix_host[(bs[m] + k) * n_mels + m];
    std::vector<float2> tw(n_fft);
    for (int k = 0; k < n_fft; ++k) {
        const double a = -2.0 * M_PI * k / n_fft;
        tw[k] = make_float2(static_cast<float>(cos(a)), static_cast<float>(sin(a)));
    }
    const size_t o_win = 0, o_tw = o_win + n_fft * 4, o_bs = o_tw + n_fft * 8, o_bl = o_bs + n_mels * 4,
                 o_bw = o_bl + n_mels * 4, total = o_bw + bw.size() * 4;
    uint8_t* base = nullptr;
    if (cudaMalloc(&base, total) != cudaSuccess) {
        delete fb;
        set_error("fbank_create: cudaMalloc failed");
        return SBK_ERR_NOMEM;
    }
    fb->arena = base;
    cudaMemcpy(base + o_win, window_host, n_fft * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(base + o_tw, tw.data(), n_fft * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(base + o_bs, bs.data(), n_mels * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(base + o_bl, bl.data(), n_mels * 4, cudaMemcpyHostToDevice);
    SBK_CUDA_CHECK(cudaMemcpy(base + o_bw, bw.data(), bw.size() * 4, cudaMemcpyHostToDevice));
    d.window = reinterpret_cast<float*>(base + o_win);
    d.twiddle = reinterpret_cast<float2*>(base + o_tw);
    d.band_start = reinterpret_cast<int*>(base + o_bs);
    d.band_len = reinterpret_cast<int*>(base + o_bl);
    d.band_w = reinterpret_cast<float*>(base + o_bw);
    *out = fb;
    return SBK_OK;
}

void fbank_destroy(Fbank* fb) {
    if (!fb) return;
    cudaFree(fb->arena);
    delete fb;
}

int fbank_num_frames(const Fbank* fb, int L) { return 1 + L / fb->d.hop; }

static int make_wav_map(CUtensorMap* m, const float* wav, int B, int L);

// wav [B, L] fp32 device -> out [B, T_f, n_mels] fp32 device. utt_max: [B] int scratch.
// If mean/std given, the global CMVN is fused into the finalize pass.
int fbank_forward(const Fbank* fb, const float* wav, int B, int L, float* out, int* utt_max, const float* mean,
                  const float* stdv, float eps, cudaStream_t stream) {
    const FbankDev& d = fb->d;
    SBK_REQUIRE(B > 0 && L > 0, "fbank_forward: empty input B=%d L=%d", B, L);
    const int T_f = 1 + L / d.hop;
    const int seg_len = (FB_FRAMES - 1) * d.hop + d.n_fft;
    const int seg_pad = (seg_len + 255) & ~255;
    const size_t smem = static_cast<size_t>(seg_pad) * 4 + 2ull * (FB_FRAMES / 2) * d.n_fft * 8 + d.n_fft * 8ull;
    SBK_REQUIRE(smem <= 200 * 1024, "fbank_forward: tile does not fit shared memory (hop=%d n_fft=%d)", d.hop, d.n_fft);
    CUtensorMap wmap;
    memset(&wmap, 0, sizeof(wmap));
    int use_tma = (L % 4 == 0) && ((reinterpret_cast<uintptr_t>(wav) & 15) == 0);
    if (use_tma && make_wav_map(&wmap, wav, B, L) != SBK_OK) use_tma = 0;
    SBK_CUDA_CHECK(cudaFuncSetAttribute(fbank_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fbank_init_max_kernel<<<ceil_div(B, 128), 128, 0, stream>>>(utt_max, B);
    dim3 grid(ceil_div(T_f, FB_FRAMES), B);
    fbank_tile_kernel<<<grid, FB_THREADS, smem, stream>>>(wmap, wav, use_tma, B, L, T_f, d, out, utt_max);
    SBK_LAUNCH_CHECK();
    const size_t total = static_cast<size_t>(B) * T_f * d.n_mels;
    const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, SBK_NUM_SMS * 8));
    fbank_finalize_kernel<<<blocks, 256, 0, stream>>>(out, out, utt_max, d.top_db, T_f * d.n_mels, d.n_mels, mean, stdv,
                                                      eps, total);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int global_norm_forward(const float* x, float* out, int B, int T, int F, const float* mean, const float* stdv,
                        float eps, cudaStream_t stream) {
    const size_t total = static_cast<size_t>(B) * T * F;
    if (total == 0) return SBK_OK;
    const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, SBK_NUM_SMS * 8));
    fbank_finalize_kernel<<<blocks, 256, 0, stream>>>(x, out, nullptr, 0.0f, T * F, F, mean, stdv, eps, total);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int sentence_norm_forward(const float* x, float* out, const float* rel_len, int B, int T, int F, int std_norm,
                          int avoid_padding_norm, float eps, cudaStream_t stream) {
    if (B == 0 || T == 0) return SBK_OK;
    sentence_norm_kernel<<<B, 256, 2 * F * sizeof(float), stream>>>(x, out, rel_len, T, F, std_norm,
                                                                   avoid_padding_norm, eps);
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

}  // namespace sbk

// ---- TMA map over the fp32 wav batch (needs the driver entry point from tma_host.cu)
#include <cudaTypedefs.h>
namespace sbk {
int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_cols);
static int make_wav_map(CUtensorMap* m, const float* wav, int B, int L) { return make_tmap_2d_f32(m, wav, B, L, 256); }
}  // namespace sbk
