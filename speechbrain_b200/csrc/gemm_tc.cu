// wgmma / TMA GEMM for the Conformer encoder (and decoder prefill, decode-step projections):
//
//     out = epilogue( A[M,K] (fp16, K-major) x W[N,K]^T (fp16, K-major) ), fp32 accumulate in registers
//
// Replaces the reference's F.linear / nn.Linear / Conv1d(k=1) call sites
// (nnet/attention.py:623,739,932-936,1344; Conformer.py:126-157; TransformerASR.py:308-316).
//
// One BM x BN output tile per CTA (BM = 64 or 128; main loop: gemm_mainloop.cuh).  The epilogue runs row-wise on
// 32-column chunks of the staged accumulator tile, so it handles any N and every epilogue mode, including partial column
// chunks.  With BN <= 128 two CTAs fit per SM, so one CTA's epilogue overlaps the other's main loop.
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "gemm_mainloop.cuh"
#include "sbk_internal.h"

namespace sbk {

template <int BM, int BN, int STAGES>
struct GemmSmem {
    static constexpr int TOTAL = WgRing<BM, BN, STAGES>::END + 1024;  // + alignment slack
};

template <int BM, int BN, int STAGES>
__global__ void __launch_bounds__(WgRoles<BM>::THREADS, (BN <= 128 ? 2 : 1))
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmEpilogue epi, int M, int N, int K) {
    using R = WgRing<BM, BN, STAGES>;
    constexpr int CONSUMERS = WgRoles<BM>::CONSUMERS;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
    const int num_kb = (K + WG_BK - 1) / WG_BK;

    // Before pdl_wait() (launched with programmatic stream serialisation, see common.cuh): barrier init, tensor-map
    // prefetch, the first stages' weight loads and the bias.  Activations, the residual, the step counter and every
    // global write come after it.
    wg_init<BM, BN, STAGES>(smem, &tmap_a, &tmap_b);
    EpiPrefetch pre;
    if (threadIdx.x >= CONSUMERS) {
        wg_produce<BM, BN, STAGES>(smem, &tmap_a, &tmap_b, m0, n0, num_kb);
    } else {
        constexpr bool prefetch = BN == 32;  // while the main loop runs
        if constexpr (prefetch)
            if (threadIdx.x < BM) epilogue_prefetch_bias(epi, pre, m0 + threadIdx.x, n0, M, N);
        pdl_wait();  // the consumers' own: the producer's wait does not order this thread's reads and writes
        if constexpr (prefetch)
            if (threadIdx.x < BM) epilogue_prefetch_resid(epi, pre, m0 + threadIdx.x, n0);
        wg_consume_and_stage<BM, BN, STAGES>(smem, num_kb);
    }
    if (threadIdx.x < CONSUMERS) {
        const int r = threadIdx.x & (BM - 1);
#pragma unroll 1
        for (int c = threadIdx.x / BM; c < BN / 32; c += CONSUMERS / BM) {
            uint32_t acc[32];
            wg_load_row32(smem_u32(smem) + r * R::STG_PITCH + c * 128, acc);
            epilogue_chunk(epi, acc, m0 + r, n0 + c * 32, M, N, pre);
        }
    }
}

// pdl: launch with programmatic stream serialisation (the decode-step projections); the kernel's pre-wait section obeys
// the rules of common.cuh either way.
template <int BM, int BN, int STAGES>
static int launch_gemm(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
                       cudaStream_t stream, bool pdl) {
    using S = GemmSmem<BM, BN, STAGES>;
    CUtensorMap ta, tb;
    int rc = make_tmap_2d_f16(&ta, A, M, K, lda, BM, WG_BK);
    if (rc) return rc;
    rc = make_tmap_2d_f16(&tb, W, N, K, ldw, BN, WG_BK);
    if (rc) return rc;
    auto kern = gemm_tc_kernel<BM, BN, STAGES>;
    SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    dim3 grid(ceil_div(N, BN), ceil_div(M, BM));
    GemmProfile* prof = gemm_profile();
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (prof->enabled) {
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0, stream);
    }
    SBK_CUDA_CHECK(launch_pdl(kern, grid, dim3(WgRoles<BM>::THREADS), S::TOTAL, stream, pdl, ta, tb, epi, M, N, K));
    if (prof->enabled) {
        cudaEventRecord(e1, stream);
        prof->ev.push_back(e0);
        prof->ev.push_back(e1);
        prof->flops.push_back(2.0 * M * N * K);
        prof->shape.insert(prof->shape.end(), {M, N, K, epi.mode});
    }
    SBK_LAUNCH_CHECK();
    return SBK_OK;
}

int gemm_f16_small(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
                   cudaStream_t stream) {
    SBK_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_f16_small: empty problem M=%d N=%d K=%d", M, N, K);
    SBK_REQUIRE((K % 8) == 0 && (lda % 8) == 0 && (ldw % 8) == 0, "gemm_f16_small: K/lda/ldw must be multiples of 8");
    SBK_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
                "gemm_f16_small: operands must be 16-byte aligned");
    SBK_REQUIRE(epi.mode == EPI_F16 || epi.mode == EPI_F32 || epi.mode == EPI_RESID || epi.mode == EPI_QKV_CACHE,
                "gemm_f16_small: epilogue mode %d not supported", epi.mode);
    if (epi.mode == EPI_QKV_CACHE)
        SBK_REQUIRE(epi.qkv_d % 32 == 0 && N == 3 * epi.qkv_d && epi.kcache && epi.vcache && epi.step_ptr,
                    "gemm_f16_small: bad EPI_QKV_CACHE arguments");
    // few, latency-bound CTAs: narrow N tiles spread the weight stream over more SMs; the ring holds a whole K = 512 panel.
    // 64-row tiles (one consumer warpgroup): twice the CTAs of 128-row tiles, each streaming half the activations -- at
    // 96 - 224 rows they measured faster for every decode shape (FFN2 K = 2048 and the vocabulary head included).
    if (N > 2048) return launch_gemm<64, 64, 6>(A, lda, W, ldw, epi, M, N, K, stream, true);
    return launch_gemm<64, 32, 8>(A, lda, W, ldw, epi, M, N, K, stream, true);
}

int gemm_f16(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
             cudaStream_t stream) {
    SBK_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_f16: empty problem M=%d N=%d K=%d", M, N, K);
    SBK_REQUIRE((K % 8) == 0 && (lda % 8) == 0 && (ldw % 8) == 0, "gemm_f16: K/lda/ldw must be multiples of 8");
    SBK_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
                "gemm_f16: operands must be 16-byte aligned");
    if (epi.mode == EPI_GLU || epi.mode == EPI_ROPE)
        SBK_REQUIRE(N % 32 == 0, "gemm_f16: GLU/RoPE epilogues need N %% 32 == 0");
    if (epi.mode == EPI_ROPE) SBK_REQUIRE(epi.head_dim % 32 == 0, "gemm_f16: RoPE epilogue needs head_dim %% 32 == 0");
    if (N % 256 == 0) return gemm_f16_wide(A, lda, W, ldw, epi, M, N, K, stream);
    return launch_gemm<128, 128, 3>(A, lda, W, ldw, epi, M, N, K, stream, false);
}

}  // namespace sbk
