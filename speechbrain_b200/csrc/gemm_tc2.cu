// Wide-tile wgmma GEMM for N % 256 == 0: out = epilogue(A[M,K] x W[N,K]^T), fp16 in / fp32 accumulate.
//
// One 128 x 256 output tile per CTA (main loop: gemm_mainloop.cuh; each consumer warpgroup issues two m64n128k16 per k
// step), a 4-stage ring of 48 KB stages.  Versus the 128 x 128 tiles of gemm_tc.cu this halves the L2 -> SM traffic of
// the A operand per FLOP, which is what bounds these K = 512..2048 GEMMs.  The grid runs n fastest, so the CTAs that
// share the rows of A are resident together.
// Epilogue: the 8 consumer warps each own 32 rows x 128 columns of the staged tile and run the warp-cooperative,
// coalesced epilogue (gemm_epilogue.cuh) on it chunk by chunk, the staged rows doubling as its staging area.
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "gemm_mainloop.cuh"
#include "sbk_internal.h"

namespace sbk {

constexpr int G2_BN = 256;       // columns per tile (default; template parameter BN of the kernel)
constexpr int G2_STAGES = 4;
// shared-memory map: [ring | barriers] [BN floats: the tile's bias vector] (+ alignment slack)
template <int BN, int ST>
__host__ __device__ constexpr int g2_bias_offset() { return (WgRing<BN, ST>::END + 15) / 16 * 16; }
template <int BN, int ST>
__host__ __device__ constexpr int g2_smem() { return g2_bias_offset<BN, ST>() + BN * 4 + 1024; }

template <int MODE, int ACT, int BN = G2_BN, int ST = G2_STAGES>
__global__ void __launch_bounds__(WG_THREADS, 1)
gemm_tc2_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmEpilogue epi, int M, int N, int K) {
    using R = WgRing<BN, ST>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int n0 = blockIdx.x * BN, m0 = blockIdx.y * WG_BM;
    const int num_kb = (K + WG_BK - 1) / WG_BK;

    wg_init<BN, ST>(smem, &tmap_a, &tmap_b);
    if (threadIdx.x >= WG_CONSUMERS) {
        wg_produce<BN, ST>(smem, &tmap_a, &tmap_b, m0, n0, 0, num_kb);
        return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rg = warp & 3;                 // rows rg * 32 .. + 31 of the tile
    constexpr int PART_COLS = BN / 2, CHUNKS = PART_COLS / 32;
    const int c0 = (warp >> 2) * PART_COLS;  // this warp's half of the columns
    const int row_base = m0 + rg * 32;
    // the tile's bias vector -> shared memory (read by every lane of every chunk: a broadcast instead of an L2 round trip);
    // visible after the consumer barriers of the main loop
    float* sbias = reinterpret_cast<float*>(smem + g2_bias_offset<BN, ST>());
    for (int j = threadIdx.x; j < BN; j += WG_CONSUMERS) sbias[j] = epi.bias ? __ldg(epi.bias + n0 + j) : 0.0f;
    // residual / RoPE-table operands of the first chunk are fetched before the main loop, so their memory round trip
    // overlaps it; each chunk then fetches the next one's ahead of its own math
    float4 res[8];
    float4 rcs[4], rsn[4];
    if constexpr (MODE == EPI_RESID) epilogue_resid_prefetch(epi, res, row_base, n0 + c0, M, lane);
    if constexpr (MODE == EPI_ROPE) epilogue_rope_prefetch(epi, rcs, rsn, row_base, n0 + c0, lane);
    wg_consume_and_stage<BN, ST>(smem, num_kb);
    uint8_t* stg = smem + rg * 32 * R::STG_PITCH + c0 * 4;
#pragma unroll 1
    for (int c = 0; c < CHUNKS; ++c) {
        uint32_t acc[32];
        wg_load_row32(smem_u32(stg + lane * R::STG_PITCH + c * 128), acc);
        epilogue_chunk_coalesced<MODE, ACT, R::STG_PITCH>(epi, acc, stg + c * 128, row_base, n0 + c0 + c * 32, M, lane, res,
                                                          c + 1 < CHUNKS ? n0 + c0 + (c + 1) * 32 : -1, rcs, rsn,
                                                          sbias + c0 + c * 32);
    }
}

int gemm_f16_wide(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
                  cudaStream_t stream) {
    CUtensorMap ta, tb;
    int rc = make_tmap_2d_f16(&ta, A, M, K, lda, WG_BM, WG_BK);
    if (rc) return rc;
    // optional 128 x 128 tiles with a 4-stage ring for the fp32-output modes (N = 512 GEMMs: twice the CTAs) -> opt-in
    static const bool bn128_env = getenv("SBK_GEMM_BN128") != nullptr;
    const bool bn128 = bn128_env && (epi.mode == EPI_RESID || epi.mode == EPI_F32) && N % 128 == 0 && N <= 1024;
    const int bn = bn128 ? 128 : G2_BN;
    rc = make_tmap_2d_f16(&tb, W, N, K, ldw, bn, WG_BK);
    if (rc) return rc;
    void (*kern)(const CUtensorMap, const CUtensorMap, const GemmEpilogue, int, int, int) = nullptr;
    int smem = 0;
#define G2_PICK(MODE, ACT)                                                        \
    do {                                                                          \
        kern = gemm_tc2_kernel<MODE, ACT>;                                        \
        smem = g2_smem<G2_BN, G2_STAGES>();                                       \
    } while (0)
#define G2_PICK_BN128(MODE)                                                       \
    do {                                                                          \
        kern = gemm_tc2_kernel<MODE, ACT_NONE, 128, 4>;                           \
        smem = g2_smem<128, 4>();                                                 \
    } while (0)
    // SiLU / GLU-gate sigmoid through one tanh.approx MUFU per element (default) or the exact-form EX2 + RCP (SBK_SILU_EXACT=1)
    static const bool fast_act = getenv("SBK_SILU_EXACT") == nullptr;
    switch (epi.mode) {
        case EPI_F16:
            if (epi.act == ACT_SILU && fast_act) G2_PICK(EPI_F16, ACT_SILU_FAST);
            else if (epi.act == ACT_SILU) G2_PICK(EPI_F16, ACT_SILU);
            else if (epi.act == ACT_GELU) G2_PICK(EPI_F16, ACT_GELU);
            else if (epi.act == ACT_NONE) G2_PICK(EPI_F16, ACT_NONE);
            else { set_error("gemm_f16_wide: activation %d not built", epi.act); return SBK_ERR_ARG; }
            break;
        case EPI_F32:
            if (bn128) G2_PICK_BN128(EPI_F32);
            else G2_PICK(EPI_F32, ACT_NONE);
            break;
        case EPI_RESID:
            if (bn128) G2_PICK_BN128(EPI_RESID);
            else G2_PICK(EPI_RESID, ACT_NONE);
            break;
        case EPI_GLU:
            if (fast_act) G2_PICK(EPI_GLU, ACT_SILU_FAST);
            else G2_PICK(EPI_GLU, ACT_NONE);
            break;
        case EPI_ROPE: G2_PICK(EPI_ROPE, ACT_NONE); break;
        default: set_error("gemm_f16_wide: bad epilogue mode %d", epi.mode); return SBK_ERR_ARG;
    }
#undef G2_PICK
#undef G2_PICK_BN128
    SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    GemmProfile* prof = gemm_profile();
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (prof->enabled) {
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0, stream);
    }
    kern<<<dim3(N / bn, ceil_div(M, WG_BM)), WG_THREADS, smem, stream>>>(ta, tb, epi, M, N, K);
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

}  // namespace sbk
