// TMA + wgmma main loop of the GEMM kernels of gemm_tc.cu:
//
//     acc = A[m0 .. m0 + BM, k-blocks] x W[n0 .. n0 + BN, k-blocks]^T    (fp16 operands, fp32 accumulate in registers)
//
// BM / 64 consumer warpgroups (warpgroup g owns tile rows 64 g .. 64 g + 63) and one TMA producer warp (one elected
// lane) behind them.  A ring of STAGES (A BM x 128 B | W BN x 128 B, both 128B-swizzled K-major) is guarded by
// full / empty mbarriers; a consumer warpgroup frees a stage as soon as the wgmma that read it has retired
// (wait_group 1 keeps one k-block of MMAs in flight behind the next stage's).  After the loop the accumulators are
// staged as an fp32 [BM][BN] tile over the (then idle) ring, so that the epilogues can work on rows of 32 columns.
// Every output row's k-summation is the same m64nBNk16 chain whatever BM is.
#pragma once
#include "common.cuh"

namespace sbk {

constexpr int WG_BK = 64;

template <int BM>
struct WgRoles {
    static_assert(BM == 64 || BM == 128, "one or two consumer warpgroups");
    static constexpr int CONSUMERS = 2 * BM;  // 128 threads per 64 rows
    static constexpr int THREADS = CONSUMERS + 32;
};

template <int BN>
struct WgAcc {
    static constexpr int WN = BN < 128 ? BN : 128;  // wgmma width: BN = 256 issues two n128 instructions per k step
    static constexpr int NI = BN / WN;
    float r[NI][WN / 2];
};

template <int BM, int BN, int STAGES>
struct WgRing {
    static constexpr int A_BYTES = BM * WG_BK * 2;
    static constexpr int B_BYTES = BN * WG_BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
    static constexpr int END = BAR_OFFSET + 2 * STAGES * 8;
    // fp32 accumulator staging row; the 16-byte pad makes 16-byte accesses of 8 consecutive rows conflict-free
    static constexpr int STG_PITCH = BN * 4 + 16;
    static_assert(STAGE_BYTES % 1024 == 0, "128B-swizzled stages must stay 1 KB aligned");
    static_assert(BM * STG_PITCH <= BAR_OFFSET, "the accumulator staging tile reuses the operand ring");
};

// consumer warpgroups only: named barrier 1
template <int BM>
__device__ __forceinline__ void wg_consumers_sync() {
    asm volatile("bar.sync 1, %0;" ::"n"(WgRoles<BM>::CONSUMERS) : "memory");
}

// all threads: barriers initialised before any role starts
template <int BM, int BN, int STAGES>
__device__ __forceinline__ void wg_init(uint8_t* smem, const CUtensorMap* ta, const CUtensorMap* tb) {
    using R = WgRing<BM, BN, STAGES>;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + R::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    if (threadIdx.x == WgRoles<BM>::CONSUMERS) {
        tma_prefetch_desc(ta);
        tma_prefetch_desc(tb);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);        // producer's expect_tx arrive
            mbar_init(&empty_bar[s], BM / 64);  // one arrive per consumer warpgroup
        }
        mbar_fence_init();
    }
    __syncthreads();
}

// producer warp: the num_kb k-blocks of rows m0 (A) and n0 (W).  The weights of the first min(STAGES, num_kb)
// k-blocks are requested before pdl_wait() -- they do not depend on the previous kernel -- and every A tile after it.
// Each stage's full barrier still expects both loads' bytes.
template <int BM, int BN, int STAGES>
__device__ __forceinline__ void wg_produce(uint8_t* smem, const CUtensorMap* ta, const CUtensorMap* tb, int m0, int n0,
                                           int num_kb) {
    using R = WgRing<BM, BN, STAGES>;
    if (threadIdx.x != WgRoles<BM>::CONSUMERS) return;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + R::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    const int pre = num_kb < STAGES ? num_kb : STAGES;
    for (int kb = 0; kb < pre; ++kb) {  // first use of each stage: nothing to wait for
        mbar_arrive_expect_tx(&full_bar[kb], R::STAGE_BYTES);
        tma_load_2d(smem + kb * R::STAGE_BYTES + R::A_BYTES, tb, &full_bar[kb], kb * WG_BK, n0);
    }
    pdl_trigger();  // after this CTA's weight loads are in flight (measured faster than triggering at the top)
    pdl_wait();
    for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        uint8_t* a_dst = smem + s * R::STAGE_BYTES;
        if (kb >= pre) {
            mbar_wait(&empty_bar[s], ((kb / STAGES) & 1) ^ 1);
            mbar_arrive_expect_tx(&full_bar[s], R::STAGE_BYTES);
            tma_load_2d(a_dst + R::A_BYTES, tb, &full_bar[s], kb * WG_BK, n0);
        }
        tma_load_2d(a_dst, ta, &full_bar[s], kb * WG_BK, m0);
    }
}

// consumer warpgroups: the whole k loop, then the accumulators -> fp32 staging tile at smem (row pitch STG_PITCH).
// Ends with the staging tile complete and visible to all consumer threads.
template <int BM, int BN, int STAGES>
__device__ __forceinline__ void wg_consume_and_stage(uint8_t* smem, int num_kb) {
    using R = WgRing<BM, BN, STAGES>;
    using Acc = WgAcc<BN>;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + R::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    const int wg = threadIdx.x >> 7;
    Acc acc;
#pragma unroll
    for (int i = 0; i < Acc::NI; ++i)
#pragma unroll
        for (int j = 0; j < Acc::WN / 2; ++j) acc.r[i][j] = 0.0f;
    for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t a_addr = smem_u32(smem + s * R::STAGE_BYTES) + wg * 64 * 128;
        const uint32_t b_addr = smem_u32(smem + s * R::STAGE_BYTES) + R::A_BYTES;
        const uint64_t da = make_kmajor_sw128_desc(a_addr);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WG_BK / 16; ++k)  // +32 B per k16 step -> +2 in (addr >> 4)
#pragma unroll
            for (int i = 0; i < Acc::NI; ++i)
                wgmma_f16<Acc::WN>(acc.r[i], da + 2 * k, make_kmajor_sw128_desc(b_addr + i * Acc::WN * 128) + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(kb - 1) % STAGES]);
    }
    wgmma_wait<0>();
    wg_consumers_sync<BM>();  // every warpgroup is done reading the ring before it is overwritten
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    uint8_t* base = smem + (wg * 64 + w * 16 + (l >> 2)) * R::STG_PITCH + (l & 3) * 8;
#pragma unroll
    for (int i = 0; i < Acc::NI; ++i)
#pragma unroll
        for (int j = 0; j < Acc::WN / 8; ++j) {
            const int col = i * Acc::WN + j * 8;
            *reinterpret_cast<float2*>(base + col * 4) = make_float2(acc.r[i][4 * j], acc.r[i][4 * j + 1]);
            *reinterpret_cast<float2*>(base + 8 * R::STG_PITCH + col * 4) = make_float2(acc.r[i][4 * j + 2], acc.r[i][4 * j + 3]);
        }
    wg_consumers_sync<BM>();
}

// 32 consecutive staged fp32 columns of one row (16-byte aligned shared-memory address)
__device__ __forceinline__ void wg_load_row32(uint32_t addr, uint32_t (&a)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 v = lds128(addr + 16 * j);
        a[4 * j] = v.x; a[4 * j + 1] = v.y; a[4 * j + 2] = v.z; a[4 * j + 3] = v.w;
    }
}

}  // namespace sbk
