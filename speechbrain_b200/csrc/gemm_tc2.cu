// Wide GEMM for N % 256 == 0 (every encoder Linear, the cross-attention K/V projection, the CTC head):
//     out = epilogue(A[M,K] x W[N,K]^T), fp16 in / fp32 accumulate.
//
// Persistent and warp-specialised:
//  * grid = as many CTAs as it takes to cover the tiles in the fewest rounds (at most one CTA per SM); CTA b takes tiles
//    b, b + grid, b + 2 grid, ... of a grouped rasterisation (pp_tile_coords).
//  * warpgroup 0 is the producer: one thread runs the TMA ring (STAGES x [A 128 x 64 | W BN x 64], 128B-swizzled) across
//    tile boundaries, so the next tile's operands arrive while the current one is still in its epilogue.
//  * warpgroups 1 and 2 are consumers with 128 fp32 accumulator registers per thread (setmaxnreg moves registers from the
//    producer to them), in one of two arrangements (PpCfg; chosen per shape in gemm_f16_wide):
//      - BN = 128, ping-pong: each consumer warpgroup owns alternate 128 x 128 tiles whole.  A pair of named barriers
//        hands the tensor pipe from one to the other: warpgroup g issues its tile's wgmmas, passes the turn, then runs its
//        epilogue while the other warpgroup's main loop runs.
//      - BN = 256, cooperative: both warpgroups work on one 128 x 256 tile, 64 rows each, one m64n256k16 per k step
//        (the W stage is read by both; the widest instruction re-reads the least A per FLOP).
//  * the epilogue works on the accumulator fragments in registers (bias, activation, GLU, residual scale) and stages
//    only what the coalesced stores need, 16 rows x 32 columns at a time, in a per-warp buffer outside the ring.
// The k-summation order of every output element is that of a plain k loop (no split-K), the same as gemm_tc.cu.
#include <stdio.h>

#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

constexpr int PP_BM = 128, PP_BK = 64;
constexpr int PP_THREADS = 384;  // warpgroup 0: producer; 1, 2: consumers
constexpr int PP_GROUP_M = 8;    // row panels per rasterisation group
constexpr int PP_A_BYTES = PP_BM * PP_BK * 2;
constexpr int PP_STG_WARP_BYTES = 16 * 160;  // 16 rows at the largest staging pitch
constexpr int PP_BAR_TURN = 2;   // ping-pong: named barriers 2, 3 = "consumer warpgroup g may issue its main loop"
constexpr int PP_CONSUMER_REGS = 232, PP_PRODUCER_REGS = 40;
static_assert(128 * PP_PRODUCER_REGS + 256 * PP_CONSUMER_REGS <= 65536, "register file");

// BN = 128: ping-pong, each consumer warpgroup owns a whole 128 x 128 tile (two m64n128k16 per k step).
// BN = 256: cooperative, the two consumer warpgroups share a 128 x 256 tile, 64 rows each (one m64n256k16 per k step).
// Both keep 128 fp32 accumulators per consumer thread.
template <int BN>
struct PpCfg {
    static constexpr bool PINGPONG = BN == 128;
    static constexpr int STAGES = BN == 128 ? 6 : 4;
    static constexpr int STAGE_BYTES = PP_A_BYTES + BN * PP_BK * 2;
    static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
    static constexpr int STG_OFFSET = BAR_OFFSET + 128;                   // full[STAGES], empty[STAGES] mbarriers, padded
    static constexpr int BIAS_OFFSET = STG_OFFSET + 8 * PP_STG_WARP_BYTES;  // per warp: the tile's BN bias values
    static constexpr int SMEM = BIAS_OFFSET + 8 * BN * 4 + 1024;          // + alignment slack
    static_assert(STAGE_BYTES % 1024 == 0, "128B-swizzled stages must stay 1 KB aligned");
    static_assert(2 * STAGES * 8 <= 128, "mbarriers overflow their slot");
    static_assert(SMEM <= 227 * 1024, "shared memory");
};

// staging row pitch (bytes) per mode: fp32 rows (F32 / RESID: float2 writes of 4 rows per half-warp and 16-byte reads of a
// whole row per quarter-warp are conflict-free at 160; ROPE reads 32 B per lane, conflict-free at 144), 64 B rows (fp16, GLU)
template <int MODE>
__host__ __device__ constexpr int pp_stg_pitch() {
    return (MODE == EPI_F32 || MODE == EPI_RESID) ? 160 : MODE == EPI_ROPE ? 144 : 80;
}

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts64(uint32_t addr, float x, float y) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
    return v;
}

// Tile t -> (m0, n0): groups of PP_GROUP_M row panels, rows fastest inside a group.  The tiles in flight at one time (a
// contiguous range of t) then read a few W column panels and the group's A row panels, all of which stay in L2.
template <int BN>
__device__ __forceinline__ void pp_tile_coords(int t, int tiles_m, int tiles_n, int& m0, int& n0) {
    const int per_group = PP_GROUP_M * tiles_n;
    const int grp = t / per_group, first_m = grp * PP_GROUP_M;
    const int rows = min(PP_GROUP_M, tiles_m - first_m);
    const int r = t - grp * per_group;
    m0 = (first_m + r % rows) * PP_BM;
    n0 = (r / rows) * BN;
}

// ------------------------------------------------------------------------------------------------- epilogue
// One warp's 16 rows x 32 columns of the tile.  Accumulator fragment (wgmma m64nN, common.cuh): a[4 jj + 2 i + c] is row
// row_base + lane / 4 + 8 i, column 8 jj + 2 (lane % 4) + c; this chunk is jj = 4 CH .. 4 CH + 3.
// Operands that the store phase reads from global memory (EPI_RESID residual, EPI_ROPE cos / sin) are fetched one chunk
// ahead, the first chunk's before the tile's main loop (pp_prefetch).  So are the tile's bias (into a per-warp copy in
// shared memory) and the EPI_RESID row scales: no global load is left on the epilogue's dependency chain.

// EPI_RESID: alpha, or 0 for a padded frame (t >= row_lens[utt]), for the thread's rows row_base + lane / 4 + {0, 8}
template <int MODE>
__device__ __forceinline__ void pp_row_alpha(const GemmEpilogue& e, float (&alpha)[2], int row_base, int M, int lane) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int row = row_base + (lane >> 2) + 8 * i;
        alpha[i] = e.alpha;
        if (MODE == EPI_RESID && e.row_lens != nullptr && row < M) {
            const int b = row / e.T, t = row - b * e.T;
            if (t >= __ldg(e.row_lens + b)) alpha[i] = 0.0f;
        }
    }
}

// EPI_RESID: 8 lanes x 16 B per row, 4 rows per instruction
__device__ __forceinline__ void pp_resid_prefetch(const GemmEpilogue& e, float4 (&res)[4], int row_base, int col0, int M,
                                                  int lane) {
    const int seg = lane & 7, rsub = lane >> 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = row_base + i * 4 + rsub;
        res[i] = row < M ? __ldcg(reinterpret_cast<const float4*>(e.resid + static_cast<size_t>(row) * e.ldo + col0 + seg * 4))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}
// EPI_ROPE: 4 lanes x 8 columns (4 rotation pairs) per row, 8 rows per instruction -> one 16-byte cos and sin load per row
__device__ __forceinline__ void pp_rope_prefetch(const GemmEpilogue& e, float4 (&rc)[2], float4 (&rs)[2], int row_base,
                                                 int col0, int lane) {
    const int dh = e.head_dim;
    const int within = col0 % (3 * dh);
    const int sect = within / dh;  // 0 q, 1 k, 2 v
    if (sect < 2) {
        const int p = ((within - sect * dh) >> 1) + (lane & 3) * 4;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int t = (row_base + i * 8 + (lane >> 2)) % e.T;
            rc[i] = __ldg(reinterpret_cast<const float4*>(e.rope_cos + static_cast<size_t>(t) * (dh >> 1) + p));
            rs[i] = __ldg(reinterpret_cast<const float4*>(e.rope_sin + static_cast<size_t>(t) * (dh >> 1) + p));
        }
    }
}
template <int MODE>
__device__ __forceinline__ void pp_prefetch(const GemmEpilogue& e, float4 (&res)[4], float4 (&rc)[2], float4 (&rs)[2],
                                            int row_base, int col0, int M, int lane) {
    if constexpr (MODE == EPI_RESID) pp_resid_prefetch(e, res, row_base, col0, M, lane);
    if constexpr (MODE == EPI_ROPE) pp_rope_prefetch(e, rc, rs, row_base, col0, lane);
}

template <int MODE, int ACT, int CH>
__device__ __forceinline__ void pp_epilogue_chunk(const GemmEpilogue& e, const float (&a)[64], uint32_t stg, uint32_t sbias,
                                                  const float (&alpha)[2], int row_base, int col0, int M, int lane,
                                                  float4 (&res)[4], float4 (&rc)[2], float4 (&rs)[2]) {
    constexpr int P = pp_stg_pitch<MODE>();
    const int qc = 2 * (lane & 3), r0 = lane >> 2;
    float v[4][2][2];  // [8-column group q][row r0 + 8 i][column 2 (lane % 4) + c]
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 b = lds64(sbias + (32 * CH + 8 * q + qc) * 4);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            v[q][i][0] = a[4 * (4 * CH + q) + 2 * i] + b.x;
            v[q][i][1] = a[4 * (4 * CH + q) + 2 * i + 1] + b.y;
        }
    }
    // ---- maths in registers, then this chunk's output (or, for EPI_RESID / EPI_ROPE, its fp32 operand) -> staging rows
    if constexpr (MODE == EPI_F16) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    if constexpr (ACT == ACT_SILU_FAST) v[q][i][c] = silu_fast(v[q][i][c]);
                    else if constexpr (ACT == ACT_GELU) v[q][i][c] = gelu_erf_f(v[q][i][c]);
                    else if constexpr (ACT == ACT_RELU) v[q][i][c] = fmaxf(v[q][i][c], 0.0f);
                }
                sts32(stg + (r0 + 8 * i) * P + (8 * q + qc) * 2, pack_half2(v[q][i][0], v[q][i][1]));
            }
    } else if constexpr (MODE == EPI_GLU) {  // weight rows interleaved [16 values | 16 gates] per 32 columns: the gate of
                                             // value column j (group q) is column j + 16 (group q + 2) of the same thread
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float o[2];
#pragma unroll
                for (int c = 0; c < 2; ++c) o[c] = v[q][i][c] * sigmoid_fast(v[q + 2][i][c]);
                sts64(stg + (r0 + 8 * i) * P + (8 * q + qc) * 4, o[0], o[1]);
            }
    } else {  // EPI_F32, EPI_RESID (alpha-scaled; the residual is added in the store phase), EPI_ROPE (rotated there)
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                if constexpr (MODE == EPI_RESID) sts64(stg + (r0 + 8 * i) * P + (8 * q + qc) * 4, v[q][i][0] * alpha[i], v[q][i][1] * alpha[i]);
                else sts64(stg + (r0 + 8 * i) * P + (8 * q + qc) * 4, v[q][i][0], v[q][i][1]);
            }
    }
    __syncwarp();
    // ---- coalesced write-back: each instruction covers whole row segments
    if constexpr (MODE == EPI_F32 || MODE == EPI_RESID) {
        const int seg = lane & 7, rsub = lane >> 3;
        float* outp = reinterpret_cast<float*>(e.out);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = i * 4 + rsub;
            const int row = row_base + r;
            if (row < M) {
                float4 val = u4_as_f4(lds128(stg + r * P + seg * 16));
                if constexpr (MODE == EPI_RESID) {
                    val.x += res[i].x; val.y += res[i].y; val.z += res[i].z; val.w += res[i].w;
                }
                *reinterpret_cast<float4*>(outp + static_cast<size_t>(row) * e.ldo + col0 + seg * 4) = val;
            }
        }
    } else if constexpr (MODE == EPI_ROPE) {  // columns = per-head [q(dh) | k(dh) | v(dh)], dh % 32 == 0
        const int seg = lane & 3, rsub = lane >> 2;
        const int dh = e.head_dim;
        const int sect = (col0 % (3 * dh)) / dh;  // 0 q (rotated, scaled), 1 k (rotated), 2 v
        const float sc = sect == 0 ? e.alpha : 1.0f;
        __half* outp = reinterpret_cast<__half*>(e.out);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = i * 8 + rsub;
            const int row = row_base + r;
            float4 x0 = u4_as_f4(lds128(stg + r * P + seg * 32));
            float4 x1 = u4_as_f4(lds128(stg + r * P + seg * 32 + 16));
            if (sect < 2) {
                const float4 c = rc[i], s4 = rs[i];
                const float a0 = (x0.x * c.x - x0.y * s4.x) * sc, a1 = (x0.y * c.x + x0.x * s4.x) * sc;
                const float a2 = (x0.z * c.y - x0.w * s4.y) * sc, a3 = (x0.w * c.y + x0.z * s4.y) * sc;
                const float b0 = (x1.x * c.z - x1.y * s4.z) * sc, b1 = (x1.y * c.z + x1.x * s4.z) * sc;
                const float b2 = (x1.z * c.w - x1.w * s4.w) * sc, b3 = (x1.w * c.w + x1.z * s4.w) * sc;
                x0 = make_float4(a0, a1, a2, a3);
                x1 = make_float4(b0, b1, b2, b3);
            }
            if (row < M)
                *reinterpret_cast<uint4*>(outp + static_cast<size_t>(row) * e.ldo + col0 + seg * 8) =
                    make_uint4(pack_half2(x0.x, x0.y), pack_half2(x0.z, x0.w), pack_half2(x1.x, x1.y), pack_half2(x1.z, x1.w));
        }
    } else {  // 64 B per row (32 fp16, or 16 fp32 GLU outputs): 4 lanes x 16 B per row, 8 rows per instruction
        const int seg = lane & 3, rsub = lane >> 2;
        if (MODE == EPI_F16 && e.kv_heads > 0) {
            // cross-attention K/V scatter: column c of the [layer][K (d) | V (d)] row goes to
            // layer[c / 2d] part[(c % 2d) / d][utt][head][t][64], so that the decode-step attention streams one contiguous
            // T x 128 B block per (utterance, head)
            const int d = e.kv_heads * 64;
            const int layer = col0 / (2 * d), within = col0 - layer * 2 * d;
            const int part = within / d, cc = within - part * d, head = cc >> 6, dcol = cc & 63;
            __half* pbase = reinterpret_cast<__half*>(e.out) + static_cast<size_t>(layer) * e.kv_layer_stride +
                            static_cast<size_t>(part) * e.kv_part_stride;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = i * 8 + rsub;
                const int row = row_base + r;
                if (row < M) {
                    const int b = row / e.T, t = row - b * e.T;
                    __half* dst = pbase + ((static_cast<size_t>(b) * e.kv_heads + head) * e.T + t) * 64 + dcol + seg * 8;
                    *reinterpret_cast<uint4*>(dst) = lds128(stg + r * P + seg * 16);
                }
            }
        } else {
            // byte offset of this chunk inside a row: fp16 -> col0 * 2 ; GLU fp32 (16 columns) -> (col0 / 2) * 4
            uint8_t* outp = reinterpret_cast<uint8_t*>(e.out);
            const size_t row_pitch = MODE == EPI_GLU ? static_cast<size_t>(e.ldo) * 4 : static_cast<size_t>(e.ldo) * 2;
            const size_t col_off = static_cast<size_t>(col0) * 2;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = i * 8 + rsub;
                const int row = row_base + r;
                if (row < M)
                    *reinterpret_cast<uint4*>(outp + static_cast<size_t>(row) * row_pitch + col_off + seg * 16) =
                        lds128(stg + r * P + seg * 16);
            }
        }
    }
    __syncwarp();  // the staging rows are reused by the next chunk
}

// 128 accumulator columns (fragment a): this warp's 16 rows x 128 columns, chunk by chunk, each fetching the next one's operands
template <int MODE, int ACT>
__device__ __forceinline__ void pp_epilogue_rows(const GemmEpilogue& e, const float (&a)[64], uint32_t stg, uint32_t sbias,
                                                 const float (&alpha)[2], int row_base, int n0, int M, int lane,
                                                 float4 (&res)[4], float4 (&rc)[2], float4 (&rs)[2], bool has_next,
                                                 int next_row_base, int next_n0) {
    pp_epilogue_chunk<MODE, ACT, 0>(e, a, stg, sbias, alpha, row_base, n0, M, lane, res, rc, rs);
    pp_prefetch<MODE>(e, res, rc, rs, row_base, n0 + 32, M, lane);
    pp_epilogue_chunk<MODE, ACT, 1>(e, a, stg, sbias, alpha, row_base, n0 + 32, M, lane, res, rc, rs);
    pp_prefetch<MODE>(e, res, rc, rs, row_base, n0 + 64, M, lane);
    pp_epilogue_chunk<MODE, ACT, 2>(e, a, stg, sbias, alpha, row_base, n0 + 64, M, lane, res, rc, rs);
    pp_prefetch<MODE>(e, res, rc, rs, row_base, n0 + 96, M, lane);
    pp_epilogue_chunk<MODE, ACT, 3>(e, a, stg, sbias, alpha, row_base, n0 + 96, M, lane, res, rc, rs);
    if (has_next) pp_prefetch<MODE>(e, res, rc, rs, next_row_base, next_n0, M, lane);
}

// ------------------------------------------------------------------------------------------------- kernel
template <int MODE, int ACT, int BN>
__global__ void __launch_bounds__(PP_THREADS, 1)
gemm_tc2_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmEpilogue epi, int M, int N, int K) {
    using C = PpCfg<BN>;
    constexpr int ST = C::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + ST;
    const int num_kb = (K + PP_BK - 1) / PP_BK;
    const int tiles_m = (M + PP_BM - 1) / PP_BM, tiles_n = N / BN, tiles = tiles_m * tiles_n;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < ST; ++s) {
            mbar_init(&full_bar[s], 1);                      // producer's expect_tx arrive
            mbar_init(&empty_bar[s], C::PINGPONG ? 1 : 2);   // the consumer warpgroup(s) that read the stage
        }
        mbar_fence_init();
    }
    __syncthreads();
    const int wg = threadIdx.x >> 7;
    if (wg == 0) {  // ---- producer: the ring, in tile order, across tile boundaries
        setmaxnreg_dec<PP_PRODUCER_REGS>();
        if (threadIdx.x == 0) {
            int it = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                int m0, n0;
                pp_tile_coords<BN>(t, tiles_m, tiles_n, m0, n0);
                for (int kb = 0; kb < num_kb; ++kb, ++it) {
                    const int s = it % ST;
                    mbar_wait(&empty_bar[s], ((it / ST) & 1) ^ 1);
                    mbar_arrive_expect_tx(&full_bar[s], C::STAGE_BYTES);
                    uint8_t* dst = smem + s * C::STAGE_BYTES;
                    tma_load_2d(dst, &tmap_a, &full_bar[s], kb * PP_BK, m0);
                    tma_load_2d(dst + PP_A_BYTES, &tmap_b, &full_bar[s], kb * PP_BK, n0);
                }
            }
        }
        return;
    }
    // ---- consumers.  Ping-pong: warpgroup g takes the CTA's tiles g, g + 2, g + 4, ... (local index j); cooperative: both
    // take every tile of the CTA, warpgroup g rows 64 g .. 64 g + 63.
    setmaxnreg_inc<PP_CONSUMER_REGS>();
    const int g = wg - 1;
    const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const uint32_t stg = smem_u32(smem + C::STG_OFFSET + (g * 4 + warp) * PP_STG_WARP_BYTES);
    const uint32_t sbias = smem_u32(smem + C::BIAS_OFFSET + (g * 4 + warp) * BN * 4);
    constexpr int STEP = C::PINGPONG ? 2 : 1;
    int j = C::PINGPONG ? g : 0;
    for (int t = blockIdx.x + (C::PINGPONG ? g : 0) * gridDim.x; t < tiles; t += STEP * gridDim.x, j += STEP) {
        int m0, n0;
        pp_tile_coords<BN>(t, tiles_m, tiles_n, m0, n0);
        // the two 128-column accumulator halves: (rows rb[h], columns cb[h])
        const int rb0 = m0 + (C::PINGPONG ? 0 : 64 * g) + warp * 16, rb1 = C::PINGPONG ? rb0 + 64 : rb0;
        const int cb1 = C::PINGPONG ? n0 : n0 + 128;
        float4 res[4], rc[2], rs[2];
        pp_prefetch<MODE>(epi, res, rc, rs, rb0, n0, M, lane);
        float4 bias4[BN / 128];
#pragma unroll
        for (int q = 0; q < BN / 128; ++q)
            bias4[q] = epi.bias != nullptr ? __ldg(reinterpret_cast<const float4*>(epi.bias + n0 + 128 * q) + lane)
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
        float alpha[2][2];
        if constexpr (MODE == EPI_RESID) {
            pp_row_alpha<MODE>(epi, alpha[0], rb0, M, lane);
            pp_row_alpha<MODE>(epi, alpha[1], rb1, M, lane);
        }
        float acc[2][64];  // ping-pong: [m64 half h: tile rows 64 h ..][fragment]; cooperative: one m64n256 fragment
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int x = 0; x < 64; ++x) acc[h][x] = 0.0f;
        if (C::PINGPONG && j > 0) named_bar_sync(PP_BAR_TURN + g, 256);  // the other warpgroup has issued its main loop
        int it = j * num_kb;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % ST;
            mbar_wait(&full_bar[s], (it / ST) & 1);
            const uint32_t a_addr = smem_u32(smem + s * C::STAGE_BYTES);
            const uint64_t db = make_kmajor_sw128_desc(a_addr + PP_A_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < PP_BK / 16; ++k) {  // +32 B per k16 step -> +2 in (addr >> 4)
                if constexpr (C::PINGPONG) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        wgmma_f16<128>(acc[h], make_kmajor_sw128_desc(a_addr + h * 64 * 128) + 2 * k, db + 2 * k, 1u);
                } else {
                    wgmma_f16<256>(reinterpret_cast<float(&)[128]>(acc), make_kmajor_sw128_desc(a_addr + g * 64 * 128) + 2 * k,
                                   db + 2 * k, 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % ST]);
        }
        if (C::PINGPONG && t + gridDim.x < tiles) named_bar_arrive(PP_BAR_TURN + (g ^ 1), 256);  // the next tile may start
        wgmma_wait<0>();
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % ST]);
#pragma unroll
        for (int q = 0; q < BN / 128; ++q)  // (this warp's reads of the previous tile's copy are done)
            sts128(sbias + q * 512 + lane * 16, f4_as_u4(bias4[q]));
        __syncwarp();
        pp_epilogue_rows<MODE, ACT>(epi, acc[0], stg, sbias, alpha[0], rb0, n0, M, lane, res, rc, rs, true, rb1, cb1);
        pp_epilogue_rows<MODE, ACT>(epi, acc[1], stg, sbias + (cb1 - n0) * 4, alpha[1], rb1, cb1, M, lane, res, rc, rs, false,
                                    0, 0);
    }
}

using WideKernel = void (*)(const CUtensorMap, const CUtensorMap, const GemmEpilogue, int, int, int);
// SiLU and the GLU gate's sigmoid: one tanh.approx MUFU per element
template <int BN>
static WideKernel pick_wide_kernel(const GemmEpilogue& epi) {
    switch (epi.mode) {
        case EPI_F16:
            if (epi.act == ACT_SILU) return gemm_tc2_kernel<EPI_F16, ACT_SILU_FAST, BN>;
            if (epi.act == ACT_GELU) return gemm_tc2_kernel<EPI_F16, ACT_GELU, BN>;
            if (epi.act == ACT_RELU) return gemm_tc2_kernel<EPI_F16, ACT_RELU, BN>;  // ReLU TransformerLM FFN
            if (epi.act == ACT_NONE) return gemm_tc2_kernel<EPI_F16, ACT_NONE, BN>;
            return nullptr;
        case EPI_F32: return gemm_tc2_kernel<EPI_F32, ACT_NONE, BN>;
        case EPI_RESID: return gemm_tc2_kernel<EPI_RESID, ACT_NONE, BN>;
        case EPI_GLU: return gemm_tc2_kernel<EPI_GLU, ACT_SILU_FAST, BN>;
        case EPI_ROPE: return gemm_tc2_kernel<EPI_ROPE, ACT_NONE, BN>;
        default: return nullptr;
    }
}

int gemm_f16_wide(const void* A, int lda, const void* W, int ldw, const GemmEpilogue& epi, int M, int N, int K,
                  cudaStream_t stream) {
    // Tile shape per shape class (M = 8032, one H100 SXM at a 400 W power limit, tools/gemm_overhead.py): fp32 outputs at K <= 1024
    // (out-proj, conv pw2, input linear) run ping-pong 128 x 128 tiles, whose heavier write-back then hides under the other
    // warpgroup's main loop (N = 512 / 1024 / 2048, K = 512: 11.7 / 25.2 / 49.3 us vs 12.2 / 29.7 / 56.5 us cooperative).
    // Everything else runs cooperative 128 x 256 tiles with m64n256k16: per FLOP they move less operand data through shared
    // memory (FFN1 N = 2048, K = 512: 44.0 vs 51.9 us; FFN2 N = 512, K = 2048: 36.4 vs 40.3 us).
    const int bn = (epi.mode == EPI_F32 || epi.mode == EPI_RESID) && K <= 1024 ? 128 : 256;
    CUtensorMap ta, tb;
    int rc = make_tmap_2d_f16(&ta, A, M, K, lda, PP_BM, PP_BK);
    if (rc) return rc;
    rc = make_tmap_2d_f16(&tb, W, N, K, ldw, bn, PP_BK);
    if (rc) return rc;
    const WideKernel kern = bn == 128 ? pick_wide_kernel<128>(epi) : pick_wide_kernel<256>(epi);
    if (kern == nullptr) { set_error("gemm_f16_wide: epilogue mode %d / activation %d not built", epi.mode, epi.act); return SBK_ERR_ARG; }
    const int smem = bn == 128 ? PpCfg<128>::SMEM : PpCfg<256>::SMEM;
    SBK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    // fewest rounds of tiles per CTA with at most one CTA per SM, then as few CTAs as give that many rounds: the SMs left
    // over are free for the kernels of other streams
    int dev = 0, sms = 0;
    SBK_CUDA_CHECK(cudaGetDevice(&dev));
    SBK_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int tiles = ceil_div(M, PP_BM) * (N / bn);
    const int rounds = ceil_div(tiles, sms);
    const int grid = ceil_div(tiles, rounds);
    GemmProfile* prof = gemm_profile();
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (prof->enabled) {
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0, stream);
    }
    kern<<<grid, PP_THREADS, smem, stream>>>(ta, tb, epi, M, N, K);
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
