// Shared device helpers for the sm_90a kernels: mbarrier, TMA, wgmma, warp
// reductions. Hand-written PTX wrappers (no CUTLASS dependency).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define SBK_OK 0
#define SBK_ERR_CUDA -1
#define SBK_ERR_ARG -2
#define SBK_ERR_UNSUPPORTED -3
#define SBK_ERR_NOMEM -4

namespace sbk {

void set_error(const char* fmt, ...);

#define SBK_CUDA_CHECK(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            sbk::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return SBK_ERR_CUDA;                                                          \
        }                                                                                 \
    } while (0)

// returns a failed call's error code
#define RC(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

// every kernel launch goes through this: counts launches (bench.py "gpu_launches") and checks the launch
void count_launch();
#define SBK_LAUNCH_CHECK()                   \
    do {                                     \
        sbk::count_launch();                 \
        SBK_CUDA_CHECK(cudaGetLastError());  \
    } while (0)

#define SBK_REQUIRE(cond, ...)            \
    do {                                  \
        if (!(cond)) {                    \
            sbk::set_error(__VA_ARGS__);  \
            return SBK_ERR_ARG;           \
        }                                 \
    } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// SMs of the target GPU (H100 SXM): caps the grids of grid-stride kernels at a few waves
constexpr int SBK_NUM_SMS = 132;

// ---------------------------------------------------------------- programmatic dependent launch
// A kernel launched by launch_pdl may start while its predecessor in the stream is still running; pdl_wait() blocks
// until that predecessor has completed and its writes are visible (a no-op when the kernel was launched without the
// attribute).  pdl_trigger() lets the successor start launching.  Rules for the code a kernel runs before pdl_wait(),
// which may overlap not only the predecessor but, through its early trigger, kernels further back in the stream:
//   * read only data no kernel of the decode loop writes (weights, biases, LayerNorm parameters, the cross-attention
//     K/V ckv16, the fp16 encoder states enc16 the folded cross-attention reads, enc_len), and that data must come from
//     kernels that never trigger early (project_cross_kv, abs_len_kernel);
//   * write nothing to global memory: a predecessor that is still running could read the overwritten values;
//   * never read step, dx, dh16, dq16, datt16, df16, the self-attention K/V caches, logits or tokens.
// Every kernel launched this way executes pdl_wait() in at least one thread, so its completion implies its
// predecessor's, and a chain of such kernels stays ordered.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                              Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

// ---------------------------------------------------------------- warp utils
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- ldmatrix (8 x 8 fp16 tiles from shared memory)
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

// ---------------------------------------------------------------- mma.sync (warp MMA)
// D[16 x 8] += A[16 x 16] * B[8 x 16]^T, fp16 in, fp32 accumulate; a: the four A registers, b0 / b1: the two B registers
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------- cp.async (global -> shared, bypassing registers)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// copies src_bytes (0 or 16) and zero-fills the rest of the 16 bytes: src_bytes 0 writes zeros without reading src
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// 8-byte copy through L1 (.cg takes 16-byte copies only)
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// generic-proxy writes to shared memory (cp.async, st.shared) made visible to the async proxy wgmma reads through
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates (c0 = innermost element index, c1 = row index).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// 1-D bulk copy global -> shared (bytes multiple of 16, 16-byte aligned both sides).
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle, rows of 64 fp16 (128 B); 8-row groups are
// 1024 B apart (SBO).  sm_90 layout (PTX ISA "Matrix Descriptor Format"): start>>4 [0,14), LBO>>4 [16,30),
// SBO>>4 [32,46), swizzle mode [62,64) with SWIZZLE_128B = 1.
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(1) << 16;             // LBO (ignored for swizzled K-major)
    d |= static_cast<uint64_t>(1024 >> 4) << 32;     // SBO
    d |= static_cast<uint64_t>(1) << 62;             // SWIZZLE_128B
    return d;
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T for one warpgroup, both operands K-major in shared memory, fp16 in, fp32
// accumulate in registers.  Fragment of thread t (warp w = t / 32, lane l): d[4 j + 2 i + c] is row 16 w + l / 4 + 8 i,
// column 8 j + 2 (l % 4) + c.
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<256>(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t}"
        :
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}

// ---------------------------------------------------------------- fp32 -> fp16 with saturation
// F2FP.SATFINITE: values beyond +-65504 clamp to the largest finite half instead of becoming inf (and NaN one op later).
// fp16 operands were chosen for the 1e-3 parity bar (DESIGN.md 2); every activation that is stored in fp16 (LayerNorm
// outputs, FFN hidden, q/k/v, attention output, conv-module intermediates) goes through these, so an out-of-range
// activation of a trained checkpoint degrades gracefully; same cost as the plain conversion (one instruction).
__device__ __forceinline__ __half2 floats2half2_sat(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return *reinterpret_cast<__half2*>(&r);
}
__device__ __forceinline__ __half float2half_sat(float x) {
    const __half2 h = floats2half2_sat(x, 0.0f);
    return __low2half(h);
}
// the bits of floats2half2_sat(lo, hi), for 32-bit stores and mma operands
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    const __half2 h = floats2half2_sat(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// ---------------------------------------------------------------- misc math
// MUFU.EX2 + MUFU.RCP (approximate reciprocal, ~1 ulp) instead of an IEEE division: the GEMM epilogues are
// instruction-bound, and a full-precision divide costs ~8 extra instructions per element.
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// exp(x) = 2^(x log2 e) on the SFU, flush-to-zero: without -use_fast_math `__expf` wraps ex2.approx in a denormal
// range check + two scalings (5 instructions); results below 1.2e-38 are irrelevant for sigmoid / softmax weights
__device__ __forceinline__ float exp_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
    return y;
}
__device__ __forceinline__ float sigmoid_f(float x) { return rcp_approx(1.0f + exp_ftz(-x)); }
// One MUFU instead of two (EX2 + RCP): sigmoid(x) = 0.5 + 0.5 tanh(x / 2) with the hardware tanh (abs. error ~5e-4 on
// tanh, i.e. 2.5e-4 on the sigmoid: below the fp16 rounding of the value it feeds).  The SiLU / GLU GEMM epilogues were
// bound by the SFU pipe with the two-MUFU form.
__device__ __forceinline__ float tanh_approx(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(0.5f, tanh_approx(0.5f * x), 0.5f); }
__device__ __forceinline__ float silu_fast(float x) {
    const float h = 0.5f * x;
    return fmaf(h, tanh_approx(h), h);
}
// explicit shared-space 16-byte accesses (a generic pointer makes the compiler emit LD.E / ST.E with 64-bit addressing)
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint4 f4_as_u4(float4 f) {
    return make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w));
}
__device__ __forceinline__ float4 u4_as_f4(uint4 u) {
    return make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
}
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// One merge step of an arg-max, in torch.argmax's order: NaN counts as the largest value, and the lower index wins ties.
// True when (v, i) replaces (best, bi); start from (-INFINITY, INT_MAX).  A row of NaN (the logits of an utterance with no
// encoder frame) thus gives its first index, as the reference does, instead of the start index.
__device__ __forceinline__ bool argmax_takes(float v, int i, float best, int bi) {
    if (isnan(v)) return !isnan(best) || i < bi;
    return !isnan(best) && (v > best || (v == best && i < bi));
}

// ordered-int encoding so that atomicMax on int orders floats correctly
__device__ __forceinline__ int float_to_ordered(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float ordered_to_float(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF); }

// Order-preserving unsigned key of a score, for radix_select: a larger score gives a larger key, -inf the smallest, every
// NaN (whatever its sign) the largest key (argmax_takes's order), -0 the key of +0.  Key 0 is never produced.
__device__ __forceinline__ uint32_t score_key(float s) {
    if (isnan(s)) return 0xFFFFFFFFu;
    const uint32_t u = __float_as_uint(s == 0.0f ? 0.0f : s);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint64_t score_key(double s) {
    if (isnan(s)) return ~0ull;
    const uint64_t u = static_cast<uint64_t>(__double_as_longlong(s == 0.0 ? 0.0 : s));
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
// the score of a float key (the NaN key gives a NaN)
__device__ __forceinline__ float key_score(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

template <typename Key>
struct KthKey {
    Key key;    // the k-th largest key
    int ties;   // how many keys equal to it belong to the top k (the others of the top k are larger)
};

// Block-wide radix select, 8 bits per pass: the k-th largest of the nonzero keys key_of(0), ..., key_of(n - 1) (key 0:
// not a candidate; there must be at least k others).  Every thread of the block calls it.
template <typename Key, typename KeyOf>
__device__ __forceinline__ KthKey<Key> radix_select(int n, int k, KeyOf key_of) {
    __shared__ int s_hist[256];
    __shared__ int s_sel[2];
    Key prefix = 0, mask = 0;
    int rem = k;
    for (int shift = 8 * static_cast<int>(sizeof(Key)) - 8; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
        for (int u = threadIdx.x; u < n; u += blockDim.x) {
            const Key key = key_of(u);
            if (key != 0 && (key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {   // walk the bins from the top until the bin that holds the rem-th largest key
            int acc = 0, d = 255;
            for (; d > 0; --d) {
                if (acc + s_hist[d] >= rem) break;
                acc += s_hist[d];
            }
            s_sel[0] = d;
            s_sel[1] = rem - acc;
        }
        __syncthreads();
        prefix |= static_cast<Key>(s_sel[0]) << shift;
        mask |= static_cast<Key>(255) << shift;
        rem = s_sel[1];
    }
    return {prefix, rem};
}

// Host: encode a 2-D row-major fp16 tensor [rows, cols] as a TMA map with box
// [box_rows, 64 cols] and 128B swizzle. Implemented in tma_host.cu.
int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                     uint32_t box_rows, uint32_t box_cols);

}  // namespace sbk
