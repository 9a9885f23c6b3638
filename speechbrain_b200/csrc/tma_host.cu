// Host side of TMA: build CUtensorMap descriptors through the driver entry point
// (resolved at run time so the library links without libcuda on GPU-less build boxes).
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"
#include "sbk_internal.h"

namespace sbk {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }

// ---- launch accounting + optional per-GEMM timing (bench.py roofline leg)
static long long g_launches = 0;
static bool g_capturing = false;
static long long g_capture_count = 0;
void count_launch() {
    if (g_capturing) ++g_capture_count;
    else ++g_launches;
}
void launch_count_begin_capture() { g_capturing = true; g_capture_count = 0; }
long long launch_count_end_capture() { g_capturing = false; return g_capture_count; }
void launch_count_add(long long n) { g_launches += n; }
long long launch_count() { return g_launches; }

static GemmProfile g_prof;
GemmProfile* gemm_profile() { return &g_prof; }

static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    return fn;
}

int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                     uint32_t box_rows, uint32_t box_cols) {
    auto fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
        return SBK_ERR_CUDA;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_elems * 2};  // bytes, dim 1
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu stride=%llu", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)row_stride_elems);
        return SBK_ERR_CUDA;
    }
    return SBK_OK;
}

// fp32 [rows, cols] row-major, box [1, box_cols], no swizzle; OOB (incl. negative coords) reads 0.
int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_cols) {
    auto fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
        return SBK_ERR_CUDA;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {cols * 4};
    cuuint32_t box[2] = {box_cols, 1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(f32) failed (%d)", (int)r);
        return SBK_ERR_CUDA;
    }
    return SBK_OK;
}

}  // namespace sbk
