// Shared device helpers for the sm_90a kernels: error plumbing, tile-rect math, and thin
// wrappers over the PTX the kernels use (mbarrier, cp.async.bulk = TMA 1-D bulk copies).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/grendel_gs_b200.h"

#define GS_HD __host__ __device__ __forceinline__
#define GS_D __device__ __forceinline__

// ---- host-side error plumbing (capi.cu owns the storage) ------------------------------------
void gs_set_error(const char *fmt, ...);
#define GS_CUDA_TRY(expr)                                                                      \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            gs_set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(_e)); \
            return GS_ECUDA;                                                                   \
        }                                                                                      \
    } while (0)
#define GS_LAUNCH_CHECK() GS_CUDA_TRY(cudaGetLastError())
#define GS_REQUIRE(cond, msg)                                           \
    do {                                                                \
        if (!(cond)) {                                                  \
            gs_set_error("invalid argument: %s (%s)", msg, #cond);      \
            return GS_EINVAL;                                           \
        }                                                               \
    } while (0)

// ---- per-stage device timing (capi.cu) -------------------------------------------------------------
extern bool g_gs_profile_on;
extern int g_gs_debug_flags;  // gs_debug_set: GS_DEBUG_* bits, test-only switches
void gs_prof_mark(int stage, bool begin, cudaStream_t stream);
struct GsStageTimer {  // RAII: events around the launches of one stage when profiling is enabled
    int stage; cudaStream_t stream;
    GsStageTimer(int st, cudaStream_t s) : stage(st), stream(s) { if (g_gs_profile_on) gs_prof_mark(stage, true, stream); }
    ~GsStageTimer() { if (g_gs_profile_on) gs_prof_mark(stage, false, stream); }
};

// ---- tile rectangle of a splat ----------------------------------------------------------------
// Same IEEE fp32 operation sequence as oracle/gs_oracle.c:get_rect -> tile indices are bit-exact.
GS_D void gs_get_rect(float px, float py, int r, int gx, int gy, int &x0, int &y0, int &x1, int &y1) {
    const float rr = (float)r;
    x0 = min(gx, max(0, (int)(__fdiv_rn(__fsub_rn(px, rr), (float)GS_BLOCK_X))));
    y0 = min(gy, max(0, (int)(__fdiv_rn(__fsub_rn(py, rr), (float)GS_BLOCK_Y))));
    x1 = min(gx, max(0, (int)(__fdiv_rn(__fadd_rn(__fadd_rn(px, rr), (float)(GS_BLOCK_X - 1)), (float)GS_BLOCK_X))));
    y1 = min(gy, max(0, (int)(__fdiv_rn(__fadd_rn(__fadd_rn(py, rr), (float)(GS_BLOCK_Y - 1)), (float)GS_BLOCK_Y))));
}

// ---- the reference's ground-truth unit ---------------------------------------------------------------------------
// The reference forms its ground truth as original_image / 255.0 on a CUDA uint8 tensor (gaussian_renderer/
// loss_distribution.py:232, 938, 1469, 1833, 1933, 2107, 2224, 2269, 2561; train_internal.py:472-474; render.py:128).
// On the device torch's true division by a scalar multiplies by the scalar's fp32 reciprocal, so that value is
// fl32(g * fl32(1/255)), not the IEEE quotient fl32(g / 255): the two differ by one ulp on 126 of the 256 bytes.
GS_D float gs_gt_unit(uint8_t g) { return __fmul_rn((float)g, 1.0f / 255.0f); }

// ---- several views (cameras) binned and blended by ONE launch per stage --------------------------------
// The splats of view v are rows [start[v], start[v+1]) of the concatenated splat arrays; its tiles are
// [v*T, (v+1)*T) of the concatenated tile arrays (compute_locally, ranges) and of the sort key.  A rank that owns a
// tile-row strip of each of the B cameras of a step (workload_division.py:852-941) bins and blends all of them
// together; B = 1 is the reference's per-camera call.  Passed by value (kernel parameter space).
struct GsViews {
    int n;                          // number of views
    int T;                          // tiles per view
    int start[GS_MAX_VIEWS + 1];
};
GS_D int gs_view_of(const GsViews &v, int i) {  // largest k with start[k] <= i
    int lo = 0, hi = v.n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (v.start[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// ---- mbarrier + TMA bulk copy (cp.async.bulk) wrappers -------------------------------------------
GS_D uint32_t gs_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

GS_D void gs_mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(gs_smem_u32(bar)), "r"(count));
}
// make mbarrier.init visible to the async (TMA) proxy
GS_D void gs_fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// order generic-proxy shared-memory writes before async-proxy (TMA) reads of the same bytes
GS_D void gs_fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

GS_D void gs_mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(gs_smem_u32(bar)), "r"(bytes)
                 : "memory");
}
GS_D void gs_mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "GS_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra GS_DONE_%=;\n"
        "bra GS_WAIT_%=;\n"
        "GS_DONE_%=:\n"
        "}\n" ::"r"(gs_smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier.
// dst/src 16-byte aligned, bytes a multiple of 16.
GS_D void gs_bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     gs_smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(gs_smem_u32(bar))
                 : "memory");
}
// TMA 1-D bulk copy shared -> global (bulk-group completion).
GS_D void gs_bulk_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst),
                 "r"(gs_smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
GS_D void gs_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
GS_D void gs_bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// streaming loads/stores for data touched once
GS_D float4 gs_ldg_stream(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
