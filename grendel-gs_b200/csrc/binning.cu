// Tile binning: CUDA stages 21-24 (local tile count), 30 (scan), 40 (duplicate with keys),
// 50 (radix sort), 60 (tile ranges) of /root/reference/analyze_statistic.py:1976-1980, i.e. the
// first half of GaussianRasterizer.render_gaussians (/root/reference/gaussian_renderer/__init__.py:1271).
//
// All of this is integer / byte work bound by HBM traffic.  The scan and the sorts are CUB device
// primitives (the reference's stages 30 and 50 are CUB calls too).
//
// The published algorithm sorts R (splat, tile) instances by the 64-bit key  tile << 32 | depth bits
// (45 significant bits at 1080p = 6 onesweep passes over 12 B/instance).  The same
// order is produced here by two cheaper stable sorts:
//   1. the P splats are sorted ONCE by their 32-bit depth key (culled splats get 0xFFFFFFFF), value = splat index;
//   2. instances are emitted in that depth order with a 32-bit TILE key, and one stable radix sort over only the
//      ceil(log2 T) tile bits (2 passes over 8 B/instance) groups them by tile.
// A stable sort by depth followed by a stable sort by tile IS the stable sort by (tile, depth): the sorted id
// list, the tile ranges and hence the blend order are identical to the 64-bit sort, entry for entry
// (tests/test_gpu_parity.py::test_tile_binning_bit_exact rebuilds the 64-bit keys and compares with the oracle).
#include <cub/cub.cuh>

#include "common.cuh"
#include <atomic>
#include <cfloat>
#include <mutex>

#define BIN_THREADS 256

// Stages 21-24: per-splat number of LOCAL tiles its rectangle touches, its depth sort key, and the packed
// 48-byte record the blend kernels gather:
//   r0 = (mx, my, a', b')      a' = -A/2, b' = -B, c' = -C/2  so that  power = a'dx^2 + b'dx dy + c'dy^2
//   r1 = (c', opacity, thr, red)     thr = ln(1/(255*opacity)): power < thr  <=>  alpha < 1/255 -- THE per-pixel test of the
//                                    blend kernels (no second test on the computed alpha: the exponent decides)
//   r2 = (green, blue, ex, ey)       half extents of the bounding box of {power >= thr} (+0.5 px slack),
//                                    used by the blend kernels to cull splats per 4x4 / 8x4 pixel block
GS_D uint32_t count_local_tiles(int i, int W, int H, const float *__restrict__ means2D, const int32_t *__restrict__ radii,
                                const uint8_t *__restrict__ compute_locally, const GsViews &views) {
    const int gx = (W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    const int r = radii[i];
    uint32_t n = 0;
    if (r > 0) {
        const float2 m = *reinterpret_cast<const float2 *>(means2D + 2 * i);
        int x0, y0, x1, y1;
        gs_get_rect(m.x, m.y, r, gx, gy, x0, y0, x1, y1);
        const uint8_t *mask = compute_locally + (size_t)gs_view_of(views, i) * views.T;
        for (int y = y0; y < y1; y++) {
            const uint8_t *row = mask + y * gx;
            for (int x = x0; x < x1; x++) n += row[x] ? 1u : 0u;
        }
    }
    return n;
}

__global__ void __launch_bounds__(BIN_THREADS)
k_count_tiles(int P, int W, int H, const float *__restrict__ means2D, const float *__restrict__ conic_opacity,
              const float *__restrict__ rgb, const float *__restrict__ depths, const int32_t *__restrict__ radii,
              const uint8_t *__restrict__ compute_locally, uint32_t *__restrict__ touched,
              uint32_t *__restrict__ depth_key, uint32_t *__restrict__ index, float *__restrict__ rec, int no_cull,
              unsigned long long *__restrict__ total64, const GsViews views) {
    const int i = blockIdx.x * BIN_THREADS + threadIdx.x;
    const bool valid = i < P;
    // 64-bit instance total beside the 32-bit scan: a batch whose total reaches 2^32 would wrap the scan and pass the
    // R < 2^31 check with corrupted offsets (one atomic per warp)
    const uint32_t my_n = valid ? count_local_tiles(i, W, H, means2D, radii, compute_locally, views) : 0u;
    {   // one 64-bit atomic per CTA (per-warp atomics on one address cost 20 us at 2 M splats)
        __shared__ uint32_t s_sum[BIN_THREADS / 32];
        const uint32_t wsum = __reduce_add_sync(0xffffffffu, my_n);   // <= 32 * T: no overflow
        if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = wsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long t = 0ull;
#pragma unroll
            for (int w = 0; w < BIN_THREADS / 32; w++) t += s_sum[w];
            if (t) atomicAdd(total64, t);
        }
    }
    if (!valid) return;
    const uint32_t n = my_n;
    const float2 m = *reinterpret_cast<const float2 *>(means2D + 2 * i);
    touched[i] = n;
    // raw bits, as the published 64-bit key: for positive depths they sort like the values; -0, negative depths and
    // NaN sort after +inf, in bit order (tests/test_binning_gpu.py::test_depth_orders_bit_exact)
    depth_key[i] = n > 0 ? __float_as_uint(depths[i]) : 0xffffffffu;
    index[i] = (uint32_t)i;
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0, r2 = r0;
    if (n > 0) {
        const float4 co = *reinterpret_cast<const float4 *>(conic_opacity + 4 * i);
        const float thr = -logf(255.0f * fmaxf(co.w, 1e-30f));
        // {d : A dx^2 + 2B dx dy + C dy^2 <= -2 thr} has half extents sqrt(t C/det), sqrt(t A/det)
        // det = AC - B^2 cancels catastrophically for needle-like splats (relative error ~ulp * lambda_max/lambda_min),
        // which would shrink the box and drop real contributions: evaluate it with Kahan's FMA-compensated ab - cd,
        // exact to ~1.5 ulp, and widen the box by 2 % on top of the half-pixel slack.
        const float t = -2.f * thr;
        const float bb = co.y * co.y, bb_err = __fmaf_rn(co.y, co.y, -bb);
        const float det = __fmaf_rn(co.x, co.z, -bb) - bb_err;
        float ex = -1.f, ey = -1.f;  // never contributes
        // t == 0 is a live splat: fl(1/255) is the one opacity whose 255 o rounds to exactly 1 (thr = -0), and it lies
        // above 1/255, so the pixel on its mean (power = +0) blends it -- as the alpha >= 1/255 test does
        // a subnormal det has lost that accuracy (A = 4.2e-45, C = 0.5: det = 2.1e-45 rounds to 2.8e-45 and ey came
        // out 1 % short of the true extent): below FLT_MIN the conic is treated as degenerate, never culled
        if (t >= 0.f) {
            if (!no_cull && det >= FLT_MIN && co.x > 0.f && co.z > 0.f) {
                ex = sqrtf(t * co.z / det) * 1.02f + 0.5f;
                ey = sqrtf(t * co.x / det) * 1.02f + 0.5f;
            } else {
                ex = ey = 3.0e38f;  // degenerate conic: never cull
            }
        }
        r0 = make_float4(m.x, m.y, -0.5f * co.x, -co.y);
        r1 = make_float4(-0.5f * co.z, co.w, thr, rgb[3 * i]);
        r2 = make_float4(rgb[3 * i + 1], rgb[3 * i + 2], ex, ey);
    }
    float4 *o = reinterpret_cast<float4 *>(rec + (size_t)GS_REC_FLOATS * i);
    o[0] = r0; o[1] = r1; o[2] = r2;
}

// touched counts in depth order, as an input iterator of the inclusive scan that yields the instance offsets
struct TouchedInDepthOrder {
    const uint32_t *order, *touched;
    __host__ __device__ __forceinline__ uint32_t operator()(int s) const { return touched[order[s]]; }
};

// Stage 40: one (tile, splat id) pair per (splat, local tile), emitted in DEPTH order of the splats.
__global__ void __launch_bounds__(BIN_THREADS)
k_duplicate(int P, int W, int H, const float *__restrict__ means2D, const int32_t *__restrict__ radii,
            const uint8_t *__restrict__ compute_locally, const uint32_t *__restrict__ order,
            const uint32_t *__restrict__ offsets, uint32_t *__restrict__ tile_keys, uint32_t *__restrict__ ids,
            const GsViews views) {
    const int s = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (s >= P) return;
    uint32_t off = (s == 0) ? 0u : offsets[s - 1];
    if (offsets[s] == off) return;  // culled or no local tile
    const uint32_t i = order[s];
    const int gx = (W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    const float2 m = *reinterpret_cast<const float2 *>(means2D + 2 * (size_t)i);
    int x0, y0, x1, y1;
    gs_get_rect(m.x, m.y, radii[i], gx, gy, x0, y0, x1, y1);
    const int t0 = gs_view_of(views, (int)i) * views.T;  // first tile of this splat's view
    for (int y = y0; y < y1; y++)
        for (int x = x0; x < x1; x++) {
            const int t = t0 + y * gx + x;
            if (!compute_locally[t]) continue;
            tile_keys[off] = (uint32_t)t;
            ids[off] = i;
            off++;
        }
}

// Stage 60: [start,end) of every tile in the sorted list.  One thread per TILE finds its two boundaries by binary search
// (2 x ~23 dependent L2 reads for T = 8160 threads) instead of one thread per INSTANCE comparing neighbours (R = 5.7 M
// threads, 18 us on c2); every tile is written -- (0,0) when it is empty, as the neighbour compare left it -- so the
// ranges need no memset.
GS_D uint32_t lower_bound_u32(const uint32_t *__restrict__ keys, uint32_t n, uint32_t v) {
    uint32_t lo = 0, hi = n;   // first index with keys[index] >= v
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (__ldg(keys + mid) < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__global__ void __launch_bounds__(BIN_THREADS)
k_tile_ranges(int64_t R, int T, const uint32_t *__restrict__ tile_keys, uint32_t *__restrict__ ranges) {
    const int t = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (t >= T) return;
    const uint32_t a = lower_bound_u32(tile_keys, (uint32_t)R, (uint32_t)t);
    const uint32_t b = lower_bound_u32(tile_keys, (uint32_t)R, (uint32_t)t + 1u);
    reinterpret_cast<uint2 *>(ranges)[t] = a < b ? make_uint2(a, b) : make_uint2(0u, 0u);
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static size_t count_cub_bytes(int P) {
    size_t scan = 0, sort = 0;
    const int n = P > 0 ? P : 1;
    {
        cub::CountingInputIterator<int> idx(0);
        cub::TransformInputIterator<uint32_t, TouchedInDepthOrder, cub::CountingInputIterator<int>> in(
            idx, TouchedInDepthOrder{nullptr, nullptr});
        cub::DeviceScan::InclusiveSum(nullptr, scan, in, (uint32_t *)nullptr, n);
    }
    cub::DeviceRadixSort::SortPairs(nullptr, sort, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (const uint32_t *)nullptr, (uint32_t *)nullptr, n, 0, 32);
    return align_up(scan > sort ? scan : sort, 256);
}

// temp layout: 5 arrays of P uint32 (touched, depth_key, depth_key_sorted, index, one spare) + CUB scratch
extern "C" size_t gs_render_count_temp_bytes(int P) {
    return 5 * align_up((size_t)(P > 0 ? P : 1) * sizeof(uint32_t), 256) + count_cub_bytes(P) + 256;
}

// host copy of the view table; validates it (monotone, within GS_MAX_VIEWS)
static int make_views(int num_views, const int32_t *view_start, int T, GsViews &v) {
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views must be in [1, GS_MAX_VIEWS]");
    GS_REQUIRE(view_start != nullptr && view_start[0] == 0, "view_start[0] must be 0");
    GS_REQUIRE((long long)T * num_views < (1ll << 31), "too many tiles");
    v.n = num_views;
    v.T = T;
    for (int k = 0; k <= GS_MAX_VIEWS; k++) v.start[k] = view_start[k <= num_views ? k : num_views];
    for (int k = 0; k < num_views; k++) GS_REQUIRE(v.start[k] <= v.start[k + 1], "view_start must be non-decreasing");
    return GS_OK;
}

// The instance total travels to the host through a small ring of pinned 8-byte slots owned by the library, so that the
// launch half of the count can return before the device has produced it (the caller prepares the next launch meanwhile).
#define GS_COUNT_SLOTS 64
static unsigned long long *g_count_slots = nullptr;
static cudaEvent_t g_count_events[GS_COUNT_SLOTS];
static std::atomic<unsigned> g_count_next{0};
static std::mutex g_count_mutex;

static unsigned long long *count_slot() {
    {
        std::lock_guard<std::mutex> lock(g_count_mutex);
        if (!g_count_slots) {
            if (cudaHostAlloc((void **)&g_count_slots, GS_COUNT_SLOTS * sizeof(unsigned long long), cudaHostAllocDefault) != cudaSuccess) {
                g_count_slots = nullptr;
                return nullptr;
            }
            for (int i = 0; i < GS_COUNT_SLOTS; i++)
                if (cudaEventCreateWithFlags(&g_count_events[i], cudaEventDisableTiming) != cudaSuccess) {
                    cudaFreeHost(g_count_slots);
                    g_count_slots = nullptr;
                    return nullptr;
                }
        }
    }
    return g_count_slots + (g_count_next.fetch_add(1) % GS_COUNT_SLOTS);
}

extern "C" int gs_render_count_launch(int num_views, const int32_t *view_start, int P1, int image_height, int image_width,
                                      const float *means2D, const float *conic_opacity, const float *rgb,
                                      const float *depths, const int32_t *radii, const uint8_t *compute_locally,
                                      uint32_t *order, uint32_t *offsets, float *rec, void *temp, size_t temp_bytes,
                                      void **ticket, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    GS_REQUIRE(image_height > 0 && image_width > 0, "sizes");
    GS_REQUIRE(ticket != nullptr, "ticket");
    *ticket = nullptr;
    const int32_t one_view[2] = {0, P1};
    if (view_start == nullptr) {   // the single-camera form: one view of P1 splats
        GS_REQUIRE(num_views == 1 && P1 >= 0, "view_start may only be NULL for one view");
        view_start = one_view;
    }
    GsViews views;
    {
        const int gx = (image_width + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (image_height + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
        const int rc = make_views(num_views, view_start, gx * gy, views);
        if (rc != GS_OK) return rc;
    }
    const int P = views.start[num_views];
    unsigned long long *slot = count_slot();
    GS_REQUIRE(slot != nullptr, "pinned host slot for the instance count");
    *slot = 0ull;
    *ticket = slot;
    if (P == 0) {
        GS_CUDA_TRY(cudaEventRecord(g_count_events[slot - g_count_slots], stream));
        return GS_OK;
    }
    GS_REQUIRE(means2D && conic_opacity && rgb && depths && radii && compute_locally && order && offsets && rec && temp,
               "null pointer");
    GS_REQUIRE(((uintptr_t)rec & 15) == 0 && ((uintptr_t)conic_opacity & 15) == 0 && ((uintptr_t)means2D & 7) == 0,
               "alignment");
    if (temp_bytes < gs_render_count_temp_bytes(P)) {
        gs_set_error("gs_render_count: temp too small (%zu < %zu)", temp_bytes, gs_render_count_temp_bytes(P));
        return GS_ENOMEM;
    }
    const size_t stride = align_up((size_t)P * sizeof(uint32_t), 256);
    char *base = (char *)temp;
    uint32_t *touched = (uint32_t *)base, *dkey = (uint32_t *)(base + stride), *dkey_sorted = (uint32_t *)(base + 2 * stride),
             *index = (uint32_t *)(base + 3 * stride);
    void *cub_temp = base + 5 * stride;
    size_t cub_bytes = count_cub_bytes(P);
    unsigned long long *total64 = (unsigned long long *)(base + 5 * stride + cub_bytes);  // the last 256 bytes of temp
    GS_CUDA_TRY(cudaMemsetAsync(total64, 0, sizeof(unsigned long long), stream));
    const int grid = (P + BIN_THREADS - 1) / BIN_THREADS;
    {
        GsStageTimer timer(GS_STAGE_COUNT_TILES, stream);
        k_count_tiles<<<grid, BIN_THREADS, 0, stream>>>(P, image_width, image_height, means2D, conic_opacity, rgb, depths,
                                                        radii, compute_locally, touched, dkey, index, rec,
                                                        (g_gs_debug_flags & GS_DEBUG_NO_BLOCK_CULL) ? 1 : 0, total64, views);
        GS_LAUNCH_CHECK();
    }
    // the total is complete after the FIRST kernel: it is copied to the host now and an event marks the copy, so that
    // gs_render_count_read returns while the depth sort and the scan are still running and the caller can enqueue the
    // duplicate / sort / blend launches behind them -- the stream never runs dry behind the operator's host sync
    GS_CUDA_TRY(cudaMemcpyAsync(slot, total64, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    GS_CUDA_TRY(cudaEventRecord(g_count_events[slot - g_count_slots], stream));
    {
        GsStageTimer timer(GS_STAGE_SORT, stream);  // depth order of the splats (stable: ties keep index order)
        GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_temp, cub_bytes, dkey, dkey_sorted, index, order, P, 0, 32, stream));
    }
    {
        GsStageTimer timer(GS_STAGE_SCAN, stream);
        // the scan reads touched[order[s]] through a transform iterator: no gathered copy, no extra launch
        cub::CountingInputIterator<int> idx(0);
        cub::TransformInputIterator<uint32_t, TouchedInDepthOrder, cub::CountingInputIterator<int>> in(
            idx, TouchedInDepthOrder{order, touched});
        GS_CUDA_TRY(cub::DeviceScan::InclusiveSum(cub_temp, cub_bytes, in, offsets, P, stream));
    }
    return GS_OK;
}

extern "C" int gs_render_count_read(void *ticket, int64_t *R_host, void *stream_) {
    GS_REQUIRE(ticket != nullptr && R_host != nullptr, "ticket / R_host");
    *R_host = 0;
    (void)stream_;
    const ptrdiff_t idx = (unsigned long long *)ticket - g_count_slots;
    GS_REQUIRE(g_count_slots != nullptr && idx >= 0 && idx < GS_COUNT_SLOTS, "not a ticket of gs_render_count_launch");
    GS_CUDA_TRY(cudaEventSynchronize(g_count_events[idx]));
    const unsigned long long total = *(volatile unsigned long long *)ticket;
    if (total >= (1ull << 31)) {  // the 32-bit scan (and the int32 instance indices downstream) cannot hold it
        gs_set_error("gs_render_count: %llu splat-tile instances in one call (limit 2^31 - 1): render fewer views per call",
                     total);
        return GS_EINVAL;
    }
    *R_host = (int64_t)total;
    return GS_OK;
}

extern "C" int gs_render_count_batched(int num_views, const int32_t *view_start, int image_height, int image_width,
                                       const float *means2D, const float *conic_opacity, const float *rgb,
                                       const float *depths, const int32_t *radii, const uint8_t *compute_locally,
                                       uint32_t *order, uint32_t *offsets, float *rec, void *temp, size_t temp_bytes,
                                       int64_t *R_host, void *stream_) {
    GS_REQUIRE(R_host != nullptr, "R_host");
    *R_host = 0;
    GS_REQUIRE(view_start != nullptr, "view_start[0] must be 0");
    void *ticket = nullptr;
    const int rc = gs_render_count_launch(num_views, view_start, 0, image_height, image_width, means2D, conic_opacity, rgb,
                                          depths, radii, compute_locally, order, offsets, rec, temp, temp_bytes, &ticket,
                                          stream_);
    if (rc != GS_OK) return rc;
    return gs_render_count_read(ticket, R_host, stream_);
}

extern "C" int gs_render_count(int P, int image_height, int image_width, const float *means2D,
                               const float *conic_opacity, const float *rgb, const float *depths, const int32_t *radii,
                               const uint8_t *compute_locally, uint32_t *order, uint32_t *offsets, float *rec,
                               void *temp, size_t temp_bytes, int64_t *R_host, void *stream) {
    GS_REQUIRE(P >= 0, "sizes");
    const int32_t one_view[2] = {0, P};
    return gs_render_count_batched(1, one_view, image_height, image_width, means2D, conic_opacity, rgb, depths, radii,
                                   compute_locally, order, offsets, rec, temp, temp_bytes, R_host, stream);
}

static int tile_bits(int T) {
    int b = 0;
    while ((1ll << b) < (long long)T) b++;
    return b > 0 ? b : 1;
}

extern "C" size_t gs_render_sort_temp_bytes(int64_t R) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (const uint32_t *)nullptr, (uint32_t *)nullptr, R > 0 ? R : 1, 0, 32);
    return align_up(bytes, 256) + 256;
}

// Implemented in blend.cu
int gs_launch_blend_forward(int num_views, int64_t R, int H, int W, const float *rec, const float *bg,
                            const uint8_t *compute_locally, const uint32_t *ranges, const uint32_t *ids_sorted,
                            float *image, float *final_T, uint32_t *n_contrib, int64_t *stats, void *seg_ws,
                            size_t seg_ws_bytes, cudaStream_t stream);

extern "C" int gs_render_forward_batched(int num_views, const int32_t *view_start, int64_t R, int image_height,
                                         int image_width, const float *means2D, const int32_t *radii,
                                         const uint8_t *compute_locally, const uint32_t *order, const uint32_t *offsets,
                                         const float *rec, const float *bg, uint32_t *tiles_unsorted,
                                         uint32_t *ids_unsorted, uint32_t *tiles_sorted, uint32_t *ids_sorted,
                                         void *sort_temp, size_t sort_temp_bytes, uint32_t *ranges, float *image,
                                         float *final_T, uint32_t *n_contrib, int64_t *stats, void *seg_ws,
                                         size_t seg_ws_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    GS_REQUIRE(R >= 0 && image_height > 0 && image_width > 0, "sizes");
    GS_REQUIRE(R < (1ll << 31), "more than 2^31 splat-tile instances");
    GS_REQUIRE(compute_locally && bg && ranges && image && final_T && n_contrib, "null pointer");
    const int gx = (image_width + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (image_height + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    GsViews views;
    {
        const int rc = make_views(num_views, view_start, gx * gy, views);
        if (rc != GS_OK) return rc;
    }
    const int P = views.start[num_views];
    const int T = gx * gy * num_views;  // tiles of all views
    GS_REQUIRE(ranges != nullptr && ((uintptr_t)ranges & 7) == 0, "ranges must be 8-byte aligned");
    if (R == 0) GS_CUDA_TRY(cudaMemsetAsync(ranges, 0, sizeof(uint32_t) * 2 * (size_t)T, stream));
    if (R > 0) {
        GS_REQUIRE(means2D && radii && order && offsets && rec && tiles_unsorted && ids_unsorted && tiles_sorted &&
                       ids_sorted && sort_temp,
                   "null pointer");
        if (sort_temp_bytes < gs_render_sort_temp_bytes(R)) {
            gs_set_error("gs_render_forward: sort temp too small");
            return GS_ENOMEM;
        }
        {
            GsStageTimer timer(GS_STAGE_DUPLICATE, stream);
            k_duplicate<<<(P + BIN_THREADS - 1) / BIN_THREADS, BIN_THREADS, 0, stream>>>(
                P, image_width, image_height, means2D, radii, compute_locally, order, offsets, tiles_unsorted, ids_unsorted,
                views);
            GS_LAUNCH_CHECK();
        }
        {
            GsStageTimer timer(GS_STAGE_SORT, stream);  // stable sort on the tile bits only
            GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_temp, sort_temp_bytes, tiles_unsorted, tiles_sorted,
                                                        ids_unsorted, ids_sorted, (int)R, 0, tile_bits(T), stream));
        }
        {
            GsStageTimer timer(GS_STAGE_RANGES, stream);
            k_tile_ranges<<<(T + BIN_THREADS - 1) / BIN_THREADS, BIN_THREADS, 0, stream>>>(R, T, tiles_sorted, ranges);
            GS_LAUNCH_CHECK();
        }
    }
    return gs_launch_blend_forward(num_views, R, image_height, image_width, rec, bg, compute_locally, ranges, ids_sorted,
                                   image, final_T, n_contrib, stats, seg_ws, seg_ws_bytes, stream);
}

extern "C" int gs_render_forward(int P, int64_t R, int image_height, int image_width, const float *means2D,
                                 const int32_t *radii, const uint8_t *compute_locally, const uint32_t *order,
                                 const uint32_t *offsets, const float *rec, const float *bg, uint32_t *tiles_unsorted,
                                 uint32_t *ids_unsorted, uint32_t *tiles_sorted, uint32_t *ids_sorted, void *sort_temp,
                                 size_t sort_temp_bytes, uint32_t *ranges, float *image, float *final_T,
                                 uint32_t *n_contrib, int64_t *stats, void *seg_ws, size_t seg_ws_bytes, void *stream) {
    GS_REQUIRE(P >= 0, "sizes");
    const int32_t one_view[2] = {0, P};
    return gs_render_forward_batched(1, one_view, R, image_height, image_width, means2D, radii, compute_locally, order,
                                     offsets, rec, bg, tiles_unsorted, ids_unsorted, tiles_sorted, ids_sorted, sort_temp,
                                     sort_temp_bytes, ranges, image, final_T, n_contrib, stats, seg_ws, seg_ws_bytes, stream);
}
