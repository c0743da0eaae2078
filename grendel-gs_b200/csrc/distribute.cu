// Splat -> strip-owner routing and all-to-all staging.
//   gs_get_local2j_ids_bool        /root/reference/gaussian_renderer/workload_division.py:721-744
//   gs_get_local2j_ids_bool_rects  workload_division.py:471-484 (legacy "adjust_mode6")
//   gs_mask_scan/pack/unpack       replace the per-(destination, camera) nonzero() + index_select + cat
//                                  glue of gaussian_renderer/__init__.py:590-607,651-658
// Pure integer / byte work, HBM bound: 12 B read and world_size bytes written per splat.
#include <cstring>

#include <cub/cub.cuh>

#include "common.cuh"

#define DT_THREADS 256
#define ROW_FLOATS 11

__global__ void __launch_bounds__(DT_THREADS)
k_local2j(int P, int W, int H, int world_size, const float *__restrict__ means2D, const int32_t *__restrict__ radii,
          const int32_t *__restrict__ strategy, uint8_t *__restrict__ out) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x;
    if (i >= P) return;
    const int gx = (W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    const int r = radii[i];
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (r > 0) {
        const float2 m = *reinterpret_cast<const float2 *>(means2D + 2 * i);
        gs_get_rect(m.x, m.y, r, gx, gy, x0, y0, x1, y1);
    }
    for (int j = 0; j < world_size; j++) {
        const int lo_j = strategy[j], hi_j = strategy[j + 1];
        bool hit = false;
        if (x1 > x0)
            for (int y = y0; y < y1 && !hit; y++) hit = max(y * gx + x0, lo_j) < min(y * gx + x1, hi_j);
        out[(size_t)i * world_size + j] = hit ? 1 : 0;
    }
}

__global__ void __launch_bounds__(DT_THREADS)
k_local2j_rects(int P, int W, int H, int world_size, const float *__restrict__ means2D,
                const int32_t *__restrict__ radii, const int32_t *__restrict__ rects, uint8_t *__restrict__ out) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x;
    if (i >= P) return;
    const int gx = (W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    const int r = radii[i];
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (r > 0) {
        const float2 m = *reinterpret_cast<const float2 *>(means2D + 2 * i);
        gs_get_rect(m.x, m.y, r, gx, gy, x0, y0, x1, y1);
    }
    for (int j = 0; j < world_size; j++) {
        const int32_t *q = rects + 4 * j;
        const bool hit = r > 0 && max(y0, q[0]) < min(y1, q[1]) && max(x0, q[2]) < min(x1, q[3]);
        out[(size_t)i * world_size + j] = hit ? 1 : 0;
    }
}

extern "C" int gs_get_local2j_ids_bool(int P, int image_height, int image_width, int world_size, const float *means2D,
                                       const int32_t *radii, const int32_t *strategy, uint8_t *out, void *stream) {
    GS_REQUIRE(P >= 0 && world_size > 0 && image_height > 0 && image_width > 0, "sizes");
    if (P == 0) return GS_OK;
    GS_REQUIRE(means2D && radii && strategy && out, "null pointer");
    GsStageTimer timer(GS_STAGE_LOCAL2J, (cudaStream_t)stream);
    k_local2j<<<(P + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, (cudaStream_t)stream>>>(
        P, image_width, image_height, world_size, means2D, radii, strategy, out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

extern "C" int gs_get_local2j_ids_bool_rects(int P, int image_height, int image_width, int world_size,
                                             const float *means2D, const int32_t *radii, const int32_t *rects,
                                             uint8_t *out, void *stream) {
    GS_REQUIRE(P >= 0 && world_size > 0 && image_height > 0 && image_width > 0, "sizes");
    if (P == 0) return GS_OK;
    GS_REQUIRE(means2D && radii && rects && out, "null pointer");
    k_local2j_rects<<<(P + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, (cudaStream_t)stream>>>(
        P, image_width, image_height, world_size, means2D, radii, rects, out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// ---- all-to-all staging ---------------------------------------------------------------------
// Row = means2D(2) rgb(3) conic_opacity(4) radius-as-float depth   (gaussian_renderer/__init__.py:651-658)
// Gradient row = d means2D(2) d rgb(3) d conic_opacity(4).
// gs_route_scan: exclusive ranks of the flagged entries of a (P, ncols) byte mask in column-major order (also used
// with ncols = 1 by the sparse gradient all-reduce below).
#define GRAD_FLOATS 9
#define MAX_COLS 16

struct MaskColMajor {  // element e = c*P + i of the column-major traversal of the (P, ncols) mask
    const uint8_t *mask;
    int P, ncols;
    __host__ __device__ int32_t operator()(int e) const {
        const int c = e / P, i = e - c * P;
        return mask[(size_t)i * ncols + c] ? 1 : 0;
    }
};

struct Cols { int32_t v[MAX_COLS]; };

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" size_t gs_route_scan_temp_bytes(int P, int ncols) {
    size_t b = 0;
    const int n = (P > 0 ? P : 1) * (ncols > 0 ? ncols : 1);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t *)nullptr, (int32_t *)nullptr, n);
    return align_up(b, 256) + 256;
}

__global__ void k_colstart(int P, int ncols, const uint8_t *__restrict__ mask, const int32_t *__restrict__ gpos,
                           int32_t *__restrict__ colstart) {
    const int c = threadIdx.x;
    if (c < ncols) colstart[c] = gpos[(size_t)c * P];
    if (c == ncols) colstart[ncols] = gpos[(size_t)ncols * P - 1] + (mask[(size_t)(P - 1) * ncols + (ncols - 1)] ? 1 : 0);
}

// gpos: (ncols*P) int32, exclusive rank of every (column, splat) in the column-major flag stream;
// colstart: (ncols+1) int32, colstart[c] = gpos of column c's first element, colstart[ncols] = total flags;
// so column c holds colstart[c+1]-colstart[c] rows and splat i's row inside it is gpos[c*P+i]-colstart[c].
extern "C" int gs_route_scan(int P, int ncols, const uint8_t *mask, int32_t *gpos, int32_t *colstart, void *temp,
                             size_t temp_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    GS_REQUIRE(P >= 0 && ncols > 0 && ncols <= MAX_COLS, "sizes (at most 16 destination columns)");
    GS_REQUIRE(colstart != nullptr, "colstart");
    if (P == 0) {
        GS_CUDA_TRY(cudaMemsetAsync(colstart, 0, sizeof(int32_t) * (ncols + 1), stream));
        return GS_OK;
    }
    GS_REQUIRE(mask && gpos && temp, "null pointer");
    GS_REQUIRE((long long)P * ncols < (1ll << 31), "P*ncols overflows int32");
    cub::CountingInputIterator<int> idx(0);
    cub::TransformInputIterator<int32_t, MaskColMajor, cub::CountingInputIterator<int>> it(idx, MaskColMajor{mask, P, ncols});
    GsStageTimer timer(GS_STAGE_PACK, stream);
    GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, it, gpos, P * ncols, stream));
    k_colstart<<<1, 32, 0, stream>>>(P, ncols, mask, gpos, colstart);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// ---- batched exchange: ALL cameras of a step in one launch per stage ------------------------------------
// The per-camera calls above cost O(B) launches and Python round trips per step; with B = W = 8 that is the
// scaling limiter, not NVLink (SURVEY.md section 5.1: 5-25 k splats per (src,dst) pair, latency dominated).
// Here the flag stream is laid out [destination rank j][camera k][splat i]; ONE exclusive scan over it yields the
// row of every (j,k,i) in the send buffer directly, because that order IS the all_to_all_single send layout
// (per destination: cameras in batch order, splats in index order -- gaussian_renderer/__init__.py:590-607).
#define XB 16   // max cameras per step
#define XW 16   // max ranks
#define XSEG 128

struct XIn { const float *m2[XB]; const float *rgb[XB]; const float *co[XB]; const int32_t *rad[XB]; const float *dep[XB]; };
struct XOut { float *m2[XB]; float *rgb[XB]; float *co[XB]; int32_t *rad[XB]; float *dep[XB]; };
struct XRows { int16_t lo[XB * XW]; int16_t hi[XB * XW]; };
struct XSegs { int32_t recv_start[XSEG]; int32_t dst_start[XSEG]; uint8_t cam[XSEG]; int n; };

__global__ void __launch_bounds__(DT_THREADS)
k_xchg_flags(int B, int P, int Wr, int W, int H, XIn in, XRows rows, uint8_t *__restrict__ flags) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x, k = blockIdx.y;
    if (i >= P) return;
    const int gx = (W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    const int r = in.rad[k][i];
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (r > 0) {
        const float2 m = *reinterpret_cast<const float2 *>(in.m2[k] + 2 * i);
        gs_get_rect(m.x, m.y, r, gx, gy, x0, y0, x1, y1);
    }
    for (int j = 0; j < Wr; j++) {
        const int lo = rows.lo[k * XW + j], hi = rows.hi[k * XW + j];
        const bool hit = x1 > x0 && max(y0, lo) < min(y1, hi);
        flags[((size_t)j * B + k) * P + i] = hit ? 1 : 0;
    }
}

struct FlagToInt {
    const uint8_t *f;
    __host__ __device__ int32_t operator()(int e) const { return f[e]; }
};

__global__ void k_xchg_counts(int n_cols, int P, const uint8_t *__restrict__ flags, const int32_t *__restrict__ gpos,
                              int32_t *__restrict__ counts) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;  // column = j*B + k
    if (c >= n_cols) return;
    const size_t last = (size_t)(c + 1) * P - 1;
    const int32_t end = gpos[last] + (flags[last] ? 1 : 0);
    counts[c] = end - gpos[(size_t)c * P];
}

extern "C" size_t gs_xchg_temp_bytes(int B, int P, int W) {
    size_t b = 0;
    const long long n = (long long)(B > 0 ? B : 1) * (P > 0 ? P : 1) * (W > 0 ? W : 1);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t *)nullptr, (int32_t *)nullptr, (int)n);
    return align_up(b, 256) + 256;
}

static int fill_in(XIn &in, int B, const void *const *m2, const void *const *rgb, const void *const *co,
                   const void *const *rad, const void *const *dep) {
    for (int k = 0; k < XB; k++) {
        in.m2[k] = (k < B && m2) ? (const float *)m2[k] : nullptr;
        in.rgb[k] = (k < B && rgb) ? (const float *)rgb[k] : nullptr;
        in.co[k] = (k < B && co) ? (const float *)co[k] : nullptr;
        in.rad[k] = (k < B && rad) ? (const int32_t *)rad[k] : nullptr;
        in.dep[k] = (k < B && dep) ? (const float *)dep[k] : nullptr;
    }
    return GS_OK;
}

// row_lo_host/row_hi_host: (B*W) HOST ints, tile-row range [lo,hi) of camera k owned by rank j (lo>=hi: none).
// flags: (W*B*P) uint8, gpos: (W*B*P) int32, counts: (W*B) int32 laid out [j][k].
extern "C" int gs_xchg_route(int B, int P, int W, int image_height, int image_width,
                             const void *const *means2D_ptrs_host, const void *const *radii_ptrs_host,
                             const int32_t *row_lo_host, const int32_t *row_hi_host, uint8_t *flags, int32_t *gpos,
                             int32_t *counts, void *temp, size_t temp_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    GS_REQUIRE(B > 0 && B <= XB && W > 0 && W <= XW && P >= 0, "sizes (<= 16 cameras, <= 16 ranks)");
    GS_REQUIRE(counts != nullptr, "counts");
    if (P == 0) {
        GS_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int32_t) * B * W, stream));
        return GS_OK;
    }
    GS_REQUIRE((long long)B * P * W < (1ll << 31), "B*P*W overflows int32");
    GS_REQUIRE(means2D_ptrs_host && radii_ptrs_host && row_lo_host && row_hi_host && flags && gpos && temp, "null pointer");
    XIn in;
    fill_in(in, B, means2D_ptrs_host, nullptr, nullptr, radii_ptrs_host, nullptr);
    XRows rows;
    for (int k = 0; k < XB; k++)
        for (int j = 0; j < XW; j++) {
            const bool v = k < B && j < W;
            rows.lo[k * XW + j] = v ? (int16_t)row_lo_host[k * W + j] : 0;
            rows.hi[k * XW + j] = v ? (int16_t)row_hi_host[k * W + j] : 0;
        }
    {
        GsStageTimer timer(GS_STAGE_LOCAL2J, stream);
        dim3 grid((P + DT_THREADS - 1) / DT_THREADS, B);
        k_xchg_flags<<<grid, DT_THREADS, 0, stream>>>(B, P, W, image_width, image_height, in, rows, flags);
        GS_LAUNCH_CHECK();
    }
    GsStageTimer timer(GS_STAGE_PACK, stream);
    const int n = B * P * W;
    cub::CountingInputIterator<int> idx(0);
    cub::TransformInputIterator<int32_t, FlagToInt, cub::CountingInputIterator<int>> it(idx, FlagToInt{flags});
    GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, it, gpos, n, stream));
    k_xchg_counts<<<(B * W + 63) / 64, 64, 0, stream>>>(B * W, P, flags, gpos, counts);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

__global__ void __launch_bounds__(DT_THREADS)
k_xchg_pack(int B, int P, int Wr, XIn in, const uint8_t *__restrict__ flags, const int32_t *__restrict__ gpos,
            float *__restrict__ out) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x, k = blockIdx.y;
    if (i >= P) return;
    bool any = false;
    for (int j = 0; j < Wr; j++) any |= flags[((size_t)j * B + k) * P + i] != 0;
    if (!any) return;
    const float2 m = *reinterpret_cast<const float2 *>(in.m2[k] + 2 * i);
    const float4 co = *reinterpret_cast<const float4 *>(in.co[k] + 4 * i);
    const float r0 = in.rgb[k][3 * i], r1 = in.rgb[k][3 * i + 1], r2 = in.rgb[k][3 * i + 2];
    const float rad = (float)in.rad[k][i], dep = in.dep[k][i];
    for (int j = 0; j < Wr; j++) {
        const size_t e = ((size_t)j * B + k) * P + i;
        if (!flags[e]) continue;
        float *o = out + (size_t)gpos[e] * ROW_FLOATS;
        o[0] = m.x; o[1] = m.y; o[2] = r0; o[3] = r1; o[4] = r2;
        o[5] = co.x; o[6] = co.y; o[7] = co.z; o[8] = co.w; o[9] = rad; o[10] = dep;
    }
}

extern "C" int gs_xchg_pack(int B, int P, int W, const uint8_t *flags, const int32_t *gpos,
                            const void *const *means2D_ptrs_host, const void *const *rgb_ptrs_host,
                            const void *const *conic_opacity_ptrs_host, const void *const *radii_ptrs_host,
                            const void *const *depths_ptrs_host, float *send_rows, void *stream) {
    GS_REQUIRE(B > 0 && B <= XB && W > 0 && W <= XW && P >= 0, "sizes");
    if (P == 0) return GS_OK;
    GS_REQUIRE(flags && gpos && means2D_ptrs_host && rgb_ptrs_host && conic_opacity_ptrs_host && radii_ptrs_host &&
                   depths_ptrs_host && send_rows, "null pointer");
    XIn in;
    fill_in(in, B, means2D_ptrs_host, rgb_ptrs_host, conic_opacity_ptrs_host, radii_ptrs_host, depths_ptrs_host);
    GsStageTimer timer(GS_STAGE_PACK, (cudaStream_t)stream);
    dim3 grid((P + DT_THREADS - 1) / DT_THREADS, B);
    k_xchg_pack<<<grid, DT_THREADS, 0, (cudaStream_t)stream>>>(B, P, W, in, flags, gpos, send_rows);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

__device__ __forceinline__ int xseg_find(const XSegs &s, int r) {
    int lo = 0, hi = s.n - 1;  // last segment with recv_start <= r (empty segments share a start; any is fine
    while (lo < hi) {          // as long as r falls inside it, so prefer the LAST one that starts at or before r)
        const int mid = (lo + hi + 1) >> 1;
        if (s.recv_start[mid] <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(DT_THREADS)
k_xchg_unpack(int total, XSegs segs, const float *__restrict__ rows, XOut out) {
    const int r = blockIdx.x * DT_THREADS + threadIdx.x;
    if (r >= total) return;
    const int s = xseg_find(segs, r);
    const int k = segs.cam[s], i = segs.dst_start[s] + (r - segs.recv_start[s]);
    const float *q = rows + (size_t)r * ROW_FLOATS;
    out.m2[k][2 * i] = q[0]; out.m2[k][2 * i + 1] = q[1];
    out.rgb[k][3 * i] = q[2]; out.rgb[k][3 * i + 1] = q[3]; out.rgb[k][3 * i + 2] = q[4];
    *reinterpret_cast<float4 *>(out.co[k] + 4 * i) = make_float4(q[5], q[6], q[7], q[8]);
    out.rad[k][i] = (int32_t)q[9];
    out.dep[k][i] = q[10];
}

static int fill_segs(XSegs &s, int nseg, const int32_t *recv_start, const int32_t *seg_len, const int32_t *cam,
                     const int32_t *dst_start) {
    // keep only non-empty segments so that the binary search over recv_start is unambiguous
    GS_REQUIRE(nseg >= 0 && recv_start && seg_len && cam && dst_start, "segments");
    s.n = 0;
    for (int q = 0; q < nseg; q++) {
        if (seg_len[q] <= 0) continue;
        GS_REQUIRE(s.n < XSEG, "too many (source, camera) segments (max 128)");
        s.recv_start[s.n] = recv_start[q];
        s.dst_start[s.n] = dst_start[q];
        s.cam[s.n] = (uint8_t)cam[q];
        s.n++;
    }
    for (int q = s.n; q < XSEG; q++) { s.recv_start[q] = 0x7fffffff; s.dst_start[q] = 0; s.cam[q] = 0; }
    return GS_OK;
}

// Segments (source rank i, camera k) of the recv buffer, in recv order: first row, length, camera, first row
// inside camera k's output tensors.  All four are HOST int32 arrays of length nseg.
extern "C" int gs_xchg_unpack(int nseg, const int32_t *seg_recv_start_host, const int32_t *seg_len_host,
                              const int32_t *seg_cam_host, const int32_t *seg_dst_start_host, int total_rows,
                              const float *recv_rows, int B, void *const *means2D_ptrs_host, void *const *rgb_ptrs_host,
                              void *const *conic_opacity_ptrs_host, void *const *radii_ptrs_host,
                              void *const *depths_ptrs_host, void *stream) {
    GS_REQUIRE(B > 0 && B <= XB && total_rows >= 0, "sizes");
    if (total_rows == 0) return GS_OK;
    XSegs s;
    int rc = fill_segs(s, nseg, seg_recv_start_host, seg_len_host, seg_cam_host, seg_dst_start_host);
    if (rc != GS_OK) return rc;
    GS_REQUIRE(recv_rows && means2D_ptrs_host && rgb_ptrs_host && conic_opacity_ptrs_host && radii_ptrs_host &&
                   depths_ptrs_host, "null pointer");
    XOut out;
    for (int k = 0; k < XB; k++) {
        out.m2[k] = k < B ? (float *)means2D_ptrs_host[k] : nullptr;
        out.rgb[k] = k < B ? (float *)rgb_ptrs_host[k] : nullptr;
        out.co[k] = k < B ? (float *)conic_opacity_ptrs_host[k] : nullptr;
        out.rad[k] = k < B ? (int32_t *)radii_ptrs_host[k] : nullptr;
        out.dep[k] = k < B ? (float *)depths_ptrs_host[k] : nullptr;
    }
    GsStageTimer timer(GS_STAGE_UNPACK, (cudaStream_t)stream);
    k_xchg_unpack<<<(total_rows + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, (cudaStream_t)stream>>>(total_rows, s,
                                                                                                       recv_rows, out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// backward of unpack: per-camera gradients -> 9-float rows in recv order (a camera without gradient: NULL -> zeros)
__global__ void __launch_bounds__(DT_THREADS)
k_xchg_pack_grad(int total, XSegs segs, XIn g, float *__restrict__ rows) {
    const int r = blockIdx.x * DT_THREADS + threadIdx.x;
    if (r >= total) return;
    const int s = xseg_find(segs, r);
    const int k = segs.cam[s], i = segs.dst_start[s] + (r - segs.recv_start[s]);
    float *q = rows + (size_t)r * GRAD_FLOATS;
    float v[GRAD_FLOATS];
#pragma unroll
    for (int t = 0; t < GRAD_FLOATS; t++) v[t] = 0.f;
    if (g.m2[k]) { v[0] = g.m2[k][2 * i]; v[1] = g.m2[k][2 * i + 1]; }
    if (g.rgb[k]) { v[2] = g.rgb[k][3 * i]; v[3] = g.rgb[k][3 * i + 1]; v[4] = g.rgb[k][3 * i + 2]; }
    if (g.co[k]) {
        const float4 c = *reinterpret_cast<const float4 *>(g.co[k] + 4 * i);
        v[5] = c.x; v[6] = c.y; v[7] = c.z; v[8] = c.w;
    }
#pragma unroll
    for (int t = 0; t < GRAD_FLOATS; t++) q[t] = v[t];
}

extern "C" int gs_xchg_pack_grad(int nseg, const int32_t *seg_recv_start_host, const int32_t *seg_len_host,
                                 const int32_t *seg_cam_host, const int32_t *seg_dst_start_host, int total_rows, int B,
                                 const void *const *d_means2D_ptrs_host, const void *const *d_rgb_ptrs_host,
                                 const void *const *d_conic_opacity_ptrs_host, float *grad_rows, void *stream) {
    GS_REQUIRE(B > 0 && B <= XB && total_rows >= 0, "sizes");
    if (total_rows == 0) return GS_OK;
    XSegs s;
    int rc = fill_segs(s, nseg, seg_recv_start_host, seg_len_host, seg_cam_host, seg_dst_start_host);
    if (rc != GS_OK) return rc;
    GS_REQUIRE(grad_rows && d_means2D_ptrs_host && d_rgb_ptrs_host && d_conic_opacity_ptrs_host, "null pointer");
    XIn g;
    fill_in(g, B, d_means2D_ptrs_host, d_rgb_ptrs_host, d_conic_opacity_ptrs_host, nullptr, nullptr);
    GsStageTimer timer(GS_STAGE_UNPACK, (cudaStream_t)stream);
    k_xchg_pack_grad<<<(total_rows + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, (cudaStream_t)stream>>>(total_rows, s,
                                                                                                          g, grad_rows);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// backward of pack: every (camera, local splat) sums the gradient rows returned by the ranks it was sent to
__global__ void __launch_bounds__(DT_THREADS)
k_xchg_scatter_grad(int B, int P, int Wr, const uint8_t *__restrict__ flags, const int32_t *__restrict__ gpos,
                    const float *__restrict__ rows, XOut d) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x, k = blockIdx.y;
    if (i >= P) return;
    float a[GRAD_FLOATS];
#pragma unroll
    for (int q = 0; q < GRAD_FLOATS; q++) a[q] = 0.f;
    for (int j = 0; j < Wr; j++) {
        const size_t e = ((size_t)j * B + k) * P + i;
        if (!flags[e]) continue;
        const float *r = rows + (size_t)gpos[e] * GRAD_FLOATS;
#pragma unroll
        for (int q = 0; q < GRAD_FLOATS; q++) a[q] += r[q];
    }
    d.m2[k][2 * i] = a[0]; d.m2[k][2 * i + 1] = a[1];
    d.rgb[k][3 * i] = a[2]; d.rgb[k][3 * i + 1] = a[3]; d.rgb[k][3 * i + 2] = a[4];
    *reinterpret_cast<float4 *>(d.co[k] + 4 * i) = make_float4(a[5], a[6], a[7], a[8]);
}

extern "C" int gs_xchg_scatter_grad(int B, int P, int W, const uint8_t *flags, const int32_t *gpos,
                                    const float *grad_rows, void *const *d_means2D_ptrs_host,
                                    void *const *d_rgb_ptrs_host, void *const *d_conic_opacity_ptrs_host, void *stream) {
    GS_REQUIRE(B > 0 && B <= XB && W > 0 && W <= XW && P >= 0, "sizes");
    if (P == 0) return GS_OK;
    GS_REQUIRE(flags && gpos && grad_rows && d_means2D_ptrs_host && d_rgb_ptrs_host && d_conic_opacity_ptrs_host,
               "null pointer");
    XOut d;
    for (int k = 0; k < XB; k++) {
        d.m2[k] = k < B ? (float *)d_means2D_ptrs_host[k] : nullptr;
        d.rgb[k] = k < B ? (float *)d_rgb_ptrs_host[k] : nullptr;
        d.co[k] = k < B ? (float *)d_conic_opacity_ptrs_host[k] : nullptr;
        d.rad[k] = nullptr; d.dep[k] = nullptr;
    }
    GsStageTimer timer(GS_STAGE_PACK, (cudaStream_t)stream);
    dim3 grid((P + DT_THREADS - 1) / DT_THREADS, B);
    k_xchg_scatter_grad<<<grid, DT_THREADS, 0, (cudaStream_t)stream>>>(B, P, W, flags, gpos, grad_rows, d);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// ---- NVLink peer memory for the direct-placement exchange below ---------------------------------------------------
// all_to_all_single moves a rank's rows through NCCL's point-to-point channels: two device copies (pack into the send
// buffer, NCCL from there into the peer's receive buffer) and a few channels per peer pair, far above the NVLink wire
// time of the rows.  Here every rank's receive region and gradient region are cudaMalloc allocations exported through
// CUDA IPC and mapped by all peers: the pack kernel stores each splat straight into its final row of the destination's
// receive region, and the backward loads the gradient rows straight from the destinations' gradient regions.
// Ordering: the host enqueues a 4-byte all-reduce after the kernel; it completes on a rank once every peer's kernel has
// finished, so the consumer that follows it in stream order sees all rows.  Buffers are reused every step: a peer only
// writes after it has received this rank's counts of the NEXT step, which this rank sends after its consumers ran.
extern "C" int gs_peer_alloc(size_t bytes, void **dev_ptr, void *ipc_handle_64) {
    GS_REQUIRE(bytes > 0 && dev_ptr && ipc_handle_64, "arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    void *p = nullptr;
    GS_CUDA_TRY(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        gs_set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
        return GS_ECUDA;
    }
    memcpy(ipc_handle_64, &h, 64);
    *dev_ptr = p;
    return GS_OK;
}

extern "C" int gs_peer_open(const void *ipc_handle_64, void **peer_ptr) {
    GS_REQUIRE(ipc_handle_64 && peer_ptr, "arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle_64, 64);
    GS_CUDA_TRY(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return GS_OK;
}

extern "C" int gs_peer_close(void *peer_ptr) {
    if (peer_ptr) GS_CUDA_TRY(cudaIpcCloseMemHandle(peer_ptr));
    return GS_OK;
}

extern "C" int gs_peer_free(void *dev_ptr) {
    if (dev_ptr) GS_CUDA_TRY(cudaFree(dev_ptr));
    return GS_OK;
}

// ---- sparse per-Gaussian gradient all-reduce staging (replicated-Gaussian data parallelism) ------------------
// /root/reference/scene/gaussian_model.py:1332-1391 (get_sparse_ids / sync_gradients_sparsely): rows whose
// _xyz.grad is non-zero on ANY rank are compacted, all-reduced and scattered back -- per parameter, i.e. 1 + 6
// collectives and 12 gather/scatter kernels.  Here the six gradients of a touched Gaussian travel as ONE row of
// 14 + rest = 11 + 3 K floats (xyz 3, features_dc 3, features_rest rest = 3 (K - 1): 45 at the default max_sh_degree
// 3, scaling 3, rotation 4, opacity 1), so the step is: mask kernel -> all-reduce(MAX) of the byte mask -> scan ->
// pack -> ONE all-reduce(SUM) -> unpack.  (The reference lists this "fused_sparse" mode as NotImplemented,
// gaussian_model.py:1438-1439.)
#define SG_FIXED_FLOATS 14   // xyz, features_dc, scaling, rotation, opacity

__global__ void __launch_bounds__(DT_THREADS)
k_sparse_mask(int P, const float *__restrict__ xyz_grad, uint8_t *__restrict__ mask) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x;
    if (i >= P) return;
    mask[i] = (xyz_grad[3 * i] != 0.f || xyz_grad[3 * i + 1] != 0.f || xyz_grad[3 * i + 2] != 0.f) ? 1 : 0;
}

extern "C" int gs_sparse_grad_mask(int P, const float *xyz_grad, uint8_t *mask, void *stream) {
    GS_REQUIRE(P >= 0, "P");
    if (P == 0) return GS_OK;
    GS_REQUIRE(xyz_grad && mask, "null pointer");
    k_sparse_mask<<<(P + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, (cudaStream_t)stream>>>(P, xyz_grad, mask);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

struct SgPtrs { float *p[6]; };

template <bool PACK>
__global__ void __launch_bounds__(DT_THREADS)
k_sparse_rows(int P, int rest, const uint8_t *__restrict__ mask, const int32_t *__restrict__ pos, SgPtrs g,
              float *__restrict__ rows) {
    const int i = blockIdx.x * DT_THREADS + threadIdx.x;
    if (i >= P || !mask[i]) return;
    float *r = rows + (size_t)pos[i] * (SG_FIXED_FLOATS + rest);
    const int width[6] = {3, 3, rest, 3, 4, 1};
    int o = 0;
#pragma unroll
    for (int t = 0; t < 6; t++) {
        float *src = g.p[t] + (size_t)i * width[t];
        for (int q = 0; q < width[t]; q++) {
            if (PACK) r[o + q] = src[q]; else src[q] = r[o + q];
        }
        o += width[t];
    }
}

template <bool PACK>
static int sparse_rows(int P, int rest_floats, const uint8_t *mask, const int32_t *pos, void *const *grads_host,
                       float *rows, void *stream) {
    GS_REQUIRE(P >= 0, "P");
    GS_REQUIRE(rest_floats == 0 || rest_floats == 9 || rest_floats == 24 || rest_floats == 45,
               "rest_floats must be 3 ((max_sh_degree + 1)^2 - 1): 0, 9, 24 or 45");
    if (P == 0) return GS_OK;
    GS_REQUIRE(mask && pos && grads_host && rows, "null pointer");
    SgPtrs g;
    for (int t = 0; t < 6; t++) {
        g.p[t] = (float *)grads_host[t];
        GS_REQUIRE(g.p[t] != nullptr || (t == 2 && rest_floats == 0), "null gradient");
    }
    k_sparse_rows<PACK><<<(P + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, (cudaStream_t)stream>>>(
        P, rest_floats, mask, pos, g, rows);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// grads_host: HOST array of the six device gradient pointers in GaussianModel order
// (_xyz, _features_dc, _features_rest, _scaling, _rotation, _opacity); pos: exclusive scan of mask (gs_route_scan
// with ncols = 1); rows: (n_touched, 14 + rest_floats).
extern "C" int gs_sparse_grad_pack_rows(int P, int rest_floats, const uint8_t *mask, const int32_t *pos,
                                        void *const *grads_host, float *rows, void *stream) {
    return sparse_rows<true>(P, rest_floats, mask, pos, grads_host, rows, stream);
}

extern "C" int gs_sparse_grad_unpack_rows(int P, int rest_floats, const uint8_t *mask, const int32_t *pos,
                                          const float *rows, void *const *grads_host, void *stream) {
    return sparse_rows<false>(P, rest_floats, mask, pos, grads_host, const_cast<float *>(rows), stream);
}

extern "C" int gs_sparse_grad_pack(int P, const uint8_t *mask, const int32_t *pos, void *const *grads_host,
                                   float *rows, void *stream) {
    return gs_sparse_grad_pack_rows(P, 45, mask, pos, grads_host, rows, stream);
}

extern "C" int gs_sparse_grad_unpack(int P, const uint8_t *mask, const int32_t *pos, const float *rows,
                                     void *const *grads_host, void *stream) {
    return gs_sparse_grad_unpack_rows(P, 45, mask, pos, rows, grads_host, stream);
}

// ---- direct-placement exchange ---------------------------------------------------------------------------------------
// The row-staged exchange above materialises a dense [destination][camera][splat] flag array, a W*B*P-element scan
// (64 MB of positions at W = B = 8), a row-major staging layout and an unpack pass on the receiver, all of it traffic
// the rows themselves do not need.  Here:
//   * routing is recomputed from (means2D, radius) wherever it is needed (12 B per splat) instead of being stored;
//   * positions come from per-CTA hit counts ([destination][camera][block of 256 splats]: W*B*P/256 integers, scanned
//     in microseconds) plus a ballot prefix inside the CTA -- the order is still the reference's (per destination:
//     cameras in batch order, splats in index order; per receiver: sources in rank order);
//   * the pack kernel stores every field straight into its FINAL place in the destination rank's structure-of-arrays
//     receive region (means2D | rgb | conic_opacity | radii | depths, `cap` rows each), i.e. the tensors the render reads:
//     no staging rows, no unpack;
//   * backward, the source PULLS: the receiver's render backward leaves its gradients in its own peer-visible region
//     (d means2D | d rgb | d conic_opacity) and the owner of a splat loads the rows of its (at most few) destinations over
//     NVLink and sums them -- no pack kernel on the receiver, no atomics.
#define XR_NB(P) (((P) + DT_THREADS - 1) / DT_THREADS)

struct XrGeom {           // what a rank needs to recompute "which strip owners does splat i of camera k reach"
    const float *m2[XB];
    const int32_t *rad[XB];
    XRows rows;
    int B, P, Wr, W, H;
};
struct XrPeers { char *base[XW]; int32_t row0[XW * XB]; long long cap; };  // row0[j*B+k]: my first row in rank j's camera k

GS_D uint32_t xr_hits(const XrGeom &g, int k, int i, bool valid) {
    if (!valid) return 0u;
    const int r = g.rad[k][i];
    if (r <= 0) return 0u;
    const int gx = (g.W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (g.H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    int x0, y0, x1, y1;
    const float2 m = *reinterpret_cast<const float2 *>(g.m2[k] + 2 * (size_t)i);
    gs_get_rect(m.x, m.y, r, gx, gy, x0, y0, x1, y1);
    uint32_t h = 0u;
    if (x1 > x0)
        for (int j = 0; j < g.Wr; j++)
            if (max(y0, (int)g.rows.lo[k * XW + j]) < min(y1, (int)g.rows.hi[k * XW + j])) h |= 1u << j;
    return h;
}

__global__ void __launch_bounds__(DT_THREADS)
k_xr_count(XrGeom g, int32_t *__restrict__ blkcnt) {
    __shared__ int32_t s_cnt[DT_THREADS / 32][XW];
    const int i = blockIdx.x * DT_THREADS + threadIdx.x, k = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t h = xr_hits(g, k, i, i < g.P);
    for (int j = 0; j < g.Wr; j++) {
        const int c = __popc(__ballot_sync(0xffffffffu, (h >> j) & 1u));
        if (lane == 0) s_cnt[warp][j] = c;
    }
    __syncthreads();
    if ((int)threadIdx.x < g.Wr) {
        int c = 0;
#pragma unroll
        for (int w = 0; w < DT_THREADS / 32; w++) c += s_cnt[w][threadIdx.x];
        blkcnt[((size_t)threadIdx.x * g.B + k) * gridDim.x + blockIdx.x] = c;
    }
}

__global__ void k_xr_totals(int n_cols, int NB, const int32_t *__restrict__ blkcnt, const int32_t *__restrict__ blkbase,
                            int32_t *__restrict__ counts) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;  // column = j*B + k
    if (c >= n_cols) return;
    const size_t last = (size_t)(c + 1) * NB - 1;
    counts[c] = blkbase[last] + blkcnt[last] - blkbase[(size_t)c * NB];
}

// per-CTA position of this thread's row for destination j: rows of the CTA's hits in thread order
struct XrRank { int32_t warp_base[DT_THREADS / 32]; };
GS_D int xr_local_rank(uint32_t h, int j, int warp, int lane, int32_t (*s_wcnt)[XW]) {
    const uint32_t b = __ballot_sync(0xffffffffu, (h >> j) & 1u);
    int r = __popc(b & ((1u << lane) - 1u));
    for (int w = 0; w < warp; w++) r += s_wcnt[w][j];
    return r;
}

// Destination rows computed ON THE DEVICE from the all-gathered counts cnt[i][k][j] (source, camera, destination), so that the
// pack kernel can be enqueued before the host has read the counts (exchange.direct_rows is the host restatement):
//   row0[j*B+k] = sum_{k' < k} sum_i cnt[i][k'][j]  +  sum_{i < me} cnt[i][k][j];   row0[W*B] = 1 if some rank would receive
// more than `cap` rows (then the pack writes nothing and every rank -- same counts, same decision -- takes the fallback).
__global__ void k_xr_rows(int W, int B, int me, const int32_t *__restrict__ cnt, long long cap, int32_t *__restrict__ row0) {
    const int c = threadIdx.x;
    if (c < W * B) {
        const int j = c / B, k = c % B;
        long long r = 0;
        for (int kk = 0; kk < k; kk++)
            for (int i = 0; i < W; i++) r += cnt[((size_t)i * B + kk) * W + j];
        for (int i = 0; i < me; i++) r += cnt[((size_t)i * B + k) * W + j];
        row0[c] = (int32_t)r;
    }
    if (c == 0) {
        int over = 0;
        for (int j = 0; j < W; j++) {
            long long t = 0;
            for (int i = 0; i < W; i++)
                for (int k = 0; k < B; k++) t += cnt[((size_t)i * B + k) * W + j];
            if (t > cap) over = 1;
        }
        row0[W * B] = over;
    }
}

__global__ void __launch_bounds__(DT_THREADS)
k_xr_pack(XrGeom g, XIn in, const int32_t *__restrict__ blkbase, XrPeers peers, const int32_t *__restrict__ row0_dev) {
    __shared__ int32_t s_wcnt[DT_THREADS / 32][XW];
    __shared__ float s_rgb[DT_THREADS / 32][96];
    if (row0_dev[g.Wr * g.B] != 0) return;   // over capacity: nothing is written (uniform)
    const int i = blockIdx.x * DT_THREADS + threadIdx.x, k = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool valid = i < g.P;
    const uint32_t h = xr_hits(g, k, i, valid);
    uint32_t any = __reduce_or_sync(0xffffffffu, h);
    for (int j = 0; j < g.Wr; j++) {
        const int c = __popc(__ballot_sync(0xffffffffu, (h >> j) & 1u));
        if (lane == 0) s_wcnt[warp][j] = c;
    }
    __syncthreads();
    if (any == 0u) return;
    float2 m = make_float2(0.f, 0.f);
    float4 co = make_float4(0.f, 0.f, 0.f, 0.f);
    float r0 = 0.f, r1 = 0.f, r2 = 0.f, dep = 0.f;
    int rad = 0;
    if (h) {
        m = *reinterpret_cast<const float2 *>(in.m2[k] + 2 * (size_t)i);
        co = *reinterpret_cast<const float4 *>(in.co[k] + 4 * (size_t)i);
        r0 = in.rgb[k][3 * (size_t)i]; r1 = in.rgb[k][3 * (size_t)i + 1]; r2 = in.rgb[k][3 * (size_t)i + 2];
        rad = in.rad[k][i]; dep = in.dep[k][i];
    }
    const long long cap = peers.cap;
    while (any) {
        const int j = __ffs(any) - 1;
        any &= any - 1u;
        // the warp's hits for destination j are consecutive rows: every field is one contiguous span, written with
        // consecutive lanes on consecutive addresses (rgb, 12 B per row, goes through a shared-memory transpose: strided
        // 4-byte stores are partial sectors on NVLink).  Visibility to the peer: kernel completion + the stream-ordered
        // barrier the caller enqueues -- no per-thread system fence.
        const uint32_t bal = __ballot_sync(0xffffffffu, (h >> j) & 1u);
        const int wr = __popc(bal & ((1u << lane) - 1u)), wn = __popc(bal);
        int lr = wr;
        for (int w = 0; w < warp; w++) lr += s_wcnt[w][j];
        const bool hit = (h >> j) & 1u;
        const size_t col = (size_t)j * g.B + k;
        const long long row = (long long)row0_dev[col] + (blkbase[col * gridDim.x + blockIdx.x] - blkbase[col * gridDim.x]) + lr;
        float *b = reinterpret_cast<float *>(peers.base[j]);
        if (hit) {
            *reinterpret_cast<float2 *>(b + 2 * row) = m;
            *reinterpret_cast<float4 *>(b + 5 * cap + 4 * row) = co;
            reinterpret_cast<int32_t *>(b + 9 * cap)[row] = rad;
            (b + 10 * cap)[row] = dep;
            s_rgb[warp][3 * wr] = r0; s_rgb[warp][3 * wr + 1] = r1; s_rgb[warp][3 * wr + 2] = r2;
        }
        const long long row_w = __shfl_sync(0xffffffffu, row - wr, __ffs(bal) - 1);   // first row of the warp's span
        __syncwarp();
        float *q = b + 2 * cap + 3 * row_w;
        for (int t = lane; t < 3 * wn; t += 32) q[t] = s_rgb[warp][t];
        __syncwarp();
    }
}

__global__ void __launch_bounds__(DT_THREADS)
k_xr_pull_grad(XrGeom g, const int32_t *__restrict__ blkbase, XrPeers peers, XOut out) {
    __shared__ int32_t s_wcnt[DT_THREADS / 32][XW];
    const int i = blockIdx.x * DT_THREADS + threadIdx.x, k = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool valid = i < g.P;
    const uint32_t h = xr_hits(g, k, i, valid);
    uint32_t any = __reduce_or_sync(0xffffffffu, h);
    for (int j = 0; j < g.Wr; j++) {
        const int c = __popc(__ballot_sync(0xffffffffu, (h >> j) & 1u));
        if (lane == 0) s_wcnt[warp][j] = c;
    }
    __syncthreads();
    float2 dm = make_float2(0.f, 0.f);
    float4 dco = make_float4(0.f, 0.f, 0.f, 0.f);
    float d0 = 0.f, d1 = 0.f, d2 = 0.f;
    const long long cap = peers.cap;
    while (any) {   // ascending destination rank: the summation order of the reference's index_add over received blocks
        const int j = __ffs(any) - 1;
        any &= any - 1u;
        const int lr = xr_local_rank(h, j, warp, lane, s_wcnt);
        if (!((h >> j) & 1u)) continue;
        const size_t col = (size_t)j * g.B + k;
        const long long row = (long long)peers.row0[col] + (blkbase[col * gridDim.x + blockIdx.x] - blkbase[col * gridDim.x]) + lr;
        const float *b = reinterpret_cast<const float *>(peers.base[j]);
        const float2 a = *reinterpret_cast<const float2 *>(b + 2 * row);
        const float4 q = *reinterpret_cast<const float4 *>(b + 2 * cap + 4 * row);   // d rgb, padded to 16 B per row
        const float4 c = *reinterpret_cast<const float4 *>(b + 6 * cap + 4 * row);
        dm.x += a.x; dm.y += a.y;
        d0 += q.x; d1 += q.y; d2 += q.z;
        dco.x += c.x; dco.y += c.y; dco.z += c.z; dco.w += c.w;
    }
    if (valid) {
        *reinterpret_cast<float2 *>(out.m2[k] + 2 * (size_t)i) = dm;
        float *q = out.rgb[k] + 3 * (size_t)i;
        q[0] = d0; q[1] = d1; q[2] = d2;
        *reinterpret_cast<float4 *>(out.co[k] + 4 * (size_t)i) = dco;
    }
}

static int xr_geom(XrGeom &g, int B, int P, int W, int H, int Wimg, const void *const *m2, const void *const *rad,
                   const int32_t *row_lo, const int32_t *row_hi) {
    GS_REQUIRE(B > 0 && B <= XB && W > 0 && W <= XW && P >= 0, "sizes (<= 16 cameras, <= 16 ranks)");
    GS_REQUIRE(H > 0 && Wimg > 0 && m2 && rad && row_lo && row_hi, "geometry");
    g.B = B; g.P = P; g.Wr = W; g.W = Wimg; g.H = H;
    for (int k = 0; k < XB; k++) {
        g.m2[k] = k < B ? (const float *)m2[k] : nullptr;
        g.rad[k] = k < B ? (const int32_t *)rad[k] : nullptr;
        for (int j = 0; j < XW; j++) {
            const bool v = k < B && j < W;
            g.rows.lo[k * XW + j] = v ? (int16_t)row_lo[k * W + j] : 0;
            g.rows.hi[k * XW + j] = v ? (int16_t)row_hi[k * W + j] : 0;
        }
    }
    return GS_OK;
}

static int xr_peers(XrPeers &p, int B, int W, void *const *bases, const int32_t *row0, long long cap) {
    GS_REQUIRE(bases && row0 && cap > 0 && (cap & 3) == 0, "peer tables (capacity must be a multiple of 4 rows)");
    p.cap = cap;
    for (int j = 0; j < XW; j++) {
        p.base[j] = j < W ? (char *)bases[j] : nullptr;
        GS_REQUIRE(j >= W || p.base[j] != nullptr, "null peer buffer");
    }
    for (int c = 0; c < XW * XB; c++) p.row0[c] = c < W * B ? row0[c] : 0;
    return GS_OK;
}

extern "C" size_t gs_xr_temp_bytes(int B, int P, int W) {
    size_t b = 0;
    const long long n = (long long)(B > 0 ? B : 1) * (W > 0 ? W : 1) * XR_NB(P > 0 ? P : 1);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t *)nullptr, (int32_t *)nullptr, (int)n);
    return align_up(b, 256) + 256;
}

// blkcnt, blkbase: (W*B*ceil(P/256)) int32 each, laid out [destination j][camera k][block]; counts: (W*B) int32 [j][k].
extern "C" int gs_xr_count(int B, int P, int W, int image_height, int image_width, const void *const *means2D_ptrs_host,
                           const void *const *radii_ptrs_host, const int32_t *row_lo_host, const int32_t *row_hi_host,
                           int32_t *blkcnt, int32_t *blkbase, int32_t *counts, void *temp, size_t temp_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    XrGeom g;
    int rc = xr_geom(g, B, P, W, image_height, image_width, means2D_ptrs_host, radii_ptrs_host, row_lo_host, row_hi_host);
    if (rc != GS_OK) return rc;
    GS_REQUIRE(counts != nullptr, "counts");
    if (P == 0) {
        GS_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int32_t) * B * W, stream));
        return GS_OK;
    }
    GS_REQUIRE(blkcnt && blkbase && temp, "null pointer");
    const int NB = XR_NB(P);
    GsStageTimer timer(GS_STAGE_LOCAL2J, stream);
    k_xr_count<<<dim3(NB, B), DT_THREADS, 0, stream>>>(g, blkcnt);
    GS_LAUNCH_CHECK();
    GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, blkcnt, blkbase, W * B * NB, stream));
    k_xr_totals<<<(B * W + 63) / 64, 64, 0, stream>>>(B * W, NB, blkcnt, blkbase, counts);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// peer_recv_ptrs_host[j]: rank j's receive region (11 * cap floats: means2D | rgb | conic_opacity | radii | depths) as
// mapped into this process.  The destination rows are computed on the device: counts_all_dev = the all-gathered counts
// (W*B*W int32, [source i][camera k][destination j], as all_gather_into_tensor of every rank's (B,W) table leaves them),
// me = this rank, row0_dev = (W*B + 1) int32 scratch that receives the rows and the over-capacity flag.  The caller needs
// no host copy of the counts to launch it: the launch goes out right behind the all-gather and the host reads the
// counts while it runs.
extern "C" int gs_xr_pack_dev(int B, int P, int W, int image_height, int image_width, const void *const *means2D_ptrs_host,
                              const void *const *rgb_ptrs_host, const void *const *conic_opacity_ptrs_host,
                              const void *const *radii_ptrs_host, const void *const *depths_ptrs_host,
                              const int32_t *row_lo_host, const int32_t *row_hi_host, const int32_t *blkbase,
                              void *const *peer_recv_ptrs_host, const int32_t *counts_all_dev, int me, int32_t *row0_dev,
                              long long cap_rows, void *stream) {
    XrGeom g;
    int rc = xr_geom(g, B, P, W, image_height, image_width, means2D_ptrs_host, radii_ptrs_host, row_lo_host, row_hi_host);
    if (rc != GS_OK) return rc;
    GS_REQUIRE(counts_all_dev && row0_dev && me >= 0 && me < W, "device counts / row table / rank");
    GS_REQUIRE(W * B <= 256, "W * B <= 256");
    XrPeers peers;
    int32_t zeros[XW * XB] = {0};   // k_xr_pack reads its rows from row0_dev
    rc = xr_peers(peers, B, W, peer_recv_ptrs_host, zeros, cap_rows);
    if (rc != GS_OK) return rc;
    k_xr_rows<<<1, 256, 0, (cudaStream_t)stream>>>(W, B, me, counts_all_dev, cap_rows, row0_dev);
    GS_LAUNCH_CHECK();
    if (P == 0) return GS_OK;
    GS_REQUIRE(rgb_ptrs_host && conic_opacity_ptrs_host && depths_ptrs_host && blkbase, "null pointer");
    XIn in;
    fill_in(in, B, means2D_ptrs_host, rgb_ptrs_host, conic_opacity_ptrs_host, radii_ptrs_host, depths_ptrs_host);
    GsStageTimer timer(GS_STAGE_PACK, (cudaStream_t)stream);
    k_xr_pack<<<dim3(XR_NB(P), B), DT_THREADS, 0, (cudaStream_t)stream>>>(g, in, blkbase, peers, row0_dev);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// peer_grad_ptrs_host[j]: rank j's gradient region (10 * cap floats: d means2D (2) | d rgb padded to 4 | d conic_opacity (4)); the outputs
// are the (B,P,.) gradients of this rank's projected splats: the sum over the destinations each splat was sent to.
extern "C" int gs_xr_pull_grad(int B, int P, int W, int image_height, int image_width, const void *const *means2D_ptrs_host,
                               const void *const *radii_ptrs_host, const int32_t *row_lo_host, const int32_t *row_hi_host,
                               const int32_t *blkbase, void *const *peer_grad_ptrs_host, const int32_t *dst_row0_host,
                               long long cap_rows, void *const *d_means2D_ptrs_host, void *const *d_rgb_ptrs_host,
                               void *const *d_conic_opacity_ptrs_host, void *stream) {
    XrGeom g;
    int rc = xr_geom(g, B, P, W, image_height, image_width, means2D_ptrs_host, radii_ptrs_host, row_lo_host, row_hi_host);
    if (rc != GS_OK) return rc;
    if (P == 0) return GS_OK;
    GS_REQUIRE(blkbase && d_means2D_ptrs_host && d_rgb_ptrs_host && d_conic_opacity_ptrs_host, "null pointer");
    XrPeers peers;
    rc = xr_peers(peers, B, W, peer_grad_ptrs_host, dst_row0_host, cap_rows);
    if (rc != GS_OK) return rc;
    XOut out;
    for (int k = 0; k < XB; k++) {
        out.m2[k] = k < B ? (float *)d_means2D_ptrs_host[k] : nullptr;
        out.rgb[k] = k < B ? (float *)d_rgb_ptrs_host[k] : nullptr;
        out.co[k] = k < B ? (float *)d_conic_opacity_ptrs_host[k] : nullptr;
        out.rad[k] = nullptr; out.dep[k] = nullptr;
    }
    GsStageTimer timer(GS_STAGE_UNPACK, (cudaStream_t)stream);
    k_xr_pull_grad<<<dim3(XR_NB(P), B), DT_THREADS, 0, (cudaStream_t)stream>>>(g, blkbase, peers, out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}
