// Held-out view metrics: the L1 and PSNR that training_report prints (train_internal.py:461-481), from per-tile-row sums.
//   x^ = clamp(x, 0, 1)  (train_internal.py:471; NaN stays NaN, as torch.clamp leaves it)
//   g^ = g / 255          (:472-474, the uint8 ground truth; the fp32 quotient the reference forms)
//   S1[v,c] = sum |x^ - g^|,  S2[v,c] = sum (x^ - g^)^2          (fp64; x^ - g^ of two fp32 values is exact in fp64,
//                                                                 so a render equal to the ground truth scores 0)
//   L1_v   = (S1[v,0] + S1[v,1] + S1[v,2]) / (3 H W)             (l1_loss(...).mean(), utils/loss_utils.py:18-19)
//   PSNR_v = mean_c 20 log10(1 / sqrt(S2[v,c] / (H W)))          (psnr(...).mean(), utils/image_utils.py:19-21: per
//                                                                 channel, then averaged -- not the PSNR of the pooled MSE)
// k_eval_sums writes one (3, 2) slot per (view, tile row).  A slot is a function of that tile row's pixels alone, summed
// in an order fixed by (W, the row's height): it does not depend on the batch, the rank or the strip boundaries.  Every
// tile row is owned by exactly one rank and the slots of the others are +0.0, so an all-reduce(SUM) of the slots is exact
// in any order, and k_eval_finalize adds each view's slots in row order: the metrics are the same bits at any world size,
// strip division and batch size.
//
// HBM bound: 12 B of image + 3 B of ground truth per local pixel, 48 B of slots per tile row.
#include "common.cuh"

#define EV_THREADS 512
#define EV_UNROLL 4

// The views of one k_eval_sums launch; passed by value.
struct EvalViews {
    int row0[GS_MAX_VIEWS], row1[GS_MAX_VIEWS];     // local pixel rows [row0, row1); row0 == row1: none
    int gt_row0[GS_MAX_VIEWS], gt_rows[GS_MAX_VIEWS];  // the GT buffer holds image rows [gt_row0, gt_row0 + gt_rows)
    const uint8_t *gt[GS_MAX_VIEWS];
};

// grid (TILE_Y, B): one CTA per (tile row, view).  Thread t adds the pixels t, t + EV_THREADS, ... of the row's
// contiguous 16 x W block in each channel, in fp64; then a fixed xor tree per warp and warp 0 over the warps in order.
__global__ void __launch_bounds__(EV_THREADS)
k_eval_sums(int H, int W, const EvalViews ev, const float *__restrict__ image, double *__restrict__ slots) {
    __shared__ double s_g[256];
    __shared__ double s_red[6][EV_THREADS / 32];
    const int ty = blockIdx.x, view = blockIdx.y, TY = gridDim.x;
    double *out = slots + ((size_t)view * TY + ty) * 6;
    const int y0 = ty * GS_BLOCK_Y, y1 = min(y0 + GS_BLOCK_Y, H);
    if (y0 < ev.row0[view] || y1 > ev.row1[view]) {  // not a local tile row (row0 and row1 are tile aligned, or H)
        if (threadIdx.x < 6) out[threadIdx.x] = 0.0;
        return;
    }
    for (int i = threadIdx.x; i < 256; i += EV_THREADS) s_g[i] = (double)__fdiv_rn((float)i, 255.f);
    __syncthreads();
    const size_t HW = (size_t)H * W, GP = (size_t)ev.gt_rows[view] * W;
    const int n = (y1 - y0) * W;
    const float *__restrict__ x = image + (size_t)view * 3 * HW + (size_t)y0 * W;
    const uint8_t *__restrict__ g = ev.gt[view] + (size_t)(y0 - ev.gt_row0[view]) * W;
    double a[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // (S1, S2) per channel
    for (int base = threadIdx.x; base < n; base += EV_UNROLL * EV_THREADS) {
        float xv[EV_UNROLL][3];
        uint8_t gv[EV_UNROLL][3];
#pragma unroll
        for (int u = 0; u < EV_UNROLL; u++) {
            const int i = base + u * EV_THREADS;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                xv[u][c] = i < n ? __ldg(x + c * HW + i) : 0.f;
                gv[u][c] = i < n ? __ldg(g + c * GP + i) : (uint8_t)0;
            }
        }
#pragma unroll
        for (int u = 0; u < EV_UNROLL; u++) {
            if (base + u * EV_THREADS >= n) break;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float v = xv[u][c];
                const float vc = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);  // NaN fails both tests and stays NaN
                const double d = (double)vc - s_g[gv[u][c]];
                a[2 * c] += fabs(d);
                a[2 * c + 1] += d * d;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 6; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < 6; k++) s_red[k][warp] = a[k];
    __syncthreads();
    if (threadIdx.x < 6) {
        double s = 0.0;
        for (int w = 0; w < EV_THREADS / 32; w++) s += s_red[threadIdx.x][w];
        out[threadIdx.x] = s;
    }
}

// One CTA of 32 threads per view: thread k < 6 adds slot value k of the view's tile rows in row order; thread 0 forms
// (L1, PSNR).  An MSE of 0 gives +inf, as the reference's 20 log10(1 / sqrt(0)) does.
__global__ void __launch_bounds__(32)
k_eval_finalize(int TY, double hw, const double *__restrict__ slots, double *__restrict__ out) {
    __shared__ double s_sum[6];
    const int view = blockIdx.x;
    if (threadIdx.x < 6) {
        const double *p = slots + (size_t)view * TY * 6 + threadIdx.x;
        double s = 0.0;
        for (int r = 0; r < TY; r++) s += p[(size_t)6 * r];
        s_sum[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const double l1 = (s_sum[0] + s_sum[2] + s_sum[4]) / (3.0 * hw);
        double psnr = 0.0;
        for (int c = 0; c < 3; c++) psnr += 20.0 * log10(1.0 / sqrt(s_sum[2 * c + 1] / hw));
        out[2 * view] = l1;
        out[2 * view + 1] = psnr / 3.0;
    }
}

extern "C" int gs_eval_slot_count(int num_views, int image_height) {
    if (num_views < 1 || num_views > GS_MAX_VIEWS || image_height < 1) return 0;
    return num_views * ((image_height + GS_BLOCK_Y - 1) / GS_BLOCK_Y) * 6;
}

extern "C" int gs_eval_sums_batched(int num_views, int image_height, int image_width, const float *image,
                                    const void *const *gt_u8_ptrs_host, const int32_t *gt_row0_host,
                                    const int32_t *gt_rows_host, const int32_t *row0_host, const int32_t *row1_host,
                                    double *slots, void *stream_) {
    const int H = image_height, W = image_width;
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views must be in [1, GS_MAX_VIEWS]");
    GS_REQUIRE(H > 0 && W > 0, "sizes");
    GS_REQUIRE(image && slots, "null image or slots pointer");
    GS_REQUIRE(gt_u8_ptrs_host && gt_row0_host && gt_rows_host && row0_host && row1_host, "null host array");
    EvalViews ev;
    for (int v = 0; v < GS_MAX_VIEWS; v++) {
        ev.row0[v] = ev.row1[v] = ev.gt_row0[v] = ev.gt_rows[v] = 0;
        ev.gt[v] = nullptr;
        if (v >= num_views) continue;
        const int r0 = row0_host[v], r1 = row1_host[v], g0 = gt_row0_host[v], gr = gt_rows_host[v];
        GS_REQUIRE(r0 >= 0 && r1 <= H && r0 <= r1, "rows [row0, row1) must lie in [0, H)");
        GS_REQUIRE(r0 % GS_BLOCK_Y == 0 && (r1 % GS_BLOCK_Y == 0 || r1 == H), "row0 must be a multiple of 16, row1 too or H");
        if (r0 == r1) continue;
        GS_REQUIRE(gt_u8_ptrs_host[v] != nullptr, "null ground-truth pointer for a view with rows");
        GS_REQUIRE(g0 >= 0 && gr >= 0 && g0 <= r0 && r1 <= g0 + gr && g0 + gr <= H,
                   "the ground truth must hold rows [row0, row1): gt_row0 <= row0, row1 <= gt_row0 + gt_rows <= H");
        ev.row0[v] = r0; ev.row1[v] = r1; ev.gt_row0[v] = g0; ev.gt_rows[v] = gr;
        ev.gt[v] = (const uint8_t *)gt_u8_ptrs_host[v];
    }
    const int TY = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    k_eval_sums<<<dim3(TY, num_views), EV_THREADS, 0, (cudaStream_t)stream_>>>(H, W, ev, image, slots);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

extern "C" int gs_eval_finalize(int num_views, int image_height, int image_width, const double *slots, double *out,
                                void *stream_) {
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views must be in [1, GS_MAX_VIEWS]");
    GS_REQUIRE(image_height > 0 && image_width > 0, "sizes");
    GS_REQUIRE(slots && out, "null slots or out pointer");
    const int TY = (image_height + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    k_eval_finalize<<<num_views, 32, 0, (cudaStream_t)stream_>>>(TY, (double)image_height * image_width, slots, out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}
