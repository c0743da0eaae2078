// Held-out view metrics: the L1 and PSNR that training_report prints (train_internal.py:461-481), from per-tile-row sums.
//   x^ = clamp(x, 0, 1)  (train_internal.py:471; NaN stays NaN, as torch.clamp leaves it)
//   g^ = g / 255          (:472-474, the uint8 ground truth divided on the device: fl32(g * fl32(1/255)), gs_gt_unit)
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
    for (int i = threadIdx.x; i < 256; i += EV_THREADS) s_g[i] = (double)gs_gt_unit((uint8_t)i);
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

// ---- image metrics: metrics.py's SSIM and PSNR of the 8-bit renders render.py writes --------------------------------
// q = uint8(clamp(fl(fl(clamp(x, 0, 1) * 255) + 0.5), 0, 255)): render.py's clamp, then save_image's
// mul(255).add_(0.5).clamp_(0, 255).to(uint8) -- two separately rounded fp32 operations and a truncating conversion.  A NaN
// render maps to 0 here (torch's NaN -> uint8 cast is undefined).  A ground truth saved the same way comes back as itself,
// so the 8-bit ground truth g is read directly.
// a = fl32(q / 255), b = fl32(g / 255) (tf.to_tensor), promoted to fp64.  Per pixel and channel, the SSIM map of _ssim
// (utils/loss_utils.py:56-80) in fp64: the separable 11-tap window below, zero outside the image, C1 = 0.01^2,
// C2 = 0.03^2.  SSIM_v = sum of the map / (3 H W); S = sum (q - g)^2 (an exact integer in fp64) and
// PSNR_v = 20 log10(1 / sqrt(S / (255^2 3 H W))) -- the MSE pooled over the channels, as psnr on (1,3,H,W) pools it.
// k_image_metric_sums writes one (sum of the map, S) slot per (view, tile row).  A pixel's map value depends only on the
// 8-bit values of its 11 x 11 neighbourhood and a slot is summed in an order fixed by (W, the row's height), so, as for
// k_eval_sums, one all-reduce(SUM) of the slots over the ranks is exact and the metrics are the same bits at any world size,
// strip division and batch size.
#define IM_HALO 5
#define IM_TAPS (2 * IM_HALO + 1)
#define IM_CW 32                              // output columns per chunk
#define IM_ROWS (GS_BLOCK_Y + 2 * IM_HALO)    // input rows of a tile row: 26
#define IM_IN_W (IM_CW + 2 * IM_HALO)         // input columns of a chunk: 42
#define IM_THREADS 512                        // one thread per output pixel of a 16 x 32 chunk
#define QU_THREADS 256

// gaussian(11, 1.5) of utils/loss_utils.py:26-33 as torch builds it on the CPU (fp32 taps over their fp32 sum,
// 3.7592328), promoted to fp64.  Not loss.cu's window, whose sequential sum lands 1 ulp low on 9 of the 11 taps.
__constant__ double c_ssim_w[IM_TAPS] = {
    0x1.0d956cp-10, 0x1.f1fe02p-8, 0x1.26eb18p-5, 0x1.bff0fep-4, 0x1.b43c3ep-3, 0x1.10656p-2,
    0x1.b43c3ep-3,  0x1.bff0fep-4, 0x1.26eb18p-5, 0x1.f1fe02p-8, 0x1.0d956cp-10};

GS_D uint8_t quantize_u8(float x) {
    const float c = fminf(fmaxf(x, 0.f), 1.f);                 // fmaxf(NaN, 0) = 0: NaN -> 0
    const float t = __fadd_rn(__fmul_rn(c, 255.f), 0.5f);      // no FMA contraction: torch rounds the product first
    return (uint8_t)__float2uint_rz(fminf(t, 255.f));
}

// The views of one k_quantize_u8 launch; passed by value.
struct QuantViews {
    int row0[GS_MAX_VIEWS], row1[GS_MAX_VIEWS];          // rows [row0, row1) to quantize; row0 == row1: none
    int out_row0[GS_MAX_VIEWS], out_rows[GS_MAX_VIEWS];  // the output holds image rows [out_row0, out_row0 + out_rows)
    uint8_t *out[GS_MAX_VIEWS];
};

// grid (x, B, 3): view blockIdx.y, channel blockIdx.z; a grid-stride loop over the channel's rows.
__global__ void __launch_bounds__(QU_THREADS)
k_quantize_u8(int H, int W, const QuantViews qv, const float *__restrict__ image) {
    const int v = blockIdx.y, c = blockIdx.z;
    const size_t n = (size_t)(qv.row1[v] - qv.row0[v]) * W;
    const float *__restrict__ x = image + ((size_t)v * 3 + c) * H * W + (size_t)qv.row0[v] * W;
    uint8_t *__restrict__ o = qv.out[v] + (size_t)c * qv.out_rows[v] * W + (size_t)(qv.row0[v] - qv.out_row0[v]) * W;
    for (size_t i = (size_t)blockIdx.x * QU_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * QU_THREADS)
        o[i] = quantize_u8(__ldg(x + i));
}

// The views of one k_image_metric_sums launch; passed by value.
struct MetricViews {
    int row0[GS_MAX_VIEWS], row1[GS_MAX_VIEWS];          // local pixel rows [row0, row1); row0 == row1: none
    int win_row0[GS_MAX_VIEWS], win_rows[GS_MAX_VIEWS];  // the window holds image rows [win_row0, win_row0 + win_rows)
    const uint8_t *win[GS_MAX_VIEWS];                    // (6, win_rows, W): q in channels 0-2, g in 3-5
};

// grid (TILE_Y, B): one CTA per (tile row, view).  The CTA walks the row in chunks of 32 columns from column 0; per chunk
// and channel it stages the fp64 values a and b of the 26 x 42 neighbourhood (zero outside the image), runs the row pass
// of the five moments (a, b, a^2, b^2, ab) over the 26 rows, then the column pass, one output pixel per thread.  Thread
// (r, j) adds its pixel's map value and squared 8-bit difference of each chunk and channel in that order; then a fixed
// xor tree per warp and warp 0 over the warps in order.
#define IM_SMEM_BYTES ((2 * IM_ROWS * IM_IN_W + 5 * IM_ROWS * IM_CW) * (int)sizeof(double))
__global__ void __launch_bounds__(IM_THREADS)
k_image_metric_sums(int H, int W, const MetricViews mv, double *__restrict__ slots) {
    extern __shared__ double im_smem[];
    double (*s_ab)[IM_ROWS][IM_IN_W] = reinterpret_cast<double (*)[IM_ROWS][IM_IN_W]>(im_smem);   // [2]: a, b
    double (*s_h)[IM_ROWS][IM_CW] = reinterpret_cast<double (*)[IM_ROWS][IM_CW]>(im_smem + 2 * IM_ROWS * IM_IN_W);  // [5]
    __shared__ double s_val[256];
    __shared__ double s_red[2][IM_THREADS / 32];
    const int ty = blockIdx.x, view = blockIdx.y, TY = gridDim.x;
    double *out = slots + ((size_t)view * TY + ty) * 2;
    const int y0 = ty * GS_BLOCK_Y, y1 = min(y0 + GS_BLOCK_Y, H);
    if (y0 < mv.row0[view] || y1 > mv.row1[view]) {  // not a local tile row (row0 and row1 are tile aligned, or H)
        if (threadIdx.x < 2) out[threadIdx.x] = 0.0;
        return;
    }
    // the IEEE quotient, not gs_gt_unit: metrics.py's tf.to_tensor divides on the CPU
    for (int i = threadIdx.x; i < 256; i += IM_THREADS) s_val[i] = (double)__fdiv_rn((float)i, 255.f);
    const uint8_t *__restrict__ win = mv.win[view];
    const size_t WP = (size_t)mv.win_rows[view] * W;
    const int wr0 = mv.win_row0[view];
    const int tr = threadIdx.x / IM_CW, tc = threadIdx.x % IM_CW;
    double acc_map = 0.0, acc_sse = 0.0;
    for (int x0 = 0; x0 < W; x0 += IM_CW) {
        for (int c = 0; c < 3; c++) {
            __syncthreads();  // the table is written; the previous column pass is done with s_ab and s_h
            for (int i = threadIdx.x; i < 2 * IM_ROWS * IM_IN_W; i += IM_THREADS) {
                const int k = i / (IM_ROWS * IM_IN_W), rem = i % (IM_ROWS * IM_IN_W);
                const int r = rem / IM_IN_W, col = rem % IM_IN_W;
                const int y = y0 - IM_HALO + r, x = x0 - IM_HALO + col;
                s_ab[k][r][col] = (y >= 0 && y < H && x >= 0 && x < W)
                                      ? s_val[win[(3 * k + c) * WP + (size_t)(y - wr0) * W + x]] : 0.0;
            }
            __syncthreads();
            for (int i = threadIdx.x; i < IM_ROWS * IM_CW; i += IM_THREADS) {
                const int r = i / IM_CW, j = i % IM_CW;
                double m1 = 0.0, m2 = 0.0, m11 = 0.0, m22 = 0.0, m12 = 0.0;
#pragma unroll
                for (int k = 0; k < IM_TAPS; k++) {
                    const double w = c_ssim_w[k], a = s_ab[0][r][j + k], b = s_ab[1][r][j + k];
                    m1 = fma(w, a, m1);
                    m2 = fma(w, b, m2);
                    m11 = fma(w, a * a, m11);
                    m22 = fma(w, b * b, m22);
                    m12 = fma(w, a * b, m12);
                }
                s_h[0][r][j] = m1; s_h[1][r][j] = m2; s_h[2][r][j] = m11; s_h[3][r][j] = m22; s_h[4][r][j] = m12;
            }
            __syncthreads();
            const int y = y0 + tr, x = x0 + tc;
            if (y < y1 && x < W) {
                double mu1 = 0.0, mu2 = 0.0, e11 = 0.0, e22 = 0.0, e12 = 0.0;
#pragma unroll
                for (int k = 0; k < IM_TAPS; k++) {
                    const double w = c_ssim_w[k];
                    mu1 = fma(w, s_h[0][tr + k][tc], mu1);
                    mu2 = fma(w, s_h[1][tr + k][tc], mu2);
                    e11 = fma(w, s_h[2][tr + k][tc], e11);
                    e22 = fma(w, s_h[3][tr + k][tc], e22);
                    e12 = fma(w, s_h[4][tr + k][tc], e12);
                }
                // each operation rounded on its own, as _ssim writes them: no FMA contraction, so a == b gives
                // numerator == denominator and a map of exactly 1 (a render whose 8-bit image is the ground truth)
                const double mu1_sq = __dmul_rn(mu1, mu1), mu2_sq = __dmul_rn(mu2, mu2), mu1_mu2 = __dmul_rn(mu1, mu2);
                const double s11 = __dsub_rn(e11, mu1_sq), s22 = __dsub_rn(e22, mu2_sq), s12 = __dsub_rn(e12, mu1_mu2);
                const double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
                const double num = __dmul_rn(__dadd_rn(2.0 * mu1_mu2, C1), __dadd_rn(2.0 * s12, C2));
                const double den = __dmul_rn(__dadd_rn(__dadd_rn(mu1_sq, mu2_sq), C1), __dadd_rn(__dadd_rn(s11, s22), C2));
                acc_map += num / den;
                const size_t at = (size_t)(y - wr0) * W + x;
                const int d = (int)win[c * WP + at] - (int)win[(3 + c) * WP + at];
                acc_sse += (double)(d * d);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        acc_map += __shfl_xor_sync(0xffffffffu, acc_map, o);
        acc_sse += __shfl_xor_sync(0xffffffffu, acc_sse, o);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        s_red[0][warp] = acc_map;
        s_red[1][warp] = acc_sse;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        double s = 0.0;
        for (int w = 0; w < IM_THREADS / 32; w++) s += s_red[threadIdx.x][w];
        out[threadIdx.x] = s;
    }
}

// One CTA of 32 threads per view: threads 0 and 1 add the view's map sums and S in row order; thread 0 forms
// (SSIM, PSNR).  S = 0 gives +inf, as 20 log10(1 / sqrt(0)) does.
__global__ void __launch_bounds__(32)
k_image_metric_finalize(int TY, double n3hw, const double *__restrict__ slots, double *__restrict__ out) {
    __shared__ double s_sum[2];
    const int view = blockIdx.x;
    if (threadIdx.x < 2) {
        const double *p = slots + (size_t)view * TY * 2 + threadIdx.x;
        double s = 0.0;
        for (int r = 0; r < TY; r++) s += p[(size_t)2 * r];
        s_sum[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        out[2 * view] = s_sum[0] / n3hw;
        out[2 * view + 1] = 20.0 * log10(1.0 / sqrt(s_sum[1] / (255.0 * 255.0 * n3hw)));
    }
}

extern "C" int gs_quantize_u8_batched(int num_views, int image_height, int image_width, const float *image,
                                      const int32_t *row0_host, const int32_t *row1_host, void *const *out_u8_ptrs_host,
                                      const int32_t *out_row0_host, const int32_t *out_rows_host, void *stream_) {
    const int H = image_height, W = image_width;
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views must be in [1, GS_MAX_VIEWS]");
    GS_REQUIRE(H > 0 && W > 0, "sizes");
    GS_REQUIRE(image, "null image pointer");
    GS_REQUIRE(row0_host && row1_host && out_u8_ptrs_host && out_row0_host && out_rows_host, "null host array");
    QuantViews qv;
    size_t most = 0;
    for (int v = 0; v < GS_MAX_VIEWS; v++) {
        qv.row0[v] = qv.row1[v] = qv.out_row0[v] = qv.out_rows[v] = 0;
        qv.out[v] = nullptr;
        if (v >= num_views) continue;
        const int r0 = row0_host[v], r1 = row1_host[v], o0 = out_row0_host[v], orows = out_rows_host[v];
        GS_REQUIRE(r0 >= 0 && r1 <= H && r0 <= r1, "rows [row0, row1) must lie in [0, H)");
        if (r0 == r1) continue;
        GS_REQUIRE(out_u8_ptrs_host[v] != nullptr, "null output pointer for a view with rows");
        GS_REQUIRE(o0 >= 0 && orows >= 0 && o0 <= r0 && r1 <= o0 + orows && o0 + orows <= H,
                   "the output must hold rows [row0, row1): out_row0 <= row0, row1 <= out_row0 + out_rows <= H");
        qv.row0[v] = r0; qv.row1[v] = r1; qv.out_row0[v] = o0; qv.out_rows[v] = orows;
        qv.out[v] = (uint8_t *)out_u8_ptrs_host[v];
        most = max(most, (size_t)(r1 - r0) * W);
    }
    if (most == 0) return GS_OK;  // no view has rows: nothing to write
    const unsigned bx = (unsigned)min((most + QU_THREADS - 1) / QU_THREADS, (size_t)4096);
    k_quantize_u8<<<dim3(bx, num_views, 3), QU_THREADS, 0, (cudaStream_t)stream_>>>(H, W, qv, image);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

extern "C" int gs_image_metric_sums_batched(int num_views, int image_height, int image_width,
                                            const void *const *win_u8_ptrs_host, const int32_t *win_row0_host,
                                            const int32_t *win_rows_host, const int32_t *row0_host,
                                            const int32_t *row1_host, double *slots, void *stream_) {
    const int H = image_height, W = image_width;
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views must be in [1, GS_MAX_VIEWS]");
    GS_REQUIRE(H > 0 && W > 0, "sizes");
    GS_REQUIRE(slots, "null slots pointer");
    GS_REQUIRE(win_u8_ptrs_host && win_row0_host && win_rows_host && row0_host && row1_host, "null host array");
    MetricViews mv;
    for (int v = 0; v < GS_MAX_VIEWS; v++) {
        mv.row0[v] = mv.row1[v] = mv.win_row0[v] = mv.win_rows[v] = 0;
        mv.win[v] = nullptr;
        if (v >= num_views) continue;
        const int r0 = row0_host[v], r1 = row1_host[v], w0 = win_row0_host[v], wr = win_rows_host[v];
        GS_REQUIRE(r0 >= 0 && r1 <= H && r0 <= r1, "rows [row0, row1) must lie in [0, H)");
        GS_REQUIRE(r0 % GS_BLOCK_Y == 0 && (r1 % GS_BLOCK_Y == 0 || r1 == H), "row0 must be a multiple of 16, row1 too or H");
        if (r0 == r1) continue;
        GS_REQUIRE(win_u8_ptrs_host[v] != nullptr, "null window pointer for a view with rows");
        GS_REQUIRE(w0 >= 0 && wr >= 0 && w0 <= max(0, r0 - IM_HALO) && min(H, r1 + IM_HALO) <= w0 + wr && w0 + wr <= H,
                   "the window must hold the halo of the local rows: rows [max(0, row0 - 5), min(H, row1 + 5))");
        mv.row0[v] = r0; mv.row1[v] = r1; mv.win_row0[v] = w0; mv.win_rows[v] = wr;
        mv.win[v] = (const uint8_t *)win_u8_ptrs_host[v];
    }
    const int TY = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    GS_CUDA_TRY(cudaFuncSetAttribute(k_image_metric_sums, cudaFuncAttributeMaxDynamicSharedMemorySize, IM_SMEM_BYTES));
    k_image_metric_sums<<<dim3(TY, num_views), IM_THREADS, IM_SMEM_BYTES, (cudaStream_t)stream_>>>(H, W, mv, slots);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

extern "C" int gs_image_metric_finalize(int num_views, int image_height, int image_width, const double *slots,
                                        double *out, void *stream_) {
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views must be in [1, GS_MAX_VIEWS]");
    GS_REQUIRE(image_height > 0 && image_width > 0, "sizes");
    GS_REQUIRE(slots && out, "null slots or out pointer");
    const int TY = (image_height + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    k_image_metric_finalize<<<num_views, 32, 0, (cudaStream_t)stream_>>>(TY, 3.0 * image_height * image_width, slots,
                                                                         out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}
