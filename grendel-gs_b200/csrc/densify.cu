// Densification step in three launches (SURVEY.md 8f rank 4): select -> scan -> gather.
// /root/reference/scene/gaussian_model.py:1005-1044 (densify_and_prune) runs densify_and_clone (:973-1003),
// densify_and_split (:922-971) and two prune_points (:816-835) as ~150 torch kernels: every step boolean-indexes or
// concatenates all six parameters and both Adam moments (cat_tensors_to_optimizer :837-881, _prune_optimizer :789-814)
// and reads a count back to the host each time.  The END STATE of that sequence is, in this order:
//     [ originals that are neither split nor pruned | clones | split children, copy 1 | split children, copy 2 ]
// (each block in index order, the final opacity / world-size prune applied to every block), with the Adam moments of
// the survivors carried over and those of new Gaussians zero.  So:
//   1. k_densify_flags: per Gaussian, the five decisions (keep, clone, child 1, child 2, "was selected for split") as
//      five byte planes -- the concatenation of the first four planes IS the output order;
//   2. one exclusive scan over the 5 P flags: a flag's rank is its output row (planes 0-3) or its index into the
//      split's block of normal draws (plane 4); the plane totals go back to the host once;
//   3. k_densify_gather: every tensor (6 parameters, 12 moments, send_to_gpui_cnt) is read once and written to its
//      output rows, with the split's two transforms applied on the fly (position: R(q) (s * z) + x, scale:
//      log(s * fl32(1 / 1.6))).
// Byte / index work plus a few transcendentals: HBM bound, ~(3 x 236 + 4 W) B read and written per Gaussian.
#include <cub/cub.cuh>

#include "common.cuh"

#define DN_THREADS 256
#define DN_PLANES 5
// a split child's scale is get_scaling / (0.8 N) with N = 2.  On CUDA, torch divides a tensor by a Python scalar by
// multiplying with the scalar's fp32 reciprocal, fl32(1 / 1.6f) = 0.625f; a true division by 1.6f rounds differently for
// about 15 % of fp32 scales (measured over every fp32 in [2^-14, 256) on an H100).
#define DN_CHILD_SCALE (1.0f / 1.6f)

struct PlaneToInt {
    const uint8_t *f;
    __host__ __device__ int32_t operator()(int e) const { return f[e]; }
};

static size_t dn_align(size_t v) { return (v + 255) / 256 * 256; }

static size_t dn_scan_bytes(int P) {
    size_t b = 0;
    const int n = DN_PLANES * (P > 0 ? P : 1);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t *)nullptr, (int32_t *)nullptr, n);
    return dn_align(b);
}

// temp layout: flags (5 P bytes) | pos (5 P int32) | totals (8 int32) | scan scratch
extern "C" size_t gs_densify_temp_bytes(int P) {
    const size_t n = (size_t)DN_PLANES * (size_t)(P > 0 ? P : 1);
    return dn_align(n) + dn_align(4 * n) + 256 + dn_scan_bytes(P) + 256;
}

__global__ void __launch_bounds__(DN_THREADS)
k_densify_flags(int P, const float *__restrict__ accum, const float *__restrict__ denom,
                const float *__restrict__ scaling, const float *__restrict__ opacity, float max_grad, float min_opacity,
                float dense_thr, float big_thr, int use_screen, uint8_t *__restrict__ flags) {
    const int i = blockIdx.x * DN_THREADS + threadIdx.x;
    if (i >= P) return;
    float grad = __fdiv_rn(accum[i], denom[i]);          // grads = xyz_gradient_accum / denom      (:1018)
    if (isnan(grad)) grad = 0.f;                          // grads[grads.isnan()] = 0.0              (:1019)
    const float s0 = expf(scaling[3 * i]), s1 = expf(scaling[3 * i + 1]), s2 = expf(scaling[3 * i + 2]);
    const float smax = fmaxf(s0, fmaxf(s1, s2));
    const bool hot = fabsf(grad) >= max_grad;             // torch.norm(grads, dim=-1) >= grad_threshold (:975-977)
    const bool sel_clone = hot && smax <= dense_thr;      // (:978-982)
    const bool sel_split = grad >= max_grad && smax > dense_thr;   // (:927-932); clones have zero padded_grad
    const float opa = __fdiv_rn(1.f, 1.f + expf(-opacity[i]));
    const bool faint = opa < min_opacity;                 // (:1026)
    const bool prune_orig = faint || (use_screen && smax > big_thr);   // (:1037-1040)
    // a child's scale is stored as log(s / (0.8 N)) (:949-951) and read back through exp (:110-111)
    const float c0 = expf(logf(__fmul_rn(s0, DN_CHILD_SCALE))), c1 = expf(logf(__fmul_rn(s1, DN_CHILD_SCALE))),
                c2 = expf(logf(__fmul_rn(s2, DN_CHILD_SCALE)));
    const bool prune_child = faint || (use_screen && fmaxf(c0, fmaxf(c1, c2)) > big_thr);
    flags[i] = (!sel_split && !prune_orig) ? 1 : 0;
    flags[(size_t)P + i] = (sel_clone && !prune_orig) ? 1 : 0;
    const uint8_t child = (sel_split && !prune_child) ? 1 : 0;
    flags[(size_t)2 * P + i] = child;
    flags[(size_t)3 * P + i] = child;
    flags[(size_t)4 * P + i] = sel_split ? 1 : 0;
}

__global__ void k_densify_totals(int P, const uint8_t *__restrict__ flags, const int32_t *__restrict__ pos,
                                 int32_t *__restrict__ totals) {
    const int c = threadIdx.x;
    if (c < DN_PLANES) totals[c] = pos[(size_t)c * P];   // first output row / first draw of plane c
    if (c == DN_PLANES) totals[DN_PLANES] = pos[(size_t)DN_PLANES * P - 1] + flags[(size_t)DN_PLANES * P - 1];
}

// counts_host (HOST, 6 int32): rows kept, clones, children copy 1, children copy 2, S = Gaussians selected for the split
// (the split consumes 2 S rows of `noise`), and the new number of Gaussians.  Synchronises `stream`.
extern "C" int gs_densify_select(int P, const float *xyz_gradient_accum, const float *denom, const float *scaling_raw,
                                 const float *opacity_raw, float max_grad, float min_opacity, double extent,
                                 double percent_dense, int use_screen_size, void *temp, size_t temp_bytes,
                                 int32_t *counts_host, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    GS_REQUIRE(P > 0, "P");
    GS_REQUIRE((long long)DN_PLANES * P < (1ll << 31), "5 P overflows int32");
    GS_REQUIRE(xyz_gradient_accum && denom && scaling_raw && opacity_raw && temp && counts_host, "null pointer");
    if (temp_bytes < gs_densify_temp_bytes(P)) {
        gs_set_error("gs_densify_select: temp too small");
        return GS_ENOMEM;
    }
    const size_t n = (size_t)DN_PLANES * P;
    uint8_t *flags = (uint8_t *)temp;
    int32_t *pos = (int32_t *)((char *)temp + dn_align(n));
    int32_t *totals = (int32_t *)((char *)pos + dn_align(4 * n));
    void *scratch = (char *)totals + 256;
    size_t scratch_bytes = dn_scan_bytes(P);
    // the thresholds are Python doubles in the reference (percent_dense * extent, 0.1 * extent), rounded to fp32 once
    // when compared with fp32 tensors: form the product in double from the unrounded inputs, then round
    const float dense_thr = (float)(percent_dense * extent), big_thr = (float)(0.1 * extent);
    k_densify_flags<<<(P + DN_THREADS - 1) / DN_THREADS, DN_THREADS, 0, stream>>>(
        P, xyz_gradient_accum, denom, scaling_raw, opacity_raw, max_grad, min_opacity, dense_thr, big_thr,
        use_screen_size ? 1 : 0, flags);
    GS_LAUNCH_CHECK();
    cub::CountingInputIterator<int> idx(0);
    cub::TransformInputIterator<int32_t, PlaneToInt, cub::CountingInputIterator<int>> it(idx, PlaneToInt{flags});
    GS_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scratch, scratch_bytes, it, pos, (int)n, stream));
    k_densify_totals<<<1, 32, 0, stream>>>(P, flags, pos, totals);
    GS_LAUNCH_CHECK();
    int32_t t[DN_PLANES + 1];
    GS_CUDA_TRY(cudaMemcpyAsync(t, totals, sizeof(t), cudaMemcpyDeviceToHost, stream));
    GS_CUDA_TRY(cudaStreamSynchronize(stream));
    counts_host[0] = t[1] - t[0];   // kept originals
    counts_host[1] = t[2] - t[1];   // clones
    counts_host[2] = t[3] - t[2];   // children, copy 1
    counts_host[3] = t[4] - t[3];   // children, copy 2
    counts_host[4] = t[5] - t[4];   // S
    counts_host[5] = t[4];          // new number of Gaussians
    return GS_OK;
}

#define DN_MAX_TENSORS 24
enum { DN_COPY = 0, DN_XYZ = 1, DN_SCALING = 2, DN_MOMENT = 3 };

struct DnTensors {
    const float *src[DN_MAX_TENSORS];
    float *dst[DN_MAX_TENSORS];
    int width[DN_MAX_TENSORS];
    int kind[DN_MAX_TENSORS];
};

__global__ void __launch_bounds__(DN_THREADS)
k_densify_gather(int P, int S, const DnTensors t, const float *__restrict__ scaling,
                 const float *__restrict__ rotation, const float *__restrict__ noise, const uint8_t *__restrict__ flags,
                 const int32_t *__restrict__ pos, int split_base) {
    const int k = blockIdx.y;
    const int d = t.width[k], kind = t.kind[k];
    const long long e = (long long)blockIdx.x * DN_THREADS + threadIdx.x;
    if (e >= (long long)P * d) return;
    const int i = (int)(e / d), col = (int)(e - (long long)i * d);
    const float v = t.src[k][e];
    float *dst = t.dst[k];
    if (flags[i]) dst[(size_t)pos[i] * d + col] = v;                                             // survivor: as is
    if (flags[(size_t)P + i]) dst[(size_t)pos[(size_t)P + i] * d + col] = kind == DN_MOMENT ? 0.f : v;   // clone
    if (flags[(size_t)2 * P + i]) {                                                               // two children
        const int rank = pos[(size_t)4 * P + i] - split_base;   // index among the S Gaussians selected for the split
        float c[2] = {v, v};
        if (kind == DN_MOMENT) {
            c[0] = c[1] = 0.f;
        } else if (kind == DN_SCALING) {
            c[0] = c[1] = logf(__fmul_rn(expf(v), DN_CHILD_SCALE));   // scaling_inverse_activation(get_scaling / (0.8 N))
        } else if (kind == DN_XYZ) {
            // new_xyz = R(q) (s * z) + xyz, R of utils/general_utils.py:416-438 on the RAW quaternion
            const float q0 = rotation[4 * i], q1 = rotation[4 * i + 1], q2 = rotation[4 * i + 2], q3 = rotation[4 * i + 3];
            const float nrm = sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
            const float w = q0 / nrm, x = q1 / nrm, y = q2 / nrm, z = q3 / nrm;
            float r0, r1, r2;   // row `col` of R
            if (col == 0) { r0 = 1.f - 2.f * (y * y + z * z); r1 = 2.f * (x * y - w * z); r2 = 2.f * (x * z + w * y); }
            else if (col == 1) { r0 = 2.f * (x * y + w * z); r1 = 1.f - 2.f * (x * x + z * z); r2 = 2.f * (y * z - w * x); }
            else { r0 = 2.f * (x * z - w * y); r1 = 2.f * (y * z + w * x); r2 = 1.f - 2.f * (x * x + y * y); }
            const float s0 = expf(scaling[3 * i]), s1 = expf(scaling[3 * i + 1]), s2 = expf(scaling[3 * i + 2]);
#pragma unroll
            for (int copy = 0; copy < 2; copy++) {
                const float *zz = noise + 3 * ((size_t)copy * S + rank);   // stds.repeat(N,1): copy-major blocks of S rows
                c[copy] = (r0 * (s0 * zz[0]) + r1 * (s1 * zz[1]) + r2 * (s2 * zz[2])) + v;   // v = xyz[i][col]
            }
        }
        dst[(size_t)pos[(size_t)2 * P + i] * d + col] = c[0];
        dst[(size_t)pos[(size_t)3 * P + i] * d + col] = c[1];
    }
}

// After gs_densify_select (same temp, untouched; S and new_P are its counts[4] and counts[5]).  src_host / dst_host:
// HOST arrays of num_tensors device pointers to (P, width) inputs and (new_P, width) outputs of 4-byte elements; kind:
// 0 copy (f_dc, f_rest, opacity, rotation, send_to_gpui_cnt), 1 position, 2 log-scale, 3 Adam moment (zero for new
// Gaussians).  noise: (2 S, 3) standard-normal draws (torch.normal's role at scene/gaussian_model.py:936-938), may be
// NULL if S == 0.
extern "C" int gs_densify_gather(int P, int S, int new_P, int num_tensors, const void *const *src_host,
                                 void *const *dst_host, const int32_t *width_host, const int32_t *kind_host,
                                 const float *scaling_raw, const float *rotation_raw, const float *noise, const void *temp,
                                 void *stream) {
    GS_REQUIRE(P > 0 && S >= 0 && new_P >= 0 && num_tensors > 0 && num_tensors <= DN_MAX_TENSORS, "sizes");
    GS_REQUIRE(src_host && dst_host && width_host && kind_host && scaling_raw && rotation_raw && temp, "null pointer");
    GS_REQUIRE(S == 0 || noise != nullptr, "noise");
    const size_t n = (size_t)DN_PLANES * P;
    const uint8_t *flags = (const uint8_t *)temp;
    const int32_t *pos = (const int32_t *)((const char *)temp + dn_align(n));
    DnTensors t;
    int widest = 0;
    for (int k = 0; k < DN_MAX_TENSORS; k++) {
        const bool v = k < num_tensors;
        t.src[k] = v ? (const float *)src_host[k] : nullptr;
        t.dst[k] = v ? (float *)dst_host[k] : nullptr;
        t.width[k] = v ? width_host[k] : 0;
        t.kind[k] = v ? kind_host[k] : 0;
        if (!v) continue;
        // an output of new_P == 0 rows may have no storage (a NULL pointer): nothing is written to it
        GS_REQUIRE(t.src[k] && (t.dst[k] || new_P == 0) && t.width[k] > 0 && t.kind[k] >= DN_COPY && t.kind[k] <= DN_MOMENT, "tensor table");
        GS_REQUIRE((t.kind[k] != DN_XYZ && t.kind[k] != DN_SCALING) || t.width[k] == 3, "position / scale rows have 3 elements");
        widest = t.width[k] > widest ? t.width[k] : widest;
    }
    if (new_P == 0) return GS_OK;
    // pos is ONE exclusive scan over all five planes: plane 4 (the draw indices) starts where the output rows end
    const int split_base = new_P;
    const long long blocks = ((long long)P * widest + DN_THREADS - 1) / DN_THREADS;
    GS_REQUIRE(blocks < (1ll << 31), "too many elements");
    dim3 grid((unsigned)blocks, (unsigned)num_tensors);
    k_densify_gather<<<grid, DN_THREADS, 0, (cudaStream_t)stream>>>(P, S, t, scaling_raw, rotation_raw, noise, flags, pos,
                                                                      split_base);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// ---- densification statistics: the reference's densification.py:15-24 + scene/gaussian_model.py:1046-1052 ----------
// Per camera k of the batch, in batch order, over the Gaussians with radii_k > 0:
//     max_radii2D = torch.max(max_radii2D, radii_k);  xyz_gradient_accum += ||means2D_k.grad[:, :2]||;  denom += 1
// Every masked read / write there is a nonzero (a host sync).  Here one thread per Gaussian walks the views in the same
// order, so the fp32 sum is the reference's sequence; rows visible in no view are neither loaded nor stored.
struct DsViews {
    const float2 *grad[GS_MAX_VIEWS];
    const int32_t *radii[GS_MAX_VIEWS];
};

// torch.norm(g, dim=-1) of a 2-vector on the device: the two squares are rounded, then summed (tests/
// test_densify_stats_gpu.py, test_norm_form, checks this against torch on inputs where the FMA forms differ)
GS_D float ds_norm(float2 g) { return __fsqrt_rn(__fadd_rn(__fmul_rn(g.x, g.x), __fmul_rn(g.y, g.y))); }

__global__ void __launch_bounds__(DN_THREADS)
k_densify_stats(int B, int P, const DsViews v, float *__restrict__ accum, float *__restrict__ denom,
                float *__restrict__ max_radii) {
    const int i = blockIdx.x * DN_THREADS + threadIdx.x;
    if (i >= P) return;
    float a = 0.f, d = 0.f, m = 0.f;
    bool seen = false;
    for (int k = 0; k < B; k++) {
        const int r = v.radii[k][i];
        if (r <= 0) continue;                              // visibility_filter = radii > 0
        const float2 g = v.grad[k][i];
        if (!seen) {
            a = accum[i]; d = denom[i]; m = max_radii[i];
            seen = true;
        }
        const float f = __int2float_rn(r);                 // torch's int32 -> float32 promotion rounds to nearest
        m = (isnan(m) || m > f) ? m : f;                   // torch.max: a NaN operand is returned as is
        a = __fadd_rn(a, ds_norm(g));
        d = __fadd_rn(d, 1.f);
    }
    if (seen) {
        accum[i] = a; denom[i] = d; max_radii[i] = m;
    }
}

extern "C" int gs_densify_stats(int num_views, int P, const void *const *grad_host, const void *const *radii_host,
                                float *xyz_gradient_accum, float *denom, float *max_radii2D, void *stream) {
    GS_REQUIRE(num_views >= 1 && num_views <= GS_MAX_VIEWS, "num_views");
    GS_REQUIRE(P >= 0, "P");
    GS_REQUIRE(grad_host && radii_host && xyz_gradient_accum && denom && max_radii2D, "null pointer");
    DsViews v;
    for (int k = 0; k < GS_MAX_VIEWS; k++) {
        const bool in = k < num_views;
        v.grad[k] = in ? (const float2 *)grad_host[k] : nullptr;
        v.radii[k] = in ? (const int32_t *)radii_host[k] : nullptr;
        if (!in) continue;
        GS_REQUIRE(v.grad[k] && v.radii[k], "null pointer");
        GS_REQUIRE(((uintptr_t)v.grad[k] & 7) == 0, "means2D gradients must be 8-byte aligned (float2 loads)");
        GS_REQUIRE(((uintptr_t)v.radii[k] & 3) == 0, "radii must be 4-byte aligned");
    }
    GS_REQUIRE((((uintptr_t)xyz_gradient_accum | (uintptr_t)denom | (uintptr_t)max_radii2D) & 3) == 0,
               "statistics must be 4-byte aligned");
    if (P == 0) return GS_OK;
    k_densify_stats<<<(P + DN_THREADS - 1) / DN_THREADS, DN_THREADS, 0, (cudaStream_t)stream>>>(
        num_views, P, v, xyz_gradient_accum, denom, max_radii2D);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// Opacity reset (scene/gaussian_model.py:555-561 with replace_tensor_to_optimizer :771-787):
//     o = inverse_sigmoid(torch.min(sigmoid(o), ones_like * 0.01));  exp_avg = exp_avg_sq = 0
// in torch's CUDA arithmetic, one rounding per operation: sigmoid is 1 / (1 + expf(-o)), ones * 0.01 is 0.01f, min
// returns a NaN operand, inverse_sigmoid is logf(m / (1 - m)).  Every element takes the round trip (logit of a
// sigmoid is not the identity in fp32), at or below 0.01 too.
GS_D float ro_reset(float o) {
    const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-o)));
    const float m = (isnan(s) || s < 0.01f) ? s : 0.01f;
    return logf(__fdiv_rn(m, __fsub_rn(1.f, m)));
}

__global__ void __launch_bounds__(DN_THREADS)
k_reset_opacity(long long P, float *__restrict__ o, float *__restrict__ m, float *__restrict__ v, int vec) {
    const long long base = ((long long)blockIdx.x * DN_THREADS + threadIdx.x) * 4;
    if (base >= P) return;
    if (vec && base + 4 <= P) {
        float4 x = *reinterpret_cast<float4 *>(o + base);
        x.x = ro_reset(x.x); x.y = ro_reset(x.y); x.z = ro_reset(x.z); x.w = ro_reset(x.w);
        *reinterpret_cast<float4 *>(o + base) = x;
        if (m) {
            *reinterpret_cast<float4 *>(m + base) = make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4 *>(v + base) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        return;
    }
    const int cnt = (int)min(4ll, P - base);
    for (int q = 0; q < cnt; q++) {
        o[base + q] = ro_reset(o[base + q]);
        if (m) { m[base + q] = 0.f; v[base + q] = 0.f; }
    }
}

extern "C" int gs_reset_opacity(int P, float *opacity_raw, float *exp_avg, float *exp_avg_sq, void *stream) {
    GS_REQUIRE(P >= 0, "P");
    GS_REQUIRE(!exp_avg == !exp_avg_sq, "exp_avg and exp_avg_sq: both or neither");
    if (P == 0) return GS_OK;
    GS_REQUIRE(opacity_raw, "null pointer");
    const uintptr_t all = (uintptr_t)opacity_raw | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq;
    GS_REQUIRE((all & 3) == 0, "tensors must be 4-byte aligned");
    const long long per_block = (long long)DN_THREADS * 4;
    k_reset_opacity<<<(unsigned)((P + per_block - 1) / per_block), DN_THREADS, 0, (cudaStream_t)stream>>>(
        P, opacity_raw, exp_avg, exp_avg_sq, (all & 15) == 0 ? 1 : 0);
    GS_LAUNCH_CHECK();
    return GS_OK;
}
