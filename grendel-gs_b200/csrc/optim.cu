// Fused Adam step over the Gaussian parameter tensors (SURVEY.md 8f rank 3): ONE launch updates up to
// GS_ADAM_MAX_TENSORS tensors, each with its own learning rate / betas / eps, instead of the ~8 foreach kernels per
// step of torch.optim.Adam plus the six `param.grad /= bsz` passes in front of it
// (/root/reference/train_internal.py:316-329; optimizer built at scene/gaussian_model.py:257-292, six groups,
// eps 1e-15).  Arithmetic is torch.optim.Adam's (no weight decay, no amsgrad, maximize off), in its operation order:
//     g      = grad * grad_scale
//     m      = m + (1 - beta1) (g - m)                    (lerp; g - (g - m) beta1 when 1 - beta1 >= 0.5)
//     v      = v beta2 + (1 - beta2) g g                  (mul, addcmul)
//     denom  = sqrt(v) / sqrt(1 - beta2^t) + eps
//     p      = p - (lr / (1 - beta1^t)) m / denom         (addcdiv)
// Pure streaming work, HBM bound: 16 B read + 12 B written per element (59 elements = 1652 B per Gaussian).
#include <cmath>

#include "common.cuh"

#define AD_THREADS 256

struct AdamTensors {
    float *p[GS_ADAM_MAX_TENSORS];
    const float *g[GS_ADAM_MAX_TENSORS];
    float *m[GS_ADAM_MAX_TENSORS];
    float *v[GS_ADAM_MAX_TENSORS];
    long long n[GS_ADAM_MAX_TENSORS];
    float w1[GS_ADAM_MAX_TENSORS];         // 1 - beta1
    float beta2[GS_ADAM_MAX_TENSORS];
    float w2[GS_ADAM_MAX_TENSORS];         // 1 - beta2
    float bc2_sqrt[GS_ADAM_MAX_TENSORS];   // sqrt(1 - beta2^t)
    float eps[GS_ADAM_MAX_TENSORS];
    float step_size[GS_ADAM_MAX_TENSORS];  // lr / (1 - beta1^t)
    int vec[GS_ADAM_MAX_TENSORS];          // all four pointers 16-byte aligned: float4 path
};

GS_D void adam_one(float &p, float g, float &m, float &v, float gs, float w1, float beta2, float w2, float bc2_sqrt,
                   float eps, float step_size) {
    g = g * gs;
    // torch's lerp (ATen/native/Lerp.h): m + w (g - m) for |w| < 0.5, else g - (g - m) (1 - w)
    m = w1 < 0.5f ? __fmaf_rn(w1, g - m, m) : __fmaf_rn(-(g - m), 1.f - w1, g);
    v = __fmaf_rn(w2, g * g, v * beta2);
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
    // addcdiv_(m, denom, value=-step_size) on CUDA is one fma: p + (-step_size) (m / denom), rounded once
    p = __fmaf_rn(-step_size, __fdiv_rn(m, denom), p);
}

__global__ void __launch_bounds__(AD_THREADS)
k_adam(const AdamTensors t, float grad_scale) {
    const int k = blockIdx.y;
    const long long n = t.n[k];
    const long long base = ((long long)blockIdx.x * AD_THREADS + threadIdx.x) * 4;
    if (base >= n) return;
    const float w1 = t.w1[k], beta2 = t.beta2[k], w2 = t.w2[k], bc2 = t.bc2_sqrt[k], eps = t.eps[k], ss = t.step_size[k];
    float *p = t.p[k] + base, *m = t.m[k] + base, *v = t.v[k] + base;
    const float *g = t.g[k] + base;
    if (t.vec[k] && base + 4 <= n) {
        float4 P = *reinterpret_cast<float4 *>(p), M = *reinterpret_cast<float4 *>(m), V = *reinterpret_cast<float4 *>(v);
        const float4 G = *reinterpret_cast<const float4 *>(g);
        adam_one(P.x, G.x, M.x, V.x, grad_scale, w1, beta2, w2, bc2, eps, ss);
        adam_one(P.y, G.y, M.y, V.y, grad_scale, w1, beta2, w2, bc2, eps, ss);
        adam_one(P.z, G.z, M.z, V.z, grad_scale, w1, beta2, w2, bc2, eps, ss);
        adam_one(P.w, G.w, M.w, V.w, grad_scale, w1, beta2, w2, bc2, eps, ss);
        *reinterpret_cast<float4 *>(p) = P;
        *reinterpret_cast<float4 *>(m) = M;
        *reinterpret_cast<float4 *>(v) = V;
    } else {
        const int cnt = (int)min(4ll, n - base);
        for (int q = 0; q < cnt; q++) {
            float P = p[q], M = m[q], V = v[q];
            adam_one(P, g[q], M, V, grad_scale, w1, beta2, w2, bc2, eps, ss);
            p[q] = P; m[q] = M; v[q] = V;
        }
    }
}

// num_tensors <= GS_ADAM_MAX_TENSORS.  All *_host arguments are HOST arrays of num_tensors entries: device pointers
// (params / grads / exp_avg / exp_avg_sq, fp32, contiguous, numel[k] elements; a NULL grad skips the tensor, like a
// parameter whose .grad is None) and per-tensor hyper-parameters (doubles: they are Python floats in the reference and
// 1 - beta2^t loses 1e-5 relative if beta2 is rounded to fp32 first).  step[k] >= 1 is the value of the tensor's step
// counter AFTER this update (torch increments before use).  grad_scale multiplies every gradient first (the
// reference's `param.grad /= args.bsz`, train_internal.py:319-324).  Updates params, exp_avg, exp_avg_sq in place.
extern "C" int gs_adam_step(int num_tensors, const int64_t *numel_host, void *const *params_host,
                            const void *const *grads_host, void *const *exp_avg_host, void *const *exp_avg_sq_host,
                            const double *lr_host, const double *beta1_host, const double *beta2_host,
                            const double *eps_host, const int64_t *step_host, float grad_scale, void *stream) {
    GS_REQUIRE(num_tensors >= 0 && num_tensors <= GS_ADAM_MAX_TENSORS, "num_tensors");
    if (num_tensors == 0) return GS_OK;
    GS_REQUIRE(numel_host && params_host && grads_host && exp_avg_host && exp_avg_sq_host && lr_host && beta1_host &&
                   beta2_host && eps_host && step_host, "null pointer");
    AdamTensors t;
    long long longest = 0;
    for (int k = 0; k < GS_ADAM_MAX_TENSORS; k++) {
        t.p[k] = nullptr; t.g[k] = nullptr; t.m[k] = nullptr; t.v[k] = nullptr; t.n[k] = 0;
        t.w1[k] = t.beta2[k] = t.w2[k] = t.eps[k] = t.step_size[k] = 0.f; t.bc2_sqrt[k] = 1.f; t.vec[k] = 0;
        if (k >= num_tensors || grads_host[k] == nullptr || numel_host[k] <= 0) continue;
        GS_REQUIRE(params_host[k] && exp_avg_host[k] && exp_avg_sq_host[k], "null tensor pointer");
        GS_REQUIRE(step_host[k] >= 1, "step must be >= 1 (the counter after this update)");
        GS_REQUIRE(beta1_host[k] >= 0.0 && beta1_host[k] < 1.0 && beta2_host[k] >= 0.0 && beta2_host[k] < 1.0, "betas");
        t.p[k] = (float *)params_host[k]; t.g[k] = (const float *)grads_host[k];
        t.m[k] = (float *)exp_avg_host[k]; t.v[k] = (float *)exp_avg_sq_host[k];
        t.n[k] = numel_host[k];
        // scalars are formed in double like the Python floats of torch/optim/adam.py, then rounded once to fp32
        const double b1 = beta1_host[k], b2 = beta2_host[k], st = (double)step_host[k];
        const double bc1 = 1.0 - pow(b1, st), bc2 = 1.0 - pow(b2, st);
        t.w1[k] = (float)(1.0 - b1);
        t.beta2[k] = (float)b2;
        t.w2[k] = (float)(1.0 - b2);
        t.bc2_sqrt[k] = (float)sqrt(bc2);
        t.eps[k] = (float)eps_host[k];
        t.step_size[k] = (float)(lr_host[k] / bc1);
        t.vec[k] = ((((uintptr_t)t.p[k] | (uintptr_t)t.g[k] | (uintptr_t)t.m[k] | (uintptr_t)t.v[k]) & 15) == 0) ? 1 : 0;
        longest = t.n[k] > longest ? t.n[k] : longest;
    }
    if (longest == 0) return GS_OK;
    const long long per_block = (long long)AD_THREADS * 4;
    const long long blocks = (longest + per_block - 1) / per_block;
    GS_REQUIRE(blocks < (1ll << 31), "tensor too large");
    dim3 grid((unsigned)blocks, (unsigned)num_tensors);
    k_adam<<<grid, AD_THREADS, 0, (cudaStream_t)stream>>>(t, grad_scale);
    GS_LAUNCH_CHECK();
    return GS_OK;
}
