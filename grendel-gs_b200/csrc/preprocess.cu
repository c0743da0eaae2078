// Per-splat projection: stages "10 preprocess" / "b20 preprocess", the forward and backward of
// GaussianRasterizer.preprocess_gaussians (gaussian_renderer/__init__.py:949-958 of the reference).  Three forms share
// one set of stage functions:
//   k_preprocess_{fwd,bwd}<false,K>   activated inputs, SH as one (P,K,3) block        gs_preprocess_{forward,backward}
//   k_preprocess_{fwd,bwd}<true,K>    the six raw GaussianModel parameters, activations fused in          ..._raw
//   k_preprocess_{fwd,bwd}_batched<K> raw parameters, all B cameras of a step per launch, each splat read once  ..._batched
// K = (max_sh_degree + 1)^2 in {1, 4, 9, 16} is the number of SH coefficients the model stores (--sh_degree of the
// reference, scene/gaussian_model.py:51-53, 150-156).  A K-coefficient kernel does the K = 16 kernel's fp32 operations
// minus the terms whose basis value is zero (coefficients beyond the active degree), so with the stored coefficients
// zero-padded to 16 both give the same bits.
// Compiled with -fmad=false: radius, tile rectangle and depth key follow the IEEE fp32 operation sequence that
// oracle/gs_oracle.c repeats, so tile indices are bit-exact; the kernels are HBM-bound, so losing FMA costs nothing.
// A CTA's SH rows (12 K bytes per splat) come into shared memory by TMA bulk copies issued before the projection math, and
// dL/dSH leaves by TMA bulk stores.  cams (batched): (B, 40) floats per camera: viewmatrix[16], projmatrix[16]
// (transposed storage, scene/cameras.py:84-99), campos[3], tanfovx, tanfovy, 3 pad.
#include <initializer_list>
#include <type_traits>
#include "common.cuh"

#define PP_THREADS 128
#define PB_BWD_THREADS 64
#define PB_MAX_CAMS 64
#define DC_FLOATS 3
#define CAM_FLOATS 40

static __device__ __constant__ float c_SH_C0 = 0.28209479177387814f;
static __device__ __constant__ float c_SH_C1 = 0.4886025119029199f;
static __device__ __constant__ float c_SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                            -1.0925484305920792f, 0.5462742152960396f};
static __device__ __constant__ float c_SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                            0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                            -0.5900435899266435f};

// ---- camera ---------------------------------------------------------------------------------------------------------
struct Cam { float V[16], PM[16], cp[3]; };

GS_D void load_cam(Cam &c, const float *viewmatrix, const float *projmatrix, const float *campos) {
#pragma unroll
    for (int k = 0; k < 16; k++) { c.V[k] = __ldg(viewmatrix + k); c.PM[k] = __ldg(projmatrix + k); }
    c.cp[0] = __ldg(campos); c.cp[1] = __ldg(campos + 1); c.cp[2] = __ldg(campos + 2);
}

GS_D void load_cam_row(Cam &c, float &tanfovx, float &tanfovy, const float *__restrict__ row) {
    load_cam(c, row, row + 16, row + 32);
    tanfovx = __ldg(row + 35); tanfovy = __ldg(row + 36);
}

// ---- per-splat parameters and the GaussianModel activations (scene/gaussian_model.py:109-129) ------------------------
GS_D float3 ld3(const float *a) { return make_float3(a[0], a[1], a[2]); }
GS_D void st3(float *a, const float3 v) { a[0] = v.x; a[1] = v.y; a[2] = v.z; }
GS_D float3 add3(const float3 a, const float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
GS_D float sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// v / max(|v|, 1e-12); denom is kept for the backward
GS_D float4 normalize4(const float4 r, float &denom) {
    const float n = sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
    denom = fmaxf(n, 1e-12f);
    return make_float4(r.x / denom, r.y / denom, r.z / denom, r.w / denom);
}

// normalize': d r = (dq - q (q . dq)) / |r|
GS_D float4 normalize4_backward(const float4 q, const float4 dq, float denom) {
    const float dot = q.x * dq.x + q.y * dq.y + q.z * dq.z + q.w * dq.w;
    return make_float4((dq.x - q.x * dot) / denom, (dq.y - q.y * dot) / denom, (dq.z - q.z * dot) / denom,
                       (dq.w - q.w * dot) / denom);
}

// Scale and unit quaternion of splat i; RAW: from the log-scale and the unnormalised quaternion (den = its norm).
template <bool RAW>
GS_D void load_scale_rot(const float *scale, const float *rot, int i, float3 &sc, float4 &q, float &den) {
    const float4 r = *reinterpret_cast<const float4 *>(rot + 4 * i);
    if constexpr (RAW) {
        sc = make_float3(expf(scale[3 * i]), expf(scale[3 * i + 1]), expf(scale[3 * i + 2]));
        q = normalize4(r, den);
    } else { sc = ld3(scale + 3 * i); q = r; }
}

// ---- SH rows in shared memory ---------------------------------------------------------------------------------------
// The CTA's SH rows (flat index f = 3 * coefficient + channel, f < 3 K) lie in one block of 3 K floats per splat or,
// SPLIT (the raw parameters), in a block of the 3 dc floats per splat followed by a block of the 3 (K - 1) rest floats
// (none at K = 1: the rest pointers are then never read or written, and may be NULL).
template <bool SPLIT, int K> constexpr int N0 = SPLIT ? DC_FLOATS : 3 * K;       // floats per splat in the first block
template <bool SPLIT, int K> constexpr int N1 = SPLIT ? 3 * (K - 1) : 0;         // ... and in the rest block

template <int THREADS, bool SPLIT, int K>
struct ShRow {  // thread t's row
    float *s;
    int t;
    GS_D float &operator[](int f) const {
        constexpr int n0 = N0<SPLIT, K>;
        return f < n0 ? s[t * n0 + f] : s[THREADS * n0 + t * N1<SPLIT, K> + (f - n0)];
    }
};

// Bring the rows of the CTA's nvalid splats into s_sh.  Returns true when they come by TMA on the mbarrier, false when
// by plain loads: a bulk copy's size must be a multiple of 16 B, which a ragged tail block of n floats per splat misses
// when n is not a multiple of 4 and its splat count is not a multiple of 4 (the dc block of the split forms, and the
// unsplit block at K = 1 and K = 9).
template <int THREADS, bool SPLIT, int K>
GS_D bool stage_sh(float *s_sh, uint64_t *bar, const float *sh, const float *sh_rest, int base, int nvalid) {
    constexpr int n0 = N0<SPLIT, K>, n1 = N1<SPLIT, K>;
    float *s_dc = s_sh, *s_rest = s_sh + THREADS * n0;
    const bool tma = (n0 % 4 == 0 && n1 % 4 == 0) || (nvalid & 3) == 0;
    if (threadIdx.x == 0) { gs_mbar_init(bar, 1); gs_fence_mbar_init(); }
    __syncthreads();
    if (tma) {
        if (threadIdx.x == 0) {
            gs_mbar_arrive_expect_tx(bar, (uint32_t)nvalid * (n0 + n1) * 4u);
            gs_bulk_g2s(s_dc, sh + (size_t)base * n0, (uint32_t)nvalid * n0 * 4u, bar);
            if constexpr (n1 > 0) gs_bulk_g2s(s_rest, sh_rest + (size_t)base * n1, (uint32_t)nvalid * n1 * 4u, bar);
        }
    } else {
        for (int k = threadIdx.x; k < nvalid * n0; k += THREADS) s_dc[k] = sh[(size_t)base * n0 + k];
        if constexpr (n1 > 0)
            for (int k = threadIdx.x; k < nvalid * n1; k += THREADS) s_rest[k] = sh_rest[(size_t)base * n1 + k];
    }
    return tma;
}

// Every thread waits: the CTA must not retire with the bulk copy in flight.
GS_D void wait_sh(bool tma, uint64_t *bar) { if (tma) gs_mbar_wait(bar, 0); else __syncthreads(); }

// Write the CTA's dL/dSH rows from s_sh to d_sh (and d_sh_rest): TMA bulk stores, or plain stores after plain loads.
template <int THREADS, bool SPLIT, int K>
GS_D void store_sh(float *d_sh, float *d_sh_rest, float *s_sh, bool tma, int base, int nvalid) {
    constexpr int n0 = N0<SPLIT, K>, n1 = N1<SPLIT, K>;
    float *s_dc = s_sh, *s_rest = s_sh + THREADS * n0;
    gs_fence_proxy_async_smem();
    __syncthreads();
    if (tma) {
        if (threadIdx.x == 0) {
            gs_bulk_s2g(d_sh + (size_t)base * n0, s_dc, (uint32_t)nvalid * n0 * 4u);
            if constexpr (n1 > 0) gs_bulk_s2g(d_sh_rest + (size_t)base * n1, s_rest, (uint32_t)nvalid * n1 * 4u);
            gs_bulk_commit();
            gs_bulk_wait_read0();
        }
    } else {
        for (int k = threadIdx.x; k < nvalid * n0; k += THREADS) d_sh[(size_t)base * n0 + k] = s_dc[k];
        if constexpr (n1 > 0)
            for (int k = threadIdx.x; k < nvalid * n1; k += THREADS) d_sh_rest[(size_t)base * n1 + k] = s_rest[k];
    }
}

// ---- projection -----------------------------------------------------------------------------------------------------
GS_D void quat_to_R(const float4 q, float R[9]) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - r * z); R[2] = 2.f * (x * z + r * y);
    R[3] = 2.f * (x * y + r * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - r * x);
    R[6] = 2.f * (x * z - r * y); R[7] = 2.f * (y * z + r * x); R[8] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = (R S)(R S)^T; L = R diag(mod*s) row-major, S6 = xx,xy,xz,yy,yz,zz
GS_D void cov3d_from(const float3 sc, float mod, const float4 q, float L[9], float S[6]) {
    float R[9];
    quat_to_R(q, R);
    const float s0 = mod * sc.x, s1 = mod * sc.y, s2 = mod * sc.z;
    L[0] = R[0] * s0; L[1] = R[1] * s1; L[2] = R[2] * s2;
    L[3] = R[3] * s0; L[4] = R[4] * s1; L[5] = R[5] * s2;
    L[6] = R[6] * s0; L[7] = R[7] * s1; L[8] = R[8] * s2;
    S[0] = L[0] * L[0] + L[1] * L[1] + L[2] * L[2];
    S[1] = L[0] * L[3] + L[1] * L[4] + L[2] * L[5];
    S[2] = L[0] * L[6] + L[1] * L[7] + L[2] * L[8];
    S[3] = L[3] * L[3] + L[4] * L[4] + L[5] * L[5];
    S[4] = L[3] * L[6] + L[4] * L[7] + L[5] * L[8];
    S[5] = L[6] * L[6] + L[7] * L[7] + L[8] * L[8];
}

// SH basis of utils/sh_utils.py:57-120
GS_D void sh_basis(int deg, float x, float y, float z, float b[16]) {
    b[0] = c_SH_C0;
#pragma unroll
    for (int k = 1; k < 16; k++) b[k] = 0.f;
    if (deg > 0) {
        b[1] = -c_SH_C1 * y; b[2] = c_SH_C1 * z; b[3] = -c_SH_C1 * x;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = c_SH_C2[0] * xy; b[5] = c_SH_C2[1] * yz; b[6] = c_SH_C2[2] * (2.f * zz - xx - yy);
            b[7] = c_SH_C2[3] * xz; b[8] = c_SH_C2[4] * (xx - yy);
            if (deg > 2) {
                b[9] = c_SH_C3[0] * y * (3.f * xx - yy);
                b[10] = c_SH_C3[1] * xy * z;
                b[11] = c_SH_C3[2] * y * (4.f * zz - xx - yy);
                b[12] = c_SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
                b[13] = c_SH_C3[4] * x * (4.f * zz - xx - yy);
                b[14] = c_SH_C3[5] * z * (xx - yy);
                b[15] = c_SH_C3[6] * x * (xx - 3.f * yy);
            }
        }
    }
}

// Projection of one splat; returns false when culled. Shared by forward and backward so both see
// identical intermediates.
struct Proj {
    float tx, ty, tz;          // view space
    float hx, hy, hw, pw;      // clip space and 1/(w+eps)
    float L[9], S[6];
    float cx, cy, xmul, ymul;  // guard-band clamped view x,y and their gradient gates
    float J00, J02, J11, J12;
    float T0[3], T1[3], u0[3], u1[3];
    float a, b, c, det;
};

// COV_READY: o.L / o.S (camera independent) were filled by the caller -- the batched kernels compute them once per
// splat and project it into B cameras.
template <bool COV_READY = false>
GS_D bool project(const Cam &cam, const float3 p, const float3 sc, float mod, const float4 q, float fx, float fy,
                  float tanfovx, float tanfovy, Proj &o) {
    const float *V = cam.V, *PM = cam.PM;
    o.tx = V[0] * p.x + V[4] * p.y + V[8] * p.z + V[12];
    o.ty = V[1] * p.x + V[5] * p.y + V[9] * p.z + V[13];
    o.tz = V[2] * p.x + V[6] * p.y + V[10] * p.z + V[14];
    if (o.tz <= 0.2f) return false;
    o.hx = PM[0] * p.x + PM[4] * p.y + PM[8] * p.z + PM[12];
    o.hy = PM[1] * p.x + PM[5] * p.y + PM[9] * p.z + PM[13];
    o.hw = PM[3] * p.x + PM[7] * p.y + PM[11] * p.z + PM[15];
    o.pw = 1.0f / (o.hw + 0.0000001f);
    if (!COV_READY) cov3d_from(sc, mod, q, o.L, o.S);
    const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
    const float txtz = o.tx / o.tz, tytz = o.ty / o.tz;
    o.cx = fminf(limx, fmaxf(-limx, txtz)) * o.tz;
    o.cy = fminf(limy, fmaxf(-limy, tytz)) * o.tz;
    o.xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    o.ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    o.J00 = fx / o.tz; o.J02 = -(fx * o.cx) / (o.tz * o.tz);
    o.J11 = fy / o.tz; o.J12 = -(fy * o.cy) / (o.tz * o.tz);
    o.T0[0] = o.J00 * V[0] + o.J02 * V[2]; o.T0[1] = o.J00 * V[4] + o.J02 * V[6]; o.T0[2] = o.J00 * V[8] + o.J02 * V[10];
    o.T1[0] = o.J11 * V[1] + o.J12 * V[2]; o.T1[1] = o.J11 * V[5] + o.J12 * V[6]; o.T1[2] = o.J11 * V[9] + o.J12 * V[10];
    const float *S = o.S;
    o.u0[0] = S[0] * o.T0[0] + S[1] * o.T0[1] + S[2] * o.T0[2];
    o.u0[1] = S[1] * o.T0[0] + S[3] * o.T0[1] + S[4] * o.T0[2];
    o.u0[2] = S[2] * o.T0[0] + S[4] * o.T0[1] + S[5] * o.T0[2];
    o.u1[0] = S[0] * o.T1[0] + S[1] * o.T1[1] + S[2] * o.T1[2];
    o.u1[1] = S[1] * o.T1[0] + S[3] * o.T1[1] + S[4] * o.T1[2];
    o.u1[2] = S[2] * o.T1[0] + S[4] * o.T1[1] + S[5] * o.T1[2];
    o.a = o.T0[0] * o.u0[0] + o.T0[1] * o.u0[1] + o.T0[2] * o.u0[2] + 0.3f;
    o.b = o.T0[0] * o.u1[0] + o.T0[1] * o.u1[1] + o.T0[2] * o.u1[2];
    o.c = o.T1[0] * o.u1[0] + o.T1[1] * o.u1[1] + o.T1[2] * o.u1[2] + 0.3f;
    o.det = o.a * o.c - o.b * o.b;
    return o.det != 0.f;
}

// ---- forward stages -------------------------------------------------------------------------------------------------
// What the forward writes for one splat in one camera (pixel centre, depth, radius, conic + opacity); zero if culled.
struct Footprint { float2 xy; float depth; int rad; float4 co; };

// Radius, pixel centre and conic of a projected splat.  Returns false, leaving fp untouched, when its tile rectangle
// is empty; the caller fills in the opacity.
GS_D bool screen(const Proj &pr, int W, int H, Footprint &fp) {
    const int gx = (W + GS_BLOCK_X - 1) / GS_BLOCK_X, gy = (H + GS_BLOCK_Y - 1) / GS_BLOCK_Y;
    const float det_inv = 1.0f / pr.det;
    const float mid = 0.5f * (pr.a + pr.c);
    const float disc = sqrtf(fmaxf(0.1f, mid * mid - pr.det));
    const float lam = fmaxf(mid + disc, mid - disc);
    const int rad = (int)ceilf(3.f * sqrtf(lam));
    const float ndcx = pr.hx * pr.pw, ndcy = pr.hy * pr.pw;
    const float ix = ((ndcx + 1.f) * (float)W - 1.f) * 0.5f;
    const float iy = ((ndcy + 1.f) * (float)H - 1.f) * 0.5f;
    int x0, y0, x1, y1;
    gs_get_rect(ix, iy, rad, gx, gy, x0, y0, x1, y1);
    if ((x1 - x0) * (y1 - y0) == 0) return false;
    fp = {make_float2(ix, iy), pr.tz, rad, make_float4(pr.c * det_inv, -pr.b * det_inv, pr.a * det_inv, 0.f)};
    return true;
}

// Unit view direction from the camera centre to p; len is the distance.
GS_D float3 view_dir(const float3 p, const float *cp, float &len) {
    const float dx = p.x - cp[0], dy = p.y - cp[1], dz = p.z - cp[2];
    len = sqrtf(dx * dx + dy * dy + dz * dz);
    return make_float3(dx / len, dy / len, dz / len);
}

// Colour of a visible splat: its SH of degree D along the view direction, + 0.5, clamped at 0.  cm gets the clamp
// bits (1, 2, 4 = r, g, b) that mask the backward.  The row holds K coefficients, D <= sqrt(K) - 1.
template <int K, class Row>
GS_D float3 sh_forward(int D, const float3 p, const float *cp, const Row sh, uint8_t &cm) {
    float len;
    const float3 d = view_dir(p, cp, len);
    float bas[16];
    sh_basis(D, d.x, d.y, d.z, bas);
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int f = 0; f < 3 * K; f++) acc[f % 3] += bas[f / 3] * sh[f];
    float c0 = acc[0] + 0.5f, c1 = acc[1] + 0.5f, c2 = acc[2] + 0.5f;
    cm = 0;
    if (c0 < 0.f) { cm |= 1; c0 = 0.f; }
    if (c1 < 0.f) { cm |= 2; c1 = 0.f; }
    if (c2 < 0.f) { cm |= 4; c2 = 0.f; }
    return make_float3(c0, c1, c2);
}

template <class Idx>
GS_D void store_footprint(Idx o, const Footprint &fp, const float3 c, uint8_t cm, float *means2D, float *depths,
                          int32_t *radii, float *conic_opacity, float *rgb, uint8_t *clamped) {
    *reinterpret_cast<float2 *>(means2D + 2 * o) = fp.xy;
    depths[o] = fp.depth;
    radii[o] = fp.rad;
    *reinterpret_cast<float4 *>(conic_opacity + 4 * o) = fp.co;
    st3(rgb + 3 * o, c);
    clamped[o] = cm;
}

// ---- backward stages ------------------------------------------------------------------------------------------------
// Gradients of one camera's screen-space outputs, back through the projection.
struct CovGrad {
    float3 m_cov;   // mean gradient through the 2D covariance: cov2D -> T -> J -> view-space mean
    float3 m_2d;    // mean gradient through means2D and the perspective divide
    float G[6];     // dL/dSigma, symmetric: xx, xy, xz, yy, yz, zz
};

GS_D CovGrad cov2d_backward(const Proj &pr, const Cam &cam, float fx, float fy, const float4 gco, const float2 g2) {
    const float *V = cam.V, *PM = cam.PM;
    CovGrad o;
    // conic (A,B,C) = (c,-b,a)/det  ->  cov2D (a,b,c)
    const float a = pr.a, b = pr.b, c = pr.c, det = pr.det;
    float dLda = 0.f, dLdb = 0.f, dLdc = 0.f;
    if (det != 0.f) {
        const float d2 = 1.0f / (det * det);
        dLda = d2 * (-c * c * gco.x + b * c * gco.y - b * b * gco.z);
        dLdb = d2 * (2.f * b * c * gco.x - (det + 2.f * b * b) * gco.y + 2.f * a * b * gco.z);
        dLdc = d2 * (-b * b * gco.x + a * b * gco.y - a * a * gco.z);
    }
    // cov2D -> T -> J -> view-space mean
    float dT0[3], dT1[3];
#pragma unroll
    for (int r = 0; r < 3; r++) {
        dT0[r] = 2.f * dLda * pr.u0[r] + dLdb * pr.u1[r];
        dT1[r] = 2.f * dLdc * pr.u1[r] + dLdb * pr.u0[r];
    }
    const float dJ00 = dT0[0] * V[0] + dT0[1] * V[4] + dT0[2] * V[8];
    const float dJ02 = dT0[0] * V[2] + dT0[1] * V[6] + dT0[2] * V[10];
    const float dJ11 = dT1[0] * V[1] + dT1[1] * V[5] + dT1[2] * V[9];
    const float dJ12 = dT1[0] * V[2] + dT1[1] * V[6] + dT1[2] * V[10];
    const float tzi = 1.0f / pr.tz, tzi2 = tzi * tzi, tzi3 = tzi2 * tzi;
    const float dtx = pr.xmul * (-fx * tzi2) * dJ02;
    const float dty = pr.ymul * (-fy * tzi2) * dJ12;
    const float dtz = -fx * tzi2 * dJ00 - fy * tzi2 * dJ11 + 2.f * fx * pr.cx * tzi3 * dJ02 +
                      2.f * fy * pr.cy * tzi3 * dJ12;
    o.m_cov = make_float3(V[0] * dtx + V[1] * dty + V[2] * dtz, V[4] * dtx + V[5] * dty + V[6] * dtz,
                          V[8] * dtx + V[9] * dty + V[10] * dtz);
    // means2D (per NDC unit) -> mean3D through the perspective divide
    const float dhx = g2.x * pr.pw, dhy = g2.y * pr.pw;
    const float dhw = -(g2.x * pr.hx + g2.y * pr.hy) * pr.pw * pr.pw;
    o.m_2d = make_float3(PM[0] * dhx + PM[1] * dhy + PM[3] * dhw, PM[4] * dhx + PM[5] * dhy + PM[7] * dhw,
                         PM[8] * dhx + PM[9] * dhy + PM[11] * dhw);
    // cov2D = T Sigma T^T -> Sigma
    const int rr[6] = {0, 0, 0, 1, 1, 2}, ss[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; e++) {
        const int r = rr[e], s = ss[e];
        o.G[e] = pr.T0[r] * pr.T0[s] * dLda + 0.5f * (pr.T0[r] * pr.T1[s] + pr.T0[s] * pr.T1[r]) * dLdb +
                 pr.T1[r] * pr.T1[s] * dLdc;
    }
    return o;
}

// dL/dSigma -> gradients of the activated scale (gs) and of the unit quaternion (dq), through Sigma = L L^T,
// L = R diag(mod*s).
GS_D void sigma_backward(const float G[6], const float4 q, const float3 sc, float mod, const float L[9], float3 &gs,
                         float4 &dq) {
    const float Gm[3][3] = {{G[0], G[1], G[2]}, {G[1], G[3], G[4]}, {G[2], G[4], G[5]}};
    float R[9];
    quat_to_R(q, R);
    const float s[3] = {mod * sc.x, mod * sc.y, mod * sc.z};
    float dLm[9];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int k = 0; k < 3; k++)
            dLm[3 * r + k] = 2.f * (Gm[r][0] * L[k] + Gm[r][1] * L[3 + k] + Gm[r][2] * L[6 + k]);
    float dR[9], gsk[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        gsk[k] = mod * (dLm[k] * R[k] + dLm[3 + k] * R[3 + k] + dLm[6 + k] * R[6 + k]);
        dR[k] = dLm[k] * s[k]; dR[3 + k] = dLm[3 + k] * s[k]; dR[6 + k] = dLm[6 + k] * s[k];
    }
    gs = make_float3(gsk[0], gsk[1], gsk[2]);
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    dq.x = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
    dq.y = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] + r * dR[7] -
                  2.f * x * dR[8]);
    dq.z = 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] + z * dR[7] -
                  2.f * y * dR[8]);
    dq.w = 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] + y * dR[5] +
                  x * dR[6] + y * dR[7]);
}

// Colour gradient g_rgb (3 floats; channels clamped in the forward get none) -> dL/dSH of the row and the gradient
// through the view direction into the mean, which is returned.  ACCUM (several cameras): the dL/dSH of the
// coefficients in use is added to row g.  Otherwise every slot of row sh is overwritten with its gradient (zero beyond
// degree D) and g is not touched.  The rows hold K coefficients, D <= sqrt(K) - 1.
template <bool ACCUM, int K, class Row>
GS_D float3 sh_backward(int D, const float3 p, const float *cp, uint8_t cm, const float *g_rgb, const Row sh,
                        const Row g) {
    float len;
    const float3 d = view_dir(p, cp, len);
    const float x = d.x, y = d.y, z = d.z;
    float bas[16];
    sh_basis(D, x, y, z, bas);
    const float dc[3] = {(cm & 1) ? 0.f : g_rgb[0], (cm & 2) ? 0.f : g_rgb[1], (cm & 4) ? 0.f : g_rgb[2]};
    const int ncoef = (D + 1) * (D + 1);
    float s[16] = {};  // dL/d(basis value), per coefficient
#pragma unroll
    for (int j = 0; j < 3 * K; j += 4) {
        float v[4];  // four loads, then four stores: on a contiguous row both vectorise
#pragma unroll
        for (int e = 0; e < 4; e++)
            if (j + e < 3 * K) v[e] = sh[j + e];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int f = j + e, k = f / 3, ch = f % 3;
            if (f >= 3 * K) break;
            if constexpr (ACCUM) {
                if (k < ncoef) { s[k] += v[e] * dc[ch]; g[f] += bas[k] * dc[ch]; }
            } else {
                s[k] += (k < ncoef) ? v[e] * dc[ch] : 0.f;
                sh[f] = (k < ncoef) ? bas[k] * dc[ch] : 0.f;
            }
        }
    }
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;
    if (D > 0) {
        ddx += -c_SH_C1 * s[3]; ddy += -c_SH_C1 * s[1]; ddz += c_SH_C1 * s[2];
        if (D > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            ddx += c_SH_C2[0] * y * s[4] + c_SH_C2[2] * 2.f * -x * s[6] + c_SH_C2[3] * z * s[7] +
                   c_SH_C2[4] * 2.f * x * s[8];
            ddy += c_SH_C2[0] * x * s[4] + c_SH_C2[1] * z * s[5] + c_SH_C2[2] * 2.f * -y * s[6] +
                   c_SH_C2[4] * 2.f * -y * s[8];
            ddz += c_SH_C2[1] * y * s[5] + c_SH_C2[2] * 4.f * z * s[6] + c_SH_C2[3] * x * s[7];
            if (D > 2) {
                ddx += c_SH_C3[0] * s[9] * 6.f * xy + c_SH_C3[1] * s[10] * yz + c_SH_C3[2] * s[11] * -2.f * xy +
                       c_SH_C3[3] * s[12] * -6.f * xz + c_SH_C3[4] * s[13] * (-3.f * xx + 4.f * zz - yy) +
                       c_SH_C3[5] * s[14] * 2.f * xz + c_SH_C3[6] * s[15] * 3.f * (xx - yy);
                ddy += c_SH_C3[0] * s[9] * 3.f * (xx - yy) + c_SH_C3[1] * s[10] * xz +
                       c_SH_C3[2] * s[11] * (-3.f * yy + 4.f * zz - xx) + c_SH_C3[3] * s[12] * -6.f * yz +
                       c_SH_C3[4] * s[13] * -2.f * xy + c_SH_C3[5] * s[14] * -2.f * yz +
                       c_SH_C3[6] * s[15] * -6.f * xy;
                ddz += c_SH_C3[1] * s[10] * xy + c_SH_C3[2] * s[11] * 8.f * yz +
                       c_SH_C3[3] * s[12] * 3.f * (2.f * zz - xx - yy) + c_SH_C3[4] * s[13] * 8.f * xz +
                       c_SH_C3[5] * s[14] * (xx - yy);
            }
        }
    }
    const float dot = x * ddx + y * ddy + z * ddz;
    return make_float3((ddx - x * dot) / len, (ddy - y * dot) / len, (ddz - z * dot) / len);
}

// ---- single-camera kernels ------------------------------------------------------------------------------------------
// RAW = false: scale, rotation (unit), opacity as the rasterizer takes them and sh = the (P,K,3) block (sh_rest and
// d_sh_rest unused).  RAW = true: the GaussianModel parameters, sh / sh_rest = _features_dc / _features_rest.
template <bool RAW, int K>
__global__ void __launch_bounds__(PP_THREADS) k_preprocess_fwd(
    int P, int D, const float *__restrict__ xyz, const float *__restrict__ sh, const float *__restrict__ sh_rest,
    const float *__restrict__ scale, float mod, const float *__restrict__ rot, const float *__restrict__ opac,
    const float *__restrict__ viewmatrix, const float *__restrict__ projmatrix, const float *__restrict__ campos,
    int W, int H, float tanfovx, float tanfovy, float *__restrict__ means2D, float *__restrict__ depths,
    int32_t *__restrict__ radii, float *__restrict__ conic_opacity, float *__restrict__ rgb, uint8_t *__restrict__ clamped) {
    __shared__ __align__(128) float s_sh[PP_THREADS * 3 * K];
    __shared__ __align__(8) uint64_t s_bar;
    const int base = blockIdx.x * PP_THREADS, nvalid = min(PP_THREADS, P - base);
    const bool tma = stage_sh<PP_THREADS, RAW, K>(s_sh, &s_bar, sh, sh_rest, base, nvalid);
    const int i = base + threadIdx.x;
    bool vis = false;
    Footprint fp = {};
    float3 p = make_float3(0.f, 0.f, 0.f);
    Cam cam;
    if (i < P) {
        load_cam(cam, viewmatrix, projmatrix, campos);
        p = ld3(xyz + 3 * i);
        const float tz = cam.V[2] * p.x + cam.V[6] * p.y + cam.V[10] * p.z + cam.V[14];
        if (tz > 0.2f) {  // a splat behind the near plane needs no scale / rotation loads
            float3 sc; float4 q; float den;
            load_scale_rot<RAW>(scale, rot, i, sc, q, den);
            const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
            Proj pr;
            if (project(cam, p, sc, mod, q, fx, fy, tanfovx, tanfovy, pr) && screen(pr, W, H, fp)) {
                vis = true;
                fp.co.w = RAW ? sigmoid(opac[i]) : opac[i];
            }
        }
    }
    wait_sh(tma, &s_bar);
    if (i >= P) return;
    float3 c = make_float3(0.f, 0.f, 0.f); uint8_t cm = 0;
    if (vis) c = sh_forward<K>(D, p, cam.cp, ShRow<PP_THREADS, RAW, K>{s_sh, (int)threadIdx.x}, cm);
    store_footprint(i, fp, c, cm, means2D, depths, radii, conic_opacity, rgb, clamped);
}

template <bool RAW, int K>
__global__ void __launch_bounds__(PP_THREADS) k_preprocess_bwd(
    int P, int D, const float *__restrict__ xyz, const float *__restrict__ sh, const float *__restrict__ sh_rest,
    const float *__restrict__ scale, float mod, const float *__restrict__ rot, const float *__restrict__ opac,
    const float *__restrict__ viewmatrix, const float *__restrict__ projmatrix, const float *__restrict__ campos,
    int W, int H, float tanfovx, float tanfovy, const int32_t *__restrict__ radii, const uint8_t *__restrict__ clamped,
    const float *__restrict__ g_means2D, const float *__restrict__ g_conic_opacity, const float *__restrict__ g_rgb,
    float *__restrict__ d_xyz, float *__restrict__ d_sh, float *__restrict__ d_sh_rest, float *__restrict__ d_scale,
    float *__restrict__ d_rot, float *__restrict__ d_opac) {
    __shared__ __align__(128) float s_sh[PP_THREADS * 3 * K];
    __shared__ __align__(8) uint64_t s_bar;
    const int base = blockIdx.x * PP_THREADS, nvalid = min(PP_THREADS, P - base);
    const bool tma = stage_sh<PP_THREADS, RAW, K>(s_sh, &s_bar, sh, sh_rest, base, nvalid);
    const int i = base + threadIdx.x;
    const bool act = (i < P) && (radii[i] > 0);
    float3 p = make_float3(0.f, 0.f, 0.f), gm = p, gs = p;
    float4 gq = make_float4(0.f, 0.f, 0.f, 0.f);
    float gop = 0.f;
    Cam cam;
    if (act) {
        load_cam(cam, viewmatrix, projmatrix, campos);
        p = ld3(xyz + 3 * i);
        float3 sc; float4 q; float den;
        load_scale_rot<RAW>(scale, rot, i, sc, q, den);
        const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
        Proj pr;
        project(cam, p, sc, mod, q, fx, fy, tanfovx, tanfovy, pr);
        const float4 gco = *reinterpret_cast<const float4 *>(g_conic_opacity + 4 * i);
        const CovGrad cg = cov2d_backward(pr, cam, fx, fy, gco, *reinterpret_cast<const float2 *>(g_means2D + 2 * i));
        gm = add3(cg.m_cov, cg.m_2d);
        float4 dq;
        sigma_backward(cg.G, q, sc, mod, pr.L, gs, dq);
        if constexpr (RAW) {
            const float op = sigmoid(opac[i]);
            gop = gco.w * op * (1.f - op);                                 // sigmoid'
            gs = make_float3(gs.x * sc.x, gs.y * sc.y, gs.z * sc.z);       // exp'
            gq = normalize4_backward(q, dq, den);
        } else { gop = gco.w; gq = dq; }
    }
    wait_sh(tma, &s_bar);
    // colour -> SH coefficients (written in place over the staged rows) and view direction
    if (i < P) {
        const ShRow<PP_THREADS, RAW, K> row{s_sh, (int)threadIdx.x};
        if (act) {
            gm = add3(gm, sh_backward<false, K>(D, p, cam.cp, clamped[i], g_rgb + 3 * i, row, row));
        } else {
#pragma unroll
            for (int f = 0; f < 3 * K; f++) row[f] = 0.f;
        }
        st3(d_xyz + 3 * i, gm); st3(d_scale + 3 * i, gs);
        *reinterpret_cast<float4 *>(d_rot + 4 * i) = gq;
        d_opac[i] = gop;
    }
    store_sh<PP_THREADS, RAW, K>(d_sh, d_sh_rest, s_sh, tma, base, nvalid);
}

// ---- batched kernels: B cameras, each Gaussian read once ------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(PP_THREADS) k_preprocess_fwd_batched(
    int B, int P, int D, const float *__restrict__ xyz, const float *__restrict__ f_dc, const float *__restrict__ f_rest,
    const float *__restrict__ scaling, float mod, const float *__restrict__ rotation, const float *__restrict__ opacity,
    const float *__restrict__ cams, int W, int H, float *__restrict__ means2D, float *__restrict__ depths,
    int32_t *__restrict__ radii, float *__restrict__ conic_opacity, float *__restrict__ rgb, uint8_t *__restrict__ clamped) {
    __shared__ __align__(128) float s_sh[PP_THREADS * 3 * K];
    __shared__ __align__(8) uint64_t s_bar;
    const int base = blockIdx.x * PP_THREADS, nvalid = min(PP_THREADS, P - base);
    const bool tma = stage_sh<PP_THREADS, true, K>(s_sh, &s_bar, f_dc, f_rest, base, nvalid);
    const int i = base + threadIdx.x;
    float3 p = make_float3(0.f, 0.f, 0.f), sc = p;
    float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
    float op = 0.f;
    Proj pr;
    if (i < P) {
        p = ld3(xyz + 3 * i);
        float den;
        load_scale_rot<true>(scaling, rotation, i, sc, q, den);
        op = sigmoid(opacity[i]);
        cov3d_from(sc, mod, q, pr.L, pr.S);  // camera independent
    }
    wait_sh(tma, &s_bar);
    if (i >= P) return;
    const ShRow<PP_THREADS, true, K> row{s_sh, (int)threadIdx.x};
    for (int k = 0; k < B; k++) {
        Cam cam; float tanfovx, tanfovy;
        load_cam_row(cam, tanfovx, tanfovy, cams + (size_t)k * CAM_FLOATS);
        const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
        Footprint fp = {};
        float3 c = make_float3(0.f, 0.f, 0.f); uint8_t cm = 0;
        if (project<true>(cam, p, sc, mod, q, fx, fy, tanfovx, tanfovy, pr) && screen(pr, W, H, fp)) {
            fp.co.w = op;
            c = sh_forward<K>(D, p, cam.cp, row, cm);
        }
        store_footprint((size_t)k * P + i, fp, c, cm, means2D, depths, radii, conic_opacity, rgb, clamped);
    }
}

template <int K>
__global__ void __launch_bounds__(PB_BWD_THREADS) k_preprocess_bwd_batched(
    int B, int P, int D, const float *__restrict__ xyz, const float *__restrict__ f_dc, const float *__restrict__ f_rest,
    const float *__restrict__ scaling, float mod, const float *__restrict__ rotation, const float *__restrict__ opacity,
    const float *__restrict__ cams, int W, int H, const int32_t *__restrict__ radii, const uint8_t *__restrict__ clamped,
    const float *__restrict__ g_means2D, const float *__restrict__ g_conic_opacity, const float *__restrict__ g_rgb,
    float *__restrict__ d_xyz, float *__restrict__ d_dc, float *__restrict__ d_rest, float *__restrict__ d_scaling,
    float *__restrict__ d_rotation, float *__restrict__ d_opacity) {
    __shared__ __align__(128) float s_sh[PB_BWD_THREADS * 3 * K];   // SH coefficients of the CTA's splats
    __shared__ __align__(128) float s_g[PB_BWD_THREADS * 3 * K];    // dL/dSH accumulated over the cameras
    __shared__ __align__(8) uint64_t s_bar;
    const int base = blockIdx.x * PB_BWD_THREADS, nvalid = min(PB_BWD_THREADS, P - base);
    const bool tma = stage_sh<PB_BWD_THREADS, true, K>(s_sh, &s_bar, f_dc, f_rest, base, nvalid);
    const int i = base + threadIdx.x;
    const ShRow<PB_BWD_THREADS, true, K> row{s_sh, (int)threadIdx.x}, grow{s_g, (int)threadIdx.x};
#pragma unroll
    for (int f = 0; f < 3 * K; f++) grow[f] = 0.f;
    float3 p = make_float3(0.f, 0.f, 0.f), sc = p;
    float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
    float den = 1.f, op = 0.f;
    Proj pr;
    if (i < P) {
        p = ld3(xyz + 3 * i);
        load_scale_rot<true>(scaling, rotation, i, sc, q, den);
        op = sigmoid(opacity[i]);
        cov3d_from(sc, mod, q, pr.L, pr.S);
    }
    wait_sh(tma, &s_bar);
    if (i < P) {
        float3 gm = make_float3(0.f, 0.f, 0.f);
        float gop = 0.f, G[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // dL/dSigma summed over the cameras
        for (int k = 0; k < B; k++) {
            const size_t o = (size_t)k * P + i;
            if (radii[o] <= 0) continue;
            Cam cam; float tanfovx, tanfovy;
            load_cam_row(cam, tanfovx, tanfovy, cams + (size_t)k * CAM_FLOATS);
            const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
            project<true>(cam, p, sc, mod, q, fx, fy, tanfovx, tanfovy, pr);
            const float4 gco = *reinterpret_cast<const float4 *>(g_conic_opacity + 4 * o);
            gop += gco.w;
            const CovGrad cg = cov2d_backward(pr, cam, fx, fy, gco, *reinterpret_cast<const float2 *>(g_means2D + 2 * o));
            gm = add3(add3(gm, cg.m_cov), cg.m_2d);
#pragma unroll
            for (int e = 0; e < 6; e++) G[e] += cg.G[e];
            gm = add3(gm, sh_backward<true, K>(D, p, cam.cp, clamped[o], g_rgb + 3 * o, row, grow));
        }
        // Sigma -> (scale, rotation) once, with the accumulated dL/dSigma
        float3 gs; float4 dq;
        sigma_backward(G, q, sc, mod, pr.L, gs, dq);
        st3(d_xyz + 3 * i, gm);
        st3(d_scaling + 3 * i, make_float3(gs.x * sc.x, gs.y * sc.y, gs.z * sc.z));  // exp'
        *reinterpret_cast<float4 *>(d_rotation + 4 * i) = normalize4_backward(q, dq, den);
        d_opacity[i] = gop * op * (1.f - op);  // sigmoid'
    }
    store_sh<PB_BWD_THREADS, true, K>(d_dc, d_rest, s_g, tma, base, nvalid);
}

// ---- C ABI ----------------------------------------------------------------------------------------------------------
// Checks shared by the entry points: GS_EINVAL with the error set, or GS_OK.  B is the camera count (1 for the
// single-camera forms).  rest: the features_rest pointers of the split forms, unused (and allowed to be NULL) when the
// model stores degree 0 only.  With P == 0 nothing past the sizes is checked, and launch() does nothing.
static int check_args(int B, int P, int sh_degree, int max_sh_degree, bool image_ok,
                      std::initializer_list<const void *> ptrs, std::initializer_list<const void *> aligned16,
                      const void *aligned8, std::initializer_list<const void *> rest = {}) {
    GS_REQUIRE(B > 0 && B <= PB_MAX_CAMS && P >= 0, "sizes");
    GS_REQUIRE(max_sh_degree >= 0 && max_sh_degree <= 3, "max_sh_degree must be 0..3");
    GS_REQUIRE(sh_degree >= 0 && sh_degree <= max_sh_degree, "sh_degree must be 0..max_sh_degree");
    if (P == 0) return GS_OK;
    GS_REQUIRE(image_ok, "image size");
    for (const void *p : ptrs) GS_REQUIRE(p != nullptr, "null pointer");
    for (const void *p : aligned16) GS_REQUIRE(((uintptr_t)p & 15) == 0, "16-byte alignment");
    GS_REQUIRE(((uintptr_t)aligned8 & 7) == 0, "8-byte alignment");
    if (max_sh_degree > 0)
        for (const void *p : rest) {
            GS_REQUIRE(p != nullptr, "null features_rest pointer with max_sh_degree > 0");
            GS_REQUIRE(((uintptr_t)p & 15) == 0, "16-byte alignment");
        }
    return GS_OK;
}

template <class... Params, class... Args>
static int launch(int stage, int P, int threads, void *stream, void (*kernel)(Params...), Args... args) {
    if (P == 0) return GS_OK;
    GsStageTimer timer(stage, (cudaStream_t)stream);
    kernel<<<(P + threads - 1) / threads, threads, 0, (cudaStream_t)stream>>>(args...);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// f(std::integral_constant<int, K>) with K = (max_sh_degree + 1)^2, the instantiation for the stored coefficients
template <class F>
static int with_coefficients(int max_sh_degree, F f) {
    switch (max_sh_degree) {
    case 0: return f(std::integral_constant<int, 1>{});
    case 1: return f(std::integral_constant<int, 4>{});
    case 2: return f(std::integral_constant<int, 9>{});
    default: return f(std::integral_constant<int, 16>{});
    }
}

extern "C" int gs_preprocess_forward_sh(
    int P, int sh_degree, int max_sh_degree, const float *means3D, const float *scales, float scale_modifier,
    const float *rotations, const float *opacities, const float *shs, const float *viewmatrix, const float *projmatrix,
    const float *campos, int image_width, int image_height, float tanfovx, float tanfovy, float *means2D, float *depths,
    int32_t *radii, float *conic_opacity, float *rgb, uint8_t *clamped, void *stream) {
    // unlike the other entry points, this one has always refused an empty image even when P == 0
    GS_REQUIRE(image_width > 0 && image_height > 0, "image size");
    if (int rc = check_args(1, P, sh_degree, max_sh_degree, true, {means3D, scales, rotations, opacities, shs,
                            viewmatrix, projmatrix, campos, means2D, depths, radii, conic_opacity, rgb, clamped},
                            {shs, rotations, conic_opacity}, means2D)) return rc;
    return with_coefficients(max_sh_degree, [&](auto k) {
        return launch(GS_STAGE_PREPROCESS_FWD, P, PP_THREADS, stream, k_preprocess_fwd<false, decltype(k)::value>, P,
                      sh_degree, means3D, shs, (const float *)nullptr, scales, scale_modifier, rotations, opacities,
                      viewmatrix, projmatrix, campos, image_width, image_height, tanfovx, tanfovy, means2D, depths,
                      radii, conic_opacity, rgb, clamped);
    });
}

extern "C" int gs_preprocess_forward(
    int P, int sh_degree, const float *means3D, const float *scales, float scale_modifier, const float *rotations,
    const float *opacities, const float *shs, const float *viewmatrix, const float *projmatrix, const float *campos,
    int image_width, int image_height, float tanfovx, float tanfovy, float *means2D, float *depths, int32_t *radii,
    float *conic_opacity, float *rgb, uint8_t *clamped, void *stream) {
    return gs_preprocess_forward_sh(P, sh_degree, 3, means3D, scales, scale_modifier, rotations, opacities, shs,
                                    viewmatrix, projmatrix, campos, image_width, image_height, tanfovx, tanfovy, means2D,
                                    depths, radii, conic_opacity, rgb, clamped, stream);
}

extern "C" int gs_preprocess_backward_sh(
    int P, int sh_degree, int max_sh_degree, const float *means3D, const float *scales, float scale_modifier,
    const float *rotations, const float *shs, const float *viewmatrix, const float *projmatrix, const float *campos,
    int image_width, int image_height, float tanfovx, float tanfovy, const int32_t *radii, const uint8_t *clamped,
    const float *dL_dmeans2D, const float *dL_dconic_opacity, const float *dL_drgb, float *dL_dmeans3D,
    float *dL_dscales, float *dL_drotations, float *dL_dopacities, float *dL_dshs, void *stream) {
    if (int rc = check_args(1, P, sh_degree, max_sh_degree, true, {means3D, scales, rotations, shs, viewmatrix,
                            projmatrix, campos, radii, clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dmeans3D,
                            dL_dscales, dL_drotations, dL_dopacities, dL_dshs},
                            {shs, dL_dshs, rotations, dL_drotations, dL_dconic_opacity}, dL_dmeans2D)) return rc;
    return with_coefficients(max_sh_degree, [&](auto k) {
        return launch(GS_STAGE_PREPROCESS_BWD, P, PP_THREADS, stream, k_preprocess_bwd<false, decltype(k)::value>, P,
                      sh_degree, means3D, shs, (const float *)nullptr, scales, scale_modifier, rotations,
                      (const float *)nullptr, viewmatrix, projmatrix, campos, image_width, image_height, tanfovx,
                      tanfovy, radii, clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dmeans3D, dL_dshs,
                      (float *)nullptr, dL_dscales, dL_drotations, dL_dopacities);
    });
}

extern "C" int gs_preprocess_backward(
    int P, int sh_degree, const float *means3D, const float *scales, float scale_modifier, const float *rotations,
    const float *shs, const float *viewmatrix, const float *projmatrix, const float *campos, int image_width,
    int image_height, float tanfovx, float tanfovy, const int32_t *radii, const uint8_t *clamped,
    const float *dL_dmeans2D, const float *dL_dconic_opacity, const float *dL_drgb, float *dL_dmeans3D,
    float *dL_dscales, float *dL_drotations, float *dL_dopacities, float *dL_dshs, void *stream) {
    return gs_preprocess_backward_sh(P, sh_degree, 3, means3D, scales, scale_modifier, rotations, shs, viewmatrix,
                                     projmatrix, campos, image_width, image_height, tanfovx, tanfovy, radii, clamped,
                                     dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dmeans3D, dL_dscales, dL_drotations,
                                     dL_dopacities, dL_dshs, stream);
}

extern "C" int gs_preprocess_forward_raw_sh(
    int P, int sh_degree, int max_sh_degree, const float *xyz, const float *features_dc, const float *features_rest,
    const float *scaling, float scale_modifier, const float *rotation, const float *opacity, const float *viewmatrix,
    const float *projmatrix, const float *campos, int image_width, int image_height, float tanfovx, float tanfovy,
    float *means2D, float *depths, int32_t *radii, float *conic_opacity, float *rgb, uint8_t *clamped, void *stream) {
    if (int rc = check_args(1, P, sh_degree, max_sh_degree, image_width > 0 && image_height > 0, {xyz, features_dc,
                            scaling, rotation, opacity, viewmatrix, projmatrix, campos, means2D, depths, radii,
                            conic_opacity, rgb, clamped},
                            {features_dc, rotation, conic_opacity}, means2D, {features_rest})) return rc;
    return with_coefficients(max_sh_degree, [&](auto k) {
        return launch(GS_STAGE_PREPROCESS_FWD, P, PP_THREADS, stream, k_preprocess_fwd<true, decltype(k)::value>, P,
                      sh_degree, xyz, features_dc, features_rest, scaling, scale_modifier, rotation, opacity,
                      viewmatrix, projmatrix, campos, image_width, image_height, tanfovx, tanfovy, means2D, depths,
                      radii, conic_opacity, rgb, clamped);
    });
}

extern "C" int gs_preprocess_forward_raw(
    int P, int sh_degree, const float *xyz, const float *features_dc, const float *features_rest, const float *scaling,
    float scale_modifier, const float *rotation, const float *opacity, const float *viewmatrix, const float *projmatrix,
    const float *campos, int image_width, int image_height, float tanfovx, float tanfovy, float *means2D, float *depths,
    int32_t *radii, float *conic_opacity, float *rgb, uint8_t *clamped, void *stream) {
    return gs_preprocess_forward_raw_sh(P, sh_degree, 3, xyz, features_dc, features_rest, scaling, scale_modifier,
                                        rotation, opacity, viewmatrix, projmatrix, campos, image_width, image_height,
                                        tanfovx, tanfovy, means2D, depths, radii, conic_opacity, rgb, clamped, stream);
}

extern "C" int gs_preprocess_backward_raw_sh(
    int P, int sh_degree, int max_sh_degree, const float *xyz, const float *features_dc, const float *features_rest,
    const float *scaling, float scale_modifier, const float *rotation, const float *opacity, const float *viewmatrix,
    const float *projmatrix, const float *campos, int image_width, int image_height, float tanfovx, float tanfovy,
    const int32_t *radii, const uint8_t *clamped, const float *dL_dmeans2D, const float *dL_dconic_opacity,
    const float *dL_drgb, float *dL_dxyz, float *dL_dfeatures_dc, float *dL_dfeatures_rest, float *dL_dscaling,
    float *dL_drotation, float *dL_dopacity, void *stream) {
    if (int rc = check_args(1, P, sh_degree, max_sh_degree, true, {xyz, features_dc, scaling, rotation, opacity,
                            viewmatrix, projmatrix, campos, radii, clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb,
                            dL_dxyz, dL_dfeatures_dc, dL_dscaling, dL_drotation, dL_dopacity},
                            {features_dc, dL_dfeatures_dc, rotation, dL_drotation, dL_dconic_opacity}, dL_dmeans2D,
                            {features_rest, dL_dfeatures_rest})) return rc;
    return with_coefficients(max_sh_degree, [&](auto k) {
        return launch(GS_STAGE_PREPROCESS_BWD, P, PP_THREADS, stream, k_preprocess_bwd<true, decltype(k)::value>, P,
                      sh_degree, xyz, features_dc, features_rest, scaling, scale_modifier, rotation, opacity,
                      viewmatrix, projmatrix, campos, image_width, image_height, tanfovx, tanfovy, radii, clamped,
                      dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dxyz, dL_dfeatures_dc, dL_dfeatures_rest,
                      dL_dscaling, dL_drotation, dL_dopacity);
    });
}

extern "C" int gs_preprocess_backward_raw(
    int P, int sh_degree, const float *xyz, const float *features_dc, const float *features_rest, const float *scaling,
    float scale_modifier, const float *rotation, const float *opacity, const float *viewmatrix, const float *projmatrix,
    const float *campos, int image_width, int image_height, float tanfovx, float tanfovy, const int32_t *radii,
    const uint8_t *clamped, const float *dL_dmeans2D, const float *dL_dconic_opacity, const float *dL_drgb,
    float *dL_dxyz, float *dL_dfeatures_dc, float *dL_dfeatures_rest, float *dL_dscaling, float *dL_drotation,
    float *dL_dopacity, void *stream) {
    return gs_preprocess_backward_raw_sh(P, sh_degree, 3, xyz, features_dc, features_rest, scaling, scale_modifier,
                                         rotation, opacity, viewmatrix, projmatrix, campos, image_width, image_height,
                                         tanfovx, tanfovy, radii, clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb,
                                         dL_dxyz, dL_dfeatures_dc, dL_dfeatures_rest, dL_dscaling, dL_drotation,
                                         dL_dopacity, stream);
}

extern "C" int gs_preprocess_forward_batched_sh(
    int B, int P, int sh_degree, int max_sh_degree, const float *xyz, const float *features_dc,
    const float *features_rest, const float *scaling, float scale_modifier, const float *rotation,
    const float *opacity, const float *cams, int image_width, int image_height, float *means2D, float *depths,
    int32_t *radii, float *conic_opacity, float *rgb, uint8_t *clamped, void *stream) {
    if (int rc = check_args(B, P, sh_degree, max_sh_degree, image_width > 0 && image_height > 0, {xyz, features_dc,
                            scaling, rotation, opacity, cams, means2D, depths, radii, conic_opacity, rgb, clamped},
                            {features_dc, rotation, conic_opacity}, means2D, {features_rest})) return rc;
    return with_coefficients(max_sh_degree, [&](auto k) {
        return launch(GS_STAGE_PREPROCESS_FWD, P, PP_THREADS, stream, k_preprocess_fwd_batched<decltype(k)::value>, B,
                      P, sh_degree, xyz, features_dc, features_rest, scaling, scale_modifier, rotation, opacity, cams,
                      image_width, image_height, means2D, depths, radii, conic_opacity, rgb, clamped);
    });
}

extern "C" int gs_preprocess_forward_batched(
    int B, int P, int sh_degree, const float *xyz, const float *features_dc, const float *features_rest,
    const float *scaling, float scale_modifier, const float *rotation, const float *opacity, const float *cams,
    int image_width, int image_height, float *means2D, float *depths, int32_t *radii, float *conic_opacity,
    float *rgb, uint8_t *clamped, void *stream) {
    return gs_preprocess_forward_batched_sh(B, P, sh_degree, 3, xyz, features_dc, features_rest, scaling,
                                            scale_modifier, rotation, opacity, cams, image_width, image_height,
                                            means2D, depths, radii, conic_opacity, rgb, clamped, stream);
}

extern "C" int gs_preprocess_backward_batched_sh(
    int B, int P, int sh_degree, int max_sh_degree, const float *xyz, const float *features_dc,
    const float *features_rest, const float *scaling, float scale_modifier, const float *rotation,
    const float *opacity, const float *cams, int image_width, int image_height, const int32_t *radii,
    const uint8_t *clamped, const float *dL_dmeans2D, const float *dL_dconic_opacity, const float *dL_drgb,
    float *dL_dxyz, float *dL_dfeatures_dc, float *dL_dfeatures_rest, float *dL_dscaling, float *dL_drotation,
    float *dL_dopacity, void *stream) {
    if (int rc = check_args(B, P, sh_degree, max_sh_degree, true, {xyz, features_dc, scaling, rotation, opacity, cams,
                            radii, clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dxyz, dL_dfeatures_dc,
                            dL_dscaling, dL_drotation, dL_dopacity},
                            {features_dc, dL_dfeatures_dc, rotation, dL_drotation, dL_dconic_opacity}, dL_dmeans2D,
                            {features_rest, dL_dfeatures_rest})) return rc;
    return with_coefficients(max_sh_degree, [&](auto k) {
        return launch(GS_STAGE_PREPROCESS_BWD, P, PB_BWD_THREADS, stream, k_preprocess_bwd_batched<decltype(k)::value>,
                      B, P, sh_degree, xyz, features_dc, features_rest, scaling, scale_modifier, rotation, opacity,
                      cams, image_width, image_height, radii, clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dxyz,
                      dL_dfeatures_dc, dL_dfeatures_rest, dL_dscaling, dL_drotation, dL_dopacity);
    });
}

extern "C" int gs_preprocess_backward_batched(
    int B, int P, int sh_degree, const float *xyz, const float *features_dc, const float *features_rest,
    const float *scaling, float scale_modifier, const float *rotation, const float *opacity, const float *cams,
    int image_width, int image_height, const int32_t *radii, const uint8_t *clamped, const float *dL_dmeans2D,
    const float *dL_dconic_opacity, const float *dL_drgb, float *dL_dxyz, float *dL_dfeatures_dc,
    float *dL_dfeatures_rest, float *dL_dscaling, float *dL_drotation, float *dL_dopacity, void *stream) {
    return gs_preprocess_backward_batched_sh(B, P, sh_degree, 3, xyz, features_dc, features_rest, scaling,
                                             scale_modifier, rotation, opacity, cams, image_width, image_height, radii,
                                             clamped, dL_dmeans2D, dL_dconic_opacity, dL_drgb, dL_dxyz,
                                             dL_dfeatures_dc, dL_dfeatures_rest, dL_dscaling, dL_drotation,
                                             dL_dopacity, stream);
}
