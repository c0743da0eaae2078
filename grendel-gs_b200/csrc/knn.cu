// simple_knn._C.distCUDA2 (/root/reference/scene/gaussian_model.py:20,163-166): mean SQUARED distance of every point to
// its 3 nearest neighbours, used once at start-up to initialise the Gaussian scales (log sqrt of it).  The reference's
// module is an absent submodule (bkerbl/simple-knn @ 44f7642, .SUBMODULES.json:24-28); its published algorithm is an
// EXACT 3-NN (Morton order + box pruning only skip work), self excluded by index, duplicates counted at distance 0.
//
// Two kernels compute that definition with the same fp32 arithmetic (DESIGN.md 5i):
//  * gs_knn3_mean_dist2_range, the production search: 63-bit Morton keys, a CUB radix sort, leaves of 32 consecutive
//    sorted points under an implicit KN_FANOUT-ary tree of exact AABBs, and one warp per 32 sorted queries walking the
//    tree together.  A box is skipped only when its fp32 lower bound is >= the lane's third-best distance, and the
//    bound is the point distance's own operation sequence applied to the gap to the box, so the skip is exact.
//    O(N log N) in practice.  simple_knn._C routes CUDA tensors here.
//  * gs_knn3_mean_dist2, the exhaustive tiled brute force (every thread owns one query and streams all N points through
//    shared memory, O(N^2)).  Kept as the reference the search is tested against bit for bit.
#include <algorithm>
#include <cfloat>

#include <cub/cub.cuh>

#include "common.cuh"

#define KN_THREADS 256
#define KN_LEAF 32             // points per leaf = one warp's lanes
#define KN_FANOUT 8            // children per tree node above the leaves
#define KN_MAX_LEVELS 16       // 2^31 points: 2^26 leaves, 10 levels at fan-out 8
#define KN_BBOX_BLOCKS 1024    // partial bounding boxes of the first reduction pass
#define KN_FULL 0xffffffffu

// ---- the arithmetic both kernels share -----------------------------------------------------------------------------
// The squared distance exactly as nvcc compiled the exhaustive kernel's `dx * dx + dy * dy + dz * dz` of `q - p` for
// sm_90a: FADD per axis, then FMUL dy * dy, FFMA dx, FFMA dz (the PTX is mul.f32 on dy, then fma.rn.f32 with dx, then
// with dz).  Written out so that neither kernel depends on contraction choices and the exhaustive kernel keeps its bits.
GS_D float kn_dist2(float qx, float qy, float qz, float px, float py, float pz) {
    const float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// Lower bound of kn_dist2(q, p) over every p with lo <= p <= hi per axis, lo and hi being point coordinates: the same
// sequence on the per-axis gap.  Rounding to nearest is monotone and odd, so |fl(q - p)| >= fl(gap) for every such p,
// and the squares and FMAs of non-negative values keep that order.
GS_D float kn_gap(float q, float lo, float hi) {
    return q < lo ? __fsub_rn(lo, q) : (q > hi ? __fsub_rn(q, hi) : 0.f);
}
GS_D float kn_box_dist2(float qx, float qy, float qz, float4 lo, float4 hi) {
    const float gx = kn_gap(qx, lo.x, hi.x), gy = kn_gap(qy, lo.y, hi.y), gz = kn_gap(qz, lo.z, hi.z);
    return __fmaf_rn(gz, gz, __fmaf_rn(gx, gx, __fmul_rn(gy, gy)));
}

// b0 <= b1 <= b2 are the three smallest values inserted (FLT_MAX while fewer).  Strict comparisons: the final three
// are the three smallest of the multiset whatever the insertion order, and a value >= b2 never changes them.
GS_D void kn_insert(float d, float &b0, float &b1, float &b2) {
    if (d < b2) {
        if (d < b1) {
            b2 = b1;
            if (d < b0) { b1 = b0; b0 = d; } else { b1 = d; }
        } else {
            b2 = d;
        }
    }
}

// fewer than 3 other points: average the neighbours that exist (N == 1: 0)
GS_D float kn_mean(int N, float b0, float b1, float b2) {
    const int k = min(3, N - 1);
    float s = 0.f;
    if (k >= 1) s += b0;
    if (k >= 2) s += b1;
    if (k >= 3) s += b2;
    return k > 0 ? s / (float)k : 0.f;
}

// ---- the exhaustive reference ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(KN_THREADS)
k_knn3_mean_dist2(int N, const float *__restrict__ pts, float *__restrict__ out) {
    __shared__ float sx[KN_THREADS], sy[KN_THREADS], sz[KN_THREADS];
    const int i = blockIdx.x * KN_THREADS + threadIdx.x;
    const bool valid = i < N;
    const float qx = valid ? pts[3 * (size_t)i] : 0.f, qy = valid ? pts[3 * (size_t)i + 1] : 0.f,
                qz = valid ? pts[3 * (size_t)i + 2] : 0.f;
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
    for (int base = 0; base < N; base += KN_THREADS) {
        const int j = base + threadIdx.x;
        __syncthreads();
        if (j < N) { sx[threadIdx.x] = pts[3 * (size_t)j]; sy[threadIdx.x] = pts[3 * (size_t)j + 1]; sz[threadIdx.x] = pts[3 * (size_t)j + 2]; }
        __syncthreads();
        const int cnt = min(KN_THREADS, N - base);
        for (int t = 0; t < cnt; t++) {
            const float d = (base + t == i) ? FLT_MAX : kn_dist2(qx, qy, qz, sx[t], sy[t], sz[t]);   // self excluded by index
            kn_insert(d, b0, b1, b2);
        }
    }
    if (valid) out[i] = kn_mean(N, b0, b1, b2);
}

// points: (N,3) fp32; mean_dist2: (N) fp32.
extern "C" int gs_knn3_mean_dist2(int N, const float *points, float *mean_dist2, void *stream) {
    GS_REQUIRE(N >= 0, "N");
    if (N == 0) return GS_OK;
    GS_REQUIRE(points && mean_dist2, "null pointer");
    k_knn3_mean_dist2<<<(N + KN_THREADS - 1) / KN_THREADS, KN_THREADS, 0, (cudaStream_t)stream>>>(N, points, mean_dist2);
    GS_LAUNCH_CHECK();
    return GS_OK;
}

// ---- the Morton-tree search -----------------------------------------------------------------------------------------
// Bounding box: per-block partials (min xyz, max xyz, any non-finite coordinate), then one block over the partials.
GS_D void kn_warp_minmax(float &lx, float &ly, float &lz, float &hx, float &hy, float &hz) {
    for (int o = 16; o; o >>= 1) {
        lx = fminf(lx, __shfl_xor_sync(KN_FULL, lx, o)); ly = fminf(ly, __shfl_xor_sync(KN_FULL, ly, o));
        lz = fminf(lz, __shfl_xor_sync(KN_FULL, lz, o)); hx = fmaxf(hx, __shfl_xor_sync(KN_FULL, hx, o));
        hy = fmaxf(hy, __shfl_xor_sync(KN_FULL, hy, o)); hz = fmaxf(hz, __shfl_xor_sync(KN_FULL, hz, o));
    }
}

// box[b * 8 + 0..7] = min x y z, max x y z, 1.0 if a coordinate is not finite, 0
GS_D void kn_block_box(float lx, float ly, float lz, float hx, float hy, float hz, bool bad, float *box) {
    __shared__ float s[KN_THREADS / 32][6];
    __shared__ int s_bad;
    if (threadIdx.x == 0) s_bad = 0;
    __syncthreads();
    if (bad) s_bad = 1;
    kn_warp_minmax(lx, ly, lz, hx, hy, hz);
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s[w][0] = lx; s[w][1] = ly; s[w][2] = lz; s[w][3] = hx; s[w][4] = hy; s[w][5] = hz; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const bool has = threadIdx.x < KN_THREADS / 32;
        lx = has ? s[threadIdx.x][0] : FLT_MAX; ly = has ? s[threadIdx.x][1] : FLT_MAX; lz = has ? s[threadIdx.x][2] : FLT_MAX;
        hx = has ? s[threadIdx.x][3] : -FLT_MAX; hy = has ? s[threadIdx.x][4] : -FLT_MAX; hz = has ? s[threadIdx.x][5] : -FLT_MAX;
        kn_warp_minmax(lx, ly, lz, hx, hy, hz);
        if (threadIdx.x == 0) {
            box[0] = lx; box[1] = ly; box[2] = lz; box[3] = hx; box[4] = hy; box[5] = hz;
            box[6] = s_bad ? 1.f : 0.f; box[7] = 0.f;
        }
    }
}

__global__ void __launch_bounds__(KN_THREADS)
k_knn_bbox_partial(int N, const float *__restrict__ pts, float *__restrict__ part) {
    float lx = FLT_MAX, ly = FLT_MAX, lz = FLT_MAX, hx = -FLT_MAX, hy = -FLT_MAX, hz = -FLT_MAX;
    bool bad = false;
    for (int i = blockIdx.x * KN_THREADS + threadIdx.x; i < N; i += gridDim.x * KN_THREADS) {
        const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
        bad |= !(isfinite(x) && isfinite(y) && isfinite(z));
        lx = fminf(lx, x); ly = fminf(ly, y); lz = fminf(lz, z); hx = fmaxf(hx, x); hy = fmaxf(hy, y); hz = fmaxf(hz, z);
    }
    kn_block_box(lx, ly, lz, hx, hy, hz, bad, part + 8 * (size_t)blockIdx.x);
}

__global__ void __launch_bounds__(KN_THREADS)
k_knn_bbox_final(int nparts, const float *__restrict__ part, float *__restrict__ box) {
    float lx = FLT_MAX, ly = FLT_MAX, lz = FLT_MAX, hx = -FLT_MAX, hy = -FLT_MAX, hz = -FLT_MAX;
    bool bad = false;
    for (int b = threadIdx.x; b < nparts; b += KN_THREADS) {
        const float *p = part + 8 * b;
        lx = fminf(lx, p[0]); ly = fminf(ly, p[1]); lz = fminf(lz, p[2]);
        hx = fmaxf(hx, p[3]); hy = fmaxf(hy, p[4]); hz = fmaxf(hz, p[5]);
        bad |= p[6] != 0.f;
    }
    kn_block_box(lx, ly, lz, hx, hy, hz, bad, box);
}

// 21 bits spread to every third bit of 63
GS_D uint64_t kn_spread3(uint32_t v) {
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

// Quantised in fp64 on one scale for all axes: defined for a zero-extent axis and for extents beyond fp32's range.
GS_D uint32_t kn_cell(float v, double lo, double scale) {
    return (uint32_t)fmin(floor(((double)v - lo) * scale), (double)((1u << 21) - 1));
}

__global__ void __launch_bounds__(KN_THREADS)
k_knn_morton(int N, const float *__restrict__ pts, double lx, double ly, double lz, double scale,
             uint64_t *__restrict__ keys, int32_t *__restrict__ idx) {
    const int i = blockIdx.x * KN_THREADS + threadIdx.x;
    if (i >= N) return;
    const uint32_t cx = kn_cell(pts[3 * (size_t)i], lx, scale), cy = kn_cell(pts[3 * (size_t)i + 1], ly, scale),
                   cz = kn_cell(pts[3 * (size_t)i + 2], lz, scale);
    keys[i] = kn_spread3(cx) << 2 | kn_spread3(cy) << 1 | kn_spread3(cz);
    idx[i] = i;
}

// sorted[p] = (x, y, z, original index as int bits) of the point at sorted position p
__global__ void __launch_bounds__(KN_THREADS)
k_knn_gather(int N, const float *__restrict__ pts, const int32_t *__restrict__ order, float4 *__restrict__ sorted) {
    const int p = blockIdx.x * KN_THREADS + threadIdx.x;
    if (p >= N) return;
    const int i = order[p];
    sorted[p] = make_float4(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], __int_as_float(i));
}

// one warp per leaf: the exact AABB of its (up to) 32 points
__global__ void __launch_bounds__(KN_THREADS)
k_knn_leaves(int N, int leaves, const float4 *__restrict__ sorted, float4 *__restrict__ lo, float4 *__restrict__ hi) {
    const int leaf = (blockIdx.x * KN_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (leaf >= leaves) return;
    const int p = leaf * KN_LEAF + lane;
    float lx = FLT_MAX, ly = FLT_MAX, lz = FLT_MAX, hx = -FLT_MAX, hy = -FLT_MAX, hz = -FLT_MAX;
    if (p < N) {
        const float4 v = sorted[p];
        lx = hx = v.x; ly = hy = v.y; lz = hz = v.z;
    }
    kn_warp_minmax(lx, ly, lz, hx, hy, hz);
    if (lane == 0) { lo[leaf] = make_float4(lx, ly, lz, 0.f); hi[leaf] = make_float4(hx, hy, hz, 0.f); }
}

// node j of a level = the union of children [j F, min((j + 1) F, nchild)) of the level below
__global__ void __launch_bounds__(KN_THREADS)
k_knn_level(int n, int nchild, const float4 *__restrict__ clo, const float4 *__restrict__ chi, float4 *__restrict__ lo,
            float4 *__restrict__ hi) {
    const int j = blockIdx.x * KN_THREADS + threadIdx.x;
    if (j >= n) return;
    float4 l = clo[j * KN_FANOUT], h = chi[j * KN_FANOUT];
    for (int c = j * KN_FANOUT + 1; c < min((j + 1) * KN_FANOUT, nchild); c++) {
        const float4 a = clo[c], b = chi[c];
        l.x = fminf(l.x, a.x); l.y = fminf(l.y, a.y); l.z = fminf(l.z, a.z);
        h.x = fmaxf(h.x, b.x); h.y = fmaxf(h.y, b.y); h.z = fmaxf(h.z, b.z);
    }
    lo[j] = l; hi[j] = h;
}

struct KnTree {
    int levels;                  // level 0 = the leaves, levels - 1 = the root (one node)
    int count[KN_MAX_LEVELS];    // nodes per level
    int offset[KN_MAX_LEVELS];   // first node of the level in the lo / hi arrays
};

// selects the sorted positions whose original index lies in [q0, q1)
struct KnInRange {
    const float4 *sorted;
    int q0, q1;
    __device__ __forceinline__ bool operator()(int p) const {
        const int i = __float_as_int(sorted[p].w);
        return i >= q0 && i < q1;
    }
};

// One warp per 32 consecutive queries (sorted positions qpos[e], or e itself when qpos is null).  Each lane seeds its
// three best from its own leaf, then the warp walks the tree depth first in node order without a stack: a node is
// entered when some lane's bound is below that lane's b2, a leaf's points are loaded one per lane and broadcast.
__global__ void __launch_bounds__(KN_THREADS)
k_knn3_search(int N, int M, const int32_t *__restrict__ qpos, const float4 *__restrict__ sorted,
              const float4 *__restrict__ lo, const float4 *__restrict__ hi, KnTree tree, int q0,
              float *__restrict__ out) {
    __shared__ int s_count[KN_MAX_LEVELS], s_offset[KN_MAX_LEVELS];
    if (threadIdx.x < KN_MAX_LEVELS) { s_count[threadIdx.x] = tree.count[threadIdx.x]; s_offset[threadIdx.x] = tree.offset[threadIdx.x]; }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int e0 = (blockIdx.x * KN_THREADS + threadIdx.x) & ~31;
    if (e0 >= M) return;   // the whole warp
    const int e = e0 + lane;
    const bool valid = e < M;
    const int p = valid ? (qpos ? qpos[e] : e) : 0;
    const float4 q = sorted[p];
    const int mine = p / KN_LEAF;
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
    for (int j = mine * KN_LEAF; j < min(mine * KN_LEAF + KN_LEAF, N); j++) {
        if (j == p) continue;   // self excluded by index
        const float4 c = sorted[j];
        kn_insert(kn_dist2(q.x, q.y, q.z, c.x, c.y, c.z), b0, b1, b2);
    }
    const int top = tree.levels - 1;
    int level = top, j = 0;
    for (;;) {
        const int node = s_offset[level] + j;
        const bool want = valid && (level > 0 || j != mine) && kn_box_dist2(q.x, q.y, q.z, lo[node], hi[node]) < b2;
        if (__any_sync(KN_FULL, want)) {
            if (level > 0) {   // enter: first child
                level--;
                j *= KN_FANOUT;
                continue;
            }
            const int base = j * KN_LEAF, cnt = min(KN_LEAF, N - base);
            const float4 c = lane < cnt ? sorted[base + lane] : make_float4(0.f, 0.f, 0.f, 0.f);
            const bool other = j != mine;   // the own leaf was seeded
            for (int t = 0; t < cnt; t++) {
                const float cx = __shfl_sync(KN_FULL, c.x, t), cy = __shfl_sync(KN_FULL, c.y, t),
                            cz = __shfl_sync(KN_FULL, c.z, t);
                if (other) kn_insert(kn_dist2(q.x, q.y, q.z, cx, cy, cz), b0, b1, b2);
            }
        }
        // next node: the next sibling, else the next sibling of the nearest ancestor that has one; done at the root
        for (;;) {
            if (level == top) goto done;
            if ((j + 1) % KN_FANOUT != 0 && j + 1 < s_count[level]) { j++; break; }
            j /= KN_FANOUT;
            level++;
        }
    }
done:
    if (valid) out[__float_as_int(q.w) - q0] = kn_mean(N, b0, b1, b2);
}

// ---- workspace ------------------------------------------------------------------------------------------------------
static size_t kn_align(size_t b) { return (b + 255) & ~(size_t)255; }

static KnTree kn_tree(int N) {
    KnTree t = {};
    int n = (N + KN_LEAF - 1) / KN_LEAF, off = 0;
    t.levels = 0;
    for (;;) {
        t.count[t.levels] = n;
        t.offset[t.levels] = off;
        t.levels++;
        off += n;
        if (n == 1) break;
        n = (n + KN_FANOUT - 1) / KN_FANOUT;
    }
    return t;
}

static int kn_nodes(const KnTree &t) { return t.offset[t.levels - 1] + 1; }

// CUB scratch of the sort and the range selection, the larger of the two.  CUB sizes it for the current device, so
// the query fails in a process without a usable device.
static cudaError_t kn_cub_bytes(int N, size_t &bytes) {
    size_t sort = 0, sel = 0;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v(nullptr, nullptr);
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort, k, v, N, 0, 63);
    if (e == cudaSuccess)
        e = cub::DeviceSelect::If(nullptr, sel, cub::CountingInputIterator<int>(0), (int32_t *)nullptr,
                                  (int32_t *)nullptr, N, KnInRange{nullptr, 0, 0});
    bytes = kn_align(sort > sel ? sort : sel);
    return e;
}

// Workspace layout, every part 256-byte aligned from the first 256-byte boundary of temp:
//   bbox partials and box | keys x2 (u64) | order x2 (i32) | sorted points (float4) | node lo, hi (float4) |
//   query positions (i32) + selected count | CUB scratch
struct KnLayout {
    size_t box, keys, idx, sorted, lo, hi, qpos, cub, cub_bytes, total;
};

static cudaError_t kn_layout(int N, KnLayout &l) {
    const size_t n = (size_t)(N > 0 ? N : 1);
    const int nodes = kn_nodes(kn_tree(N > 0 ? N : 1));
    size_t o = 0;
    l.box = o;    o += kn_align(4 * 8 * (KN_BBOX_BLOCKS + 1));
    l.keys = o;   o += 2 * kn_align(8 * n);
    l.idx = o;    o += 2 * kn_align(4 * n);
    l.sorted = o; o += kn_align(16 * n);
    l.lo = o;     o += kn_align(16 * (size_t)nodes);
    l.hi = o;     o += kn_align(16 * (size_t)nodes);
    l.qpos = o;   o += kn_align(4 * (n + 1));
    l.cub = o;
    const cudaError_t e = kn_cub_bytes(N > 0 ? N : 1, l.cub_bytes);
    o += l.cub_bytes;
    l.total = o + 256;   // room to align the base
    if (e != cudaSuccess)
        gs_set_error("sizing the kNN workspace (CUB, current device) failed: %s", cudaGetErrorString(e));
    return e;
}

// 0 when the size cannot be queried (no usable device; gs_last_error() says why)
extern "C" size_t gs_knn3_temp_bytes(int N) {
    KnLayout l;
    return kn_layout(N, l) == cudaSuccess ? l.total : 0;
}

// points: (N,3) fp32, 4-byte aligned; out: (q1 - q0) fp32, out[i - q0] for query point i.  Synchronises `stream` once,
// to read the bounding box (the Morton scale) and refuse non-finite coordinates.
extern "C" int gs_knn3_mean_dist2_range(int N, const float *points, int q0, int q1, float *out, void *temp,
                                        size_t temp_bytes, void *stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    GS_REQUIRE(N >= 0, "N");
    GS_REQUIRE(0 <= q0 && q0 <= q1 && q1 <= N, "query range outside [0, N]");
    if (q0 == q1) return GS_OK;
    GS_REQUIRE(points && out && temp, "null pointer");
    GS_REQUIRE(((uintptr_t)points & 3) == 0 && ((uintptr_t)out & 3) == 0, "points / out not 4-byte aligned");
    GS_REQUIRE(((uintptr_t)temp & 15) == 0, "temp not 16-byte aligned");
    KnLayout L;
    if (kn_layout(N, L) != cudaSuccess) return GS_ECUDA;
    if (temp_bytes < L.total) {
        gs_set_error("gs_knn3_mean_dist2_range: temp too small (%zu bytes, %zu needed)", temp_bytes, L.total);
        return GS_ENOMEM;
    }
    char *base = (char *)(((uintptr_t)temp + 255) & ~(uintptr_t)255);
    float *box = (float *)(base + L.box);
    const size_t n = (size_t)N;
    uint64_t *keys0 = (uint64_t *)(base + L.keys), *keys1 = (uint64_t *)(base + L.keys + kn_align(8 * n));
    int32_t *idx0 = (int32_t *)(base + L.idx), *idx1 = (int32_t *)(base + L.idx + kn_align(4 * n));
    float4 *sorted = (float4 *)(base + L.sorted), *lo = (float4 *)(base + L.lo), *hi = (float4 *)(base + L.hi);
    int32_t *qpos = (int32_t *)(base + L.qpos);
    void *cub_temp = base + L.cub;
    const int nb = (int)std::min<long long>(KN_BBOX_BLOCKS, (N + KN_THREADS - 1) / KN_THREADS);

    k_knn_bbox_partial<<<nb, KN_THREADS, 0, stream>>>(N, points, box + 8);
    GS_LAUNCH_CHECK();
    k_knn_bbox_final<<<1, KN_THREADS, 0, stream>>>(nb, box + 8, box);
    GS_LAUNCH_CHECK();
    float hb[8];
    GS_CUDA_TRY(cudaMemcpyAsync(hb, box, sizeof(hb), cudaMemcpyDeviceToHost, stream));
    GS_CUDA_TRY(cudaStreamSynchronize(stream));
    if (hb[6] != 0.f) {
        gs_set_error("invalid argument: a point coordinate is not finite (NaN or inf)");
        return GS_EINVAL;
    }
    const double ext = std::max({(double)hb[3] - hb[0], (double)hb[4] - hb[1], (double)hb[5] - hb[2]});
    const double scale = ext > 0.0 ? (double)(1u << 21) / ext : 0.0;
    const int grid = (int)(((long long)N + KN_THREADS - 1) / KN_THREADS);
    k_knn_morton<<<grid, KN_THREADS, 0, stream>>>(N, points, hb[0], hb[1], hb[2], scale, keys0, idx0);
    GS_LAUNCH_CHECK();
    cub::DoubleBuffer<uint64_t> dk(keys0, keys1);
    cub::DoubleBuffer<int32_t> dv(idx0, idx1);
    size_t cub_bytes = L.cub_bytes;
    GS_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_temp, cub_bytes, dk, dv, N, 0, 63, stream));
    k_knn_gather<<<grid, KN_THREADS, 0, stream>>>(N, points, dv.Current(), sorted);
    GS_LAUNCH_CHECK();

    const KnTree tree = kn_tree(N);
    const int leaves = tree.count[0];
    const int leaf_blocks = (int)(((long long)leaves * KN_LEAF + KN_THREADS - 1) / KN_THREADS);   // a warp per leaf
    k_knn_leaves<<<leaf_blocks, KN_THREADS, 0, stream>>>(N, leaves, sorted, lo, hi);
    GS_LAUNCH_CHECK();
    for (int l = 1; l < tree.levels; l++) {
        k_knn_level<<<(tree.count[l] + KN_THREADS - 1) / KN_THREADS, KN_THREADS, 0, stream>>>(
            tree.count[l], tree.count[l - 1], lo + tree.offset[l - 1], hi + tree.offset[l - 1], lo + tree.offset[l],
            hi + tree.offset[l]);
        GS_LAUNCH_CHECK();
    }

    const int M = q1 - q0;
    const int32_t *queries = nullptr;   // the whole cloud: query e is sorted position e
    if (M < N) {                        // the sorted positions of [q0, q1), in sorted order: warps stay full and local
        cub_bytes = L.cub_bytes;
        GS_CUDA_TRY(cub::DeviceSelect::If(cub_temp, cub_bytes, cub::CountingInputIterator<int>(0), qpos, qpos + n, N,
                                          KnInRange{sorted, q0, q1}, stream));
        queries = qpos;
    }
    k_knn3_search<<<(int)(((long long)M + KN_THREADS - 1) / KN_THREADS), KN_THREADS, 0, stream>>>(
        N, M, queries, sorted, lo, hi, tree, q0, out);
    GS_LAUNCH_CHECK();
    return GS_OK;
}
