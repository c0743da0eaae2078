"""The 3-NN mean squared distance with the exhaustive kernel's fp32 arithmetic, in numpy: the restatement both kNN kernels
are held to.

Per pair, as nvcc compiled `dx * dx + dy * dy + dz * dz` of `q - p` for sm_90a: d = fma(dz, dz, fma(dx, dx, dy * dy))
with d_ = fl32(q_ - p_).  Per query, the three smallest distances to the other points (self excluded by index, values
>= FLT_MAX never enter), summed in ascending order from 0 in fp32 and divided by k = min(3, N - 1) in fp32."""
import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)


def fma32(a, b, c):
    """fl32(a * b + c) with one rounding, for float32 arrays.  a * b is exact in float64; the float64 sum is rounded to
    odd (Boldo & Melquiond), so its rounding to float32 is the correctly rounded value."""
    with np.errstate(over="ignore", invalid="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)          # TwoSum: s + e == p + c exactly
        odd = (s.view(np.int64) & 1) == 1
        fix = np.isfinite(s) & (e != 0) & ~odd
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def dist2_pairs(q, p):
    """(m, 3) queries x (n, 3) points, float32 -> (m, n) float32 squared distances in the kernels' arithmetic."""
    with np.errstate(over="ignore", invalid="ignore"):
        dx, dy, dz = (q[:, None, j] - p[None, :, j] for j in range(3))   # float32 subtraction, rounded once
        return fma32(dz, dz, fma32(dx, dx, dy * dy))


def mean_dist2(pts, chunk=512):
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    n = len(pts)
    k = min(3, n - 1)
    out = np.zeros(n, np.float32)
    if k <= 0:
        return out
    for s in range(0, n, chunk):
        d = np.minimum(dist2_pairs(pts[s:s + chunk], pts), FLT_MAX)
        rows = np.arange(d.shape[0])
        d[rows, rows + s] = FLT_MAX                                       # self excluded by index
        b = np.sort(np.partition(d, 2, axis=1)[:, :3] if n >= 4 else d, axis=1)[:, :3]
        if b.shape[1] < 3:
            b = np.concatenate([b, np.full((len(b), 3 - b.shape[1]), FLT_MAX, np.float32)], 1)
        with np.errstate(over="ignore"):
            acc = np.zeros(len(b), np.float32)
            for j in range(k):
                acc = acc + b[:, j]
            out[s:s + chunk] = acc / np.float32(k)
    return out
