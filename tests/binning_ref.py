"""Tile binning stated in numpy from its contract (include/grendel_gs_b200.h, the comments of csrc/binning.cu), not from
the oracle: stages 21-24 (local tile count, depth key, splat record), 30 (scan), 40 + 50 (sorted (tile, id) list) and
60 (tile ranges), single-view and batched (`view_start`).

  * rect: (px - r) / 16 and (px + r + 15) / 16 as the same fp32 operation sequence (numpy float32 adds and divides are
    correctly rounded, as __fadd_rn / __fdiv_rn are), converted to int as the device does (f2i), clamped to [0, gx];
  * local tiles per splat: from a summed-area table of compute_locally, so a total of 2^32 costs O(P), not O(R);
  * order: stable argsort of the depth key (raw fp32 depth bits; 0xFFFFFFFF for a splat without a local tile);
  * offsets: the inclusive scan of the counts in that order, modulo 2^32 (the device keeps 32 bits);
  * sorted list: one (v T + tile, id) per local tile, ordered by (v T + tile, depth bits, index); ranges: [start, end)
    per tile, (0, 0) when empty;
  * record: the exact pass-through fields, the fp64 value thr approximates, and the fp64 half extents of
    {power >= thr} against which the kernel's ex, ey must be conservative.
"""
import numpy as np

TILE = 16
F32 = np.float32
NO_TILE_KEY = 0xFFFFFFFF
INT_MIN, INT_MAX = -(2 ** 31), 2 ** 31 - 1
DEGENERATE_EXTENT = F32(3.0e38)   # ex = ey for a conic the block cull must not use
DEAD_EXTENT = F32(-1.0)           # opacity below 1/255: never contributes

# record kinds
NO_TILE, DEAD, DEGENERATE, BOX = 0, 1, 2, 3


def tiles_of(W, H):
    return (W + TILE - 1) // TILE, (H + TILE - 1) // TILE


def f2i(x):
    """fp32 -> int32 as the device's (int) cast (cvt.rzi.s32.f32): truncate toward zero, saturate to the int32 range,
    NaN -> 0.  numpy's astype leaves the out-of-range result undefined, so the saturation is spelled out."""
    x = np.atleast_1d(np.asarray(x, F32)).astype(np.float64)
    out = np.zeros(x.shape, np.int64)
    ok = ~np.isnan(x)
    out[ok] = np.clip(np.trunc(np.clip(x[ok], -2.0 ** 40, 2.0 ** 40)), INT_MIN, INT_MAX).astype(np.int64)
    return out


def rects(means2D, radii, gx, gy):
    """-> x0, y0, x1, y1 (int64, P): the tile rectangle [x0, x1) x [y0, y1) of every splat, whatever its radius."""
    m = np.asarray(means2D, F32).reshape(-1, 2)
    rr = np.asarray(radii, np.int32).astype(F32)          # (float)r: round to nearest even, as cvt.rn.f32.s32
    s, e = F32(TILE), F32(TILE - 1)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = (m - rr[:, None]) / s
        hi = ((m + rr[:, None]) + e) / s
    x0, y0 = np.clip(f2i(lo[:, 0]), 0, gx), np.clip(f2i(lo[:, 1]), 0, gy)
    x1, y1 = np.clip(f2i(hi[:, 0]), 0, gx), np.clip(f2i(hi[:, 1]), 0, gy)
    return x0, y0, x1, y1


def view_of(view_start, P):
    """View of every splat: the largest v < B with view_start[v] <= i (empty views are skipped)."""
    vs = np.asarray(view_start, np.int64)
    return np.searchsorted(vs[:-1], np.arange(P), side="right") - 1


def local_counts(means2D, radii, cl, W, H, view_start):
    """-> touched (int64, P), rect (x0, y0, x1, y1), view (P): local tiles of every splat (0 when radius <= 0)."""
    gx, gy = tiles_of(W, H)
    B = len(view_start) - 1
    P = int(view_start[-1])
    mask = np.asarray(cl, np.uint8).reshape(B, gy, gx) != 0
    sat = np.zeros((B, gy + 1, gx + 1), np.int64)
    sat[:, 1:, 1:] = mask.cumsum(1, dtype=np.int64).cumsum(2)
    v = view_of(view_start, P)
    x0, y0, x1, y1 = rects(means2D, radii, gx, gy)
    n = sat[v, y1, x1] - sat[v, y0, x1] - sat[v, y1, x0] + sat[v, y0, x0]
    n[np.asarray(radii, np.int64) <= 0] = 0
    return n, (x0, y0, x1, y1), v


def bin_splats(means2D, depths, radii, cl, W, H, view_start=None, with_list=True):
    """The whole binning contract.  view_start None = one view of all splats.  -> dict with R (int), touched (int64),
    order / offsets (uint32, P), and when with_list: tiles / ids (uint32, R) and ranges (uint32, B T x 2)."""
    P = int(np.asarray(radii).shape[0])
    if view_start is None:
        view_start = [0, P]
    gx, gy = tiles_of(W, H)
    T = gx * gy
    B = len(view_start) - 1
    n, rect, v = local_counts(means2D, radii, cl, W, H, view_start)
    dbits = np.ascontiguousarray(depths, F32).view(np.uint32).astype(np.int64)
    key = np.where(n > 0, dbits, NO_TILE_KEY)
    order = np.argsort(key, kind="stable")
    offsets = (np.cumsum(n[order]) & 0xFFFFFFFF).astype(np.uint32)
    out = dict(R=int(n.sum()), touched=n, order=order.astype(np.uint32), offsets=offsets, rect=rect, view=v, T=T, B=B)
    if not with_list:
        return out
    x0, y0, x1, y1 = rect
    live = np.nonzero(n > 0)[0]
    w, h = (x1 - x0)[live], (y1 - y0)[live]
    cnt = w * h
    sid = np.repeat(live, cnt)
    k = np.arange(int(cnt.sum()), dtype=np.int64) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    ww = np.repeat(w, cnt)
    tile = v[sid] * T + (np.repeat(y0[live], cnt) + k // ww) * gx + np.repeat(x0[live], cnt) + k % ww
    del k, ww
    keep = np.asarray(cl, np.uint8).reshape(-1)[tile] != 0
    sid, tile = sid[keep], tile[keep]
    assert sid.size == out["R"]
    # rank of a splat in (depth bits, index) order: the sorted list is ordered by (tile, rank), a unique int64 key
    rank = np.empty(P, np.int64)
    rank[np.argsort(dbits, kind="stable")] = np.arange(P)
    perm = np.argsort(tile * max(P, 1) + rank[sid])
    tiles, ids = tile[perm], sid[perm]
    counts = np.bincount(tiles, minlength=B * T)
    ends = np.cumsum(counts)
    ranges = np.where((counts > 0)[:, None], np.stack([ends - counts, ends], 1), 0).astype(np.uint32)
    out.update(tiles=tiles.astype(np.uint32), ids=ids.astype(np.uint32), ranges=ranges)
    return out


# ---- the splat record ---------------------------------------------------------------------------------------------

def fma32(a, b, c):
    """Correctly rounded fp32 a * b + c: the product is exact in fp64, the sum is rounded to odd in fp64 (TwoSum
    error, then one ulp toward it when the fp64 result is even), and round-to-odd followed by a rounding to fp32 is a
    single correct rounding (53 >= 24 + 2)."""
    a, b, c = (np.asarray(q, F32).astype(np.float64) for q in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        even = (s.view(np.int64) & 1) == 0
        s = np.where((e != 0) & even & np.isfinite(s), np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def record(means2D, conic_opacity, rgb, touched, no_cull=False):
    """-> dict: exact (P, 12) fp32 fields with NaN where the kernel's value is not bit-defined (thr, and ex / ey of a
    box), defined (P, 12) bool, kind (P), thr64 (P): the fp64 -log of the fp32 product fl(255 max(o, 1e-30)) the
    kernel forms, prod (P) that product."""
    m = np.asarray(means2D, F32).reshape(-1, 2)
    co = np.asarray(conic_opacity, F32).reshape(-1, 4)
    col = np.asarray(rgb, F32).reshape(-1, 3)
    P = m.shape[0]
    A, B, C, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    live = np.asarray(touched) > 0
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        prod = F32(255.0) * np.fmax(o, F32(1e-30))          # fmaxf: a NaN opacity gives 255e-30
        thr64 = -np.log(prod.astype(np.float64))
        bb = B * B
        det = fma32(A, C, -bb) - fma32(B, B, -bb)            # Kahan's FMA-compensated AC - B^2
    box = (det >= np.finfo(F32).tiny) & (A > 0) & (C > 0) & (not no_cull)   # a subnormal det is not accurate
    kind = np.where(~live, NO_TILE, np.where(prod < 1, DEAD, np.where(box, BOX, DEGENERATE)))
    rec = np.zeros((P, 12), F32)
    defined = np.ones((P, 12), bool)
    L = live
    rec[L, 0], rec[L, 1], rec[L, 2], rec[L, 3] = m[L, 0], m[L, 1], F32(-0.5) * A[L], -B[L]
    rec[L, 4], rec[L, 5], rec[L, 7] = F32(-0.5) * C[L], o[L], col[L, 0]
    rec[L, 8], rec[L, 9] = col[L, 1], col[L, 2]
    rec[L, 6] = np.nan
    defined[L, 6] = False
    rec[kind == DEAD, 10:12] = DEAD_EXTENT
    rec[kind == DEGENERATE, 10:12] = DEGENERATE_EXTENT
    rec[kind == BOX, 10:12] = np.nan
    defined[kind == BOX, 10:12] = False
    return dict(rec=rec, defined=defined, kind=kind, thr64=thr64, prod=prod)


def true_half_extents(rec):
    """fp64 half extents of {A dx^2 + 2 B dx dy + C dy^2 <= -2 thr} from a record's own fp32 conic (A = -2 r0.z,
    B = -r0.w, C = -2 r1.x) and thr (r1.z), and the eigenvalue ratio of the conic.  -> hx, hy, cond."""
    r = np.asarray(rec, F32).astype(np.float64)
    A, B, C, thr = -2.0 * r[:, 2], -r[:, 3], -2.0 * r[:, 4], r[:, 6]
    with np.errstate(invalid="ignore", divide="ignore"):
        det = A * C - B * B
        t = -2.0 * thr
        hx, hy = np.sqrt(t * C / det), np.sqrt(t * A / det)
        mid, rad = 0.5 * (A + C), np.sqrt(0.25 * (A - C) ** 2 + B * B)
        cond = (mid + rad) / (mid - rad)
    return hx, hy, cond
