"""The deterministic render backward and loss (csrc/blend.cu k_det_reduce / k_det_reduce_long, csrc/loss.cu
k_loss_finalize_det) stated in numpy from their documented summation orders, the workspace layouts the tests read them
out of, and scenes whose splats have range lengths chosen to order.

  * det_carve: the gs_render_det_bytes workspace -- n_long (256 bytes), the instance rows (R x 9 fp32), rank (P) and
    long_g (P) uint32, each region 256-byte aligned;
  * reduce_splat: one splat's 9 values from its (n, 9) instance rows.  n <= DR_SHORT: from +0.0f, rows in slot order.
    n > DR_SHORT: DR_THREADS thread partials (thread t adds rows t, t + 256, ... in order), an xor butterfly with offsets
    16, 8, 4, 2, 1 on every 32-lane warp (lane 0's value), then the warp sums added in warp order from +0.0f;
  * finalize_view: one view's fp64 CTA partials -> fp32 (Ll1 or ssim).  Lane l adds slots l, l + 32, ... in order, the
    same xor butterfly, then (float)(s * inv_norm);
  * loss_slots: where the _det loss forward leaves its CTA partials in temp;
  * range_length_scene / long_population: splats whose local tile counts are exactly the lengths the reduce branches
    on (0, 1, 15, 16, 17, 255, 256, 257, 4097, a whole 257 x 32-tile image) and > 1056 splats of 17-40 rows (more
    long ranges than k_det_reduce_long has persistent CTAs).
"""
import numpy as np

import binning_ref as br

F32 = np.float32
DR_SHORT = 16
DR_THREADS = 256
DR_LONG_CTAS = 1056
WARP = 32
BUTTERFLY = (16, 8, 4, 2, 1)
LS_TILE = 32
LOSS_HEADER_1 = 256               # gs_loss_forward_det: the single-view header
LOSS_HEADER_B = 2 * 8 * 64        # gs_loss_forward_batched_det: two doubles per view, GS_MAX_VIEWS views


def align256(v):
    return (int(v) + 255) // 256 * 256


def det_carve(R, P):
    """Byte offsets of the gs_render_det_bytes(R, P) workspace's regions, and its total size."""
    R, P = max(int(R), 0), max(int(P), 0)
    inst = 256
    rank = inst + align256(R * 9 * 4)
    long_g = rank + align256(P * 4)
    return dict(n_long=0, inst=inst, rank=rank, long_g=long_g, total=long_g + align256(P * 4))


def _butterfly(w):
    """xor butterfly over the last-but-one axis (32 lanes), every lane adding its partner's value at each offset."""
    lanes = np.arange(WARP)
    for o in BUTTERFLY:
        w = w + w[..., lanes ^ o, :]
    return w


def reduce_splat(rows):
    """fp32 sum of one splat's (n, 9) instance rows in the kernels' order -> (9,) float32."""
    rows = np.asarray(rows, F32).reshape(-1, 9)
    n = rows.shape[0]
    if n <= DR_SHORT:
        v = np.zeros(9, F32)
        for r in rows:
            v = v + r
        return v
    w = np.zeros((DR_THREADS, 9), F32)
    for k in range(0, n, DR_THREADS):
        blk = rows[k:k + DR_THREADS]
        w[:blk.shape[0]] = w[:blk.shape[0]] + blk
    w = _butterfly(w.reshape(DR_THREADS // WARP, WARP, 9))
    t = np.zeros(9, F32)
    for x in range(DR_THREADS // WARP):
        t = t + w[x, 0]
    return t


def range_lengths(offsets):
    """Rows per depth position: offsets[d] - offsets[d - 1] (offsets as uint32, inclusive)."""
    e = np.asarray(offsets, np.uint32).astype(np.int64)
    return e - np.concatenate([[0], e[:-1]])


def reduce_all(inst, offsets, order):
    """Every splat's 9 values: splat order[d] sums the rows [offsets[d-1], offsets[d]) of inst (R, 9) -> (P, 9).  The
    short ranges are summed column by column for all splats at once (the same adds in the same order as
    reduce_splat); the long ones one splat at a time through reduce_splat."""
    inst = np.asarray(inst, F32).reshape(-1, 9)
    order = np.asarray(order, np.int64)
    e = np.asarray(offsets, np.uint32).astype(np.int64)
    n = range_lengths(e)
    b = e - n
    P = order.size
    out_d = np.zeros((P, 9), F32)
    for k in range(DR_SHORT):
        d = np.nonzero((n > k) & (n <= DR_SHORT))[0]
        out_d[d] = out_d[d] + inst[b[d] + k]
    for d in np.nonzero(n > DR_SHORT)[0]:
        out_d[d] = reduce_splat(inst[b[d]:e[d]])
    out = np.zeros((P, 9), F32)
    out[order] = out_d
    return out


def long_set(offsets, order):
    """The splats whose range is longer than DR_SHORT (sorted ids)."""
    return np.sort(np.asarray(order, np.int64)[range_lengths(offsets) > DR_SHORT])


def finalize_view(partials, inv_norm):
    """fp64 CTA partials of one view (slots,) -> the fp32 value k_loss_finalize_det writes."""
    p = np.asarray(partials, np.float64).reshape(-1)
    s = np.zeros(WARP, np.float64)
    for k in range(0, p.size, WARP):
        blk = p[k:k + WARP]
        s[:blk.size] = s[:blk.size] + blk
    s = _butterfly(s[:, None])[:, 0]
    return F32(s[0] * inv_norm)


def loss_inv_norm(H, W):
    return 1.0 / (3.0 * float(H) * float(W))


def loss_slots(header, rows4, W):
    """Where the _det loss forward leaves its partials: -> (byte offset, slots per view).  CTA (x, y) of view v writes
    (Ll1, ssim) as two doubles at slot (v gy + y) gx + x, gx = ceil(W / 32), gy = ceil(tallest window / 32); the maps
    in front keep the atomic form's offset and are padded to 256 bytes."""
    sum_rows = sum(max(r[1] - r[0], 0) for r in rows4)
    max_rows = max([max(r[1] - r[0], 0) for r in rows4] + [0])
    gx, gy = -(-W // LS_TILE), -(-max_rows // LS_TILE)
    return header + align256(9 * sum_rows * W * 4), gx * gy


def loss_need(header, rows4, W):
    """Bytes the _det loss forward requires (its size query adds 256 spare bytes on top)."""
    off, slots = loss_slots(header, rows4, W)
    return off + 16 * len(rows4) * slots


# ---- scenes with chosen range lengths -------------------------------------------------------------------------------

def corner_splat(gx, gy, nx, ny, corner):
    """(px, py, r) of a splat whose tile rect is exactly the nx x ny tiles at `corner` ('tl', 'tr', 'bl', 'br') of a
    gx x gy grid.  Per axis with n of g tiles, r >= 8 n - 11: low side p = 16 n - r - 7 (so (p - r) / 16 truncates to
    <= 0 and (p + r + 15) / 16 = n + 1/2); high side p = 16 (g - n) + 8 + r.  All values are small integers, exact in
    fp32."""
    r = 8 * max(nx, ny) + 8

    def axis(n, g, high):
        return 16 * (g - n) + 8 + r if high else 16 * n - r - 7

    return float(axis(nx, gx, corner[1] == "r")), float(axis(ny, gy, corner[0] == "b")), r


# (label, nx, ny, corner) of range_length_scene: the tile counts the two reduce kernels branch on
RANGE_SPLATS = [("1", 1, 1, "tl"), ("15", 15, 1, "tr"), ("15", 5, 3, "bl"), ("16", 16, 1, "tl"), ("16", 4, 4, "br"),
                ("16", 1, 16, "tr"), ("17", 17, 1, "bl"), ("17", 1, 17, "tl"), ("255", 15, 17, "br"),
                ("256", 16, 16, "tr"), ("257", 257, 1, "bl"), ("4097", 241, 17, "tl"), ("whole", 257, 32, "tl")]
RANGE_W, RANGE_H = 4112, 512      # 257 x 32 tiles


def range_length_scene(seed=3, n_fill=1500):
    """RANGE_W x RANGE_H, two views of the same splats: view 0 with every tile local, view 1 with a checkerboard
    mask.  Per view the RANGE_SPLATS (wide, faint splats that reach every pixel of their rect), culled and off-screen
    splats (0 rows) and n_fill small ones.  -> (case dict as binning_cases makes them, the view-0 count promised for
    every splat of a view, -1 for the small ones)."""
    gx, gy = br.tiles_of(RANGE_W, RANGE_H)
    T = gx * gy
    rng = np.random.default_rng(seed)
    rows, label, promise = [], [], []
    for lab, nx, ny, corner in RANGE_SPLATS:
        px, py, r = corner_splat(gx, gy, nx, ny, corner)
        s = 0.6 * (r + 8)                 # alpha >= 0.15 exp(-2.8) > 1/255 at the rect's farthest pixel
        rows.append((px, py, 1 / s ** 2, 0.0, 1 / s ** 2, rng.uniform(0.15, 0.3), r))
        label.append(lab)
        promise.append(nx * ny)
    for k in range(4):
        rows.append((rng.uniform(0, RANGE_W), rng.uniform(0, RANGE_H), 0.1, 0.0, 0.1, 0.5, 0))        # culled
        rows.append((RANGE_W + 60.0 + k, -80.0, 0.1, 0.0, 0.1, 0.5, 20))                            # off-screen
        label += ["0", "0"]
        promise += [0, 0]
    mx, my = rng.uniform(0, RANGE_W, n_fill), rng.uniform(0, RANGE_H, n_fill)
    rad = rng.integers(1, 40, n_fill)
    for x, y, r in zip(mx, my, rad):
        a = 1.0 / (0.4 * r + 0.5) ** 2
        rows.append((x, y, a, 0.0, a, rng.uniform(0.05, 0.8), int(r)))
        label.append("fill")
        promise.append(-1)                # whatever its rect holds
    r = np.array(rows, np.float64)
    c = _case("range_lengths", RANGE_W, RANGE_H, r, np.array(label), rng, views=2)
    ck = np.array([((t % gx) + (t // gx)) % 2 for t in range(T)], np.uint8)
    c["cl"] = np.concatenate([np.ones(T, np.uint8), ck])
    return c, np.array(promise, np.int64)


def long_population(n=3200, W=1920, H=1080, seed=5):
    """n splats whose rect holds 17-40 local tiles (drawn, counted with binning_ref and kept in draw order)."""
    rng = np.random.default_rng(seed)
    gx, gy = br.tiles_of(W, H)
    m = np.stack([rng.uniform(0, W, 8 * n), rng.uniform(0, H, 8 * n)], 1).astype(F32)
    rad = rng.integers(24, 56, 8 * n).astype(np.int32)
    cnt, _, _ = br.local_counts(m, rad, np.ones(gx * gy, np.uint8), W, H, [0, 8 * n])
    keep = np.nonzero((cnt >= 17) & (cnt <= 40))[0][:n]
    assert keep.size == n
    s = rad[keep] / 2.5
    a = 1.0 / s ** 2
    r = np.stack([m[keep, 0], m[keep, 1], a, np.zeros(n), a, rng.uniform(0.05, 0.5, n), rad[keep]], 1)
    c = _case("long_population", W, H, r.astype(np.float64), np.full(n, "long"), rng)
    return c, cnt[keep].astype(np.int64)


def _case(name, W, H, r, label, rng, views=1):
    """rows (mx, my, A, B, C, o, radius) -> a binning_cases-style case of `views` copies of the same splats, distinct
    depths (a random permutation of 1 .. 2 in fp32 steps)."""
    P = r.shape[0]
    d = (1.0 + rng.permutation(P) / max(P, 1)).astype(F32)
    one = dict(means2D=r[:, 0:2].astype(F32), conic_opacity=r[:, 2:6].astype(F32),
               rgb=rng.uniform(0, 1, (P, 3)).astype(F32), depths=d, radii=r[:, 6].astype(np.int32))
    c = {k: np.concatenate([v] * views) for k, v in one.items()}
    gx, gy = br.tiles_of(W, H)
    c.update(name=name, W=W, H=H, vs=[P * k for k in range(views + 1)], label=np.concatenate([label] * views),
             cl=np.ones(views * gx * gy, np.uint8))
    return c
