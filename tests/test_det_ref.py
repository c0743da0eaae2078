"""CPU: tests/det_ref.py, the summation orders the deterministic GPU tests pin the kernels to, and its scenes.

  * reduce_splat / finalize_view equal a naive loop written from the documented order bit for bit, and the fp64 sum
    within the rounding bound of that order's depth; reduce_all equals reduce_splat splat by splat;
  * the orders are really different: another butterfly, another short / long split or another first lane gives other
    bits on the same data;
  * the scenes hold exactly the range lengths they promise (binning_ref), 16 and 17 among them, and the long population
    has more long ranges than k_det_reduce_long has CTAs."""
import numpy as np
import pytest

import binning_ref as br
import det_ref as dr

F32 = np.float32
U = 2.0 ** -24
LENGTHS = (0, 1, 2, 15, 16, 17, 31, 255, 256, 257, 511, 513, 4097)


def rows_of(n, seed, scale=1.0):
    """Rows with mixed signs and magnitudes (cancellation makes the order visible in the last bits)."""
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(n, 9)) * np.exp(rng.uniform(-4, 4, (n, 9))) * scale).astype(F32)


def naive_reduce(rows):
    n = len(rows)
    out = []
    for q in range(9):
        if n <= 16:
            v = F32(0.0)
            for i in range(n):
                v = F32(v + rows[i][q])
            out.append(v)
            continue
        part = []
        for t in range(256):
            w = F32(0.0)
            i = t
            while i < n:
                w = F32(w + rows[i][q])
                i += 256
            part.append(w)
        for warp in range(8):
            lanes = part[32 * warp:32 * warp + 32]
            for o in (16, 8, 4, 2, 1):
                lanes = [F32(lanes[ln] + lanes[ln ^ o]) for ln in range(32)]
            part[32 * warp:32 * warp + 32] = lanes
        t = F32(0.0)
        for warp in range(8):
            t = F32(t + part[32 * warp])
        out.append(t)
    return np.array(out, F32)


def depth(n):
    """Longest chain of fp32 adds behind one output of the kernels' order."""
    return n if n <= 16 else -(-n // 256) + 5 + 8


@pytest.mark.parametrize("n", LENGTHS)
def test_reduce_splat_is_the_documented_order(n):
    rows = rows_of(n, seed=n)
    got = dr.reduce_splat(rows)
    assert got.dtype == F32 and got.shape == (9,)
    assert np.array_equal(got.view(np.uint32), naive_reduce(rows).view(np.uint32))
    exact = rows.astype(np.float64).sum(0)
    bound = depth(n) * U * np.abs(rows.astype(np.float64)).sum(0) / (1 - depth(n) * U)
    assert (np.abs(got - exact) <= bound + 1e-45).all()
    if n == 0:
        assert (got.view(np.uint32) == 0).all()          # +0.0, not -0.0


def test_reduce_order_is_visible_in_the_bits():
    """The tests can only pin an order the data can tell apart from its neighbours."""
    rows = rows_of(4097, seed=1)
    ref = dr.reduce_splat(rows)
    flipped = dr.BUTTERFLY
    try:
        dr.BUTTERFLY = tuple(reversed(flipped))
        assert not np.array_equal(dr.reduce_splat(rows), ref)
    finally:
        dr.BUTTERFLY = flipped
    short = rows_of(16, seed=2)
    assert not np.array_equal(dr.reduce_splat(short), naive_reduce(np.concatenate([short, np.zeros((1, 9), F32)])))
    assert not np.array_equal(naive_reduce(short[::-1]), dr.reduce_splat(short))


def test_reduce_all_equals_reduce_splat_per_splat():
    rng = np.random.default_rng(7)
    n = np.array([0, 3, 16, 17, 0, 1, 300, 15, 256, 257, 2, 600, 16], np.int64)
    P = n.size
    order = rng.permutation(P)
    lens = n[rng.permutation(P)]         # lens[d]: rows of the splat at depth position d
    offsets = np.cumsum(lens).astype(np.uint32)
    inst = rows_of(int(lens.sum()), seed=8)
    got = dr.reduce_all(inst, offsets, order)
    e = offsets.astype(np.int64)
    b = e - lens
    for d in range(P):
        assert np.array_equal(got[order[d]].view(np.uint32), dr.reduce_splat(inst[b[d]:e[d]]).view(np.uint32)), d
    assert np.array_equal(dr.long_set(offsets, order), np.sort(order[lens > 16]))


def naive_finalize(p, inv_norm):
    lanes = []
    for ln in range(32):
        s = 0.0
        k = ln
        while k < len(p):
            s = s + float(p[k])
            k += 32
        lanes.append(s)
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[ln] + lanes[ln ^ o] for ln in range(32)]
    return F32(lanes[0] * inv_norm)


@pytest.mark.parametrize("slots", [0, 1, 31, 32, 33, 64, 65, 2040, 8160])
def test_finalize_view_is_the_documented_order(slots):
    rng = np.random.default_rng(slots)
    p = rng.uniform(0, 1024, slots) * np.exp(rng.uniform(-30, 0, slots))
    p[::7] = 0.0
    inv = dr.loss_inv_norm(2160, 3840)
    got = dr.finalize_view(p, inv)
    assert got.dtype == F32
    assert got.view(np.uint32) == naive_finalize(p, inv).view(np.uint32)
    exact = float(np.sum(p.astype(np.longdouble))) * inv
    assert abs(float(got) - exact) <= float(np.spacing(F32(exact))) + 1e-45
    if slots > 32:   # starting at lane 1 drops a partial: other bits
        assert naive_finalize(p[1:], inv) != got or p[0] == 0.0


def test_det_carve():
    for R, P in ((0, 0), (0, 5), (1, 1), (7, 3), (1000, 64), (12345, 6789)):
        w = dr.det_carve(R, P)
        assert w["n_long"] == 0 and w["inst"] == 256 and w["rank"] % 256 == 0 and w["long_g"] % 256 == 0
        assert w["rank"] >= w["inst"] + 36 * R and w["long_g"] >= w["rank"] + 4 * P and w["total"] >= w["long_g"] + 4 * P
        assert w["total"] == 256 + dr.align256(36 * R) + 2 * dr.align256(4 * P)


def test_loss_slots():
    W = 1920
    rows4 = [(0, 1080, 0, 1080), (0, 0, 0, 0), (37, 600, 42, 590)]
    off, slots = dr.loss_slots(dr.LOSS_HEADER_B, rows4, W)
    assert off == dr.LOSS_HEADER_B + dr.align256(9 * (1080 + 563) * W * 4)
    assert slots == 60 * 34
    assert dr.loss_need(dr.LOSS_HEADER_B, rows4, W) == off + 16 * 3 * slots


def counts_of(c):
    n, _, _ = br.local_counts(c["means2D"], c["radii"], c["cl"], c["W"], c["H"], c["vs"])
    return n


def test_range_length_scene_holds_the_promised_counts():
    c, promise = dr.range_length_scene()
    n = counts_of(c)
    P = promise.size
    assert len(c["vs"]) == 3 and c["vs"][-1] == 2 * P
    fixed = promise >= 0
    assert np.array_equal(n[:P][fixed], promise[fixed])
    lab = c["label"][:P]
    for want in ("1", "15", "16", "17", "255", "256", "257", "4097"):
        assert (n[:P][lab == want] == int(want)).all() and (lab == want).any(), want
    gx, gy = br.tiles_of(c["W"], c["H"])
    assert (n[:P][lab == "whole"] == gx * gy).all()
    assert (n[:P][lab == "0"] == 0).all()
    # view 1: the checkerboard mask keeps the tiles with odd x + y of each rect
    x0, y0, x1, y1 = br.rects(c["means2D"][P:], c["radii"][P:], gx, gy)
    for i in np.nonzero(fixed)[0]:
        odd = sum((x + y) % 2 for y in range(y0[i], y1[i]) for x in range(x0[i], x1[i]))
        assert n[P + i] == (odd if c["radii"][P + i] > 0 else 0), i
    hist = np.bincount(n[:P][fixed])
    assert hist[16] == 3 and hist[17] == 2 and hist[15] == 2
    # the sorted offsets carry the same lengths
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], c["vs"], with_list=False)
    assert np.array_equal(np.sort(dr.range_lengths(ref["offsets"])), np.sort(n))


def test_long_population_exceeds_the_persistent_ctas():
    c, promise = dr.long_population()
    n = counts_of(c)
    assert np.array_equal(n, promise)
    assert ((n >= 17) & (n <= 40)).all()
    assert (n > dr.DR_SHORT).sum() > dr.DR_LONG_CTAS * 2
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], with_list=False)
    assert dr.long_set(ref["offsets"], ref["order"]).size == n.size
