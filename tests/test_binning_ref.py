"""CPU: pins tests/binning_ref.py, the numpy statement of the tile-binning contract, against the fp32 oracle's
render_forward (tiles_touched, offsets, keys, ids, ranges) on every single-view population of tests/binning_cases.py the
oracle can take, and against a brute-force per-tile loop on tiny scenes, so the reference does not rest on the oracle
alone.  Also checks that every regime the cases claim is populated."""
from fractions import Fraction

import numpy as np
import pytest

import binning_cases as bc
import binning_ref as br
from oracle.oracle import Oracle

F32 = np.float32


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32)


def oracle_ok(c):
    """The oracle's C (int) cast is undefined outside the int32 range and for NaN; leave those splats out."""
    return ~np.isin(c["label"].astype(str), ("nonfinite", "beyond_int"))


def subset(c, keep):
    d = dict(c)
    for k in ("means2D", "conic_opacity", "rgb", "depths", "radii", "label"):
        d[k] = c[k][keep]
    d["vs"] = [0, int(keep.sum())]
    return d


def single_view_cases():
    cs = [bc.rect_case(), bc.record_case()]
    cs += [bc.size_case(P) for P in (0, 1, 255, 256, 257)]
    cs += [bc.shape_case(W, H, m) for W, H in bc.SHAPES[:7] for m in ("all", "none", "checkerboard", "single", "last")]
    return cs


@pytest.mark.parametrize("c", single_view_cases(), ids=lambda c: c["name"])
def test_reference_matches_the_oracle(o32, c):
    c = subset(c, oracle_ok(c))
    H, W = c["H"], c["W"]
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], W, H)
    o = o32.render_forward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["depths"], c["radii"], c["cl"], (0, 0, 0))
    assert ref["R"] == o["R"]
    assert np.array_equal(ref["touched"], o["tiles_touched"].astype(np.int64))
    # the oracle scans in index order; the reference's offsets are the same counts scanned in depth order
    assert np.array_equal(np.cumsum(ref["touched"]).astype(np.uint32), o["offsets"])
    assert np.array_equal(ref["offsets"], np.cumsum(o["tiles_touched"][ref["order"]].astype(np.int64)).astype(np.uint32))
    keys = (ref["tiles"].astype(np.uint64) << np.uint64(32)) | c["depths"].view(np.uint32)[ref["ids"]].astype(np.uint64)
    assert np.array_equal(keys, o["keys"])
    assert np.array_equal(ref["ids"], o["ids"])
    assert np.array_equal(ref["ranges"], o["ranges"])


def brute_force(c):
    """Every tile of every view, in order; inside a tile the splats whose fp32 rect holds it, sorted by (depth bits,
    index) with Python's sort.  -> tiles, ids, ranges, touched."""
    W, H = c["W"], c["H"]
    gx, gy = br.tiles_of(W, H)
    T = gx * gy
    vs = c["vs"]
    B = len(vs) - 1
    dbits = c["depths"].view(np.uint32)
    tiles, ids, ranges = [], [], np.zeros((B * T, 2), np.uint32)
    touched = np.zeros(len(c["radii"]), np.int64)
    sixteen, fifteen = F32(16), F32(15)
    rect = []
    for i in range(len(c["radii"])):
        px, py = (F32(q) for q in c["means2D"][i])
        r = int(c["radii"][i])
        rr = F32(r)
        with np.errstate(invalid="ignore", over="ignore"):
            lo = [br.f2i((q - rr) / sixteen)[0] for q in (px, py)]
            hi = [br.f2i(((q + rr) + fifteen) / sixteen)[0] for q in (px, py)]
        rect.append((min(gx, max(0, lo[0])), min(gy, max(0, lo[1])), min(gx, max(0, hi[0])), min(gy, max(0, hi[1])), r))
    for v in range(B):
        for t in range(T):
            if not c["cl"][v * T + t]:
                continue
            ty, tx = divmod(t, gx)
            members = [i for i in range(vs[v], vs[v + 1])
                       if rect[i][4] > 0 and rect[i][0] <= tx < rect[i][2] and rect[i][1] <= ty < rect[i][3]]
            members.sort(key=lambda i: (int(dbits[i]), i))
            if members:
                ranges[v * T + t] = (len(ids), len(ids) + len(members))
            for i in members:
                touched[i] += 1
                tiles.append(v * T + t)
                ids.append(i)
    return np.array(tiles, np.uint32), np.array(ids, np.uint32), ranges, touched


def tiny_cases():
    """48x32 (6 tiles) in 1 and 4 views: edge means, far means reaching in, non-finite means, every depth class."""
    out = []
    for B, seed in ((1, 1), (4, 2)):
        p = bc.Pop(48, 32, B=B, seed=seed)
        rng = p.rng
        for v in range(B):
            if B > 1 and v == 1:
                continue                           # an empty view between non-empty ones
            n = 40
            d = bc.SPECIAL_DEPTHS[rng.integers(0, bc.SPECIAL_DEPTHS.size, n)]
            d[::5] = F32(2.0)                      # ties
            p.add(rng.uniform(-20, 68, n), rng.uniform(-20, 52, n), rng.integers(-2, 30, n), depth=d, view=v)
            p.add([16.0, bc.ulp_step(16, -1), bc.ulp_step(32, 1), -(2.0 ** 22), np.nan, np.inf, -np.inf, 1e12],
                  [bc.ulp_step(16, 1), 8.0, 31.0, 10.0, 5.0, 5.0, 5.0, 5.0],
                  [1, 16, 7, 2 ** 22 + 20, 5, 5, 5, 2 ** 31 - 1], view=v, label="special")
        cl = np.ones(B * 6, np.uint8)
        if B > 1:
            cl[[0, 7, 13, 14, 23]] = 0
        out.append(p.finish(f"tiny_B{B}", cl))
    return out


@pytest.mark.parametrize("c", tiny_cases(), ids=lambda c: c["name"])
def test_reference_matches_a_brute_force_loop(c):
    tiles, ids, ranges, touched = brute_force(c)
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], c["vs"])
    assert ref["R"] == tiles.size > 0
    assert np.array_equal(ref["touched"], touched)
    assert np.array_equal(ref["tiles"], tiles)
    assert np.array_equal(ref["ids"], ids)
    assert np.array_equal(ref["ranges"], ranges)
    key = np.where(touched > 0, c["depths"].view(np.uint32).astype(np.int64), 0xFFFFFFFF)
    order = sorted(range(touched.size), key=lambda i: (int(key[i]), i))
    assert np.array_equal(ref["order"], np.array(order, np.uint32))
    assert np.array_equal(ref["offsets"], np.cumsum(touched[order]).astype(np.uint32))


def test_batched_reference_is_the_single_view_reference_per_view():
    for c in bc.view_cases() + [bc.depth_case(k) for k in ("runs", "special")]:
        ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], c["vs"])
        T = np.prod(br.tiles_of(c["W"], c["H"]))
        for v in range(len(c["vs"]) - 1):
            a, b = c["vs"][v], c["vs"][v + 1]
            one = br.bin_splats(c["means2D"][a:b], c["depths"][a:b], c["radii"][a:b], c["cl"][v * T:(v + 1) * T],
                                c["W"], c["H"])
            lo = np.searchsorted(ref["tiles"], v * T)
            hi = np.searchsorted(ref["tiles"], (v + 1) * T)
            assert np.array_equal(ref["tiles"][lo:hi] - v * T, one["tiles"]), (c["name"], v)
            assert np.array_equal(ref["ids"][lo:hi] - a, one["ids"]), (c["name"], v)
            assert np.array_equal(ref["touched"][a:b], one["touched"])


def test_f2i_has_the_device_conversion_semantics():
    x = np.array([0.0, -0.0, 0.9999999, -0.9999999, 2.5, -2.5, 2.0 ** 31, -(2.0 ** 31), 2.0 ** 35, -1e12, np.inf,
                  -np.inf, np.nan, 2147483520.0], F32)
    want = [0, 0, 0, 0, 2, -2, 2 ** 31 - 1, -(2 ** 31), 2 ** 31 - 1, -(2 ** 31), 2 ** 31 - 1, -(2 ** 31), 0, 2147483520]
    assert br.f2i(x).tolist() == want


def test_saturating_means_give_empty_rects():
    c = bc.rect_case()
    bad = np.isin(c["label"].astype(str), ("nonfinite", "beyond_int"))
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], with_list=False)
    assert bad.sum() >= 40 and (ref["touched"][bad] == 0).all()
    big = c["label"].astype(str) == f"radius_{2 ** 31 - 1}"   # in-image means: the whole image
    assert (ref["touched"][big] == np.prod(br.tiles_of(c["W"], c["H"]))).all()


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a, b = (rng.normal(size=3000) * 10.0 ** rng.integers(-20, 20, 3000)).astype(F32), rng.normal(size=3000).astype(F32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.normal(size=3000) * 1e-7)).astype(F32)   # heavy cancellation
    got = br.fma32(a, b, c)
    for i in range(a.size):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        g = Fraction(float(got[i]))
        # no fp32 value lies strictly closer to the exact result
        for nb in (np.nextafter(got[i], F32(np.inf)), np.nextafter(got[i], F32(-np.inf))):
            assert abs(Fraction(float(nb)) - exact) >= abs(g - exact)


def all_cases_for_regimes():
    return [bc.rect_case(), bc.depth_case("special"), bc.record_case()]


@pytest.mark.parametrize("c", all_cases_for_regimes(), ids=lambda c: c["name"])
def test_every_regime_is_populated(c):
    reg = bc.regimes(c)
    need = bc.REQUIRED["depth_special" if c["name"].startswith("depth_special") else c["name"]]
    for k in need:
        assert reg.get(k, 0) >= 3, (c["name"], k, reg.get(k, 0))


def test_view_and_size_regimes_are_populated():
    bts = {}
    for c in bc.view_cases():
        B = len(c["vs"]) - 1
        T = int(np.prod(br.tiles_of(c["W"], c["H"])))
        bts[c["name"]] = (B, T)
        counts = np.diff(c["vs"])
        if c["name"] == "view_start_empty_runs":
            assert counts[0] == 0 and counts[-1] == 0 and (counts[20:23] == 0).all() and counts.sum() > 0
        if c["name"] == "view_start_all_in_one":
            assert (counts > 0).sum() == 1
    prods = [B * T for B, T in bts.values()]
    pow2 = lambda x: x & (x - 1) == 0   # noqa: E731
    assert any(pow2(x) and B > 1 for x, (B, _) in zip(prods, bts.values()))
    assert any(pow2(x - T) and not pow2(x) for x, (_, T) in zip(prods, bts.values()))
    assert any(pow2(x + T) and not pow2(x) for x, (_, T) in zip(prods, bts.values()))
    assert {1, 64} <= {B for B, _ in bts.values()}
    big = bc.views_1080p()
    assert len(big["vs"]) == 65 and 64 * np.prod(br.tiles_of(1920, 1080)) == 522240
    for k in ("loguniform", "ulp", "equal", "runs"):
        d = bc.depth_case(k)["depths"]
        if k == "loguniform":
            assert d.min() < 2.0 ** -120 and d.max() > 2.0 ** 120
        if k == "ulp":
            assert np.unique(d).size == 7
        if k in ("equal", "runs"):
            assert np.unique(d).size <= 3
