"""Screen-space populations built to order for the tile-binning tests (CPU and GPU), with no preprocess: every splat is
(means2D, conic_opacity, rgb, depth, radius) chosen so that one regime of csrc/binning.cu sits where the case puts it.

  * rect: means on tile edges 16k and one ulp either side; fractional means whose fp32 px + r + 15 rounds onto a
    multiple of 16 (found by search); |px| of 2^20 - 2^24 with rects reaching into the image, among them means where
    the fp32 sequence and a contracted px / 16 + (r + 15) / 16 disagree; +-inf, NaN, +-1e12, +-2^35 means; radii 1,
    2^24, 2^31 - 1, 0 and negative;
  * depths: all equal, equal runs interleaved across views, one-ulp neighbours, log-uniform over [2^-126, 2^127], and
    +0.0, -0.0, negative, subnormal and +inf depths (ordered by their raw bits, as the published 64-bit key orders them);
  * views: B T = 2^k, 2^k + T and 2^k - T, 64 views of 1080p, view_start with empty first / last / consecutive views and
    with every splat in one view;
  * sizes: P = 0, 1, 255, 256, 257 and 2^21 + 5;
  * record: ordinary, axis-aligned anisotropic and needle conics (eigenvalue ratio >= 1e8), det <= 0 in fp32, A <= 0 or
    C <= 0, subnormal entries; opacities 0, 1, > 1, NaN, fl(1/255) and one ulp either side;
  * masks: all on, all off, checkerboard, one tile, the last tile only, different per view.

A case is a dict: name, W, H, vs (view_start, B + 1 ints), the five splat arrays, cl (B T uint8), label (per splat).
`regimes(case)` counts the splats of every regime the case claims; the tests assert each one populated.
"""
from fractions import Fraction

import numpy as np

import binning_ref as br

F32 = np.float32
INV255 = F32(1.0 / 255.0)


def ulp_step(v, k):
    """v moved by k fp32 steps."""
    v = F32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, F32(np.inf) if k > 0 else F32(-np.inf))
    return v


def ordinary_conics(rng, n, smin=0.5, smax=8.0):
    sx, sy, th = rng.uniform(smin, smax, n), rng.uniform(smin, smax, n), rng.uniform(0, np.pi, n)
    return conic_of(sx, sy, th)


def conic_of(sx, sy, th):
    """Inverse of the covariance R diag(sx^2, sy^2) R^T, formed in fp64 -> (A, B, C) fp64."""
    c, s = np.cos(th), np.sin(th)
    xx = c * c * sx ** 2 + s * s * sy ** 2
    yy = s * s * sx ** 2 + c * c * sy ** 2
    xy = c * s * (sx ** 2 - sy ** 2)
    det = xx * yy - xy * xy
    return yy / det, -xy / det, xx / det


class Pop:
    """Splats per view, concatenated in view order by finish()."""

    def __init__(self, W, H, B=1, seed=0):
        self.W, self.H, self.B = W, H, B
        self.rng = np.random.default_rng(seed)
        self.views = [[] for _ in range(B)]

    def add(self, mx, my, r, depth=None, conic=None, o=None, label="ordinary", view=0):
        mx = np.atleast_1d(np.asarray(mx, F32))
        n = mx.size
        my = np.broadcast_to(np.asarray(my, F32), (n,))
        r = np.broadcast_to(np.asarray(r, np.int64), (n,)).astype(np.int32)
        rng = self.rng
        depth = rng.uniform(0.5, 50.0, n) if depth is None else np.broadcast_to(np.asarray(depth, F32), (n,))
        A, B, C = ordinary_conics(rng, n) if conic is None else (np.broadcast_to(np.asarray(q), (n,)) for q in conic)
        o = rng.uniform(0.02, 1.0, n) if o is None else np.broadcast_to(np.asarray(o, F32), (n,))
        co = np.stack([np.asarray(A, F32), np.asarray(B, F32), np.asarray(C, F32), np.asarray(o, F32)], 1)
        self.views[view].append(dict(m=np.stack([mx, my], 1), r=r, d=np.asarray(depth, F32), co=co,
                                     rgb=rng.uniform(0, 1, (n, 3)).astype(F32), label=np.full(n, label, object)))

    def random(self, n, label="ordinary", rmax=40, view=0, depth=None, margin=0.1):
        W, H, rng = self.W, self.H, self.rng
        mx = rng.uniform(-margin * W, (1 + margin) * W, n)
        my = rng.uniform(-margin * H, (1 + margin) * H, n)
        self.add(mx, my, rng.integers(1, rmax + 1, n), depth=depth, label=label, view=view)

    def finish(self, name, cl=None):
        gx, gy = br.tiles_of(self.W, self.H)
        T = gx * gy
        counts, parts = [], []
        for v in self.views:
            counts.append(sum(p["r"].size for p in v))
            parts += v
        cat = (lambda k, shape, dt: np.concatenate([p[k] for p in parts]).astype(dt) if parts
               else np.zeros(shape, dt))
        c = dict(name=name, W=self.W, H=self.H, vs=[0] + np.cumsum(counts).astype(int).tolist(),
                 means2D=cat("m", (0, 2), F32), radii=cat("r", (0,), np.int32), depths=cat("d", (0,), F32),
                 conic_opacity=cat("co", (0, 4), F32), rgb=cat("rgb", (0, 3), F32),
                 label=cat("label", (0,), object))
        c["cl"] = np.ones(self.B * T, np.uint8) if cl is None else np.asarray(cl, np.uint8).reshape(-1)
        assert c["cl"].size == self.B * T
        return c


def masks(W, H):
    gx, gy = br.tiles_of(W, H)
    T = gx * gy
    ck = np.array([((t % gx) + (t // gx)) % 2 for t in range(T)], np.uint8)
    single = np.zeros(T, np.uint8)
    single[T // 2] = 1
    last = np.zeros(T, np.uint8)
    last[T - 1] = 1
    return dict(all=np.ones(T, np.uint8), none=np.zeros(T, np.uint8), checkerboard=ck, single=single, last=last)


# ---- rect rounding ----------------------------------------------------------------------------------------------

def exact_rect_axis(p, r, g):
    """[lo, hi) of one axis in exact rational arithmetic (truncation toward zero, clamped): what the fp32 sequence
    would give without rounding."""
    q = Fraction(float(p))
    lo, hi = (q - r) / 16, (q + r + 15) / 16
    tr = lambda x: int(x) if x >= 0 else -int(-x)   # noqa: E731
    return min(g, max(0, tr(lo))), min(g, max(0, tr(hi)))


def contracted_hi(p, r):
    """(int) fma(p, 1/16, fl((r + 15) / 16)): the (p + r + 15) / 16 an FMA-contracting rewrite would form."""
    rr = F32(r)
    c = (rr + F32(15)) / F32(16)
    return int(br.f2i(br.fma32(F32(p), F32(1.0 / 16.0), c))[0])


def rounding_onto(gx, rng, n):
    """Fractional (p, r) with fl(fl(p + r) + 15) a multiple 16k of the tile size while p + r + 15 < 16k exactly."""
    out = []
    while len(out) < n:
        k = int(rng.integers(2, gx))
        a = 16 * k - 15                          # the value p + r must round onto
        r = int(rng.integers(a // 2 + 1, a))     # p < r: p's ulp is finer than that of p + r
        p = F32(a - r)
        for j in range(1, 40):
            q = ulp_step(p, -j)
            if F32(q + F32(r)) != F32(a):
                break
            if exact_rect_axis(q, r, gx)[1] != min(gx, int(br.f2i((F32(q + F32(r)) + F32(15)) / F32(16))[0])):
                out.append((q, r))
                break
    return out


def contraction_sensitive(g, rng, n):
    """(p, r), |p| just below 2^24 reaching into the image, where the fp32 sequence and contracted_hi disagree.
    r = 2^24 + 2 + 4 j is exact in fp32 and r + 15 is a tie that rounds down to r + 14; p = 16k - 15 - r is exact while
    |p| < 2^24.  The sequence gives p + r + 15 = 16k (tile k), the contracted form (16k - 1) / 16 (tile k - 1)."""
    out = []
    while len(out) < n:
        k = int(rng.integers(2, g + 1))
        r = 2 ** 24 + 2 + 4 * int(rng.integers(0, (16 * k - 17) // 4))
        p = float(16 * k - 15 - r)
        if float(F32(p)) != p:
            continue
        seq = int(br.f2i((F32(F32(p) + F32(r)) + F32(15)) / F32(16))[0])
        if 0 < seq <= g and seq != contracted_hi(p, r):
            out.append((F32(p), r))
    return out


def rect_case(W=1920, H=1080, seed=11):
    p = Pop(W, H, seed=seed)
    rng = p.rng
    gx, gy = br.tiles_of(W, H)
    for k in range(0, gx + 1, 5):                  # means on tile edges and one ulp either side
        for d in (-1, 0, 1):
            x = ulp_step(16 * k, d)
            for r in (1, 7, 16, 33):
                p.add(x, rng.uniform(0, H), r, label="edge")
                p.add(rng.uniform(0, W), ulp_step(16 * min(k, gy), d), r, label="edge")
    for q, r in rounding_onto(gx, rng, 24):        # fp32 px + r + 15 rounds onto a multiple of 16
        p.add(q, rng.uniform(0, H), r, label="rounds_onto_x")
    for q, r in rounding_onto(gy, rng, 24):
        p.add(rng.uniform(0, W), q, r, label="rounds_onto_y")
    for _ in range(40):                            # far-away means whose rect reaches into the image
        mag = 2.0 ** rng.uniform(20, 24)
        x = F32(-mag)
        p.add(x, rng.uniform(0, H), int(mag) + int(rng.integers(0, W)), label="large")
        p.add(rng.uniform(0, W), F32(mag + H), int(mag) + int(rng.integers(0, H)), label="large")
    for q, r in contraction_sensitive(gx, rng, 24):
        p.add(q, rng.uniform(0, H), r, label="contraction_x")
    for q, r in contraction_sensitive(gy, rng, 24):
        p.add(rng.uniform(0, W), q, r, label="contraction_y")
    for v in (np.inf, -np.inf, np.nan):            # saturating conversions: empty rects, no loop
        for r in (1, 100, 2 ** 31 - 1):
            p.add(F32(v), rng.uniform(0, H), r, label="nonfinite")
            p.add(rng.uniform(0, W), F32(v), r, label="nonfinite")
            p.add(F32(v), F32(v), r, label="nonfinite")
    for v in (1e12, -1e12, 2.0 ** 35, -(2.0 ** 35)):
        for r in (1, 2 ** 24, 2 ** 31 - 1):
            p.add(F32(v), rng.uniform(0, H), r, label="beyond_int")
            p.add(rng.uniform(0, W), F32(v), r, label="beyond_int")
    for r in (1, 2 ** 24, 2 ** 31 - 1):            # radii
        p.add(rng.uniform(0, W, 6), rng.uniform(0, H, 6), r, label=f"radius_{r}")
    for r in (0, -1, -(2 ** 31)):
        p.add(rng.uniform(0, W, 6), rng.uniform(0, H, 6), r, label="radius_nonpositive")
    p.random(400)
    return p.finish("rect")


# ---- depths -----------------------------------------------------------------------------------------------------

SPECIAL_DEPTHS = np.array([0.0, -0.0, -1.0, -3.5e-20, 1e-45, 1e-40, np.inf, 2.0, 1.0], F32)


def depth_case(kind, seed=21):
    """256x256, three views, overlapping splats (so tile lists are long and orders matter) with depths of one kind."""
    B = 3
    p = Pop(256, 256, B=B, seed=seed + len(kind))
    rng = p.rng
    for v in range(B):
        n = 700
        if kind == "equal":
            d = np.full(n, 2.5, F32)
        elif kind == "runs":                       # runs of equal depths, the same values in every view
            d = np.repeat(np.array([1.0, 3.0, 2.0, 3.0, 1.0], F32), n // 5 + 1)[:n]
        elif kind == "ulp":
            base = F32(1.5)
            d = np.array([ulp_step(base, int(k)) for k in rng.integers(-3, 4, n)], F32)
        elif kind == "loguniform":
            d = (2.0 ** rng.uniform(-126, 127, n)).astype(F32)
        elif kind == "special":
            d = SPECIAL_DEPTHS[rng.integers(0, SPECIAL_DEPTHS.size, n)]
        p.add(rng.uniform(0, 256, n), rng.uniform(0, 256, n), rng.integers(8, 48, n), depth=d, label=kind, view=v)
    cl = np.concatenate([masks(256, 256)[m] for m in ("all", "checkerboard", "all")])
    return p.finish(f"depth_{kind}", cl)


# ---- views ------------------------------------------------------------------------------------------------------

def views_case(W, H, B, seed=31, per_view=60, name=None, counts=None, cl=None, rmax=24):
    """B views of W x H; counts: splats per view (default per_view each)."""
    p = Pop(W, H, B=B, seed=seed + 7 * B + W)
    counts = [per_view] * B if counts is None else counts
    for v, n in enumerate(counts):
        if n:
            p.random(n, label="view", view=v, rmax=rmax)
    return p.finish(name or f"views_{W}x{H}x{B}", cl)


def view_cases():
    cs = []
    for W, H, B in ((32, 32, 64), (32, 32, 63), (32, 32, 33), (64, 64, 32), (64, 64, 33), (64, 64, 31), (16, 16, 1),
                    (48, 32, 2), (80, 48, 17)):
        T = np.prod(br.tiles_of(W, H))
        cs.append(views_case(W, H, B, name=f"bt_{B * T}_{W}x{H}x{B}"))
    rng = np.random.default_rng(5)
    counts = [0, 0, 40, 0, 0, 0, 25] + [int(x) for x in rng.integers(0, 30, 55)] + [0, 0]
    counts[20:23] = [0, 0, 0]
    cs.append(views_case(64, 48, 64, counts=counts, name="view_start_empty_runs"))
    one = [0] * 64
    one[37] = 3000
    cs.append(views_case(64, 48, 64, counts=one, name="view_start_all_in_one"))
    return cs


def views_1080p(seed=41):
    """64 views of 1920x1080 (B T = 522 240: the tile sort needs 19 bits), a different mask per view."""
    W, H, B = 1920, 1080, 64
    p = Pop(W, H, B=B, seed=seed)
    for v in range(B):
        p.random(2500, label="view", view=v, rmax=60)
    gx, gy = br.tiles_of(W, H)
    T = gx * gy
    rng = p.rng
    cl = np.zeros((B, T), np.uint8)
    for v in range(B):
        cl[v] = (rng.uniform(size=T) < (v % 8) / 7.0) if v % 5 else masks(W, H)[("all", "checkerboard", "last")[v % 3]]
    return p.finish("views_1080p_x64", cl)


# ---- record -----------------------------------------------------------------------------------------------------

NEEDLE_RATIOS = (1e8, 1e9, 1e10)


def record_case(seed=51):
    W = H = 256
    p = Pop(W, H, seed=seed)
    rng = p.rng
    pos = lambda n: (rng.uniform(16, 240, n), rng.uniform(16, 240, n))   # noqa: E731
    p.add(*pos(200), 20, label="ordinary")
    for ax in (0.0, np.pi / 2):                    # axis-aligned, very different extents on x and y
        sx, sy = rng.uniform(6, 20, 60), rng.uniform(0.7, 2.0, 60)
        p.add(*pos(60), 40, conic=conic_of(sx, sy, np.full(60, ax)), label="anisotropic")
    for ratio in NEEDLE_RATIOS:                    # needles: the plain AC - B^2 cancels
        L = rng.uniform(100, 2000, 150)
        p.add(*pos(150), 60, conic=conic_of(L, L / np.sqrt(ratio), rng.uniform(0.2, 1.37, 150)), label="needle")
    a, c = rng.uniform(0.05, 0.6, 60), rng.uniform(0.05, 0.6, 60)
    b = np.sqrt(F32(a) * F32(c)) * (1 + rng.choice([0.0, 3e-8, 1e-4, 1e-2], 60)) * rng.choice([-1, 1], 60)
    p.add(*pos(60), 10, conic=(a, b, c), label="det_nonpositive")
    for A, C in ((0.0, 0.3), (-0.3, 0.2), (0.25, -1e-3), (-0.1, -0.2), (0.2, 0.0)):
        p.add(*pos(4), 10, conic=(A, 0.01, C), label="A_or_C_nonpositive")
    for A, B, C in ((1e-39, 0.0, 3e-40), (1.4e-45, 1.4e-45, 2.8e-45), (0.3, 1.4e-45, 0.2), (4.2e-45, 0.0, 0.5),
                    (1e-38, 5e-39, 1e-38)):
        p.add(*pos(4), 10, conic=(A, B, C), label="subnormal")
    for o, lab in ((INV255, "o_at"), (ulp_step(INV255, -1), "o_below"), (ulp_step(INV255, 1), "o_above"),
                   (0.0, "o_zero"), (1.0, "o_one"), (1.5, "o_gt1"), (3.0, "o_gt1"), (np.nan, "o_nan")):
        p.add(*pos(12), 12, o=o, label=lab)
    return p.finish("record")


def plain_det_overestimates(co):
    """Needles whose fp32 AC - B^2 without Kahan's compensation (plain and FMA-contracted) exceeds the fp64 determinant
    of the fp32 conic by more than 5 %: a box from that determinant is too small by more than the 2 % widening."""
    A, B, C = (co[:, q] for q in range(3))
    d64 = A.astype(np.float64) * C.astype(np.float64) - B.astype(np.float64) ** 2
    plain = (A * C) - (B * B)
    fused = br.fma32(A, C, -(B * B))
    with np.errstate(invalid="ignore", divide="ignore"):
        return (d64 > 0) & (plain > 1.05 * d64) & (fused > 1.05 * d64)


# ---- sizes and shapes -----------------------------------------------------------------------------------------------

def size_case(P, W=320, H=200, seed=61, rmax=30):
    p = Pop(W, H, seed=seed + P % 1000)
    if P:
        p.random(P, label="size", rmax=rmax)
    return p.finish(f"P{P}")


SHAPES = ((1, 1), (16, 16), (17, 17), (1, 4096), (4096, 1), (256, 256), (4112, 16), (1920, 1080), (3840, 2160))


def shape_case(W, H, mask, seed=71):
    gx, gy = br.tiles_of(W, H)
    p = Pop(W, H, seed=seed + W + 3 * H)
    p.random(min(40000, max(30, 12 * gx * gy)), label="shape", rmax=max(3, min(60, max(W, H) // 4)))
    p.add(F32((W - 1) / 2), F32((H - 1) / 2), max(W, H) + 2, label="whole_image")
    return p.finish(f"shape_{W}x{H}_{mask}", masks(W, H)[mask])


# ---- regimes ------------------------------------------------------------------------------------------------------

def regimes(c):
    """{regime: number of splats} for the regimes case c was built for; the sanity conditions of the constructed ones
    (rounding really happens, a contracted form really disagrees, depth classes are present) are checked here."""
    lab = c["label"]
    out = {str(k): int(v) for k, v in zip(*np.unique(lab.astype(str), return_counts=True))} if lab.size else {}
    m, r = c["means2D"], c["radii"]
    gx, gy = br.tiles_of(c["W"], c["H"])
    if c["name"] == "rect":
        n_onto = n_con = 0
        x0, y0, x1, y1 = br.rects(m, r, gx, gy)
        for i in range(lab.size):
            kind, _, axis = str(lab[i]).rpartition("_")
            if kind not in ("rounds_onto", "contraction"):
                continue
            ax, g = (0, gx) if axis == "x" else (1, gy)
            seq = (x0[i], x1[i]) if ax == 0 else (y0[i], y1[i])
            if kind == "rounds_onto":
                n_onto += seq != exact_rect_axis(m[i, ax], int(r[i]), g)
            else:
                n_con += min(g, max(0, contracted_hi(m[i, ax], int(r[i])))) != seq[1]
        out["rounds_onto_confirmed"], out["contraction_confirmed"] = n_onto, n_con
    if c["name"].startswith("depth_special"):
        d = c["depths"]
        bits = d.view(np.uint32)
        out.update(pos_zero=int((bits == 0).sum()), neg_zero=int((bits == 0x80000000).sum()),
                   negative=int((d < 0).sum()), subnormal=int(((d != 0) & (np.abs(d) < np.finfo(F32).tiny)).sum()),
                   inf=int(np.isinf(d).sum()))
    if c["name"] == "record":
        rec = br.record(c["means2D"], c["conic_opacity"], c["rgb"], np.ones(lab.size))
        co = c["conic_opacity"]
        out["needle_plain_det_too_large"] = int((plain_det_overestimates(co) & (lab == "needle")
                                                 & (rec["kind"] == br.BOX)).sum())
        out["det_nonpositive_fp32"] = int(((lab == "det_nonpositive") & (rec["kind"] == br.DEGENERATE)).sum())
        out["thr_exactly_zero"] = int((rec["prod"] == F32(1)).sum())
        out["dead"] = int((rec["kind"] == br.DEAD).sum())
        A, B, C = (co[:, q] for q in range(3))
        det = br.fma32(A, C, -(B * B)) - br.fma32(B, B, -(B * B))
        out["det_subnormal"] = int(((det > 0) & (det < np.finfo(F32).tiny) & (A > 0) & (C > 0)).sum())
    return out


REQUIRED = {
    "rect": ("edge", "rounds_onto_confirmed", "large", "contraction_confirmed", "nonfinite", "beyond_int", "radius_1",
             f"radius_{2 ** 24}", f"radius_{2 ** 31 - 1}", "radius_nonpositive"),
    "depth_special": ("pos_zero", "neg_zero", "negative", "subnormal", "inf"),
    "record": ("ordinary", "anisotropic", "needle", "needle_plain_det_too_large", "det_nonpositive",
               "det_nonpositive_fp32", "A_or_C_nonpositive", "subnormal", "o_at", "o_below", "o_above", "o_zero", "o_one",
               "o_gt1", "o_nan", "thr_exactly_zero", "dead", "det_subnormal"),
}
