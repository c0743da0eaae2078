"""Screen-space scenes built to order for the blend-kernel tests (CPU and GPU), and the fp64 decision walk that says
which pixels every fp32 evaluation must agree on.

Each case is made directly from (means2D, conic_opacity, rgb, depths, radii), with no preprocess, so every regime the
blend kernels branch on sits exactly where the case puts it:
  * saturation: pixels whose transmittance crosses T < 1e-4 at a chosen entry of their tile list (just before, at and
    just after 32 = one ballot group, 128 = one checkpoint segment, 256 = one staging chunk, and several segments
    deep), next to pixels of the same tile that never saturate;
  * lengths: tile lists of exactly 0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257 and 1100 entries;
  * clamp: opacity in (0.99, 1], 1 included, centred on or within 0.1 px of pixel centres (alpha = min(0.99, o G));
  * floor: opacity below, at and one ulp either side of 1/255, centred on integer pixels (power exactly +0);
  * ragged: W, H in {1, 15, 17, 33}, a splat whose rect covers the whole image, off-screen means whose rect reaches in;
  * ties: equal depth bits (stable order by index) and depths one ulp apart;
  * degenerate: conics whose fp32 determinant is <= 0 (the blend kernels never cull those per block);
  * band_edge: alpha = 1/255 circles ending within 2e-6 of a pixel block's first or last pixel (the row-band cull);
plus compute_locally masks (all, checkerboard, one tile, none) and dL/dimage patterns (a zero channel, one non-zero
pixel, large magnitudes).  The radius of a splat only chooses its tiles; a case sets it independently of the conic.

decision_walk() evaluates, in fp64, every (pixel, entry) decision a pixel's front-to-back walk takes -- the alpha floor
(power >= ln(1/(255 o))), power <= 0 and T (1 - alpha) < 1e-4 -- with its margin.  A pixel whose margin on any decision
it reaches is inside what two fp32 evaluations (the kernels' FMA'd exponent test and ex2.approx, the oracle's
expf(power) >= 1/255) may disagree on is AMBIGUOUS: the tests leave it out of the per-pixel comparisons and zero its
dL/dimage.  Everywhere else the fp32 oracle, the fp64 oracle and the kernels take the same branch at every entry.
"""
import numpy as np

TILE = 16
SEG_K = 128            # entries per checkpoint segment of the segment-parallel backward
ALPHA_MAX = 0.99
T_EPS = 1e-4
INV255 = np.float32(1.0 / 255.0)

SAT_TARGETS = (31, 32, 33, 127, 128, 129, 255, 256, 257, 384, 520, 700)
LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1100)
FLOOR_OPACITIES = np.array([0.5 * INV255, INV255 * np.float32(1 - 1e-5), np.nextafter(INV255, np.float32(0)), INV255,
                            np.nextafter(INV255, np.float32(1)), INV255 * np.float32(1 + 1e-5), 1.5 * INV255,
                            3.0 * INV255], np.float32)
CLAMP_OPACITIES = np.array([1.0, np.nextafter(np.float32(0.99), np.float32(1)), 0.9901, 0.995, 0.999], np.float32)

# relative fp32 error budgets of the decision walk (see decision_walk)
EXP_TOL = 1e-6       # exponent test: |power - thr| within EXP_TOL (1 + sum of |terms of power|)
ALPHA_TOL = 1e-6     # relative error of one alpha (ex2.approx, o * G, 0.99f against 0.99)


def tiles_of(W, H):
    return (W + TILE - 1) // TILE, (H + TILE - 1) // TILE


class _Scene:
    def __init__(self, W, H, rng):
        self.W, self.H, self.rng = W, H, rng
        self.rows, self.label = [], []

    def add(self, mx, my, A, B, C, o, depth, radius, label, rgb=None):
        rgb = self.rng.uniform(0.0, 1.0, 3) if rgb is None else rgb
        self.rows.append((mx, my, A, B, C, o, *rgb, depth, radius))
        self.label.append(label)

    def iso(self, mx, my, sigma, o, depth, radius, label, rgb=None):
        a = 1.0 / (sigma * sigma)
        self.add(mx, my, a, 0.0, a, o, depth, radius, label, rgb)


def _finish(sc, name, family, bg, cl=None, dl="normal", seed=0):
    """-> case dict.  Depths are stored as fp32: their bits are the sort key (ties and one-ulp neighbours)."""
    r = np.array(sc.rows, np.float64).reshape(-1, 11)
    gx, gy = tiles_of(sc.W, sc.H)
    c = dict(name=name, family=family, W=sc.W, H=sc.H, means2D=r[:, 0:2].astype(np.float32),
             conic_opacity=r[:, 2:6].astype(np.float32), rgb=r[:, 6:9].astype(np.float32),
             depths=r[:, 9].astype(np.float32), radii=r[:, 10].astype(np.int32), label=np.array(sc.label),
             bg=tuple(float(b) for b in bg), cl=np.ones(gx * gy, np.uint8) if cl is None else np.asarray(cl, np.uint8))
    c["dL"] = make_dl(c, dl, seed)
    return c


def make_dl(c, kind, seed=0):
    rng = np.random.default_rng(1000 + seed)
    H, W = c["H"], c["W"]
    g = rng.normal(size=(3, H, W)).astype(np.float32)
    if kind == "zero_channel":
        g[1] = 0.0
    elif kind == "large":
        g *= np.float32(1e4)
        g[:, ::7, ::5] *= np.float32(100.0)
    elif isinstance(kind, tuple) and kind[0] == "pixel":
        y, x = kind[1]
        v = g[:, y, x].copy()
        g[:] = 0.0
        g[:, y, x] = v
    return g


def _in_tile(rng, X0, Y0, lo=1.0, hi=14.9, n=None):
    return rng.uniform(X0 + lo, X0 + hi, n), rng.uniform(Y0 + lo, Y0 + hi, n)


def saturation(seed, bg):
    """64x48 (12 tiles).  Tile t: a two-splat wall (opacity 0.95-0.97) at entries target-2 and target-1 and an
    opacity-1 terminator at entry `target` over the tile's left part; background splats before and after, three
    quarters of them in the right half, so right-half pixels keep blending past the left half's termination and need
    the checkpoints of later segments."""
    rng = np.random.default_rng(seed)
    sc = _Scene(64, 48, rng)
    gx, _ = tiles_of(64, 48)
    for t, target in enumerate(SAT_TARGETS):
        X0, Y0 = (t % gx) * TILE, (t // gx) * TILE
        for k in range(target + 48):
            d = 1.0 + 1e-3 * k
            if target - 2 <= k <= target:
                o = 1.0 if k == target else rng.uniform(0.95, 0.97)
                sc.iso(X0 + 3.3 + rng.uniform(0, 0.4), Y0 + 7.2 + rng.uniform(0, 0.6), 6.0, o, d, 1, "wall")
            else:
                right = rng.uniform() < 0.75
                mx, my = _in_tile(rng, X0, Y0, 9.0 if right else 1.0)
                o = 0.002 if rng.uniform() < 0.08 else rng.uniform(0.03, 0.35)
                sc.iso(mx, my, rng.uniform(0.5, 1.2), o, d, 1, "background")
    return _finish(sc, f"saturation_bg{int(any(bg))}", "saturation", bg, seed=seed)


def lengths(seed=1, bg=(0.25, 0.5, 0.75), cl=None, name="lengths", dl="normal"):
    """64x48 (12 tiles) whose lists hold exactly LENGTHS[t] entries; every splat's rect is its own tile."""
    rng = np.random.default_rng(seed)
    sc = _Scene(64, 48, rng)
    gx, _ = tiles_of(64, 48)
    for t, n in enumerate(LENGTHS):
        X0, Y0 = (t % gx) * TILE, (t // gx) * TILE
        for k in range(n):
            mx, my = _in_tile(rng, X0, Y0)
            sc.iso(mx, my, rng.uniform(0.6, 3.0), rng.uniform(0.02, 0.6), rng.uniform(1.0, 9.0), 1, "lengths")
    return _finish(sc, name, "lengths", bg, cl=cl, dl=dl, seed=seed)


def clamp(seed=2):
    """48x48: per tile a wide veil (opacity 0.3-0.6) in front, then splats with opacity in (0.99, 1] centred on a pixel
    or within 0.1 px of one, mixed with ordinary ones: o G > 0.99 at many pixels, and a second clamped splat ends the
    pixel well below 1e-4 (after the veil) instead of on it."""
    rng = np.random.default_rng(seed)
    sc = _Scene(48, 48, rng)
    gx, gy = tiles_of(48, 48)
    for t in range(gx * gy):
        X0, Y0 = (t % gx) * TILE, (t // gx) * TILE
        sc.iso(X0 + 7.5, Y0 + 7.5, 12.0, rng.uniform(0.3, 0.6), 1.0, 1, "veil")
        for k in range(40):
            d = 2.0 + 0.01 * k
            if k % 3 != 2:
                px, py = rng.integers(1, 15, 2)
                off = np.zeros(2) if k % 2 else rng.uniform(-0.1, 0.1, 2)
                sc.iso(X0 + px + off[0], Y0 + py + off[1], rng.uniform(0.8, 2.5), rng.choice(CLAMP_OPACITIES), d, 1,
                       "clamp")
            else:
                mx, my = _in_tile(rng, X0, Y0)
                sc.iso(mx, my, rng.uniform(0.8, 2.5), rng.uniform(0.1, 0.7), d, 1, "ordinary")
    return _finish(sc, "clamp", "clamp", (0.2, 0.4, 0.6), seed=seed)


def floor(seed=3):
    """48x32: opacities around 1/255 (FLOOR_OPACITIES), half centred on integer pixels (power exactly +0 there), with
    a few ordinary splats so the pixels blend something."""
    rng = np.random.default_rng(seed)
    sc = _Scene(48, 32, rng)
    gx, gy = tiles_of(48, 32)
    for t in range(gx * gy):
        X0, Y0 = (t % gx) * TILE, (t // gx) * TILE
        for v in FLOOR_OPACITIES:
            for k in range(6):
                if k % 2:
                    mx, my = (float(q) for q in rng.integers(1, 15, 2))
                    mx, my = X0 + mx, Y0 + my
                else:
                    mx, my = _in_tile(rng, X0, Y0)
                sc.iso(mx, my, rng.uniform(0.5, 3.0), v, rng.uniform(1, 9), 1,
                       "floor_below" if v < INV255 else "floor_at_or_above")
        for k in range(16):
            mx, my = _in_tile(rng, X0, Y0)
            sc.iso(mx, my, rng.uniform(0.7, 3.0), rng.uniform(0.1, 0.6), rng.uniform(1, 9), 1, "ordinary")
    return _finish(sc, "floor", "floor", (0.1, 0.3, 0.5), seed=seed)


def ragged(W, H, seed=4):
    """W x H with W, H in {1, 15, 17, 33}: one splat covering the whole image, four off-screen means whose rect reaches
    in, and ordinary splats.  Pixels past the image edge in a partial tile carry NaN coordinates in the kernels."""
    rng = np.random.default_rng(seed + 31 * W + H)
    sc = _Scene(W, H, rng)
    big = max(W, H)
    sc.iso((W - 1) / 2, (H - 1) / 2, 0.6 * big + 1, 0.5, 5.0, big + 2, "whole_image")
    for mx, my in ((-6.0, H / 2), (W + 5.0, H / 3), (W / 2, -4.5), (W / 3, H + 3.5)):
        sc.iso(mx, my, 6.0, rng.uniform(0.3, 0.9), rng.uniform(1, 9), 10, "off_screen_reach")
    sc.iso(W + 40.0, -40.0, 2.0, 0.8, 2.0, 3, "off_screen_empty")    # rect outside the image: on no list
    for k in range(2):                                                 # culled (radius 0) on top of the image
        sc.iso((W - 1) / 2, (H - 1) / 2, 2.0, 0.9, 0.5, 0, "culled")
    for k in range(max(8, W * H // 6)):
        sc.iso(rng.uniform(-0.5, W - 0.5), rng.uniform(-0.5, H - 0.5), rng.uniform(0.5, 3.0), rng.uniform(0.05, 0.8),
               rng.uniform(1, 9), 3, "ordinary")
    return _finish(sc, f"ragged_{W}x{H}", "ragged", (0.3, 0.2, 0.1), seed=seed)


def ties(seed=5):
    """32x32: depths drawn from {1.0, 1.5, 2.0} (equal bits: the list keeps index order) and one ulp either side of
    1.5; overlapping splats of distinct colours, so any other order changes the image."""
    rng = np.random.default_rng(seed)
    sc = _Scene(32, 32, rng)
    d15 = np.float32(1.5)
    pool = np.array([1.0, d15, 2.0, np.nextafter(d15, np.float32(0)), np.nextafter(d15, np.float32(3))], np.float32)
    for k in range(240):
        d = pool[rng.integers(0, 3)] if k % 5 < 3 else pool[3 + rng.integers(0, 2)]
        sc.iso(rng.uniform(0, 31), rng.uniform(0, 31), rng.uniform(1.0, 4.0), rng.uniform(0.1, 0.6), d, 6,
               "tie" if k % 5 < 3 else "ulp_apart")
    return _finish(sc, "ties", "ties", (0.0, 0.0, 0.0), seed=seed)


def degenerate(seed=6):
    """32x32: conics with B^2 >= A C after fp32 rounding (det <= 0: a line or a hyperbola; power > 0 on part of the
    plane), among ordinary splats."""
    rng = np.random.default_rng(seed)
    sc = _Scene(32, 32, rng)
    for k in range(120):
        mx, my = rng.uniform(0.3, 30.7, 2)
        if k % 3 == 0:
            a, c = rng.uniform(0.05, 0.6, 2)
            b = np.float32(np.sqrt(np.float32(a) * np.float32(c))) * np.float32(1 + rng.choice([0.0, 3e-8, 2e-7, 1e-4]))
            sc.add(mx, my, a, b * rng.choice([-1, 1]), c, rng.uniform(0.2, 0.8), rng.uniform(1, 9), 8, "degenerate")
        else:
            sc.iso(mx, my, rng.uniform(0.7, 3.0), rng.uniform(0.1, 0.7), rng.uniform(1, 9), 4, "ordinary")
    return _finish(sc, "degenerate", "degenerate", (0.5, 0.5, 0.5), seed=seed)


def band_edge(seed=7):
    """64x64.  In each top-row tile, three integer centres whose splats' alpha = 1/255 circle ends within 2e-6
    (relative) of the first or last pixel of a pixel block on the centre row: (1, 1) reaching x = 4, (5, 7) reaching
    x = 8 and (14, 13) reaching x = 11, 3 px away (power = -4.5 A against thr = -4.5 A (1 + delta)).  The row-band cull
    keeps those blocks only through its margins (2 % + 0.05 px).  The other tiles hold ordinary splats."""
    rng = np.random.default_rng(seed)
    sc = _Scene(64, 64, rng)
    for t in range(4):
        X0 = t * TILE
        for cx, cy in ((1, 1), (5, 7), (14, 13)):
            for k in range(50):
                a = rng.uniform(0.5, 1.2)
                o = np.exp(4.5 * a * (1.0 + rng.uniform(-2e-6, 2e-6))) / 255.0
                sc.add(X0 + cx, cy, a, 0.0, a, o, rng.uniform(1, 9), 1, "band_edge")
    for t in range(4, 16):
        X0, Y0 = (t % 4) * TILE, (t // 4) * TILE
        for k in range(20):
            mx, my = _in_tile(rng, X0, Y0)
            sc.iso(mx, my, rng.uniform(0.7, 3.0), rng.uniform(0.1, 0.7), rng.uniform(1, 9), 1, "ordinary")
    return _finish(sc, "band_edge", "band_edge", (0.1, 0.1, 0.1), seed=seed)


def masks(T, gx):
    ck = np.array([((t % gx) + (t // gx)) % 2 for t in range(T)], np.uint8)
    one = np.zeros(T, np.uint8)
    one[T - 1] = 1
    return dict(all=np.ones(T, np.uint8), checkerboard=ck, single=one, none=np.zeros(T, np.uint8))


def all_cases():
    """The case list of the GPU suite (deterministic)."""
    cs = [saturation(10, (0.0, 0.0, 0.0)), saturation(11, (0.3, 0.6, 0.9))]
    gx, gy = tiles_of(64, 48)
    for k, m in masks(gx * gy, gx).items():
        cs.append(lengths(cl=m, name=f"lengths_mask_{k}"))
    cs += [clamp(), floor(), ties(), degenerate(), band_edge()]
    cs += [ragged(W, H) for W, H in ((1, 1), (15, 17), (17, 33), (33, 15), (33, 1))]
    sat = cs[1]
    for dl in ("zero_channel", "large"):
        c = dict(sat)
        c["name"], c["dL"] = f"{sat['name']}_dl_{dl}", make_dl(sat, dl, 11)
        cs.append(c)
    return cs


def single_pixel_dl(c, y, x):
    d = dict(c)
    d["name"], d["dL"] = f"{c['name']}_dl_pixel_{y}_{x}", make_dl(c, ("pixel", (y, x)), 11)
    return d


def upcast(c):
    return [np.asarray(c[k], np.float64) for k in ("means2D", "conic_opacity", "rgb")]


def decision_walk(c, fwd):
    """fp64 walk of every local tile of case c over the tile lists of fwd (an Oracle.render_forward result).

    Per pixel (H, W arrays): n_contrib (1 + index of the last blended entry), term (index of the entry whose
    T (1 - alpha) < 1e-4 ended the walk, -1 if none), ambiguous.  A decision is ambiguous when its fp64 margin is within
      * exponent test, power >= thr = ln(1/(255 o)): EXP_TOL (1 + S), S = sum of |terms| of power (FMA'd power, -logf);
        when S = 0 the mean sits on the pixel, power is +0 in every evaluation and the test is o > 1/255 exactly;
      * power <= 0: EXP_TOL S;
      * T (1 - alpha) < 1e-4: 2 E + 1e-6 relative, E = sum over the entries blended so far of
        ALPHA_TOL (1 + alpha / (1 - alpha)) (an alpha error scaled by how much it moves 1 - alpha).
    Decisions after the one that ends the walk are not taken and are not counted."""
    H, W = c["H"], c["W"]
    gx, gy = tiles_of(W, H)
    m, co, _ = upcast(c)
    ids_all, ranges, cl = fwd["ids"].astype(np.int64), fwd["ranges"], c["cl"]
    n_contrib = np.zeros((H, W), np.int64)
    term = np.full((H, W), -1, np.int64)
    amb = np.zeros((H, W), bool)
    for t in range(gx * gy):
        if not cl[t]:
            continue
        beg, end = int(ranges[t, 0]), int(ranges[t, 1])
        if end <= beg:
            continue
        ty, tx = divmod(t, gx)
        ys, xs = np.mgrid[ty * TILE:min(H, ty * TILE + TILE), tx * TILE:min(W, tx * TILE + TILE)]
        py, px = ys.reshape(-1, 1).astype(np.float64), xs.reshape(-1, 1).astype(np.float64)
        ids = ids_all[beg:end]
        A, B, C, o = (co[ids, q][None, :] for q in range(4))
        dx, dy = m[ids, 0][None, :] - px, m[ids, 1][None, :] - py
        tA, tB, tC = -0.5 * A * dx * dx, -B * dx * dy, -0.5 * C * dy * dy
        power = tA + tC + tB
        S = np.abs(tA) + np.abs(tB) + np.abs(tC)
        m1 = power + np.log(255.0 * o)
        exact = S == 0.0
        pass1 = np.where(exact, o > 1.0 / 255.0, m1 >= 0.0)
        amb1 = ~exact & (np.abs(m1) <= EXP_TOL * (1.0 + S))
        pass2 = power <= 0.0
        amb2 = ~exact & (np.abs(power) <= EXP_TOL * S)
        alpha = np.minimum(ALPHA_MAX, o * np.exp(np.minimum(power, 0.0)))
        live = pass1 & pass2
        a_eff = np.where(live, alpha, 0.0)
        Tb = np.cumprod(np.concatenate([np.ones((px.shape[0], 1)), 1.0 - a_eff[:, :-1]], 1), 1)
        testT = Tb * (1.0 - alpha)
        ends = live & (testT < T_EPS)
        L = end - beg
        k = np.arange(L)[None, :]
        first = np.where(ends.any(1), ends.argmax(1), L)[:, None]
        e = np.where(live, ALPHA_TOL * (1.0 + np.where(alpha >= ALPHA_MAX, 1.0, alpha / (1.0 - alpha))), 0.0)
        E = np.cumsum(e, 1)
        amb3 = live & (np.abs(testT / T_EPS - 1.0) <= 2.0 * E + 1e-6)
        reached = k <= first
        a_pix = ((amb1 | amb2 | amb3) & reached).any(1)
        blended = live & (k < first)
        nc = np.where(blended.any(1), L - np.argmax(blended[:, ::-1], 1), 0)
        amb[ys, xs] = a_pix.reshape(ys.shape)
        n_contrib[ys, xs] = nc.reshape(ys.shape)
        term[ys, xs] = np.where(first[:, 0] < L, first[:, 0], -1).reshape(ys.shape)
    return dict(n_contrib=n_contrib, term=term, ambiguous=amb)


def masked_dl(c, walk):
    """dL/dimage with the ambiguous pixels zeroed (their gradient contributions then vanish in every evaluation)."""
    g = np.array(c["dL"], np.float32)
    g[:, walk["ambiguous"]] = 0.0
    return g
