"""Images and ground truth for the strip loss kernels (csrc/loss.cu), by regime, and the windows they are cut into.

Regimes, each measured by `regimes()` on the data itself rather than trusted to the generator:
  equal          x == y = fl32(gt * fl32(1/255)), the reference's gt / 255.0 on the device: |x - y| has no sign, its
                 gradient must be 0 (torch's abs)
  equal_zero     x == y == 0: a black background rendered over black ground truth
  equal_one      x == y == 1 on gt 255
  ulp_above / ulp_below   x one fp32 ulp either side of y
  flat_both / flat_x / flat_y   an 11x11 neighbourhood inside the image where both / only x / only y are constant: the
                 SSIM variances vanish (both: sigma1 = sigma2 = 0)
  saturated      x > 1 (rendered rgb is not clamped above), up to ~2.5
  negative       x < 0
  checker        checkerboard ground truth 0 / 255 (maximal variance)
  smooth         a smooth rendered-like field plus noise
"""
import numpy as np
from scipy import ndimage

from eval_ref import INV255

REGIMES = ("equal", "equal_zero", "equal_one", "ulp_above", "ulp_below", "flat_both", "flat_x", "flat_y", "saturated",
           "negative", "checker", "smooth")


def gt_float(gt):
    """The ground truth as the kernel sees it: clamp(fl32(gt * fl32(1/255)), 0, 1), the reference's gt / 255.0 on the
    device (eval_ref.gt_hat)."""
    return np.clip(gt.astype(np.float32) * INV255, 0, 1)


def _smooth(rng, H, W):
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    f = np.zeros((3, H, W))
    for ch in range(3):
        for _ in range(3):
            ky, kx, ph = rng.uniform(0.002, 0.08), rng.uniform(0.002, 0.08), rng.uniform(0, 6.3)
            f[ch] += 0.15 * np.sin(ky * yy + kx * xx + ph)
    return 0.5 + f


def make_pair(H, W, seed, kind="mixed"):
    """-> (img (3,H,W) float32, gt (3,H,W) uint8).

    mixed:  x uniform in [-0.05, 1.2], gt uniform, then every element k of a fixed stride pattern is set to one of the
            exact-equality, one-ulp, saturated and negative regimes, and flat 11x11 blocks are painted where they fit.
    smooth: x and gt a smooth field plus noise (a render next to its photo), with the same scattered regimes.
    checker: checkerboard gt 0 / 255, x uniform in [-0.05, 2.5]."""
    rng = np.random.default_rng(seed)
    if kind == "checker":
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        gt = np.broadcast_to(((yy + xx) % 2 * 255).astype(np.uint8), (3, H, W)).copy()
        img = rng.uniform(-0.05, 2.5, (3, H, W)).astype(np.float32)
        img.reshape(-1)[:2] = (2.5, -0.03)[:img.size]
        return img, gt
    if kind == "smooth":
        f = _smooth(rng, H, W)
        img = (f + rng.normal(0, 0.02, f.shape)).astype(np.float32)
        gt = np.clip(np.rint(255 * (f + rng.normal(0, 0.03, f.shape))), 0, 255).astype(np.uint8)
    else:
        img = rng.uniform(-0.05, 1.2, (3, H, W)).astype(np.float32)
        gt = rng.integers(0, 256, (3, H, W), dtype=np.uint8)
    y = gt_float(gt)
    fi, fg, fy = img.reshape(-1), gt.reshape(-1), y.reshape(-1)
    # the scattered regimes: element k takes regime k % stride (sparse in a smooth field, so it stays smooth)
    slot = np.arange(fi.size) % (16 if kind == "mixed" else 997)
    fi[slot == 0] = fy[slot == 0]
    fi[slot == 1] = np.nextafter(fy[slot == 1], np.float32(np.inf))
    fi[slot == 2] = np.nextafter(fy[slot == 2], np.float32(-np.inf))
    fg[slot == 3], fi[slot == 3] = 0, 0.0
    fg[slot == 4], fi[slot == 4] = 255, 1.0
    fi[slot == 5] = rng.uniform(1.0, 2.5, int((slot == 5).sum())).astype(np.float32)
    fi[slot == 6] = rng.uniform(-0.05, 0.0, int((slot == 6).sum())).astype(np.float32)
    if fi.size > 5:
        fi[5] = 2.5
    # flat 13x13 blocks (the 11x11 neighbourhoods of their 3x3 centre pixels are flat), placed where they fit
    for (gv, xv), (y0, x0) in zip(FLAT_BLOCKS, _spots(H, W)):
        if gv is not None:
            gt[:, y0:y0 + 13, x0:x0 + 13] = gv
        if xv is not None:
            img[:, y0:y0 + 13, x0:x0 + 13] = xv
    return img, gt


# (gt value, x value) of the flat blocks in order: both flat at x == y == 0 and at x == y == 1, only x, only gt
FLAT_BLOCKS = [(0, 0.0), (255, 1.0), (None, 0.375), (100, None)]
FLAT_REGIMES = ["flat_both", "flat_both", "flat_x", "flat_y"]


def _spots(H, W):
    return [(y0, x0) for y0 in range(2, H - 12, 16) for x0 in range(2, W - 12, 16)]


def _flat(a):
    """(3,H,W) bool: the 11x11 neighbourhood lies inside the image and a is constant on it."""
    lo = ndimage.minimum_filter(a, size=(1, 11, 11), mode="nearest")
    hi = ndimage.maximum_filter(a, size=(1, 11, 11), mode="nearest")
    inside = np.zeros(a.shape, bool)
    inside[:, 5:a.shape[1] - 5, 5:a.shape[2] - 5] = True
    return inside & (lo == hi)


def regimes(img, gt):
    """-> {regime: number of elements of (img, gt) in it} (img float32, gt uint8, both (3, rows, W))."""
    y = gt_float(gt)
    fx, fy = _flat(img), _flat(y)
    ch = np.zeros(gt.shape, bool)
    g = gt.astype(np.int32)
    ch[:, :-1, :-1] = ((np.abs(g[:, :-1, :-1] - g[:, 1:, :-1]) == 255) & (np.abs(g[:, :-1, :-1] - g[:, :-1, 1:]) == 255))
    sm = np.zeros(img.shape, bool)
    if img.shape[2] > 1:
        d = np.abs(np.diff(img.astype(np.float64), axis=2))
        sm[:, :, 1:] = d < 0.1
    return dict(
        equal=int((img == y).sum()), equal_zero=int(((img == 0) & (gt == 0)).sum()),
        equal_one=int(((img == 1) & (gt == 255)).sum()),
        ulp_above=int((img == np.nextafter(y, np.float32(np.inf))).sum()),
        ulp_below=int((img == np.nextafter(y, np.float32(-np.inf))).sum()),
        flat_both=int((fx & fy).sum()), flat_x=int((fx & ~fy).sum()), flat_y=int((fy & ~fx).sum()),
        saturated=int((img > 1).sum()), negative=int((img < 0).sum()), checker=int(ch.sum()),
        smooth=int(sm.sum()) if sm.mean() > 0.9 else 0)


def claims(H, W, kind):
    """The regimes a make_pair(H, W, kind) case promises (every element count >= 1)."""
    n = 3 * H * W
    if kind == "checker":
        return {"saturated", "negative"} | ({"checker"} if H > 1 and W > 1 else set())
    scattered = ["equal", "ulp_above", "ulp_below", "equal_zero", "equal_one", "saturated", "negative"]
    out = set(scattered[:n]) | set(FLAT_REGIMES[:len(_spots(H, W))])
    if kind == "smooth":
        out.add("smooth")
    return out


def assert_populated(img, gt, want, tag=""):
    got = regimes(img, gt)
    empty = [r for r in want if got[r] == 0]
    assert not empty, (tag, empty, got)
    return got


def windows(H):
    """Window rows (row0, row1) of an H-row image: 1, 5, 16, 31, 32, 33 rows and the whole image, each starting on a
    16-row tile boundary, off one, and ending at H."""
    out = set()
    for n in (1, 5, 16, 31, 32, 33, H):
        if n > H:
            continue
        aligned = (H - n) // 32 * 16          # a tile boundary near the middle of the room left
        out |= {(aligned, aligned + n), (H - n, H)}
        if aligned + 3 <= H - n:
            out.add((aligned + 3, aligned + 3 + n))
    return sorted(out)


def count_rows(r0, r1, mode):
    """Counted rows of the window [r0, r1): 'all' = the window, 'halo' = strictly inside it (up to 5 rows off each end,
    as border.add_remote_border_rows widens a strip), 'empty' = c0 == c1 inside the window."""
    n = r1 - r0
    if mode == "all" or (mode == "halo" and n < 3):
        return r0, r1
    if mode == "halo":
        h = min(5, (n - 1) // 2)
        return r0 + h, r1 - h
    return r0 + n // 2, r0 + n // 2
