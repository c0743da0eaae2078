"""Posed cameras and region-controlled scenes for the projection parity tests (CPU and GPU).

golden_camera(i, W, H) is entry i of tests/golden/cameras.npz: rotation, translation, the translate / scale re-centring
and fovx != fovy, all produced by the reference's own camera code.  So the view matrix has a translation, campos is not
the origin, and fx != fy.

region_scene(cam, n) places every splat in VIEW space first, region by region, and maps it to world space with the
inverse view matrix.  The region of each splat (interior, guard band, near plane, behind, off-screen, flat, sub-pixel)
is then an input of the test, not an accident of the sampling.  The decisions the projection takes near a threshold are
fp32 decisions; view_coords32() recomputes the view-space coordinates in the kernel's own fp32 operation order, so
a test can tell which splats sit within a few ulps of the near plane or of the 1.3 tan(fov) guard band.
"""
import math
import os

import numpy as np

from gs_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cameras.npz")
N_GOLDEN = 6
NEAR = np.float32(0.2)      # the projection culls tz <= 0.2 (fp32)
GUARD = np.float32(1.3)     # view-space x/z and y/z are clamped to +-1.3 tan(fov)

INTERIOR, GUARD_X, GUARD_Y, GUARD_XY, GUARD_EDGE, NEAR_EDGE, NEAR_BAND, BEHIND, OFF_EMPTY, OFF_REACH, FLAT, SUBPIX = \
    range(12)
REGION_NAMES = ("interior", "guard_x", "guard_y", "guard_xy", "guard_edge", "near_edge", "near_band", "behind",
                "off_empty", "off_reach", "flat", "subpixel")
#: share of each region in a scene (interior takes the remainder)
MIX = {GUARD_X: 0.07, GUARD_Y: 0.07, GUARD_XY: 0.07, GUARD_EDGE: 0.04, NEAR_EDGE: 0.04, NEAR_BAND: 0.05, BEHIND: 0.05,
       OFF_EMPTY: 0.05, OFF_REACH: 0.05, FLAT: 0.08, SUBPIX: 0.08}
#: a milder mix for whole training steps: no needles (flat discs seen edge-on) and no splats that fill the image
MILD = {GUARD_X: 0.08, GUARD_Y: 0.08, GUARD_XY: 0.05, BEHIND: 0.05, OFF_EMPTY: 0.05, OFF_REACH: 0.05, SUBPIX: 0.08}


def golden_camera(i, width, height, sh_degree=3, uid=None):
    """Entry i of cameras.npz in the dict layout of synthetic.make_camera (viewmatrix / projmatrix stored transposed)."""
    z = np.load(GOLDEN)
    fovx, fovy = float(z[f"fovx_{i}"]), float(z[f"fovy_{i}"])
    w2v = syn.world_to_view(z[f"R_{i}"], z[f"T_{i}"], z[f"trans_{i}"], float(z[f"scale_{i}"]))
    viewmatrix = np.ascontiguousarray(w2v.T)
    proj = np.ascontiguousarray(syn.projection_matrix(syn.ZNEAR, syn.ZFAR, fovx, fovy).T)
    full = (viewmatrix.astype(np.float32) @ proj).astype(np.float32)
    campos = np.linalg.inv(viewmatrix.astype(np.float64))[3, :3].astype(np.float32)
    return dict(uid=i if uid is None else uid, image_width=int(width), image_height=int(height), FoVx=fovx, FoVy=fovy,
                tanfovx=math.tan(fovx / 2), tanfovy=math.tan(fovy / 2), viewmatrix=viewmatrix,
                projmatrix=np.ascontiguousarray(full), campos=np.ascontiguousarray(campos), sh_degree=int(sh_degree))


def focal(cam):
    return cam["image_width"] / (2 * cam["tanfovx"]), cam["image_height"] / (2 * cam["tanfovy"])


def view_coords32(cam, means3D):
    """(tx, ty, tz) in fp32, each an unfused left-to-right sum V[a] x + V[b] y + V[c] z + V[d] as project() evaluates it."""
    V = np.asarray(cam["viewmatrix"], np.float32).reshape(-1)
    p = np.asarray(means3D, np.float32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    row = lambda a, b, c, d: ((V[a] * x + V[b] * y) + V[c] * z) + V[d]
    return row(0, 4, 8, 12), row(1, 5, 9, 13), row(2, 6, 10, 14)


def _ulps(a, b):
    """Distance in ulps between fp32 values of the same sign."""
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32))


def near_threshold(cam, means3D, ulps=4):
    """Splats whose fp32 near-plane or guard-band decision is within `ulps` of flipping."""
    tx, ty, tz = view_coords32(cam, means3D)
    near = _ulps(tz, np.full_like(tz, NEAR)) <= ulps
    with np.errstate(divide="ignore", invalid="ignore"):
        rx, ry = np.abs(tx / tz), np.abs(ty / tz)
    limx = GUARD * np.float32(cam["tanfovx"])
    limy = GUARD * np.float32(cam["tanfovy"])
    front = tz > NEAR
    guard = front & ((_ulps(rx, np.full_like(rx, limx)) <= ulps) | (_ulps(ry, np.full_like(ry, limy)) <= ulps))
    return near | guard


def region_scene(cam, n, seed=0, mix=MIX, neg_dc=0.3):
    """n splats in the activated parameterisation, placed in view space by region.  -> (scene dict, region labels).
    neg_dc: share of splats whose DC term is pushed negative on a random subset of channels, so that every
    combination of the three colour-clamp bits occurs."""
    rng = np.random.default_rng(seed)
    tanx, tany = cam["tanfovx"], cam["tanfovy"]
    W, H = cam["image_width"], cam["image_height"]
    fx, fy = focal(cam)
    counts = {r: int(math.floor(f * n)) for r, f in mix.items()}
    counts[INTERIOR] = n - sum(counts.values())
    label = np.concatenate([np.full(c, r, np.int64) for r, c in sorted(counts.items())])
    label = label[rng.permutation(n)]
    sgn = lambda m: rng.choice([-1.0, 1.0], m)
    tz = rng.uniform(1.0, 8.0, n)
    rx = rng.uniform(-0.95, 0.95, n)          # x/z and y/z in units of tan(fov)
    ry = rng.uniform(-0.95, 0.95, n)
    sigma_px = np.exp(rng.normal(np.log(2.0), 0.5, n))
    flat_axis = np.full(n, -1)
    for r in range(12):
        m = label == r
        k = int(m.sum())
        if k == 0:
            continue
        if r in (GUARD_X, GUARD_Y, GUARD_XY, GUARD_EDGE):
            # centres up to 0.3 W/2 beyond the image edge: only a large splat still reaches a tile
            sigma_px[m] = rng.uniform(4.0, 40.0, k)
        if r in (GUARD_X, GUARD_XY):
            rx[m] = sgn(k) * rng.uniform(1.0, 1.6, k)
        if r in (GUARD_Y, GUARD_XY):
            ry[m] = sgn(k) * rng.uniform(1.0, 1.6, k)
        if r == GUARD_EDGE:               # x/z or y/z within ~10 ulps of the clamp
            on_x = rng.uniform(size=k) < 0.5
            edge = sgn(k) * 1.3 * (1.0 + rng.integers(-12, 13, k) * 6e-8)
            rx[m] = np.where(on_x, edge, rx[m])
            ry[m] = np.where(on_x, ry[m], edge)
        if r == NEAR_EDGE:                # tz within a few tens of ulps of 0.2, both sides
            tz[m] = 0.2 + rng.integers(-24, 25, k) * float(np.spacing(NEAR))
            rx[m] *= 0.5; ry[m] *= 0.5
        if r == NEAR_BAND:
            tz[m] = rng.uniform(0.2, 0.3, k) + 1e-6
            rx[m] *= 0.5; ry[m] *= 0.5
        if r == BEHIND:
            tz[m] = -rng.uniform(0.05, 6.0, k)
        if r == OFF_EMPTY:                # far off-screen and small: empty tile rectangle
            rx[m] = sgn(k) * rng.uniform(2.0, 4.0, k)
            sigma_px[m] = rng.uniform(0.5, 2.0, k)
        if r == OFF_REACH:                # centre 3..25 px beyond an image edge, 3-sigma radius reaching inside
            ix = np.where(rng.uniform(size=k) < 0.5, -rng.uniform(3, 25, k), W - 1 + rng.uniform(3, 25, k))
            rx[m] = ((2 * ix + 1) / W - 1)
            ry[m] *= 0.8
            sigma_px[m] = rng.uniform(10.0, 20.0, k)
        if r == FLAT:
            flat_axis[m] = rng.integers(0, 3, k)
        if r == SUBPIX:
            sigma_px[m] = rng.uniform(0.02, 0.3, k)
    tx, ty = rx * tanx * np.abs(tz), ry * tany * np.abs(tz)
    pv = np.stack([tx, ty, tz, np.ones(n)], 1)
    means3D = (pv @ np.linalg.inv(np.asarray(cam["viewmatrix"], np.float64)))[:, :3].astype(np.float32)
    s = (sigma_px * np.abs(tz) / fx)[:, None] * np.exp(rng.normal(0.0, 0.3, (n, 3)))
    for ax in range(3):
        s[flat_axis == ax, ax] *= 1e-6
    q = rng.normal(size=(n, 4))
    shs = np.concatenate([rng.normal(0.0, 1.0, (n, 1, 3)), rng.normal(0.0, 0.3, (n, 15, 3))], 1)
    neg = rng.uniform(size=n) < neg_dc
    chan = rng.uniform(size=(n, 3)) < 0.5
    shs[:, 0, :] = np.where(neg[:, None] & chan, -rng.uniform(2.0, 4.0, (n, 3)), shs[:, 0, :])
    sc = dict(means3D=means3D, scales=s.astype(np.float32),
              rotations=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32),
              opacities=rng.uniform(0.05, 0.95, (n, 1)).astype(np.float32), shs=shs.astype(np.float32))
    return sc, label
