"""-m gpu: blend decisions that fp32 arithmetic takes exactly, on pixels built to sit on them.

tests/test_blend_gpu.py leaves out of its per-pixel comparisons every pixel whose margin on a decision is inside fp32
error (blend_cases.decision_walk), since the fp64 oracle may decide such a pixel the other way.  That also leaves out
pixels whose fp32 arithmetic is exact and which every fp32 evaluation must therefore decide alike.  Here such pixels
are built on purpose:

  * transmittance exactly 1e-4: splats centred on a pixel (power = 0, G = exp(0) = 1, alpha = opacity) whose opacities
    make the fp32 product T (1 - alpha) land on fl32(1e-4) at the third splat.  The walk stops only when T (1 - alpha)
    < 1e-4 (the published `test_T < 0.0001f`), so the third splat is blended and the fourth ends the pixel: final_T =
    fl32(1e-4) and n_contrib is the third splat's place in the tile list.

Both forwards (packed and half-warp) are compared with the fp32 oracle bit for bit on those pixels, and with a numpy
fp32 evaluation of the same products.
"""
import os

import numpy as np
import pytest
import torch

import gpu_util as gu
from gs_b200 import _lib
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

T_EPS32 = np.float32(1e-4)


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32, threads=max(1, (os.cpu_count() or 8) // 2))


def _one_minus(o):
    return np.float32(1) - np.float32(o)


def exact_teps_opacities(rng, n):
    """n triples (o1, o2, o3), each below the 0.99 clamp, with fl(fl(fl(1 - o1) (1 - o2)) (1 - o3)) == fl32(1e-4).
    fl(1 - o3) moves in steps of o3's ulp, so for a given T2 = fl(fl(1 - o1) (1 - o2)) the product lands on fl32(1e-4)
    only now and then; T2 in [3e-4, 5e-3] keeps o3 in [0.67, 0.98] where the steps are fine enough to hit it often."""
    out = []
    for _ in range(200 * n):
        if len(out) == n:
            break
        o1, o2 = (np.float32(v) for v in rng.uniform(0.9, 0.99, 2))
        T2 = np.float32(_one_minus(o1) * _one_minus(o2))
        if not np.float32(3e-4) <= T2 <= np.float32(5e-3):
            continue
        o3 = np.float32(1.0 - 1e-4 / float(T2))
        for _ in range(8):
            t = np.float32(T2 * _one_minus(o3))
            if t == T_EPS32:
                out.append((o1, o2, o3))
                break
            o3 = np.nextafter(o3, np.float32(1) if t > T_EPS32 else np.float32(0))
    assert len(out) == n, len(out)
    return np.array(out, np.float32)


def teps_scene(seed=11, W=64, H=48):
    """Stacks of four splats centred on integer pixels 4 px apart, sigma 0.3 px (alpha < 1/255 one pixel away, so a
    stack touches its own pixel only): three that bring T to exactly 1e-4, then a fourth (opacity 0.5) that ends the
    pixel.  -> (means2D, conic_opacity, rgb, depths, radii, pixels (y, x), opacities)."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(2, H - 1, 4), np.arange(2, W - 1, 4), indexing="ij")
    pix = np.stack([ys.ravel(), xs.ravel()], 1)
    n = pix.shape[0]
    ops = exact_teps_opacities(rng, n)
    a = np.float32(1.0 / 0.09)
    rows = []
    for k, (y, x) in enumerate(pix):
        for j, o in enumerate((*ops[k], np.float32(0.5))):
            rows.append((x, y, a, 0.0, a, o, *rng.uniform(0, 1, 3), 1.0 + j + 1e-3 * k))
    r = np.array(rows, np.float64)
    return dict(means2D=r[:, 0:2].astype(np.float32), conic_opacity=r[:, 2:6].astype(np.float32),
                rgb=r[:, 6:9].astype(np.float32), depths=r[:, 9].astype(np.float32),
                radii=np.ones(r.shape[0], np.int32), pix=pix, ops=ops, W=W, H=H)


def _forward(c, bg, flags=0):
    old = _lib.debug_set(flags)
    try:
        return gu.render_forward(c["H"], c["W"], *(gu.to_dev(c[k]) for k in ("means2D", "conic_opacity", "rgb", "depths",
                                                                         "radii")),
                                 torch.ones(((c["H"] + 15) // 16) * ((c["W"] + 15) // 16), dtype=torch.uint8,
                                            device=gu.DEV), bg)
    finally:
        _lib.debug_set(old)


def test_transmittance_exactly_at_the_floor(o32):
    c = teps_scene()
    bg = (0.25, 0.5, 0.75)
    H, W = c["H"], c["W"]
    ref = o32.render_forward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["depths"], c["radii"],
                             np.ones(((H + 15) // 16) * ((W + 15) // 16), np.uint8), bg)
    py, px = c["pix"][:, 0], c["pix"][:, 1]
    # the regime is there: the fp32 oracle blends the third splat (T lands on 1e-4) and ends the pixel at the fourth
    assert (ref["final_T"][py, px] == T_EPS32).all()
    ids = ref["ids"].astype(np.int64)
    gx = (W + 15) // 16
    for k, (y, x) in enumerate(c["pix"]):
        t = (y // 16) * gx + x // 16
        lst = list(ids[ref["ranges"][t, 0]:ref["ranges"][t, 1]])
        assert ref["n_contrib"][y, x] == lst.index(4 * k + 2) + 1
    # numpy fp32: colour of three blended splats + T bg
    rgb = c["rgb"].reshape(-1, 4, 3)
    T = np.ones(len(py), np.float32)
    col = np.zeros((len(py), 3), np.float32)
    for j in range(3):
        al = c["ops"][:, j]
        col = col + rgb[:, j] * (al * T)[:, None]
        T = (T * (np.float32(1) - al)).astype(np.float32)
    assert (T == T_EPS32).all()
    img_np = col + T[:, None] * np.asarray(bg, np.float32)
    for flags in (0, _lib.DEBUG_FWD_HALFWARP):
        f = _forward(c, bg, flags)
        nc, fT, img = gu.npy(f["n_contrib"]), gu.npy(f["final_T"]), gu.npy(f["image"])
        assert np.array_equal(nc[py, px], ref["n_contrib"][py, px]), flags
        assert np.array_equal(fT[py, px].view(np.uint32), ref["final_T"][py, px].view(np.uint32)), flags
        np.testing.assert_allclose(img[:, py, px].T, img_np, rtol=0, atol=2e-7)
        np.testing.assert_allclose(img[:, py, px], ref["image"][:, py, px], rtol=0, atol=2e-7)
        # the walked-entries statistic counts the terminating fourth splat of each such pixel
        assert int(gu.npy(f["stats"])[1]) == int(ref["stats"][1]), flags
