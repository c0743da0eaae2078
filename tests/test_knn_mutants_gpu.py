"""-m gpu: the 3-NN search at the edges its pruning and its input check decide, against knn_ref (the numpy restatement of
the kernels' fp32 arithmetic), bit for bit.

  * a box skipped only when its bound is >= the third best: clouds where a query's third nearest point is the only
    point of a leaf, at a distance d the box's bound equals exactly, with the seeded third best one ulp above d.  A
    bound one ulp high (an inflated bound, or a rounding sequence other than the point distance's, which lies above d
    for the chosen gaps) skips that leaf, and the query's mean moves from fl(d / 3) to fl(nextup(d) / 3);
  * a non-finite coordinate on any axis, anywhere in the cloud, is refused."""
import time

import numpy as np
import pytest
import torch

import gpu_util as gu
import knn_ref
from simple_knn import _C as knn

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module", autouse=True)
def report():
    """Reports the file's runtime and peak device memory."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[knn mutants] {time.perf_counter() - t0:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 20:.1f} MiB on {torch.cuda.get_device_name(0)}")


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def dist2(q, p):
    """knn_ref's point distance of two (3,) float32 points."""
    return knn_ref.dist2_pairs(q[None, :], p[None, :])[0, 0]


def box_bound_of_point(q, p):
    """The box bound of a box holding p alone, restated: per axis the gap fl(p - q) or fl(q - p) (0 inside), then the
    point distance's own sequence fma(gz, gz, fma(gx, gx, gy * gy))."""
    g = np.where(q < p, (p - q).astype(F32), np.where(q > p, (q - p).astype(F32), F32(0))).astype(F32)
    a = knn_ref.fma32(g[0:1], g[0:1], (g[1:2] * g[1:2]).astype(F32))
    return knn_ref.fma32(g[2:3], g[2:3], a)[0]


def rounded_squares_sum(g):
    """fl(fl(fl(gx^2) + fl(gy^2)) + fl(gz^2)): the same sum with every operation rounded."""
    s = (g * g).astype(F32)
    return F32(F32(s[0] + s[1]) + s[2])


def edge_cloud(seed, q, scale):
    """33 float32 points: the query q and two copies of it (sorted positions 0..31 hold every point but the last), a
    point C at distance nextup(d) below q, 28 fillers far below q, and last a point T above q on every axis at
    distance d.  T's coordinates are the largest on every axis and its index the last, so the Morton sort puts it
    last and it is alone in the second leaf: the leaf's box is T itself and its bound from q is exactly d.  The gaps
    are chosen so that the sum of rounded squares of the gap lies above d, and so that fl(d / 3) != fl(nextup(d) / 3).
    -> (points, d)."""
    rng = np.random.default_rng(seed)
    q = np.asarray(q, F32)
    for _ in range(100_000):
        t = (q + rng.uniform(0.4, 1.2, 3) * scale).astype(F32)
        d = dist2(q, t)
        up = np.nextafter(d, F32(np.inf))
        gap = (t - q).astype(F32)
        if box_bound_of_point(q, t) != d or not rounded_squares_sum(gap) > d or F32(d / F32(3)) == F32(up / F32(3)):
            continue
        cx, cy = rng.uniform(0.4, 0.7, 2) * scale
        rest = float(up) - cx * cx - cy * cy
        if rest <= (0.1 * scale) ** 2:
            continue
        base = np.array([q[0] - cx, q[1] - cy, q[2] - np.sqrt(rest)], F32)
        for k in range(-16, 17):
            c = base.copy()
            c[2] = F32(base[2] + F32(k) * np.spacing(base[2]))
            if dist2(q, c) == up:
                break
        else:
            continue
        fill = np.stack([q[0] - scale * (20 + np.arange(28)), np.full(28, q[1] - 20 * scale),
                         np.full(28, q[2] - 20 * scale)], 1).astype(F32)
        pts = np.concatenate([q[None], q[None], q[None], c[None], fill, t[None]]).astype(F32)
        assert (pts[:-1] < t).all()
        return pts, d
    raise AssertionError("no edge configuration found")


EDGES = [(1, (0.0, 0.0, 0.0), 0.5), (2, (3.0, -2.0, 5.0), 0.3), (3, (-40.5, 17.25, 1000.0), 2.0),
         (4, (0.125, 0.0625, -0.25), 1e-3), (5, (7.0, 7.0, 7.0), 30.0), (6, (-1.0, 2.0, -3.0), 0.07)]


@pytest.mark.parametrize("seed,q,scale", EDGES)
def test_third_neighbour_exactly_at_a_box_bound(seed, q, scale):
    pts, d = edge_cloud(seed, q, scale)
    want = knn_ref.mean_dist2(pts)
    up = np.nextafter(d, F32(np.inf))
    # the edge: the query's three best are {0, 0, d}, and without T they would be {0, 0, nextup(d)}
    assert same_bits(want[:3], np.full(3, F32(d / F32(3))))
    without = knn_ref.mean_dist2(pts[:-1])
    assert same_bits(without[:3], np.full(3, F32(up / F32(3)))) and not same_bits(without[:3], want[:3])
    t = torch.from_numpy(pts).to(gu.DEV)
    assert same_bits(knn.distCUDA2(t).cpu().numpy(), want)
    assert same_bits(knn._dist2_brute(t).cpu().numpy(), want)
    assert same_bits(knn._dist2_range(t, 0, 3).cpu().numpy(), want[:3])


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_coordinate_on_every_axis_is_refused(axis, bad):
    rng = np.random.default_rng(axis)
    for n, at in ((1, 0), (5, 4), (1000, 0), (70_000, 69_999), (70_000, 33_333)):   # 70 000: many partial boxes
        p = rng.uniform(-1.0, 1.0, (n, 3)).astype(F32)
        p[at, axis] = bad
        t = torch.from_numpy(p).to(gu.DEV)
        with pytest.raises(ValueError, match="not finite"):
            knn.distCUDA2(t)
        with pytest.raises(ValueError, match="not finite"):
            knn._dist2_range(t, 0, 1)
