"""-m gpu: the projection's near-plane decision on splats placed exactly on it, in every forward entry point.

project() culls a splat whose fp32 view z is <= 0.2 (the published `p_view.z <= 0.2f` test, oracle/gs_oracle.c).  The
single-camera forwards test tz > 0.2 before they load the scale and rotation, so only the batched forward takes that
decision inside project() itself; the region scenes of tests/proj_cases.py come within a few ulps of the plane but
never land on it.  Here the splats are placed so that the kernel's own fp32 chain (proj_cases.view_coords32: unfused,
left to right) gives tz == 0.2 exactly, one ulp above and one ulp below, and every entry point must cull, keep and
write them as the fp32 oracle does.  The cameras sit at the origin and yaw (fov and yaw vary): with a translated camera
the sum's last term is the translation, so tz lands on a grid of that term's ulps, which 0.2 is not on.
"""
import numpy as np
import pytest
import torch

import gpu_util as gu
import proj_cases as pc
from gs_b200 import ops, pipeline
from gs_b200 import synthetic as syn
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

W, H = 197, 131
N_EACH = 96                       # splats per camera and per side of the plane (on, one ulp above, one ulp below)
ON, ABOVE, BELOW = 0, 1, 2
CAMS = ((60.0, 0.0), (60.0, 17.0), (50.0, -33.0), (75.0, 71.0), (40.0, 150.0), (90.0, -101.0))   # (fovx, yaw) degrees


def camera(i):
    fov, yaw = CAMS[i]
    return syn.make_camera(W, H, fovx_deg=fov, yaw_deg=yaw, uid=i)


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32, threads=4)


def _nudge_to(cam, p, target):
    """Move each fp32 mean by a few ulps along one world axis until view_coords32's tz equals `target` exactly.
    -> (means, hit mask)."""
    p = p.copy()
    hit = pc.view_coords32(cam, p)[2] == target
    for k in range(1, 65):
        for axis in range(3):
            for sgn in (1.0, -1.0):
                if hit.all():
                    return p, hit
                q = p.copy()
                q[:, axis] = p[:, axis] + sgn * k * np.spacing(np.abs(p[:, axis]))
                now = (pc.view_coords32(cam, q)[2] == target) & ~hit
                p[now] = q[now]
                hit |= now
    return p, hit


def near_plane_scene(cam, seed):
    """3 x N_EACH splats in front of the camera's image centre area: view z exactly 0.2, one ulp above, one ulp below
    (in the kernel's fp32 chain).  -> (scene dict, side labels)."""
    rng = np.random.default_rng(seed)
    targets = (pc.NEAR, np.nextafter(pc.NEAR, np.float32(1)), np.nextafter(pc.NEAR, np.float32(0)))
    inv = np.linalg.inv(np.asarray(cam["viewmatrix"], np.float64))
    means, side = [], []
    for s, t in enumerate(targets):
        m = 4 * N_EACH
        tz = np.full(m, float(t))
        tx = rng.uniform(-0.5, 0.5, m) * cam["tanfovx"] * tz
        ty = rng.uniform(-0.5, 0.5, m) * cam["tanfovy"] * tz
        p = (np.stack([tx, ty, tz, np.ones(m)], 1) @ inv)[:, :3].astype(np.float32)
        p, hit = _nudge_to(cam, p, t)
        assert hit.sum() >= N_EACH, (s, int(hit.sum()))
        means.append(p[hit][:N_EACH])
        side.append(np.full(N_EACH, s))
    means, side = np.concatenate(means), np.concatenate(side)
    n = means.shape[0]
    fx, _ = pc.focal(cam)
    s = (rng.uniform(2.0, 6.0, n) * 0.2 / fx)[:, None] * np.exp(rng.normal(0.0, 0.2, (n, 3)))
    q = rng.normal(size=(n, 4))
    sc = dict(means3D=means, scales=s.astype(np.float32),
              rotations=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32),
              opacities=rng.uniform(0.2, 0.9, (n, 1)).astype(np.float32),
              shs=np.concatenate([rng.normal(0.0, 1.0, (n, 1, 3)), rng.normal(0.0, 0.3, (n, 15, 3))], 1).astype(np.float32))
    return sc, side


def _tz(cam, sc):
    return pc.view_coords32(cam, sc["means3D"])[2]


def _check_sides(cam, sc, side, radii):
    tz = _tz(cam, sc)
    assert (tz[side == ON] == pc.NEAR).all() and (tz[side == ABOVE] > pc.NEAR).all() and (tz[side == BELOW] < pc.NEAR).all()
    radii = np.asarray(radii)
    assert (radii[side != ABOVE] == 0).all(), "a splat on or behind the near plane was kept"
    assert (radii[side == ABOVE] > 0).mean() > 0.9, "the splats one ulp in front of the plane must be visible"


@pytest.mark.parametrize("cam_id", range(len(CAMS)))
def test_near_plane_exact_single_camera(o32, cam_id):
    """gs_preprocess_forward and _raw: on the plane culled, one ulp in front kept, every output equal to the fp32
    oracle's (the integer chain bit for bit); the backward of the kept splats against the oracle's."""
    cam = camera(cam_id)
    sc, side = near_plane_scene(cam, seed=40 + cam_id)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    _check_sides(cam, sc, side, ref["radii"])
    out, d, c = gu.preprocess_forward(sc, cam)
    for k in ("radii", "clamped"):
        assert np.array_equal(gu.npy(out[k]), ref[k]), k
    for k in ("means2D", "depths"):
        assert np.array_equal(gu.npy(out[k]).view(np.uint32), ref[k].view(np.uint32)), k
    np.testing.assert_allclose(gu.npy(out["conic_opacity"]), ref["conic_opacity"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(gu.npy(out["rgb"]), ref["rgb"], rtol=1e-5, atol=1e-6)
    raw = gu.raw_parameters(sc)
    outr = gu.preprocess_forward_raw(raw, cam)
    _check_sides(cam, sc, side, gu.npy(outr["radii"]))
    P = side.size
    rng = np.random.default_rng(cam_id)
    gm, gc, gr = (rng.normal(size=(P, s)).astype(np.float32) for s in (2, 4, 3))
    rb = o32.preprocess_backward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam,
                                 ref["radii"], ref["clamped"], gm, gc, gr)
    got = gu.preprocess_backward(d, c, cam, out, gu.to_dev(gm), gu.to_dev(gc), gu.to_dev(gr))
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        a = gu.npy(got[k]).reshape(P, -1).astype(np.float64)
        e = rb[k].reshape(P, -1).astype(np.float64)
        assert (a[side != ABOVE] == 0).all(), k
        err = np.abs(a - e).max(1) / (np.abs(e).max(1) + 1e-30)
        assert err[side == ABOVE].max() <= 1e-4, (k, float(err.max()))


def test_near_plane_exact_batched():
    """gs_preprocess_forward_batched decides the near plane inside project(): for each of the six posed cameras, its
    own on-plane splats are culled and its one-ulp-in-front splats kept, and every slice equals the single-camera _raw
    call bit for bit.  The backward of the kept splats equals the sum of the single-camera backwards."""
    cams = [camera(i) for i in range(len(CAMS))]
    parts = [near_plane_scene(c, seed=70 + i) for i, c in enumerate(cams)]
    sc = {k: np.concatenate([p[0][k] for p in parts]) for k in parts[0][0]}
    own = np.concatenate([np.full(p[1].size, i) for i, p in enumerate(parts)])
    side = np.concatenate([p[1] for p in parts])
    settings = [pipeline.DeviceCamera(c, gu.DEV).settings(3) for c in cams]
    raw = [t.clone().requires_grad_(True) for t in gu.raw_parameters(sc)]
    bout = ops.preprocess_gaussians_batched(*raw, ops.pack_cameras(settings), W, H, 3)
    B, P = len(cams), side.size
    g = torch.Generator(device=gu.DEV).manual_seed(3)
    gs = [torch.randn(t.shape, device=gu.DEV, generator=g) for t in bout[:3]]
    sum((o * gg).sum() for o, gg in zip(bout[:3], gs)).backward()
    gb = [t.grad.clone() for t in raw]
    acc = [torch.zeros_like(t) for t in raw]
    for k in range(B):
        mine = own == k
        rad = gu.npy(bout[3][k])
        _check_sides(cams[k], {"means3D": sc["means3D"][mine]}, side[mine], rad[mine])
        for t in raw:
            t.grad = None
        single = ops.preprocess_gaussians_raw(*raw, settings[k])
        for a, b, name in zip(bout, single, ("means2D", "rgb", "conic_opacity", "radii", "depths")):
            assert torch.equal(a[k], b), (k, name)
        sum((o * gg[k]).sum() for o, gg in zip(single[:3], gs)).backward()
        for a, t in zip(acc, raw):
            a += t.grad
    for a, b, name in zip(gb, acc, ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity")):
        frac, _ = gu.rel_report(f"near_plane_batched.{name}", gu.npy(a), gu.npy(b))
        assert frac <= 2e-4, name
