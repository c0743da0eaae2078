"""Deterministic synthetic scenes and cameras for the BASELINE.json configurations.

Distributions follow SURVEY.md section 8(d).  Camera matrices restate the conventions of
/root/reference/utils/graphics_utils.py:42-76 (getWorld2View2, getProjectionMatrix) and
/root/reference/scene/cameras.py:84-100 (row-vector / transposed storage, znear 0.01,
zfar 100); tests/test_golden.py pins them against vectors generated from those files.
Everything here is host-side numpy: the arrays are the HOST buffers bench.py copies in.
"""
import math

import numpy as np

ZNEAR, ZFAR = 0.01, 100.0

#: BASELINE.json configs (name -> N Gaussians, width, height, world size, batch size)
CONFIGS = {
    "c1": dict(n=50_000, width=400, height=400, world=1, bsz=1),
    "c2": dict(n=2_000_000, width=1920, height=1080, world=1, bsz=1),
    "c3": dict(n=6_000_000, width=1600, height=1060, world=4, bsz=4),
    "c4": dict(n=40_000_000, width=3840, height=2160, world=8, bsz=8),
}


def world_to_view(R, t, translate=(0.0, 0.0, 0.0), scale=1.0):
    """4x4 world->view with the reference's re-centring option (graphics_utils.py:42-54)."""
    Rt = np.zeros((4, 4), np.float64)
    Rt[:3, :3] = np.asarray(R, np.float64).T
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    c2w = np.linalg.inv(Rt)
    c2w[:3, 3] = (c2w[:3, 3] + np.asarray(translate, np.float64)) * scale
    return np.linalg.inv(c2w).astype(np.float32)


def projection_matrix(znear, zfar, fovx, fovy):
    """OpenGL-style perspective with z_sign=+1 (graphics_utils.py:56-76); built in fp32 like the
    reference's torch.zeros(4,4) so the stored numbers agree bit for bit."""
    f32 = np.float32
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    bottom, left = -top, -right
    P = np.zeros((4, 4), np.float32)
    P[0, 0] = f32(2.0 * znear / (right - left))
    P[1, 1] = f32(2.0 * znear / (top - bottom))
    P[0, 2] = f32((right + left) / (right - left))
    P[1, 2] = f32((top + bottom) / (top - bottom))
    P[3, 2] = f32(1.0)
    P[2, 2] = f32(zfar / (zfar - znear))
    P[2, 3] = f32(-(zfar * znear) / (zfar - znear))
    return P


def make_camera(width, height, fovx_deg=60.0, yaw_deg=0.0, sh_degree=3, uid=0):
    """Camera at the origin looking down +z, yawed about y.  Returns the dict layout the
    operator settings use (viewmatrix / projmatrix transposed as in scene/cameras.py:84-99)."""
    fovx = math.radians(fovx_deg)
    tanx = math.tan(fovx / 2)
    tany = tanx * height / width
    fovy = 2 * math.atan(tany)
    a = math.radians(yaw_deg)
    R = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], np.float64)
    t = np.zeros(3)
    w2v = world_to_view(R, t)                                   # standard column-vector matrix
    viewmatrix = np.ascontiguousarray(w2v.T)                    # stored transposed
    proj = np.ascontiguousarray(projection_matrix(ZNEAR, ZFAR, fovx, fovy).T)
    full = (viewmatrix.astype(np.float32) @ proj.astype(np.float32)).astype(np.float32)
    campos = np.linalg.inv(viewmatrix.astype(np.float64))[3, :3].astype(np.float32)
    return dict(uid=uid, image_width=int(width), image_height=int(height), FoVx=fovx, FoVy=fovy, tanfovx=tanx,
                tanfovy=tany, viewmatrix=viewmatrix, projmatrix=np.ascontiguousarray(full),
                campos=np.ascontiguousarray(campos), sh_degree=int(sh_degree))


def make_scene(n, width, height, fovx_deg=60.0, seed=0, radius_px=6.0, max_sh_degree=3):
    """n Gaussians in the activated parameterisation the operator receives
    (scene/gaussian_model.py:109-129: exp'd scales, normalised wxyz, sigmoid'd opacity,
    SH (n,K,3) = cat(dc, rest), K = (max_sh_degree+1)^2).  A lower max_sh_degree draws the same scene and keeps the first
    K coefficients."""
    rng = np.random.default_rng(seed)
    tanx = math.tan(math.radians(fovx_deg) / 2)
    tany = tanx * height / width
    fx = width / (2 * tanx)
    z = rng.uniform(2.0, 12.0, n)
    x = rng.uniform(-1.1, 1.1, n) * z * tanx
    y = rng.uniform(-1.1, 1.1, n) * z * tany
    means3D = np.stack([x, y, z], 1).astype(np.float32)
    # sigma_px ~ s0*fx*exp(N(0,.5)); the major axis of three lognormal draws has median ~1.3x, and
    # radius = ceil(3 sqrt(sigma^2 + 0.3))
    s0 = (radius_px - 0.5) / 3.0 / 1.3 / fx
    log_s = np.log(s0 * z)[:, None] + rng.normal(0.0, 0.5, (n, 3))
    scales = np.exp(log_s).astype(np.float32)
    q = rng.normal(0.0, 1.0, (n, 4))
    rotations = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    opacities = (1.0 / (1.0 + np.exp(-rng.normal(0.0, 1.5, (n, 1))))).astype(np.float32)
    shs = np.concatenate([rng.normal(0.0, 1.0, (n, 1, 3)), rng.normal(0.0, 0.1, (n, 15, 3))], 1).astype(np.float32)
    K = (int(max_sh_degree) + 1) ** 2
    return dict(means3D=means3D, scales=scales, rotations=rotations, opacities=opacities,
                shs=np.ascontiguousarray(shs[:, :K]))


SHARD_CHUNK = 1 << 20


def make_scene_shard(n, lo, hi, width, height, fovx_deg=60.0, seed=0, radius_px=6.0):
    """Gaussians [lo, hi) of an n-Gaussian scene WITHOUT generating the rest: the scene is defined chunk by chunk
    (SHARD_CHUNK Gaussians per chunk, each from its own generator seeded (seed, chunk)), so every rank of a large
    configuration (c4: 40 M Gaussians = 9.4 GB of parameters) builds only its own shard, and the union over ranks is the
    same scene for every world size.  Same distributions as make_scene (a different sample: make_scene draws the whole
    scene from one stream)."""
    parts = []
    for c in range(lo // SHARD_CHUNK, (max(hi, lo + 1) - 1) // SHARD_CHUNK + 1):
        c0 = c * SHARD_CHUNK
        m = min(SHARD_CHUNK, n - c0)
        if m <= 0:
            break
        sc = make_scene(m, width, height, fovx_deg, seed=(seed, c), radius_px=radius_px)
        a, b = max(lo, c0) - c0, min(hi, c0 + m) - c0
        parts.append({k: v[a:b] for k, v in sc.items()})
    if not parts:
        return {k: v[:0] for k, v in make_scene(1, width, height, fovx_deg, seed=(seed, 0), radius_px=radius_px).items()}
    return {k: np.concatenate([q[k] for q in parts]) for k in parts[0]}


def make_gt_image(width, height, seed=1):
    """uint8 (3,H,W) ground truth, as the reference keeps GT on the host (scene/cameras.py:66)."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (3, height, width), dtype=np.uint8)


def make_batch_cameras(width, height, bsz, sh_degree=3):
    return [make_camera(width, height, yaw_deg=5.0 * k, sh_degree=sh_degree, uid=k) for k in range(bsz)]
