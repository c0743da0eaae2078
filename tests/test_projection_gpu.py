"""-m gpu: the projection entry points against the CPU oracle with posed cameras and region-controlled scenes.

gs_preprocess_{forward,backward}, their _raw (fused activation) and _batched forms all run project()
(csrc/preprocess.cu).  The other parity tests use a camera at the origin that only yaws, fx == fy, splats well
inside the image and scale_modifier 1.  Here every case uses a posed camera of tests/golden/cameras.npz (translation,
re-centring, fovx != fovy) and the region mix of proj_cases.region_scene: interior, the guard band on x / y / both and
within ulps of its edge, both sides of the near plane, behind, off-screen, flat discs, sub-pixel splats and negative DC
terms.  Outputs start NaN-filled: every output must be written for every splat.

Bars.  The integer-deciding forward chain (radii, depths, means2D, clamp bits) is bit-exact with the fp32 oracle: both
evaluate it as the same unfused fp32 operations.  Gradients follow test_gpu_parity: at most OUTLIER_FRAC of the entries
outside 1e-4 relative + 1e-4 x RMS of the fp32 oracle, and against the fp64 oracle no further than twice the fp32
oracle's own distance.  The near-plane and guard-band decisions are fp32 decisions, so splats within a few ulps of one
are left out of the fp64 comparison (and counted); against the fp32 oracle they must agree like every other splat.
"""
import os

import numpy as np
import pytest
import torch

import gpu_util as gu
import proj_cases as pc
from gs_b200 import _lib, ops, pipeline
from gs_b200 import synthetic as syn
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

OUTLIER_FRAC = 2e-4
W, H = 197, 131                 # ragged tiles on both axes
SIZES = (1, 129, 20011)         # 20011 = 156 x 128 + 43: a ragged tail that is not a multiple of 4 (non-TMA staging)
MODS = (1.0, 0.6, 1.7)
KEYS = ("means3D", "scales", "rotations", "opacities", "shs")
RAW = ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity")


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32, threads=max(1, (os.cpu_count() or 8) // 2))


@pytest.fixture(scope="module")
def o64():
    return Oracle(np.float64, threads=max(1, (os.cpu_count() or 8) // 2))


def _bad(got, ref, rtol=1e-4, atol_scale=1e-4):
    """Entries outside gu.rel_report's bar: |got - ref| > rtol |ref| + atol_scale rms(ref)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    rms = float(np.sqrt(np.mean(ref ** 2))) if ref.size else 0.0
    return np.abs(got - ref) > rtol * np.abs(ref) + atol_scale * rms


def _call(sc):
    return sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"]


def _activated(sc, raw):
    """The activated parameters the _raw kernels compute from `raw`: exp and sigmoid by torch (the same device expf),
    the quaternion normalised in numpy fp32 in the kernel's operation order (sqrtf of an unfused sum, max(n, 1e-12))."""
    r = gu.npy(raw[4])
    n = np.sqrt(((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2]) + r[:, 3] * r[:, 3])
    den = np.maximum(n, np.float32(1e-12))[:, None]
    return dict(means3D=sc["means3D"], scales=gu.npy(torch.exp(raw[3])), rotations=r / den,
                opacities=gu.npy(torch.sigmoid(raw[5])), shs=sc["shs"])


def _chain(g, act, raw):
    """Oracle gradients w.r.t. the activated parameters -> gradients w.r.t. the raw ones, in fp64."""
    f = lambda a: np.asarray(a, np.float64)
    q, gq = f(act["rotations"]), f(g["rotations"])
    den = np.linalg.norm(f(gu.npy(raw[4])), axis=1, keepdims=True)
    op = f(act["opacities"])
    return dict(xyz=f(g["means3D"]), f_dc=f(g["shs"])[:, :1], f_rest=f(g["shs"])[:, 1:],
                scaling=f(g["scales"]) * f(act["scales"]), rotation=(gq - q * (q * gq).sum(1, keepdims=True)) / den,
                opacity=f(g["opacities"]) * op * (1 - op))


def _assert_forward_bits(out, ref, rows=None):
    """radii, depths, means2D and clamp bits bit-exact; conic / rgb under test_preprocess_forward_parity's bars."""
    sel = (lambda a: a) if rows is None else (lambda a: a[rows])
    assert np.array_equal(sel(gu.npy(out["radii"])), sel(ref["radii"]))
    assert np.array_equal(sel(gu.npy(out["depths"])).view(np.uint32), sel(ref["depths"]).view(np.uint32))
    assert np.array_equal(sel(gu.npy(out["means2D"])).view(np.uint32), sel(ref["means2D"]).view(np.uint32))
    if "clamped" in out:        # the autograd-level operators do not return the clamp bits
        assert np.array_equal(sel(gu.npy(out["clamped"])), sel(ref["clamped"]))


def _assert_forward(out, ref):
    _assert_forward_bits(out, ref)
    np.testing.assert_allclose(gu.npy(out["conic_opacity"]), ref["conic_opacity"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(gu.npy(out["rgb"]), ref["rgb"], rtol=1e-5, atol=1e-6)


def _assert_raw_forward(out, ref, stats):
    """The _raw kernels against the oracle on the activated parameters: every splat culled or kept alike (or all but
    1e-4 of them), the integer chain bit-exact where it is, conic / rgb count-bounded as in the fused-activation test."""
    same = gu.npy(out["radii"]) == ref["radii"]
    stats["raw_same"] = min(stats.get("raw_same", 1.0), float(same.mean()))
    assert same.mean() >= 0.9999
    _assert_forward_bits(out, ref, same)
    for k in ("conic_opacity", "rgb"):
        a = gu.npy(out[k])
        assert not np.isnan(a).any(), k
        frac, _ = gu.outside(a[same], ref[k][same], rtol=1e-4, atol_scale=1e-6)
        assert frac <= 1e-3, k
    return same


def _check_sizes(cam, sc, label, ref):
    """Every region is populated where it is asserted (the large cases)."""
    vis = ref["radii"] > 0
    tx, ty, tz = pc.view_coords32(cam, sc["means3D"])
    limx = pc.GUARD * np.float32(cam["tanfovx"])
    limy = pc.GUARD * np.float32(cam["tanfovy"])
    near = label == pc.NEAR_EDGE
    assert (near & (tz <= pc.NEAR)).sum() > 20 and (near & (tz > pc.NEAR)).sum() > 20
    assert (near & vis).sum() > 0 and not (vis & (tz <= pc.NEAR)).any()
    with np.errstate(divide="ignore", invalid="ignore"):
        cx, cy = np.abs(tx / tz) > limx, np.abs(ty / tz) > limy
    for r, m in ((pc.GUARD_X, cx), (pc.GUARD_Y, cy), (pc.GUARD_XY, cx & cy)):
        assert (vis & (label == r) & m).sum() > 0, pc.REGION_NAMES[r]
    assert (vis & (label == pc.NEAR_BAND)).sum() > 0
    assert not (vis & (label == pc.BEHIND)).any()
    assert not (vis & (label == pc.OFF_EMPTY)).any()
    assert (vis & (label == pc.OFF_REACH)).sum() > 0
    assert (vis & (label == pc.FLAT)).sum() > 0 and (vis & (label == pc.SUBPIX)).sum() > 0
    assert set(ref["clamped"][vis].tolist()) == set(range(8))
    assert (vis & pc.near_threshold(cam, sc["means3D"])).sum() > 0


@pytest.mark.parametrize("P", SIZES)
@pytest.mark.parametrize("camera", range(pc.N_GOLDEN))
def test_projection_posed_camera(o32, o64, camera, P):
    """Plain and _raw entry points, forward and backward, for one posed camera x degree 0..3 x scale_modifier
    {1, 0.6, 1.7}."""
    st = dict(worst=0.0, frac=0.0, k64=0.0, o64=0.0, excluded=0, raw_frac=0.0, visible=0)
    for deg in range(4):
        for mod in MODS:
            cam = pc.golden_camera(camera, W, H, sh_degree=deg)
            seed = 1000 * camera + 10 * deg + MODS.index(mod) + P
            sc, label = pc.region_scene(cam, P, seed=seed)
            nc = (deg + 1) ** 2
            # ---- plain forward: bit-exact chain; SH coefficients above the degree do not change any output ----
            ref = o32.preprocess_forward(*_call(sc), cam, scale_modifier=mod)
            out, d, c = gu.preprocess_forward(sc, cam, mod)
            _assert_forward(out, ref)
            st["visible"] += int((ref["radii"] > 0).sum())
            if P == SIZES[-1]:
                _check_sizes(cam, sc, label, ref)
            if nc < 16:
                alt = dict(sc, shs=sc["shs"].copy())
                alt["shs"][:, nc:] = np.random.default_rng(seed).normal(0.0, 50.0, alt["shs"][:, nc:].shape)
                out2, _, _ = gu.preprocess_forward(alt, cam, mod)
                for k in out:
                    assert torch.equal(out2[k], out[k]), k
            # ---- plain backward: fp32 oracle, fp64 floor, exact zeros ----
            rng = np.random.default_rng(seed + 1)
            gm, gc, gr = (rng.normal(size=(P, s)).astype(np.float32) for s in (2, 4, 3))
            rb = o32.preprocess_backward(*_call(sc), cam, ref["radii"], ref["clamped"], gm, gc, gr, scale_modifier=mod)
            rb64 = o64.preprocess_backward(*_call(sc), cam, ref["radii"], ref["clamped"], gm, gc, gr, scale_modifier=mod)
            got = gu.preprocess_backward(d, c, cam, out, gu.to_dev(gm), gu.to_dev(gc), gu.to_dev(gr), mod)
            culled = ref["radii"] == 0
            thr = pc.near_threshold(cam, sc["means3D"]) & ~culled
            keep = ~thr
            st["excluded"] += int(thr.sum())
            for k in KEYS:
                a = gu.npy(got[k])
                assert not np.isnan(a).any(), k
                bad = _bad(a, rb[k])
                st["frac"] = max(st["frac"], float(bad.mean()))
                st["worst"] = max(st["worst"], gu.outside(a, rb[k])[1])
                assert bad.mean() <= OUTLIER_FRAC, (k, deg, mod)
                assert not bad[thr].any(), (k, "threshold-adjacent splat disagrees with the fp32 oracle")
                assert (a[culled] == 0).all(), k
                mine, _ = gu.outside(a[keep], rb64[k][keep])
                floor, _ = gu.outside(rb[k][keep], rb64[k][keep])
                st["k64"], st["o64"] = max(st["k64"], mine), max(st["o64"], floor)
                assert mine <= 2.0 * floor + OUTLIER_FRAC, (k, deg, mod, mine, floor)
            assert (gu.npy(got["shs"])[:, nc:] == 0).all()
            # ---- _raw: the same case from the raw parameters ----
            raw = gu.raw_parameters(sc)
            act = _activated(sc, raw)
            refa = o32.preprocess_forward(*_call(act), cam, scale_modifier=mod)
            outr = gu.preprocess_forward_raw(raw, cam, mod)
            same = _assert_raw_forward(outr, refa, st)
            rba = o32.preprocess_backward(*_call(act), cam, refa["radii"], refa["clamped"], gm, gc, gr, scale_modifier=mod)
            exp = _chain(rba, act, raw)
            gotr = gu.preprocess_backward_raw(raw, cam, outr, gu.to_dev(gm), gu.to_dev(gc), gu.to_dev(gr), mod)
            for t, name in zip(gotr, RAW):
                a = gu.npy(t)
                assert not np.isnan(a).any(), name
                bad = _bad(a[same], exp[name][same])
                st["raw_frac"] = max(st["raw_frac"], float(bad.mean()))
                assert bad.mean() <= OUTLIER_FRAC, (name, deg, mod)
                assert (a[gu.npy(outr["radii"]) == 0] == 0).all(), name
            assert (gu.npy(gotr[2]).reshape(P, 15, 3)[:, nc - 1:] == 0).all()
    print(f"[parity] projection cam{camera} P={P} (deg 0-3 x mod {MODS}): vs fp32 oracle worst_rel={st['worst']:.2e} "
          f"outside={st['frac']:.2e} | vs fp64: kernel outside={st['k64']:.2e} fp32 oracle outside={st['o64']:.2e} | "
          f"threshold-adjacent splats excluded from the fp64 comparison: {st['excluded']} | raw: radii identical "
          f"{st['raw_same']:.6f} outside={st['raw_frac']:.2e} | visible {st['visible']}")


def _settings(dcam, deg, mod):
    rs = dcam.settings(deg)
    rs.scale_modifier = mod
    return rs


def _batched_case(deg, mod, sizes):
    cams = [pc.golden_camera(i, W, H, sh_degree=deg) for i in range(pc.N_GOLDEN)]
    parts = [pc.region_scene(cams[i], n, seed=500 + 7 * i + deg)[0] for i, n in enumerate(sizes)]
    sc = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    settings = [_settings(pipeline.DeviceCamera(c, gu.DEV), deg, mod) for c in cams]
    return cams, sc, settings


@pytest.mark.parametrize("deg,mod", [(0, 1.0), (1, 0.6), (2, 1.7), (3, 1.0)])
def test_batched_projection_posed_cameras(o32, deg, mod):
    """gs_preprocess_*_batched over the six posed cameras (each camera's region mix, so every camera also sees the other
    cameras' splats from anywhere): slice k == the single-camera _raw call bit for bit and == the oracle for camera k;
    the backward == the sum of the six cameras' oracle gradients."""
    sizes = [3336] * 5 + [3331]                       # P = 20011
    cams, sc, settings = _batched_case(deg, mod, sizes)
    B, P = len(cams), sum(sizes)
    raw = [t.clone().requires_grad_(True) for t in gu.raw_parameters(sc)]
    act = _activated(sc, raw)
    packed = ops.pack_cameras(settings)
    bout = ops.preprocess_gaussians_batched(*raw, packed, W, H, deg, mod)
    rng = np.random.default_rng(deg)
    gm, gr, gc = (rng.normal(size=(B, P, s)).astype(np.float32) for s in (2, 3, 4))
    exp = {n: 0.0 for n in RAW}
    st = {}
    for k in range(B):
        single = ops.preprocess_gaussians_raw(*raw, settings[k])
        for a, b, name in zip(bout, single, ("means2D", "rgb", "conic_opacity", "radii", "depths")):
            assert torch.equal(a[k], b), (k, name)
        ref = o32.preprocess_forward(*_call(act), cams[k], scale_modifier=mod)
        o = dict(means2D=bout[0][k], rgb=bout[1][k], conic_opacity=bout[2][k], radii=bout[3][k], depths=bout[4][k])
        same = _assert_raw_forward(o, ref, st)
        assert (ref["radii"][same] > 0).sum() > 1000
        rb = o32.preprocess_backward(*_call(act), cams[k], ref["radii"], ref["clamped"], gm[k], gc[k], gr[k],
                                     scale_modifier=mod)
        for name, v in _chain(rb, act, raw).items():
            exp[name] = exp[name] + v
    loss = (bout[0] * gu.to_dev(gm)).sum() + (bout[1] * gu.to_dev(gr)).sum() + (bout[2] * gu.to_dev(gc)).sum()
    loss.backward()
    nc = (deg + 1) ** 2
    for t, name in zip(raw, RAW):
        frac, _ = gu.rel_report(f"batched.deg{deg}.{name}", gu.npy(t.grad), exp[name])
        assert frac <= OUTLIER_FRAC, name
    assert (gu.npy(raw[2].grad)[:, nc - 1:] == 0).all()
    print(f"[parity] batched deg {deg} mod {mod}: radii identical to the oracle for {st['raw_same']:.6f} of (camera, splat)")


def test_batched_camera_limit():
    """B = 64 (PB_MAX_CAMS) projects like the B = 6 call it repeats; B = 65 returns GS_EINVAL without a launch."""
    deg, P = 3, 2001
    cams, sc, settings = _batched_case(deg, 1.0, [334] * 5 + [331])
    raw = [t.clone().requires_grad_(True) for t in gu.raw_parameters(sc)]
    s64 = [settings[k % 6] for k in range(64)]
    out64 = ops.preprocess_gaussians_batched(*raw, ops.pack_cameras(s64), W, H, deg)
    with torch.no_grad():
        out6 = ops.preprocess_gaussians_batched(*raw, ops.pack_cameras(settings), W, H, deg)
    for k in range(64):
        for a, b in zip(out64, out6):
            assert torch.equal(a[k], b[k % 6]), k
    g = torch.Generator(device=gu.DEV).manual_seed(1)
    gs = [torch.randn(t.shape, device=gu.DEV, generator=g) for t in out64[:3]]
    sum(((o * gg).sum() for o, gg in zip(out64[:3], gs)), torch.zeros((), device=gu.DEV)).backward()
    g64 = [t.grad.clone() for t in raw]
    for t in raw:
        t.grad = None
    # the backward is linear in the incoming gradients: 64 cameras == 6 cameras with the gradients of k = j mod 6 summed
    g6 = [torch.stack([gg[j::6].sum(0) for j in range(6)]) for gg in gs]
    out6g = ops.preprocess_gaussians_batched(*raw, ops.pack_cameras(settings), W, H, deg)
    sum(((o * gg).sum() for o, gg in zip(out6g[:3], g6)), torch.zeros((), device=gu.DEV)).backward()
    for t, ref, name in zip(raw, g64, RAW):
        frac, _ = gu.rel_report(f"batched64.{name}", gu.npy(ref), gu.npy(t.grad))
        assert frac <= OUTLIER_FRAC, name
    # B = 65: rejected before any launch, every output untouched
    c65 = ops.pack_cameras(s64 + [settings[0]])
    xyz, dc, rest, scl, rot, opa = (t.detach() for t in raw)
    m2, dep, co, rgb = gu.nan(65, P, 2), gu.nan(65, P), gu.nan(65, P, 4), gu.nan(65, P, 3)
    rad = torch.full((65, P), -7, dtype=torch.int32, device=gu.DEV)
    clm = torch.full((65, P), 0xAB, dtype=torch.uint8, device=gu.DEV)
    with pytest.raises(_lib.GsError, match=r"code -1\)"):
        _lib.call("gs_preprocess_forward_batched", 65, P, deg, xyz.data_ptr(), dc.data_ptr(), rest.data_ptr(),
                  scl.data_ptr(), 1.0, rot.data_ptr(), opa.data_ptr(), c65.data_ptr(), W, H, m2.data_ptr(),
                  dep.data_ptr(), rad.data_ptr(), co.data_ptr(), rgb.data_ptr(), clm.data_ptr(), gu.stream())
    grads = [gu.nan(*t.shape) for t in raw]
    with pytest.raises(_lib.GsError, match=r"code -1\)"):
        _lib.call("gs_preprocess_backward_batched", 65, P, deg, xyz.data_ptr(), dc.data_ptr(), rest.data_ptr(),
                  scl.data_ptr(), 1.0, rot.data_ptr(), opa.data_ptr(), c65.data_ptr(), W, H, rad.data_ptr(),
                  clm.data_ptr(), m2.data_ptr(), co.data_ptr(), rgb.data_ptr(), *(t.data_ptr() for t in grads),
                  gu.stream())
    torch.cuda.synchronize()
    for t in (m2, dep, co, rgb, *grads):
        assert bool(torch.isnan(t).all())
    assert bool((rad == -7).all()) and bool((clm == 0xAB).all())


def test_whole_step_posed_camera_sh1(o32, o64):
    """pipeline.Trainer (fused activations) for one posed camera with fx != fy at active_sh_degree 1 against
    Oracle.train_step: the DeviceCamera / settings glue with a translated camera and a low SH degree."""
    Wi, Hi = 256, 192
    cam = pc.golden_camera(5, Wi, Hi, sh_degree=1)
    fx, fy = pc.focal(cam)
    assert abs(fx / fy - 1) > 0.5
    sc, _ = pc.region_scene(cam, 30000, seed=77, mix=pc.MILD)
    gt = syn.make_gt_image(Wi, Hi, seed=5)
    ref = o32.train_step(sc, cam, gt)
    ref64 = o64.train_step(sc, cam, gt)
    tr = pipeline.Trainer(sc, [cam], [torch.from_numpy(gt).pin_memory()], torch.device("cuda", 0))
    tr.params.active_sh_degree = 1
    loss = tr.step(resident=False)
    print(f"[parity] posed whole step: loss {loss:.7f} vs oracle {ref['loss']:.7f}")
    assert abs(loss - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    p = tr.params
    q = sc["rotations"].astype(np.float64)
    op = sc["opacities"].astype(np.float64)

    def chain(g):
        gq = g["rotations"].astype(np.float64)
        return dict(xyz=g["means3D"], scaling=g["scales"] * sc["scales"], opacity=g["opacities"] * op * (1 - op),
                    f_dc=g["shs"][:, :1], f_rest=g["shs"][:, 1:], rotation=gq - q * (q * gq).sum(1, keepdims=True))

    e32, e64 = chain(ref["grads"]), chain(ref64["grads"])
    for name, t in (("xyz", p._xyz), ("scaling", p._scaling), ("opacity", p._opacity), ("f_dc", p._features_dc),
                    ("f_rest", p._features_rest), ("rotation", p._rotation)):
        a = gu.npy(t.grad)
        frac, _ = gu.rel_report("posedstep." + name, a, e32[name])
        assert frac <= 5 * OUTLIER_FRAC, name
        mine, floor = gu.floor_report("posedstep." + name, a, e32[name], e64[name])
        assert mine <= 2.0 * floor + OUTLIER_FRAC, (name, mine, floor)
    assert (gu.npy(p._features_rest.grad)[:, 3:] == 0).all()      # coefficients 4..15 are above degree 1
