"""-m gpu parity tests: the CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs.  Bars (BASELINE.json north_star): tile indices bit-exact; rendered RGB and gradients
within 1e-4 relative fp32.  Because alpha >= 1/255 and T < 1e-4 are hard thresholds, two fp32
implementations may legitimately take different branches at a handful of pixels; those show up as
isolated outliers and are bounded by count (<= 2e-4 of entries) rather than hidden by a loose tolerance."""
import numpy as np
import pytest
import torch

import gpu_util as gu
from gs_b200 import synthetic as syn
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-4          # the tolerance north_star states for floating point
OUTLIER_FRAC = 2e-4  # threshold-flip outliers


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32, threads=max(1, (__import__("os").cpu_count() or 8) // 2))


@pytest.fixture(scope="module")
def o64():
    return Oracle(np.float64, threads=max(1, (__import__("os").cpu_count() or 8) // 2))


def case(n, W, H, seed=0, radius_px=7.0, yaw=3.0, sh_degree=3):
    cam = syn.make_camera(W, H, yaw_deg=yaw, sh_degree=sh_degree)
    sc = syn.make_scene(n, W, H, seed=seed, radius_px=radius_px)
    return cam, sc


@pytest.mark.parametrize("n,W,H,deg", [(20000, 320, 200, 3), (5000, 131, 77, 2), (3000, 64, 48, 1), (100, 33, 17, 0),
                                       (1, 16, 16, 3)])
def test_preprocess_forward_parity(o32, n, W, H, deg):
    cam, sc = case(n, W, H, seed=n, sh_degree=deg)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    out, _, _ = gu.preprocess_forward(sc, cam)
    # integer-deciding chain: bit-exact
    assert np.array_equal(gu.npy(out["radii"]), ref["radii"])
    assert np.array_equal(gu.npy(out["depths"]).view(np.uint32), ref["depths"].view(np.uint32))
    assert np.array_equal(gu.npy(out["means2D"]).view(np.uint32), ref["means2D"].view(np.uint32))
    assert np.array_equal(gu.npy(out["clamped"]), ref["clamped"])
    np.testing.assert_allclose(gu.npy(out["conic_opacity"]), ref["conic_opacity"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(gu.npy(out["rgb"]), ref["rgb"], rtol=1e-5, atol=1e-6)
    assert (ref["radii"] > 0).sum() > 0


def test_preprocess_backward_parity(o32):
    cam, sc = case(20000, 320, 200, seed=5)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    out, d, c = gu.preprocess_forward(sc, cam)
    rng = np.random.default_rng(1)
    gm, gc, gr = (rng.normal(size=s).astype(np.float32) for s in ((20000, 2), (20000, 4), (20000, 3)))
    rb = o32.preprocess_backward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam,
                                 ref["radii"], ref["clamped"], gm, gc, gr)
    got = gu.preprocess_backward(d, c, cam, out, gu.to_dev(gm), gu.to_dev(gc), gu.to_dev(gr))
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        frac, _ = gu.rel_report("preprocess_bwd." + k, gu.npy(got[k]), rb[k])
        assert frac <= OUTLIER_FRAC, k
    # culled splats get exact zeros
    culled = ref["radii"] == 0
    assert culled.any()
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        assert (gu.npy(got[k])[culled] == 0).all()


@pytest.mark.parametrize("n,W,H,rad", [(20000, 320, 200, 7.0), (4000, 131, 77, 14.0), (50, 40, 40, 30.0)])
def test_tile_binning_bit_exact(o32, n, W, H, rad):
    cam, sc = case(n, W, H, seed=3, radius_px=rad)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    gx = (W + 15) // 16
    masks = [np.ones(T, np.uint8)]
    strip = np.zeros(T, np.uint8); strip[gx * 2:gx * 5] = 1
    masks.append(strip)
    masks.append((np.random.default_rng(0).uniform(size=T) < 0.5).astype(np.uint8))
    for cl in masks:
        rf = o32.render_forward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], ref["depths"], ref["radii"], cl, (0, 0, 0))
        f = gu.render_forward(H, W, gu.to_dev(ref["means2D"]), gu.to_dev(ref["conic_opacity"]), gu.to_dev(ref["rgb"]),
                              gu.to_dev(ref["depths"]), gu.to_dev(ref["radii"]), gu.to_dev(cl), (0, 0, 0))
        assert f["R"] == rf["R"]
        # splats in ascending depth (stable), those without a local tile last; offsets are the scan in that order
        order = gu.npy(f["order"]).view(np.uint32)[:n]
        dkey = np.where(rf["tiles_touched"] > 0, ref["depths"].view(np.uint32), np.uint32(0xffffffff))
        assert np.array_equal(order, np.argsort(dkey, kind="stable").astype(np.uint32))
        assert np.array_equal(gu.npy(f["offsets"]).view(np.uint32)[:n], np.cumsum(rf["tiles_touched"][order]).astype(np.uint32))
        assert np.array_equal(gu.npy(f["keys"]).view(np.uint64), rf["keys"])
        assert np.array_equal(gu.npy(f["ids"]).view(np.uint32), rf["ids"])
        assert np.array_equal(gu.npy(f["ranges"]).view(np.uint32), rf["ranges"])


def _render_case(o32, n, W, H, rad, bg, seed=3, mask=None):
    cam, sc = case(n, W, H, seed=seed, radius_px=rad)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    cl = np.ones(T, np.uint8) if mask is None else mask
    rf = o32.render_forward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], ref["depths"], ref["radii"], cl, bg)
    f = gu.render_forward(H, W, gu.to_dev(ref["means2D"]), gu.to_dev(ref["conic_opacity"]), gu.to_dev(ref["rgb"]),
                          gu.to_dev(ref["depths"]), gu.to_dev(ref["radii"]), gu.to_dev(cl), bg)
    return ref, rf, f, cl


@pytest.mark.parametrize("n,W,H,rad,bg", [(20000, 320, 200, 7.0, (0.0, 0.0, 0.0)), (30000, 200, 120, 9.0, (0.2, 0.5, 0.9)),
                                          (300, 70, 35, 40.0, (1.0, 1.0, 1.0))])
def test_render_forward_parity(o32, n, W, H, rad, bg):
    ref, rf, f, cl = _render_case(o32, n, W, H, rad, bg)
    img, T_, nc = gu.npy(f["image"]), gu.npy(f["final_T"]), gu.npy(f["n_contrib"]).view(np.uint32)
    assert np.isfinite(img).all()
    err = np.abs(img - rf["image"])
    bad = err > RTOL * np.abs(rf["image"]) + 1e-5
    print(f"[parity] image: max_abs_err={err.max():.3e} outside={bad.mean():.2e} n_contrib_mismatch={(nc != rf['n_contrib']).mean():.2e}")
    assert bad.mean() <= OUTLIER_FRAC
    assert err.max() < 2e-2  # a flipped 1/255 contribution is at most ~0.004 * colour
    assert (nc != rf["n_contrib"]).mean() <= 1e-3
    np.testing.assert_allclose(np.median(np.abs(T_ - rf["final_T"])), 0, atol=1e-6)
    st = gu.npy(f["stats"])
    assert st[0] == rf["stats"][0]
    assert abs(int(st[1]) - int(rf["stats"][1])) <= 1e-3 * rf["stats"][1] + 16
    assert abs(int(st[2]) - int(rf["stats"][2])) <= 1e-3 * rf["stats"][2] + 16


def test_non_local_tiles_are_exact_zero_and_strips_sum_to_full(o32):
    n, W, H = 20000, 320, 200
    gx, gy = (W + 15) // 16, (H + 15) // 16
    ref, rf, full, _ = _render_case(o32, n, W, H, 7.0, (0, 0, 0))
    acc = torch.zeros_like(full["image"])
    Rs = 0
    for lo, hi in ((0, 4), (4, 5), (5, gy)):
        cl = np.zeros((gy, gx), np.uint8); cl[lo:hi] = 1
        _, _, part, _ = _render_case(o32, n, W, H, 7.0, (0, 0, 0), mask=cl.reshape(-1))
        img = part["image"]
        out = torch.ones((H, W), dtype=torch.bool, device=img.device); out[lo * 16:min(H, hi * 16)] = False
        assert (img[:, out] == 0).all()
        acc += img
        Rs += part["R"]
    assert Rs == full["R"]
    assert torch.equal(acc, full["image"])  # a pixel's blend order does not depend on the partition


@pytest.mark.parametrize("n,W,H,rad,bg", [(20000, 320, 200, 7.0, (0.0, 0.0, 0.0)), (3000, 96, 64, 16.0, (0.3, 0.1, 0.7))])
def test_render_backward_parity(o32, n, W, H, rad, bg):
    ref, rf, f, cl = _render_case(o32, n, W, H, rad, bg)
    g = np.random.default_rng(2).normal(size=(3, H, W)).astype(np.float32)
    rb = o32.render_backward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], bg, rf, g)
    got = gu.render_backward(f, gu.to_dev(g))
    for k in ("means2D", "conic_opacity", "rgb"):
        a = gu.npy(got[k])
        assert np.isfinite(a).all()
        frac, _ = gu.rel_report("render_bwd." + k, a, rb[k])
        assert frac <= 5 * OUTLIER_FRAC, k
        untouched = ~np.isin(np.arange(n), rf["ids"])
        assert (a[untouched] == 0).all()


@pytest.mark.parametrize("n,W,H,rad,bg", [(20000, 320, 200, 7.0, (0.0, 0.0, 0.0)), (3000, 96, 64, 16.0, (0.3, 0.1, 0.7)),
                                          (30000, 200, 120, 9.0, (0.2, 0.5, 0.9)), (60000, 100, 70, 12.0, (0.1, 0.2, 0.3))])
def test_backward_kernels_agree(o32, n, W, H, rad, bg):
    """The segment-parallel backward (default: checkpoints written by the forward, one warp per (tile, 64-entry segment))
    against the oracle AND against the tile-parallel kernel (gs_debug_set(GS_DEBUG_BWD_TILE) / no segment workspace);
    the forward's image does not depend on whether it writes checkpoints.  The last case has ~900-entry tile lists
    (many segments per tile)."""
    from gs_b200 import _lib
    ref, rf, f, cl = _render_case(o32, n, W, H, rad, bg)
    g = np.random.default_rng(2).normal(size=(3, H, W)).astype(np.float32)
    rb = o32.render_backward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], bg, rf, g)
    got = gu.render_backward(f, gu.to_dev(g))
    old = _lib.debug_set(_lib.DEBUG_BWD_TILE)
    try:
        tile = gu.render_backward(f, gu.to_dev(g))
    finally:
        _lib.debug_set(old)
    f2 = gu.render_forward(H, W, gu.to_dev(ref["means2D"]), gu.to_dev(ref["conic_opacity"]), gu.to_dev(ref["rgb"]),
                           gu.to_dev(ref["depths"]), gu.to_dev(ref["radii"]), gu.to_dev(cl), bg, seg=False)
    assert torch.equal(f2["image"], f["image"]) and torch.equal(f2["n_contrib"], f["n_contrib"])
    tile2 = gu.render_backward(f2, gu.to_dev(g))
    for k in ("means2D", "conic_opacity", "rgb"):
        a = gu.npy(got[k])
        assert np.isfinite(a).all()
        frac, _ = gu.rel_report(f"seg.{k}", a, rb[k])
        assert frac <= 5 * OUTLIER_FRAC, k
        frac2, _ = gu.rel_report(f"seg.vs_tile.{k}", a, gu.npy(tile[k]))
        assert frac2 <= 5 * OUTLIER_FRAC, k
        frac3, _ = gu.rel_report(f"tile.{k}", gu.npy(tile2[k]), rb[k])
        assert frac3 <= 5 * OUTLIER_FRAC, k
        assert (a[~np.isin(np.arange(n), rf["ids"])] == 0).all()


@pytest.mark.parametrize("n,W,H,rad,bg", [(20000, 320, 200, 7.0, (0.0, 0.0, 0.0)), (3000, 97, 61, 16.0, (0.3, 0.1, 0.7)),
                                          (60000, 100, 70, 12.0, (0.1, 0.2, 0.3))])
def test_forward_kernels_agree(o32, n, W, H, rad, bg):
    """The packed two-pixels-per-lane forward (k_blend_fwd2, default) and round 1's half-warp forward (k_blend_fwd,
    gs_debug_set(GS_DEBUG_FWD_HALFWARP)) run the same per-pixel operation sequence: image, final_T, n_contrib, the
    statistics AND the checkpoints the segment backward reads are bit-identical (ragged image edges included)."""
    from gs_b200 import _lib
    ref, rf, f, cl = _render_case(o32, n, W, H, rad, bg)
    g = gu.to_dev(np.random.default_rng(3).normal(size=(3, H, W)).astype(np.float32))
    b_new = gu.render_backward(f, g)
    old = _lib.debug_set(_lib.DEBUG_FWD_HALFWARP)
    try:
        f1 = gu.render_forward(H, W, gu.to_dev(ref["means2D"]), gu.to_dev(ref["conic_opacity"]), gu.to_dev(ref["rgb"]),
                               gu.to_dev(ref["depths"]), gu.to_dev(ref["radii"]), gu.to_dev(cl), bg)
    finally:
        _lib.debug_set(old)
    for k in ("image", "final_T", "n_contrib", "stats"):
        assert torch.equal(f[k], f1[k]), k
    b_old = gu.render_backward(f1, g)          # the segment backward on the OTHER forward's checkpoints
    for k in ("means2D", "conic_opacity", "rgb"):
        a, b = b_new[k].double(), b_old[k].double()
        assert float(((a - b).abs() > 1e-5 * b.abs() + 1e-5 * b.abs().mean()).double().mean()) <= 1e-4, k


def test_whole_step_parity_config_c1(o32, o64):
    """BASELINE.json configs[0]: 50k Gaussians, 400x400, forward + loss + backward, through the public operator.
    Whole-step gradients compound the forward's rounding through the SSIM derivative (divisions by small variances) and the
    hard thresholds; the operator-level tests above hold 1e-5.  The fp64 oracle gives the noise floor: the kernels must be
    as close to it as the fp32 oracle is."""
    import diff_gaussian_rasterization as dgr
    from gs_b200 import ops
    cam = syn.make_camera(400, 400)
    sc = syn.make_scene(50000, 400, 400)
    gt = syn.make_gt_image(400, 400)
    ref = o32.train_step(sc, cam, gt)
    p = {k: gu.to_dev(v).requires_grad_(True) for k, v in sc.items()}
    rs = dgr.GaussianRasterizationSettings(400, 400, cam["tanfovx"], cam["tanfovy"], torch.zeros(3, device="cuda"), 1.0,
                                           gu.to_dev(cam["viewmatrix"]), gu.to_dev(cam["projmatrix"]), 3,
                                           gu.to_dev(cam["campos"]), False, False)
    r = dgr.GaussianRasterizer(raster_settings=rs)
    cuda_args = {"stats_collector": {}}
    m2, rgb, co, radii, depths = r.preprocess_gaussians(p["means3D"], p["scales"], p["rotations"], p["shs"], p["opacities"], cuda_args)
    m2.retain_grad()
    img, *_ = r.render_gaussians(m2, co, rgb, depths, radii, torch.ones((25, 25), dtype=torch.bool, device="cuda"), None, cuda_args)
    l1, ss = ops.fused_l1_ssim(img, gu.to_dev(gt), 0, 400)
    loss = 0.8 * l1 + 0.2 * (1.0 - ss)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    assert abs(float(l1) - ref["Ll1"]) <= 1e-5 * ref["Ll1"] and abs(float(ss) - ref["ssim"]) <= 1e-4 * abs(ref["ssim"])
    ref64 = o64.train_step(sc, cam, gt)
    for k_t, k_o in (("means3D", "means3D"), ("scales", "scales"), ("rotations", "rotations"), ("opacities", "opacities"), ("shs", "shs")):
        frac, _ = gu.rel_report("step." + k_t, gu.npy(p[k_t].grad), ref["grads"][k_o])
        assert frac <= 5 * OUTLIER_FRAC, k_t
        mine, floor = gu.floor_report("step." + k_t, gu.npy(p[k_t].grad), ref["grads"][k_o], ref64["grads"][k_o])
        assert mine <= 2.0 * floor + OUTLIER_FRAC, (k_t, mine, floor)
    frac, _ = gu.rel_report("step.means2D.grad", gu.npy(m2.grad), ref["render_grads"]["means2D"])
    assert frac <= 5 * OUTLIER_FRAC
    sc_ = cuda_args["stats_collector"]
    assert float(sc_["forward_render_time"]) > 0 and float(sc_["backward_render_time"]) > 0
    assert isinstance(sc_["forward_render_time"] + sc_["backward_render_time"] + 0.5 * 2, float)


def test_loss_kernel_parity(o32):
    rng = np.random.default_rng(7)
    H, W, r0, r1 = 150, 211, 32, 117
    img = rng.uniform(0, 1.2, (3, H, W)).astype(np.float32)
    gt = rng.integers(0, 256, (3, r1 - r0, W), dtype=np.uint8)
    from gs_b200 import ops
    x = gu.to_dev(img).requires_grad_(True)
    l1, ss = ops.fused_l1_ssim(x, gu.to_dev(gt), r0, r1)
    (0.8 * l1 + 0.2 * (1 - ss)).backward()
    gtf = np.clip(gt.astype(np.float32) / np.float32(255), 0, 1)
    rl1, rss, rgrad = o32.loss(img[:, r0:r1], gtf, H * W, 0.2)
    assert abs(float(l1) - rl1) <= 1e-5 * rl1 and abs(float(ss) - rss) <= 1e-4 * abs(rss)
    g = gu.npy(x.grad)
    assert (g[:, :r0] == 0).all() and (g[:, r1:] == 0).all()
    frac, _ = gu.rel_report("loss.grad", g[:, r0:r1], rgrad, rtol=1e-3, atol_scale=1e-3)
    assert frac <= 1e-3


def test_local2j_and_pack_parity(o32):
    cam, sc = case(20000, 320, 200, seed=8, radius_px=12.0)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    import diff_gaussian_rasterization as dgr
    gx = 20
    div = np.array([0, 3, 4, 9, 13], np.int32) * gx
    got = dgr._C.get_local2j_ids_bool(200, 320, 1, 4, gu.to_dev(ref["means2D"]), gu.to_dev(ref["radii"]),
                                      torch.tensor(div, dtype=torch.int32, device="cuda"), {})
    exp = o32.get_local2j_ids_bool(200, 320, 4, ref["means2D"], ref["radii"], div)
    assert got.dtype == torch.bool and np.array_equal(gu.npy(got), exp)
    rects = np.array([[0, 6, 0, 9], [0, 6, 9, 20], [6, 13, 0, 20]], np.int32)
    got6 = dgr._C.get_local2j_ids_bool_adjust_mode6(200, 320, 0, 3, gu.to_dev(ref["means2D"]), gu.to_dev(ref["radii"]),
                                                    torch.tensor(rects, device="cuda"), {})
    assert np.array_equal(gu.npy(got6), o32.get_local2j_ids_bool_rects(200, 320, 3, ref["means2D"], ref["radii"], rects))


def test_empty_and_degenerate_inputs():
    import diff_gaussian_rasterization as dgr
    cam = syn.make_camera(64, 48)
    rs = dgr.GaussianRasterizationSettings(48, 64, cam["tanfovx"], cam["tanfovy"], torch.tensor([0.1, 0.2, 0.3], device="cuda"),
                                           1.0, gu.to_dev(cam["viewmatrix"]), gu.to_dev(cam["projmatrix"]), 3,
                                           gu.to_dev(cam["campos"]), False, False)
    r = dgr.GaussianRasterizer(raster_settings=rs)
    # all splats behind the camera: nothing visible, image == background on local tiles
    sc = syn.make_scene(64, 64, 48, seed=1)
    sc["means3D"][:, 2] = -5.0
    p = {k: gu.to_dev(v).requires_grad_(True) for k, v in sc.items()}
    m2, rgb, co, radii, depths = r.preprocess_gaussians(p["means3D"], p["scales"], p["rotations"], p["shs"], p["opacities"], {})
    assert (radii == 0).all()
    img, *_ = r.render_gaussians(m2, co, rgb, depths, radii, torch.ones((3, 4), dtype=torch.bool, device="cuda"), None, {})
    assert torch.allclose(img, torch.tensor([0.1, 0.2, 0.3], device="cuda")[:, None, None].expand(3, 48, 64))
    img.sum().backward()
    assert all(float(v.grad.abs().sum()) == 0 for v in p.values())
    # zero splats
    e = lambda *s: torch.zeros(*s, device="cuda")
    m2, rgb, co, radii, depths = r.preprocess_gaussians(e(0, 3), e(0, 3), e(0, 4), e(0, 16, 3), e(0, 1), {})
    img, *_ = r.render_gaussians(m2, co, rgb, depths, radii, None, None, {})
    assert img.shape == (3, 48, 64)


def test_fused_activation_preprocess_matches_torch_activations(o32):
    """gs_preprocess_*_raw == torch activations (exp / normalize / sigmoid / cat) followed by the plain operator."""
    from gs_b200 import ops, pipeline
    cam, sc = case(30003, 320, 200, seed=12)   # ragged tail: 30003 % 128 % 4 != 0 exercises the non-TMA path
    params = pipeline.GaussianParams(sc, "cuda")
    with torch.no_grad():
        params._rotation.mul_(torch.empty(30003, 1, device="cuda").uniform_(0.5, 2.0))   # unnormalised quaternions
    dcam = pipeline.DeviceCamera(cam, "cuda")
    rs = dcam.settings(3)
    a = ops.preprocess_gaussians(params.get_xyz, params.get_scaling, params.get_rotation, params.get_features,
                                 params.get_opacity, rs)
    rng = torch.Generator(device="cuda").manual_seed(0)
    gm = torch.randn(a[0].shape, device="cuda", generator=rng)
    gr = torch.randn(a[1].shape, device="cuda", generator=rng)
    gc = torch.randn(a[2].shape, device="cuda", generator=rng)
    (a[0] * gm).sum().add((a[1] * gr).sum()).add((a[2] * gc).sum()).backward()
    ref_grads = [t.grad.clone() for t in params.raw_parameters()]
    for t in params.raw_parameters():
        t.grad = None
    b = ops.preprocess_gaussians_raw(params._xyz, params._features_dc, params._features_rest, params._scaling,
                                     params._rotation, params._opacity, rs)
    (b[0] * gm).sum().add((b[1] * gr).sum()).add((b[2] * gc).sum()).backward()
    same = (a[3] == b[3]).float().mean().item()
    print(f"[parity] fused activations: radii identical for {same:.6f} of splats")
    assert same >= 0.9999
    keep = gu.npy(a[3] == b[3])
    # exp and sigmoid reproduce torch bit for bit; normalize may differ in the last ulp, which ill-conditioned
    # (needle-like) splats amplify in conic = adj(cov2D)/det -- hence a count-bounded comparison.
    for x, y, name in ((a[0], b[0], "means2D"), (a[1], b[1], "rgb"), (a[2], b[2], "conic_opacity"), (a[4], b[4], "depths")):
        frac, _ = gu.rel_report("fused.out." + name, gu.npy(y)[keep], gu.npy(x)[keep], rtol=1e-4, atol_scale=1e-6)
        assert frac <= 1e-3, name
    assert torch.equal(a[0][torch.as_tensor(keep, device="cuda")], b[0][torch.as_tensor(keep, device="cuda")])
    for t, g, name in zip(params.raw_parameters(), ref_grads, ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity")):
        frac, _ = gu.rel_report("fused." + name, gu.npy(t.grad)[keep], gu.npy(g)[keep], rtol=1e-3, atol_scale=1e-4)
        assert frac <= 1e-3, name


def test_whole_step_parity_fused_path(o32):
    """The Trainer's default (fused activations) step against the oracle, raw-parameter gradients included."""
    from gs_b200 import pipeline
    cam = syn.make_camera(400, 400)
    sc = syn.make_scene(50000, 400, 400)
    gt = syn.make_gt_image(400, 400)
    ref = o32.train_step(sc, cam, gt)
    tr = pipeline.Trainer(sc, [cam], [torch.from_numpy(gt).pin_memory()], torch.device("cuda", 0))
    loss = tr.step(resident=False)
    assert abs(loss - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    p = tr.params
    frac, _ = gu.rel_report("fusedstep.xyz", gu.npy(p._xyz.grad), ref["grads"]["means3D"])
    assert frac <= 5 * OUTLIER_FRAC
    # chain rule through the activations, evaluated in numpy on the oracle's gradients
    g_sc = ref["grads"]["scales"] * sc["scales"]
    frac, _ = gu.rel_report("fusedstep.scaling", gu.npy(p._scaling.grad), g_sc)
    assert frac <= 5 * OUTLIER_FRAC
    op = sc["opacities"]
    frac, _ = gu.rel_report("fusedstep.opacity", gu.npy(p._opacity.grad), ref["grads"]["opacities"] * op * (1 - op))
    assert frac <= 5 * OUTLIER_FRAC
    shg = ref["grads"]["shs"]
    frac, _ = gu.rel_report("fusedstep.f_dc", gu.npy(p._features_dc.grad), shg[:, :1])
    assert frac <= 5 * OUTLIER_FRAC
    frac, _ = gu.rel_report("fusedstep.f_rest", gu.npy(p._features_rest.grad), shg[:, 1:])
    assert frac <= 5 * OUTLIER_FRAC
    q = sc["rotations"]
    gq = ref["grads"]["rotations"]
    g_rot = gq - q * (q * gq).sum(1, keepdims=True)   # |q| = 1
    frac, _ = gu.rel_report("fusedstep.rotation", gu.npy(p._rotation.grad), g_rot)
    assert frac <= 5 * OUTLIER_FRAC


def test_legacy_tile_helpers_match_plain_torch():
    """Rows L3/L4: tile-mask dilation, pixel mask crop, tile gather / scatter and their autograd."""
    import diff_gaussian_rasterization as dgr
    H, W = 150, 211
    ty, tx = 10, 14
    g = torch.Generator(device="cuda").manual_seed(3)
    cl = torch.rand((ty, tx), device="cuda", generator=g) < 0.3
    touched = dgr._C.get_touched_locally(cl, H, W, 1)
    ref = torch.nn.functional.max_pool2d(cl[None, None].float(), 3, 1, 1)[0, 0] > 0
    assert touched.dtype == torch.bool and torch.equal(touched, ref)
    y0, y1, x0, x1 = 16, 112, 32, 160
    pm = dgr._C.get_pixels_compute_locally_and_in_rect(cl, H, W, y0, y1, x0, x1)
    full = cl.repeat_interleave(16, 0).repeat_interleave(16, 1)[:H, :W]
    assert torch.equal(pm, full[y0:y1, x0:x1])
    # tiles inside the rect (tile rows 1..6, cols 2..9), one on the ragged image edge
    pos = torch.tensor([[1, 2], [3, 5], [6, 9], [4, 2]], dtype=torch.int64, device="cuda")
    rect = torch.randn((3, y1 - y0, x1 - x0), device="cuda", generator=g, requires_grad=True)
    tiles = dgr.load_image_tiles_by_pos(rect, pos, H, W, [y0, y1, x0, x1], [1, 7, 2, 10])
    exp = torch.stack([rect[:, (p[0] * 16 - y0):(p[0] * 16 - y0 + 16), (p[1] * 16 - x0):(p[1] * 16 - x0 + 16)] for p in pos.tolist()])
    assert torch.equal(tiles, exp)
    w = torch.randn_like(tiles)
    (tiles * w).sum().backward()
    gref = torch.zeros_like(rect)
    for k, p in enumerate(pos.tolist()):
        gref[:, (p[0] * 16 - y0):(p[0] * 16 - y0 + 16), (p[1] * 16 - x0):(p[1] * 16 - x0 + 16)] += w[k]
    assert torch.allclose(rect.grad, gref)
    t2 = torch.randn((4, 3, 16, 16), device="cuda", generator=g, requires_grad=True)
    merged = dgr.merge_image_tiles_by_pos(pos, t2, H, W, [y0, y1, x0, x1], [1, 7, 2, 10])
    mref = torch.zeros((3, y1 - y0, x1 - x0), device="cuda")
    for k, p in enumerate(pos.tolist()):
        mref[:, (p[0] * 16 - y0):(p[0] * 16 - y0 + 16), (p[1] * 16 - x0):(p[1] * 16 - x0 + 16)] = t2[k].detach()
    assert torch.equal(merged, mref)
    w2 = torch.randn_like(merged)
    (merged * w2).sum().backward()
    assert torch.allclose(t2.grad, torch.stack([w2[:, (p[0] * 16 - y0):(p[0] * 16 - y0 + 16), (p[1] * 16 - x0):(p[1] * 16 - x0 + 16)] for p in pos.tolist()]))


def test_batched_preprocess_equals_per_camera():
    """gs_preprocess_*_batched: slice k == single-camera raw operator (bitwise for the integer-deciding outputs),
    and the accumulated parameter gradients match the sum of the per-camera backward passes."""
    from gs_b200 import ops, pipeline
    W, H, n, B = 320, 200, 20001, 3
    sc = syn.make_scene(n, W, H, seed=31, radius_px=8.0)
    cams = syn.make_batch_cameras(W, H, B)
    params = pipeline.GaussianParams(sc, "cuda")
    dcams = [pipeline.DeviceCamera(c, "cuda") for c in cams]
    settings = [d.settings(3) for d in dcams]
    g = torch.Generator(device="cuda").manual_seed(5)
    gm = torch.randn((B, n, 2), device="cuda", generator=g)
    gr = torch.randn((B, n, 3), device="cuda", generator=g)
    gc = torch.randn((B, n, 4), device="cuda", generator=g)
    outs = [ops.preprocess_gaussians_raw(params._xyz, params._features_dc, params._features_rest, params._scaling,
                                         params._rotation, params._opacity, rs) for rs in settings]
    loss = sum((o[0] * gm[k]).sum() + (o[1] * gr[k]).sum() + (o[2] * gc[k]).sum() for k, o in enumerate(outs))
    loss.backward()
    ref = [t.grad.clone() for t in params.raw_parameters()]
    for t in params.raw_parameters():
        t.grad = None
    bm2, brgb, bco, bradii, bdepths = ops.preprocess_gaussians_batched(
        params._xyz, params._features_dc, params._features_rest, params._scaling, params._rotation, params._opacity,
        ops.pack_cameras(settings), W, H, 3)
    for k, o in enumerate(outs):
        assert torch.equal(bradii[k], o[3]) and torch.equal(bdepths[k], o[4]) and torch.equal(bm2[k], o[0])
        assert torch.equal(bco[k], o[2]) and torch.equal(brgb[k], o[1])
        assert (o[3] > 0).sum() > 1000
    ((bm2 * gm).sum() + (brgb * gr).sum() + (bco * gc).sum()).backward()
    for t, r, name in zip(params.raw_parameters(), ref, ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity")):
        frac, _ = gu.rel_report("batched." + name, gu.npy(t.grad), gu.npy(r))
        assert frac <= OUTLIER_FRAC, name


def _grad_close(a, b, what):
    a, b = a.double(), b.double()
    tol = 2e-5 * b.abs() + 2e-5 * b.abs().mean()      # same pairs, different atomics order
    frac = float(((a - b).abs() > tol).double().mean())
    assert frac <= 1e-4, (what, frac)


def test_batched_render_and_loss_equal_per_camera():
    """gs_render_*_batched / gs_loss_*_batched over three cameras (ragged splat counts; one camera fully local, one a
    strip of tile rows, one with NO local tile) against the single-camera calls: images, loss terms and image gradients
    bit-identical, splat gradients equal up to the order of the atomics."""
    from types import SimpleNamespace
    from gs_b200 import ops
    W, H = 300, 170
    ty, tx = (H + 15) // 16, (W + 15) // 16
    ns = [9000, 4001, 2500]
    bg = torch.tensor([0.1, 0.3, 0.2], device="cuda")
    rs = SimpleNamespace(image_height=H, image_width=W, bg=bg)
    o = Oracle(np.float32)
    pres, masks = [], []
    for k, n in enumerate(ns):
        cam, sc = case(n, W, H, seed=60 + k, radius_px=9.0, yaw=2.0 * k)
        pres.append(o.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam))
        m = torch.zeros((ty, tx), dtype=torch.uint8, device="cuda")
        if k == 0:
            m[:] = 1
        elif k == 1:
            m[3:7] = 1
        masks.append(m)
    rows4 = [(0, H, 0, H), (48, 112, 48, 112), (0, 0, 0, 0)]
    gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=70 + k)).cuda() for k in range(3)]
    strips = [None if r[1] == r[0] else gts[k][:, r[0]:r[1]].contiguous() for k, r in enumerate(rows4)]
    lam = 0.2

    def leaves(k):
        p = pres[k]
        ts = [gu.to_dev(p[q]) for q in ("means2D", "conic_opacity", "rgb")]
        for t in ts:
            t.requires_grad_(True)
        return ts, gu.to_dev(p["depths"]), gu.to_dev(p["radii"])

    # ---- per camera -----------------------------------------------------------------------------------------
    ref_img, ref_terms, ref_grads, ref_dimg = [], [], [], []
    for k in range(3):
        (m2, co, rgb), dep, rad = leaves(k)
        img, *_ = ops.render_gaussians(m2, co, rgb, dep, rad, masks[k], rs)
        img.retain_grad()
        ref_img.append(img.detach().clone())
        if strips[k] is None:
            ref_terms.append(None)
            ref_grads.append(None)
            ref_dimg.append(None)
            continue
        l1, ss = ops.fused_l1_ssim(img, strips[k], rows4[k][0], rows4[k][1])
        ((1 - lam) * l1 + lam * (1 - ss)).backward()
        ref_terms.append((float(l1), float(ss)))
        ref_grads.append((m2.grad.clone(), co.grad.clone(), rgb.grad.clone()))
        ref_dimg.append(img.grad.clone())
    # ---- batched ----------------------------------------------------------------------------------------------
    L = [leaves(k) for k in range(3)]
    cat = [torch.cat([L[k][0][q] for k in range(3)]) for q in range(3)]
    dep, rad = torch.cat([l[1] for l in L]), torch.cat([l[2] for l in L])
    vs = [0, ns[0], ns[0] + ns[1], sum(ns)]
    imgs, stats = ops.render_gaussians_batched(cat[0], cat[1], cat[2], dep, rad, torch.stack(masks).reshape(3, -1), vs, rs)
    imgs.retain_grad()
    out = ops.fused_l1_ssim_batched(imgs, strips, rows4)
    coef = torch.tensor([1 - lam, -lam, 1 - lam, -lam, 0.0, 0.0], device="cuda")
    (torch.dot(out.reshape(-1), coef) + 2 * lam).backward()
    assert stats.shape == (3, 3) and int(stats[2].sum()) == 0 and int(stats[0, 2]) > 0
    for k in range(3):
        assert torch.equal(imgs[k], ref_img[k]), f"image of view {k}"
        if ref_terms[k] is None:
            assert float(out[k].abs().sum()) == 0.0 and float(imgs.grad[k].abs().sum()) == 0.0
            assert float(imgs[k].abs().sum()) == 0.0        # no local tile: all zeros
            for q in range(3):
                assert float(L[k][0][q].grad.abs().sum()) == 0.0
            continue
        assert abs(float(out[k, 0]) - ref_terms[k][0]) <= 1e-6 * abs(ref_terms[k][0])
        assert abs(float(out[k, 1]) - ref_terms[k][1]) <= 1e-6 * abs(ref_terms[k][1])
        assert torch.equal(imgs.grad[k], ref_dimg[k]), f"dL/dimage of view {k}"
        for q, name in enumerate(("means2D", "conic_opacity", "rgb")):
            _grad_close(L[k][0][q].grad, ref_grads[k][q], f"view {k} dL/d{name}")
    print("[parity] batched render + loss == per-camera calls (3 views, ragged, one without local tiles)")


def test_trainer_batched_render_equals_per_camera_loop():
    """Trainer.step (one batched preprocess, render and loss) against a loop of the per-camera operators: same loss, same
    parameter gradients, same screen-space gradients."""
    from gs_b200 import ops, pipeline
    W, H, n, B = 320, 208, 25000, 3
    sc = syn.make_scene(n, W, H, seed=77, radius_px=8.0)
    cams = syn.make_batch_cameras(W, H, B)
    gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=80 + k)).pin_memory() for k in range(B)]
    params = pipeline.GaussianParams(sc, "cuda")
    loss, m2s = None, []
    for k, cam in enumerate(cams):
        rs = pipeline.DeviceCamera(cam, "cuda").settings(params.active_sh_degree)
        m2, rgb, co, radii, depths = ops.preprocess_gaussians_raw(params._xyz, params._features_dc, params._features_rest,
                                                                  params._scaling, params._rotation, params._opacity, rs)
        m2.retain_grad()
        m2s.append(m2)
        image, *_ = ops.render_gaussians(m2, co, rgb, depths, radii, None, rs)
        lk = ops.fused_loss(image, gts[k].cuda(), 0, H, 0.2)
        loss = lk if loss is None else loss + lk
    loss.backward()
    tr = pipeline.Trainer(sc, cams, gts, torch.device("cuda"))
    got = tr.step(resident=False)
    assert abs(got - float(loss)) <= 2e-6 * abs(float(loss))
    for a, p, name in zip(tr.params.raw_parameters(), params.raw_parameters(),
                          ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity")):
        _grad_close(a.grad, p.grad, name)
    _grad_close(tr.means2D.grad, torch.stack([m.grad for m in m2s]), "means2D.grad (densification statistic)")
    assert tr.io_bytes_per_step() == (B * 3 * H * W, 12)   # the GT images in; the loss and ONE count read back, not B


def test_c2_scale_step_against_the_oracle(o32):
    """BASELINE.json configs[1] -- THE bench configuration (2 M Gaussians, 1920x1080, seed 0) -- forward + loss + backward
    through the public operator against the threaded fp32 oracle (tens of seconds of host time)."""
    import diff_gaussian_rasterization as dgr
    from gs_b200 import ops
    W, H, n = 1920, 1080, 2_000_000
    cam = syn.make_camera(W, H)
    sc = syn.make_scene(n, W, H, seed=0)
    gt = syn.make_gt_image(W, H)
    p = {k: gu.to_dev(v).requires_grad_(True) for k, v in sc.items()}
    rs = dgr.GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], torch.zeros(3, device="cuda"), 1.0,
                                           gu.to_dev(cam["viewmatrix"]), gu.to_dev(cam["projmatrix"]), 3,
                                           gu.to_dev(cam["campos"]), False, False)
    r = dgr.GaussianRasterizer(raster_settings=rs)
    cuda_args = {"stats_collector": {}}
    m2, rgb, co, radii, depths = r.preprocess_gaussians(p["means3D"], p["scales"], p["rotations"], p["shs"], p["opacities"], cuda_args)
    m2.retain_grad()
    gy, gx = (H + 15) // 16, (W + 15) // 16
    img, *_ = r.render_gaussians(m2, co, rgb, depths, radii, torch.ones((gy, gx), dtype=torch.bool, device="cuda"), None, cuda_args)
    l1, ss = ops.fused_l1_ssim(img, gu.to_dev(gt), 0, H)
    loss = 0.8 * l1 + 0.2 * (1.0 - ss)
    loss.backward()
    torch.cuda.synchronize()
    ref = o32.train_step(sc, cam, gt)
    assert np.array_equal(gu.npy(radii), ref["pre"]["radii"])                      # every Gaussian's integer radius
    err = np.abs(gu.npy(img.detach()) - ref["fwd"]["image"])
    print(f"[parity] c2: V={int((ref['pre']['radii'] > 0).sum())} R={int(ref['fwd']['R'])} image max_abs_err={err.max():.3e} "
          f"loss {float(loss):.7f} vs {ref['loss']:.7f}")
    # Every pixel within 2e-5 except a handful of hard-threshold flips: a pair whose alpha sits on 1/255 (or whose T sits
    # on 1e-4) is blended by one implementation and skipped by the other (ex2.approx + FMA here, expf without FMA in the
    # oracle); a flip moves a pixel by at most alpha T c <= 4e-3.  The block culling is NOT a source of flips: the same
    # render with GS_DEBUG_NO_BLOCK_CULL is bit-identical.
    from gs_b200 import _lib
    old = _lib.debug_set(_lib.DEBUG_NO_BLOCK_CULL)
    try:
        with torch.no_grad():
            img0, *_ = r.render_gaussians(m2.detach(), co.detach(), rgb.detach(), depths, radii,
                                          torch.ones((gy, gx), dtype=torch.bool, device="cuda"), None, {"stats_collector": {}})
    finally:
        _lib.debug_set(old)
    assert torch.equal(img0, img.detach()), "block culling changed the c2 image"
    n_flip = int((err > 2e-5).sum())
    print(f"[parity] c2: pixels beyond 2e-5: {n_flip} of {err.size} (max {err.max():.3e}); culled == unculled bit for bit")
    assert n_flip <= 20 and err.max() <= 4e-3
    assert abs(float(loss) - ref["loss"]) <= 1e-5 * abs(ref["loss"]), (float(loss), ref["loss"])
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        frac, _ = gu.rel_report("c2." + k, gu.npy(p[k].grad), ref["grads"][k])
        assert frac <= 5 * OUTLIER_FRAC, k
    frac, _ = gu.rel_report("c2.means2D.grad", gu.npy(m2.grad), ref["render_grads"]["means2D"])
    assert frac <= 5 * OUTLIER_FRAC


def test_full_size_properties_config_c2():
    """BASELINE.json configs[1] at full size (2 M Gaussians, 1920x1080): too big for the oracle in a test, so the
    CUDA path is checked through size-independent properties -- sortedness and bookkeeping of the binning, bit-exact
    partition invariance, exact zeros outside local tiles, forward determinism, and linearity of the backward."""
    W, H, n = 1920, 1080, 2_000_000
    cam = syn.make_camera(W, H)
    sc = syn.make_scene(n, W, H, seed=0)
    pre, d, c = gu.preprocess_forward(sc, cam)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    ones = torch.ones(gx * gy, dtype=torch.uint8, device="cuda")
    full = gu.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"], ones, (0, 0, 0))
    V = int((pre["radii"] > 0).sum())
    assert 1_500_000 < V < 1_900_000 and 4_000_000 < full["R"] < 8_000_000
    keys = full["keys"]
    assert bool((keys[1:] >= keys[:-1]).all())                          # (tile, depth) sorted
    rng_ = full["ranges"].to(torch.int64) & 0xffffffff
    assert int((rng_[:, 1] - rng_[:, 0]).sum()) == full["R"]              # ranges tile the list
    tiles = (keys >> 32)
    starts = rng_[:, 0][rng_[:, 1] > rng_[:, 0]]
    assert bool((tiles[starts] == torch.nonzero(rng_[:, 1] > rng_[:, 0]).squeeze(1)).all())
    off = full["offsets"].to(torch.int64) & 0xffffffff
    assert int(off[n - 1]) == full["R"] and bool((off[1:n] >= off[:n - 1]).all())
    img = full["image"]
    assert bool(torch.isfinite(img).all()) and float(img.min()) >= 0.0
    again = gu.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"], ones, (0, 0, 0))
    assert torch.equal(again["image"], img) and torch.equal(again["n_contrib"], full["n_contrib"])   # deterministic
    from gs_b200 import _lib
    old = _lib.debug_set(_lib.DEBUG_NO_BLOCK_CULL)          # the per-block culling never changes a (pixel, splat) decision
    try:
        raw = gu.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"], ones, (0, 0, 0))
    finally:
        _lib.debug_set(old)
    for k in ("image", "final_T", "n_contrib"):
        assert torch.equal(raw[k], full[k]), f"block culling changed {k} at c2 scale"
    del raw
    acc = torch.zeros_like(img)
    Rs = 0
    for lo, hi in ((0, 17), (17, 34), (34, 51), (51, gy)):              # the 4-rank division of SURVEY.md 8a/A8
        cl = torch.zeros((gy, gx), dtype=torch.uint8, device="cuda")
        cl[lo:hi] = 1
        part = gu.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                                 cl.reshape(-1), (0, 0, 0))
        outside = torch.ones((H, W), dtype=torch.bool, device="cuda")
        outside[lo * 16:min(H, hi * 16)] = False
        assert bool((part["image"][:, outside] == 0).all())
        acc += part["image"]
        Rs += part["R"]
    assert Rs == full["R"] and torch.equal(acc, img)
    g = torch.randn((3, H, W), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    b1 = gu.render_backward(full, g)
    b2 = gu.render_backward(full, 2.0 * g)
    for k in ("means2D", "conic_opacity", "rgb"):
        a1, a2 = b1[k], b2[k]
        assert bool(torch.isfinite(a1).all())
        scale = float(a1.abs().mean())
        assert float((a2 - 2.0 * a1).abs().max()) <= 2e-3 * float(a1.abs().max()) + 1e-3 * scale   # linear up to atomics order
        assert bool((a1[pre["radii"] == 0] == 0).all())


def test_needle_splats_survive_block_culling(o32, o64):
    """Adversarial case for the per-block culling: sub-pixel-wide splats hundreds to thousands of pixels long at
    arbitrary angles (conic determinant dominated by cancellation).  The culling must stay conservative: image and
    gradients still match the oracle, which walks every (pixel, splat) pair."""
    W, H, n = 256, 160, 400
    cam = syn.make_camera(W, H, yaw_deg=0.0)
    rng = np.random.default_rng(42)
    sc = syn.make_scene(n, W, H, seed=9, radius_px=6.0)
    sc["means3D"][:, 2] = rng.uniform(3.0, 6.0, n)
    sc["means3D"][:, 0] = rng.uniform(-1.0, 1.0, n)
    sc["means3D"][:, 1] = rng.uniform(-0.6, 0.6, n)
    long_axis = rng.uniform(2.0, 40.0, n)                       # world units: 100 .. 3000 px on screen
    sc["scales"] = np.stack([long_axis, np.full(n, 2e-4), np.full(n, 2e-4)], 1).astype(np.float32)
    ang = rng.uniform(0, np.pi, n)                              # rotate the long axis about the view direction
    sc["rotations"] = np.stack([np.cos(ang / 2), np.zeros(n), np.zeros(n), np.sin(ang / 2)], 1).astype(np.float32)
    sc["opacities"] = rng.uniform(0.05, 0.9, (n, 1)).astype(np.float32)
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    assert (ref["radii"] > 500).sum() > 50
    T = ((H + 15) // 16) * ((W + 15) // 16)
    bg = (0.1, 0.2, 0.3)
    rf = o32.render_forward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], ref["depths"], ref["radii"], np.ones(T, np.uint8), bg)
    f = gu.render_forward(H, W, gu.to_dev(ref["means2D"]), gu.to_dev(ref["conic_opacity"]), gu.to_dev(ref["rgb"]),
                          gu.to_dev(ref["depths"]), gu.to_dev(ref["radii"]), gu.to_dev(np.ones(T, np.uint8)), bg)
    assert np.array_equal(gu.npy(f["ids"]).view(np.uint32), rf["ids"])
    g = np.random.default_rng(1).normal(size=(3, H, W)).astype(np.float32)
    got = gu.render_backward(f, gu.to_dev(g))
    # (1) the cull is conservative: with it switched off the kernels blend exactly the same (pixel, splat) pairs, so
    #     image / final_T / n_contrib are bit-identical and the gradients differ only by atomics order
    from gs_b200 import _lib
    old = _lib.debug_set(_lib.DEBUG_NO_BLOCK_CULL)
    try:
        f0 = gu.render_forward(H, W, gu.to_dev(ref["means2D"]), gu.to_dev(ref["conic_opacity"]), gu.to_dev(ref["rgb"]),
                               gu.to_dev(ref["depths"]), gu.to_dev(ref["radii"]), gu.to_dev(np.ones(T, np.uint8)), bg)
        got0 = gu.render_backward(f0, gu.to_dev(g))
    finally:
        _lib.debug_set(old)
    for k in ("image", "final_T", "n_contrib"):
        assert torch.equal(f[k], f0[k]), f"block culling changed {k}"
    for k in ("means2D", "conic_opacity", "rgb"):
        a, b = got[k].double(), got0[k].double()
        tol = 1e-5 * b.abs() + 1e-5 * b.abs().mean()
        assert float(((a - b).abs() > tol).double().mean()) <= 1e-4, f"block culling changed dL/d{k}"
    # (2) and the result is the oracle's; the exponent of a needle is a difference of ~1e5-sized terms, so fp32
    #     rounding order (FMA in the kernel, none in the oracle) shows up at 1e-3 relative on a few pixels
    img = gu.npy(f["image"])
    err = np.abs(img - rf["image"])
    bad = (err > 1e-3 * np.abs(rf["image"]) + 1e-4).mean()
    print(f"[parity] needles: image max_abs_err={err.max():.3e} outside={bad:.2e} blended/pixel={rf['stats'][2] / (H * W):.1f}")
    assert rf["stats"][2] / (H * W) > 3 and bad <= 1e-2
    rb = o32.render_backward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], bg, rf, g)
    for k in ("means2D", "conic_opacity", "rgb"):
        frac, _ = gu.rel_report("needles.bwd." + k, gu.npy(got[k]), rb[k], rtol=1e-2, atol_scale=1e-2)
        assert frac <= 2e-2, k
    # (3) how ill-conditioned this input is: the SAME fp32 inputs through the fp64 oracle.  The exponent of a needle is a
    #     difference of ~1e5-sized products, so a pixel's alpha can be anything within a factor of e^(1e5 * 2^-24) -- the
    #     fp32 oracle is as far from the fp64 result as the kernel is; neither is "the" answer at those pixels.
    a64 = [x.astype(np.float64) for x in (ref["means2D"], ref["conic_opacity"], ref["rgb"], ref["depths"])]
    rf64 = o64.render_forward(H, W, a64[0], a64[1], a64[2], a64[3], ref["radii"], np.ones(T, np.uint8), bg)
    e_k, e_o = np.abs(img - rf64["image"]), np.abs(rf["image"] - rf64["image"])
    bad_k, bad_o = (e_k > 1e-3 * np.abs(rf64["image"]) + 1e-4).mean(), (e_o > 1e-3 * np.abs(rf64["image"]) + 1e-4).mean()
    print(f"[parity] needles vs the fp64 oracle: kernel image max_abs_err={e_k.max():.3e} outside={bad_k:.2e} | fp32 oracle "
          f"max_abs_err={e_o.max():.3e} outside={bad_o:.2e}")
    assert bad_k <= 2.0 * bad_o + 1e-3


@pytest.mark.parametrize("shape", ["ordinary", "anisotropic"])
def test_block_cull_is_invisible(o32, shape):
    """The row-band culling of the blend kernels (ellipse_bands) must not change a single (pixel, splat) decision: with
    GS_DEBUG_NO_BLOCK_CULL the forward produces the same image / final_T / n_contrib bit for bit, the backward the same
    gradients up to the order of the atomics -- on ordinary splats and on strongly anisotropic, rotated ones (the case
    the band extents cull hardest: 60 % of the bounding-box candidates)."""
    from gs_b200 import _lib
    W, H = 400, 240
    cam = syn.make_camera(W, H)
    sc = syn.make_scene(40_000, W, H, seed=11, radius_px=6.0 if shape == "ordinary" else 5.0)
    if shape == "anisotropic":
        sc["scales"][:, 0] *= 8.0
        sc["scales"][:, 1] /= 8.0
    ref = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    bg = (0.1, 0.2, 0.3)
    args = [gu.to_dev(ref[k]) for k in ("means2D", "conic_opacity", "rgb", "depths", "radii")]
    g = gu.to_dev(np.random.default_rng(1).normal(size=(3, H, W)).astype(np.float32))
    f = gu.render_forward(H, W, *args, gu.to_dev(np.ones(T, np.uint8)), bg)
    got = gu.render_backward(f, g)
    old = _lib.debug_set(_lib.DEBUG_NO_BLOCK_CULL)
    try:
        f0 = gu.render_forward(H, W, *args, gu.to_dev(np.ones(T, np.uint8)), bg)
        got0 = gu.render_backward(f0, g)
    finally:
        _lib.debug_set(old)
    for k in ("image", "final_T", "n_contrib"):
        assert torch.equal(f[k], f0[k]), f"block culling changed {k}"
    for k in ("means2D", "conic_opacity", "rgb"):
        a, b = got[k].double(), got0[k].double()
        tol = 1e-5 * b.abs() + 1e-5 * b.abs().mean()
        assert float(((a - b).abs() > tol).double().mean()) <= 1e-4, f"block culling changed dL/d{k}"


def test_fused_loss_node_equals_the_two_term_form():
    """ops.fused_loss (one autograd node) == (1 - lambda) Ll1 + lambda (1 - ssim) built from ops.fused_l1_ssim, value and
    image gradient, on a strip with a counted sub-window."""
    from gs_b200 import ops
    H, W, lam = 96, 160, 0.2
    g = torch.Generator(device="cuda").manual_seed(5)
    gt = torch.randint(0, 256, (3, 48, W), dtype=torch.uint8, device="cuda", generator=g)
    x1 = torch.rand((3, H, W), device="cuda", generator=g).requires_grad_(True)
    x2 = x1.detach().clone().requires_grad_(True)
    l1, ss = ops.fused_l1_ssim(x1, gt, 16, 64, 21, 59)
    a = (1.0 - lam) * l1 + lam * (1.0 - ss)
    b = ops.fused_loss(x2, gt, 16, 64, lam, 21, 59)
    (3.0 * a).backward()
    (3.0 * b).backward()
    assert abs(float(a) - float(b)) <= 1e-6 * abs(float(a))
    assert torch.allclose(x1.grad, x2.grad, rtol=1e-5, atol=1e-9)
