"""CPU tests of the oracle itself: analytic micro-cases, autograd / finite-difference pins of the
hand-written backward, partition invariance (SURVEY.md section 4 pyramid (i)-(iv))."""
import numpy as np
import pytest
import torch

import proj_cases
import torch_ref
from gs_b200 import synthetic as syn
from oracle.oracle import Oracle


@pytest.fixture(scope="module")
def o64():
    return Oracle(np.float64)


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32)


def small_case(n=400, W=80, H=56, seed=3, radius_px=9.0):
    cam = syn.make_camera(W, H, yaw_deg=7.0)
    sc = syn.make_scene(n, W, H, seed=seed, radius_px=radius_px)
    return cam, sc


def test_block_xy(o32):
    assert o32.get_block_xy() == (16, 16, 256)


def test_single_isotropic_gaussian_closed_form(o64):
    """One isotropic Gaussian on the optical axis: alpha(x,y) = o*exp(-r^2 / (2 (sigma_px^2+0.3)))."""
    W = H = 64
    cam = syn.make_camera(W, H, yaw_deg=0.0, sh_degree=0)
    z, s, op = 5.0, 0.05, 0.8
    sc = dict(means3D=np.array([[0.0, 0.0, z]]), scales=np.full((1, 3), s), rotations=np.array([[1.0, 0, 0, 0]]),
              opacities=np.array([[op]]), shs=np.zeros((1, 16, 3)))
    sc["shs"][0, 0] = (1.0 - 0.5) / 0.28209479177387814, 0.0, (0.25 - 0.5) / 0.28209479177387814
    pre = o64.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    fx = W / (2 * cam["tanfovx"])
    var = (s * fx / z) ** 2 + 0.3
    assert pre["radii"][0] == int(np.ceil(3 * np.sqrt(var)))
    np.testing.assert_allclose(pre["means2D"][0], [(W - 1) / 2, (H - 1) / 2], atol=1e-4)
    np.testing.assert_allclose(pre["conic_opacity"][0], [1 / var, 0, 1 / var, op], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(pre["rgb"][0], [1.0, 0.5, 0.25], rtol=1e-9)
    fwd = o64.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                             np.ones(16, np.uint8), (0.1, 0.2, 0.3))
    ys, xs = np.mgrid[0:H, 0:W]
    r2 = (xs - (W - 1) / 2) ** 2 + (ys - (H - 1) / 2) ** 2
    alpha = np.minimum(0.99, op * np.exp(-0.5 * r2 / var))
    alpha[alpha < 1 / 255] = 0
    # only the tiles the 3-sigma rect touches hold the Gaussian
    touched = np.zeros((H, W), bool)
    for t in range(16):
        if fwd["ranges"][t, 1] > fwd["ranges"][t, 0]:
            touched[(t // 4) * 16:(t // 4) * 16 + 16, (t % 4) * 16:(t % 4) * 16 + 16] = True
    alpha[~touched] = 0
    expect = np.stack([alpha * c + (1 - alpha) * b for c, b in zip([1.0, 0.5, 0.25], [0.1, 0.2, 0.3])])
    np.testing.assert_allclose(fwd["image"], expect, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(fwd["final_T"], 1 - alpha, rtol=1e-9, atol=1e-12)


def test_backward_matches_torch_autograd(o64):
    """Whole chain: d(sum(image*w)) / d(xyz, scale, rot, sh, opacity): oracle backward == autograd."""
    cam, sc = small_case()
    H, W = cam["image_height"], cam["image_width"]
    bg = (0.3, 0.1, 0.6)
    pre = o64.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    fwd = o64.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                             np.ones(T, np.uint8), bg)
    assert fwd["R"] > 1000 and (fwd["final_T"] < 0.5).mean() > 0.2
    wimg = np.random.default_rng(0).normal(size=(3, H, W))
    rb = o64.render_backward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], bg, fwd, wimg)
    pb = o64.preprocess_backward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam,
                                 pre["radii"], pre["clamped"], rb["means2D"], rb["conic_opacity"], rb["rgb"])
    tp = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in sc.items()}
    m2, co, col = torch_ref.preprocess(tp["means3D"], tp["scales"], tp["rotations"], tp["shs"], tp["opacities"], cam)
    m2.retain_grad(); co.retain_grad(); col.retain_grad()
    np.testing.assert_allclose(m2.detach().numpy()[pre["radii"] > 0], pre["means2D"][pre["radii"] > 0], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(co.detach().numpy()[pre["radii"] > 0], pre["conic_opacity"][pre["radii"] > 0], rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(col.detach().numpy()[pre["radii"] > 0], pre["rgb"][pre["radii"] > 0], rtol=1e-9, atol=1e-12)
    img = torch_ref.render(m2, co, col, bg, H, W, fwd)
    np.testing.assert_allclose(img.detach().numpy(), fwd["image"], rtol=1e-9, atol=1e-12)
    (img * torch.tensor(wimg)).sum().backward()
    # operator-level gradients: means2D.grad is per NDC unit = pixel gradient * (W/2, H/2)
    np.testing.assert_allclose(rb["means2D"], m2.grad.numpy() * np.array([W / 2, H / 2]), rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(rb["conic_opacity"], co.grad.numpy(), rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(rb["rgb"], col.grad.numpy(), rtol=1e-7, atol=1e-10)
    for k_o, k_t in (("means3D", "means3D"), ("scales", "scales"), ("rotations", "rotations"), ("shs", "shs"),
                     ("opacities", "opacities")):
        g = tp[k_t].grad.numpy()
        assert np.abs(g).max() > 0
        np.testing.assert_allclose(pb[k_o], g, rtol=2e-6, atol=1e-9 * np.abs(g).max(), err_msg=k_o)


def test_guard_band_clamp_is_straight_through(o64):
    """Gaussians outside the 1.3x guard band still project; their clamped ratio carries no gradient.  Every camera x SH
    degree 0..3 x scale_modifier {1, 0.6}.  "yaw": the synthetic camera at the origin with splats beyond the band on x.
    0..5: the posed cameras of cameras.npz (translated, re-centred, fx != fy) with the region mix of proj_cases (interior,
    guard band on x / y / both and at its edge, both sides of the near plane, behind, off-screen, flat, sub-pixel,
    negative DC)."""
    for camera in ["yaw"] + list(range(proj_cases.N_GOLDEN)):
        for deg in range(4):
            for mod in (1.0, 0.6):
                _guard_band_case(o64, camera, deg, mod)


def _guard_band_case(o64, camera, deg, mod):
    case = f"camera {camera}, degree {deg}, scale_modifier {mod}"
    rng = np.random.default_rng(5)
    if camera == "yaw":
        cam = syn.make_camera(96, 64, sh_degree=deg)
        n = 64
        z = rng.uniform(2, 4, n)
        x = rng.choice([-1.0, 1.0], n) * rng.uniform(1.32, 1.5, n) * z * cam["tanfovx"]
        sc = dict(means3D=np.stack([x, rng.uniform(-.2, .2, n) * z, z], 1), scales=np.exp(rng.normal(-0.5, 0.3, (n, 3))),
                  rotations=syn.make_scene(n, 96, 64, seed=1)["rotations"].astype(np.float64),
                  opacities=rng.uniform(0.3, 0.9, (n, 1)), shs=rng.normal(0, 0.5, (n, 16, 3)))
    else:
        cam = proj_cases.golden_camera(camera, 96, 64, sh_degree=deg)
        n = 400
        sc, _ = proj_cases.region_scene(cam, n, seed=10 * camera + deg)
        sc = {k: v.astype(np.float64) for k, v in sc.items()}
    W, H = cam["image_width"], cam["image_height"]
    pre = o64.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam,
                                 scale_modifier=mod)
    vis_np = pre["radii"] > 0
    tx, ty, tz = (np.asarray(c, np.float64) for c in proj_cases.view_coords32(cam, sc["means3D"]))
    beyond = vis_np & ((np.abs(tx / tz) > 1.3 * cam["tanfovx"]) | (np.abs(ty / tz) > 1.3 * cam["tanfovy"]))
    assert vis_np.sum() > 10 and beyond.sum() >= 3, case
    gm, gc, gr = rng.normal(size=(n, 2)), rng.normal(size=(n, 4)), rng.normal(size=(n, 3))
    pb = o64.preprocess_backward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam,
                                 pre["radii"], pre["clamped"], gm, gc, gr, scale_modifier=mod)
    tp = {k: torch.tensor(v, requires_grad=True) for k, v in sc.items()}
    m2, co, col = torch_ref.preprocess(tp["means3D"], tp["scales"], tp["rotations"], tp["shs"], tp["opacities"], cam,
                                       scale_modifier=mod)
    vis = torch.tensor(vis_np)
    ndc_scale = torch.tensor([2.0 / W, 2.0 / H], dtype=torch.float64)
    L = ((m2 * ndc_scale * torch.tensor(gm)).sum(1) + (co * torch.tensor(gc)).sum(1) + (col * torch.tensor(gr)).sum(1))
    L[vis].sum().backward()
    for k in ("means3D", "scales", "rotations", "shs", "opacities"):
        g = tp[k].grad.numpy()
        assert np.abs(g).max() > 0, (k, case)
        np.testing.assert_allclose(pb[k], g, rtol=1e-9, atol=1e-12 * np.abs(g).max(), err_msg=f"{k}, {case}")
    nc = (deg + 1) ** 2
    assert (pb["shs"][:, nc:] == 0).all(), case


def test_finite_differences_whole_step(o64):
    """Central differences of the scalar training loss wrt a few parameters (fp64 oracle)."""
    cam, sc = small_case(n=150, W=48, H=32, seed=11, radius_px=8.0)
    sc = {k: v.astype(np.float64) for k, v in sc.items()}
    gt = syn.make_gt_image(48, 32)
    base = o64.train_step(sc, cam, gt, bg=(0.2, 0.4, 0.1))
    rng = np.random.default_rng(0)
    vis = np.nonzero(base["pre"]["radii"] > 0)[0]
    checked = 0
    for name, gname in (("means3D", "means3D"), ("scales", "scales"), ("rotations", "rotations"),
                        ("opacities", "opacities"), ("shs", "shs")):
        for _ in range(6):
            i = rng.choice(vis)
            idx = (i,) + tuple(rng.integers(0, s) for s in sc[name].shape[1:])
            if name == "shs" and idx[1] > 15:
                continue
            h = 1e-6 * max(1.0, abs(sc[name][idx]))
            vals = []
            for sgn in (+1, -1):
                p = {k: v.copy() for k, v in sc.items()}
                p[name][idx] += sgn * h
                vals.append(o64.train_step(p, cam, gt, bg=(0.2, 0.4, 0.1))["loss"])
            fd = (vals[0] - vals[1]) / (2 * h)
            an = base["grads"][gname][idx]
            if abs(an) < 1e-9:
                continue
            # discrete decisions (alpha threshold, termination) make the loss piecewise smooth:
            # accept when analytic and numeric agree to 1e-3 relative
            assert abs(fd - an) <= 2e-3 * max(abs(an), abs(fd)) + 1e-9, (name, idx, fd, an)
            checked += 1
    assert checked >= 15


def test_partition_invariance(o32):
    """Rendering W tile-row strips and summing equals the full render bit for bit; non-local tiles stay 0
    (/root/reference/train_internal.py:466-469 relies on it)."""
    cam, sc = small_case(n=2000, W=200, H=120, seed=7, radius_px=7.0)
    H, W = 120, 200
    gx, gy = (W + 15) // 16, (H + 15) // 16
    pre = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    full = o32.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                              np.ones(gx * gy, np.uint8), (0, 0, 0))
    acc = np.zeros_like(full["image"])
    Rsum = 0
    for lo, hi in ((0, 2), (2, 3), (3, 8)):
        cl = np.zeros((gy, gx), np.uint8)
        cl[lo:hi] = 1
        part = o32.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                                  cl.reshape(-1), (0, 0, 0))
        outside = np.ones((H, W), bool)
        outside[lo * 16:min(H, hi * 16)] = False
        assert (part["image"][:, outside] == 0).all()
        acc += part["image"]
        Rsum += part["R"]
    assert Rsum == full["R"]
    assert np.array_equal(acc, full["image"])


def test_local2j_matches_tile_lists(o32):
    """get_local2j_ids_bool[i][j] <=> Gaussian i appears in some tile list of strip j."""
    cam, sc = small_case(n=1500, W=200, H=120, seed=9, radius_px=10.0)
    H, W = 120, 200
    gx, gy = (W + 15) // 16, (H + 15) // 16
    pre = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    div = [0, 3, 4, 8]
    got = o32.get_local2j_ids_bool(H, W, 3, pre["means2D"], pre["radii"], np.array(div) * gx)
    for j in range(3):
        cl = np.zeros((gy, gx), np.uint8)
        cl[div[j]:div[j + 1]] = 1
        part = o32.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                                  cl.reshape(-1), (0, 0, 0))
        expect = np.zeros(1500, bool)
        expect[part["ids"]] = True
        assert np.array_equal(got[:, j], expect)
    rects = np.array([[0, 4, 0, 6], [0, 4, 6, gx], [4, gy, 0, gx]], np.int32)
    got6 = o32.get_local2j_ids_bool_rects(H, W, 3, pre["means2D"], pre["radii"], rects)
    for j in range(3):
        cl = np.zeros((gy, gx), np.uint8)
        cl[rects[j, 0]:rects[j, 1], rects[j, 2]:rects[j, 3]] = 1
        part = o32.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                                  cl.reshape(-1), (0, 0, 0))
        expect = np.zeros(1500, bool)
        expect[part["ids"]] = True
        assert np.array_equal(got6[:, j], expect)


def test_sorted_keys_properties(o32):
    cam, sc = small_case(n=3000, W=160, H=96, seed=2)
    pre = o32.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    fwd = o32.render_forward(96, 160, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                             np.ones(60, np.uint8), (0, 0, 0))
    k = fwd["keys"]
    assert (k[1:] >= k[:-1]).all()
    assert fwd["R"] == int(fwd["tiles_touched"].sum()) == int(fwd["offsets"][-1])
    tiles = (k >> np.uint64(32)).astype(np.int64)
    for t in range(60):
        b, e = fwd["ranges"][t]
        assert (tiles[b:e] == t).all() and e - b == (tiles == t).sum()
    d = pre["depths"][fwd["ids"]].view(np.uint32)
    assert np.array_equal(d, (k & np.uint64(0xFFFFFFFF)).astype(np.uint32))


def test_loss_matches_torch(o64):
    rng = np.random.default_rng(4)
    img, gt = rng.uniform(0, 1, (3, 37, 53)), rng.uniform(0, 1, (3, 37, 53))
    l1, ss, grad = o64.loss(img, gt, 80 * 53, 0.2)
    x = torch.tensor(img, requires_grad=True)
    loss, tl1, tss = torch_ref.ssim_l1_loss(x, torch.tensor(gt), 80 * 53, 0.2)
    loss.backward()
    # the reference's 11x11 window is the fp32-rounded outer product; the separable form differs by ~1e-7 relative
    assert abs(l1 - float(tl1.detach())) < 1e-12 and abs(ss - float(tss.detach())) < 5e-6 * abs(ss)
    np.testing.assert_allclose(grad, x.grad.numpy(), rtol=1e-5, atol=1e-10)


def test_f32_oracle_close_to_f64(o32, o64):
    cam, sc = small_case(n=3000, W=160, H=96, seed=2)
    gt = syn.make_gt_image(160, 96)
    a = o32.train_step(sc, cam, gt)
    b = o64.train_step({k: v.astype(np.float64) for k, v in sc.items()}, cam, gt)
    assert np.array_equal(a["pre"]["radii"], b["pre"]["radii"])
    same = np.array_equal(a["fwd"]["ids"], b["fwd"]["ids"])
    assert same
    err = np.abs(a["fwd"]["image"] - b["fwd"]["image"])
    assert np.quantile(err, 0.999) < 2e-5
    assert abs(a["loss"] - b["loss"]) < 1e-5
