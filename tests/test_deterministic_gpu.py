"""-m gpu: the deterministic render and loss (gs_render_forward_det / gs_render_backward_det / gs_loss_forward*_det and
the operators' deterministic flag).

  * the deterministic forward is the default forward, bit for bit, in every output;
  * the deterministic backward gives the same bits on every call, writes every gradient row (culled splats read exactly
    0), does not depend on splat ids or scheduling (a permuted scene gives the permuted gradients), and is as close to
    the fp64 oracle as the atomic backward;
  * the deterministic loss gives the same bits on every call, within 1 ulp of the atomic sums;
  * six training steps with densification give the same bits twice, and a model stored at SH degree 0 / 1 / 2 the same
    bits as its zero-padded degree-3 run -- the comparison test_sh_storage_gpu.py can only make to a tolerance;
  * the drop-in operators follow torch.use_deterministic_algorithms.
Every comparison runs each call once or twice; nothing is repeated to look for a difference."""
import numpy as np
import pytest
import torch

import blend_cases as bc
import gpu_util as gu
import proj_cases as pc
from det_util import (assert_forward_unchanged, backward, bits_equal, case_view, dl_like, empty_view, forward,
                      projected_view, whole_image_scene)
from gs_b200 import _lib, densify, ops, pipeline
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

OUTLIER_FRAC = 2e-4   # test_gpu_parity's threshold-flip bar


@pytest.fixture
def det_flag():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.fixture(scope="module")
def c2():
    """The c2 workload's size: 2 M Gaussians at 1920x1080, projected once."""
    cfg = syn.CONFIGS["c2"]
    W, H = cfg["width"], cfg["height"]
    sc = syn.make_scene(cfg["n"], W, H, seed=0)
    return H, W, [projected_view(sc, syn.make_camera(W, H, yaw_deg=y)) for y in (0.0, 2.0, -3.0)]


def c1_views():
    cfg = syn.CONFIGS["c1"]
    W, H = cfg["width"], cfg["height"]
    sc = syn.make_scene(cfg["n"], W, H, seed=1)
    return H, W, [projected_view(sc, syn.make_camera(W, H, yaw_deg=y)) for y in (0.0, 4.0, -2.0)]


# ---------------------------------------------------------------------------------------------------------------------
# forward: bit-identical to the default
# ---------------------------------------------------------------------------------------------------------------------
def test_forward_unchanged_blend_cases():
    for c in bc.all_cases():
        assert_forward_unchanged([case_view(c)], c["H"], c["W"], c["bg"], c["name"])


def test_forward_unchanged_projected_c1_and_batched_with_an_empty_view():
    H, W, views = c1_views()
    assert_forward_unchanged(views[:1], H, W, (0.1, 0.2, 0.3), "c1")
    assert_forward_unchanged([views[0], empty_view(H, W), views[1], views[2]], H, W, (0.0, 0.0, 0.0), "c1.B4")


def test_forward_unchanged_c2(c2):
    H, W, views = c2
    _, b = assert_forward_unchanged(views[:1], H, W, (0.0, 0.0, 0.0), "c2")
    print(f"[det] c2 forward bit-identical, R = {b['R']}")


# ---------------------------------------------------------------------------------------------------------------------
# backward: repeatable, complete, independent of splat ids, accurate
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batched", [False, True], ids=["single", "B4"])
def test_backward_repeatable_c2(c2, batched):
    H, W, views = c2
    vs = [views[0], empty_view(H, W), views[1], views[2]] if batched else views[:1]
    f = forward(vs, H, W, (0.0, 0.0, 0.0), det=True)
    dL = dl_like(f, 3)
    g1, g2 = backward(f, dL, det=True), backward(f, dL, det=True)
    for k in g1:
        assert bool(torch.isfinite(g1[k]).all()), k
        assert bits_equal(g1[k], g2[k]), k
    ref = backward(forward(vs, H, W, (0.0, 0.0, 0.0), det=False), dL, det=False)
    for k in g1:
        frac, _ = gu.rel_report(f"det.c2.{'B4' if batched else '1'}.{k}", gu.npy(g1[k]), gu.npy(ref[k]))
        assert frac <= 5 * OUTLIER_FRAC, k


def test_backward_whole_image_splat_and_culled_rows():
    c = whole_image_scene()
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True)
    dL = dl_like(f, 5)
    g1, g2 = backward(f, dL, det=True), backward(f, dL, det=True)
    culled = torch.from_numpy(c["label"] == "culled").to(gu.DEV)
    for k in g1:
        assert bits_equal(g1[k], g2[k]), k
        assert bool((g1[k][culled] == 0).all()) and not bool(torch.signbit(g1[k][culled]).any()), k
        assert bool(torch.isfinite(g1[k]).all()), k
    assert bool((g1["rgb"][0] != 0).all())        # the whole-image splat received its sums
    ref = backward(forward([case_view(c)], c["H"], c["W"], c["bg"], det=False), dL, det=False)
    for k in g1:
        frac, _ = gu.rel_report(f"det.whole.{k}", gu.npy(g1[k]), gu.npy(ref[k]))
        assert frac <= 5 * OUTLIER_FRAC, k


def test_backward_permutation_invariance():
    H, W, views = c1_views()
    v = views[0]
    # fp32 depths of a random scene collide (ties keep index order, which a permutation changes): the later splats of
    # each tie are culled, so the depth order of every splat with a tile is unique
    radii = v[4].clone()
    vis = (radii > 0).nonzero().squeeze(1)
    d, o = torch.sort(v[3][vis], stable=True)
    tie = torch.zeros_like(d, dtype=torch.bool)
    tie[1:] = d[1:] == d[:-1]
    radii[vis[o[tie]]] = 0
    v = v[:4] + (radii, v[5])
    vis = radii > 0
    assert torch.unique(v[3][vis]).numel() == int(vis.sum()) > 40000
    f = forward([v], H, W, (0.3, 0.3, 0.3), det=True)
    dL = dl_like(f, 7)
    g = backward(f, dL, det=True)
    perm = torch.randperm(v[0].shape[0], generator=torch.Generator().manual_seed(1)).to(gu.DEV)
    vp = tuple(t[perm].contiguous() for t in v[:5]) + (v[5],)
    fp = forward([vp], H, W, (0.3, 0.3, 0.3), det=True)
    assert bits_equal(fp["image"], f["image"])
    gp = backward(fp, dL, det=True)
    for k in g:
        back = torch.empty_like(gp[k])
        back[perm] = gp[k]
        assert bits_equal(back, g[k]), k


@pytest.fixture(scope="module")
def o64():
    return Oracle(np.float64, threads=max(1, (__import__("os").cpu_count() or 8) // 2))


@pytest.mark.parametrize("n,W,H,rad,bg", [(20000, 320, 200, 7.0, (0.0, 0.0, 0.0)), (3000, 96, 64, 16.0, (0.3, 0.1, 0.7))])
def test_backward_accuracy_vs_fp64_oracle(o64, n, W, H, rad, bg):
    """As close to the fp64 oracle as the atomic backward (test_gpu_parity's bar, or the atomic backward's own distance
    where fp64 takes a different branch at a threshold), and within the same bar of the atomic backward."""
    cam = syn.make_camera(W, H, yaw_deg=3.0)
    sc = syn.make_scene(n, W, H, seed=3, radius_px=rad)
    ref = o64.preprocess_forward(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["opacities"], cam)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    cl = np.ones(T, np.uint8)
    rf = o64.render_forward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], ref["depths"], ref["radii"], cl, bg)
    g = np.random.default_rng(2).normal(size=(3, H, W))
    rb = o64.render_backward(H, W, ref["means2D"], ref["conic_opacity"], ref["rgb"], bg, rf, g)
    view = tuple(gu.to_dev(np.asarray(ref[k], np.float32)) for k in ("means2D", "conic_opacity", "rgb", "depths")) + \
        (gu.to_dev(ref["radii"].astype(np.int32)), gu.to_dev(cl))
    dL = gu.to_dev(g.astype(np.float32)).unsqueeze(0)
    det = backward(forward([view], H, W, bg, det=True), dL, det=True)
    atomic = backward(forward([view], H, W, bg, det=False), dL, det=False)
    for k in ("means2D", "conic_opacity", "rgb"):
        fd, _ = gu.rel_report(f"det.vs_fp64.{k}", gu.npy(det[k]), rb[k])
        fa, _ = gu.rel_report(f"atomic.vs_fp64.{k}", gu.npy(atomic[k]), rb[k])
        assert fd <= max(5 * OUTLIER_FRAC, 2 * fa), k
        fx, _ = gu.rel_report(f"det.vs_atomic.{k}", gu.npy(det[k]), gu.npy(atomic[k]))
        assert fx <= 5 * OUTLIER_FRAC, k


def test_refusals():
    """No deterministic form of the tile-parallel backward: a forward made without the segment workspace, or the debug
    tile kernel, is refused -- not run."""
    c = bc.all_cases()[0]
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True, seg=False)
    dL = dl_like(f, 1)
    assert f["R"] > 0
    with pytest.raises(_lib.GsError, match="segment workspace"):
        backward(f, dL, det=True)
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True)
    prev = _lib.debug_set(_lib.DEBUG_BWD_TILE)
    try:
        with pytest.raises(_lib.GsError, match="GS_DEBUG_BWD_TILE"):
            backward(f, dL, det=True)
    finally:
        _lib.debug_set(prev)


# ---------------------------------------------------------------------------------------------------------------------
# loss
# ---------------------------------------------------------------------------------------------------------------------
def _ulp_close(a, b):
    a, b = gu.npy(a).astype(np.float32), gu.npy(b).astype(np.float32)
    return bool((np.abs(a.astype(np.float64) - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b)))).all())


def test_loss_repeatable_and_within_one_ulp():
    H, W = 1080, 1920
    g = torch.Generator(device=gu.DEV).manual_seed(4)
    img = torch.rand((4, 3, H, W), device=gu.DEV, generator=g)
    gt = (torch.rand((3, H, W), device=gu.DEV, generator=g) * 255).to(torch.uint8)
    one = [torch.stack(ops.fused_l1_ssim(img[0], gt[:, 100:900].contiguous(), 100, 900, deterministic=d))
           for d in (True, True, False)]
    assert bits_equal(one[0], one[1])
    assert _ulp_close(one[0], one[2]), (one[0], one[2])
    rows4 = [(0, H, 0, H), (0, 0, 0, 0), (37, 600, 42, 590), (700, H, 700, H)]
    gts = [None if r[1] == r[0] else gt[:, r[0]:r[1]].contiguous() for r in rows4]
    bat = [ops.fused_l1_ssim_batched(img, gts, rows4, deterministic=d) for d in (True, True, False)]
    assert bits_equal(bat[0], bat[1])
    assert _ulp_close(bat[0], bat[2]), (bat[0], bat[2])
    assert bool((bat[0][1] == 0).all())
    lo = [ops.fused_loss(img[0], gt, 0, H, 0.2, deterministic=d) for d in (True, True)]
    assert bits_equal(lo[0], lo[1])


# ---------------------------------------------------------------------------------------------------------------------
# training runs: six Trainer.steps + FusedAdam + one densification
# ---------------------------------------------------------------------------------------------------------------------
TW, TH = 256, 192
SCHEDULE = (0, 0, 1, 2, 3, 3)
DENSIFY_AFTER = 3


def training_run(sc, D_max, one_view, noise, top):
    cams = [pc.golden_camera(5, TW, TH, uid=0), pc.golden_camera(4, TW, TH, uid=1)]
    gts = [torch.from_numpy(pc.syn.make_gt_image(TW, TH, seed=5 + k)).pin_memory() for k in range(2)]
    tr = pipeline.Trainer(sc, cams, gts, torch.device("cuda", 0), max_sh_degree=D_max, deterministic=True)
    opt = FusedAdam(tr.optimizer_groups(), lr=0.0, eps=1e-15)
    losses, counts = [], None
    for it, deg in enumerate(SCHEDULE):
        tr.params.active_sh_degree = min(deg, top)
        losses.append(tr.step(views=[it % 2] if one_view else None, resident=False))
        opt.step(grad_scale=1.0 if one_view else 0.5)
        if it == DENSIFY_AFTER:       # statistics and thresholds from this run's own gradients
            p = tr.params
            accum = p._xyz.grad.norm(dim=1, keepdim=True)
            extent = float(torch.exp(p._scaling.detach()).max(dim=1).values.median()) / 0.01
            res = densify.densify_and_prune(opt, accum, torch.ones_like(accum), float(torch.quantile(accum, 0.8)), 0.005,
                                            extent, 0.01, 0, noise=noise)
            tr.adopt_parameters(res)
            counts = res["counts"]
    state = {}
    for g in opt.param_groups:
        prm = g["params"][0]
        st = opt.state[prm]
        state[g["name"]] = (prm.detach(), st["exp_avg"], st["exp_avg_sq"])
    return losses, counts, state


def _scene(seed):
    cam = pc.golden_camera(5, TW, TH)
    sc, _ = pc.region_scene(cam, 30000, seed=seed, mix=pc.MILD)
    return sc


def test_training_run_is_bit_identical_twice():
    sc = _scene(91)
    noise = torch.randn((2 * 30000, 3), generator=torch.Generator().manual_seed(5)).to(gu.DEV)
    l1, c1, s1 = training_run(sc, 3, False, noise, 3)
    l2, c2_, s2 = training_run(sc, 3, False, noise, 3)
    print(f"[det] losses {l1}")
    assert l1 == l2 and c1 == c2_ and c1[1] > 0 and c1[3] > 0
    for name in s1:
        for q in range(3):
            assert bits_equal(s1[name][q], s2[name][q]), (name, q)


@pytest.mark.parametrize("one_view", [False, True], ids=["fused_batched", "one_view"])
@pytest.mark.parametrize("D_max", [0, 1, 2])
def test_training_run_equals_the_padded_run_bit_for_bit(D_max, one_view):
    """What test_sh_storage_gpu.test_training_run_equals_the_padded_run checks to a tolerance, with deterministic=True
    bit for bit over all six steps: losses, densify counts, parameters and both Adam moments."""
    K = (D_max + 1) ** 2
    sc = _scene(77 + D_max)
    padded = dict(sc, shs=sc["shs"].copy())
    padded["shs"][:, K:] = 0.0
    stored = dict(padded, shs=np.ascontiguousarray(padded["shs"][:, :K]))
    noise = torch.randn((2 * 30000, 3), generator=torch.Generator().manual_seed(D_max)).to(gu.DEV)
    lK, cK, sK = training_run(stored, D_max, one_view, noise, D_max)
    l16, c16, s16 = training_run(padded, 3, one_view, noise, D_max)
    assert lK == l16, (lK, l16)
    assert cK == c16 and cK[1] > 0 and cK[3] > 0
    for name in sK:
        for q in range(3):
            a, b = sK[name][q], s16[name][q]
            if name == "f_rest":
                assert bool((b[:, K - 1:] == 0).all()), (name, q)
                b = b[:, :K - 1]
            assert bits_equal(a, b), (name, q)


# ---------------------------------------------------------------------------------------------------------------------
# drop-in: the reference's per-camera calls under torch.use_deterministic_algorithms(True)
# ---------------------------------------------------------------------------------------------------------------------
def test_dropin_follows_the_torch_flag(det_flag):
    import diff_gaussian_rasterization as dgr
    torch.use_deterministic_algorithms(True)
    cfg = syn.CONFIGS["c1"]
    W, H = cfg["width"], cfg["height"]
    cam = syn.make_camera(W, H, yaw_deg=3.0)
    sc = syn.make_scene(cfg["n"], W, H, seed=2)
    dcam = pipeline.DeviceCamera(cam, gu.DEV)
    rs0 = dcam.settings()
    rs = dgr.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=rs0.tanfovx, tanfovy=rs0.tanfovy,
                                           bg=rs0.bg, scale_modifier=1.0, viewmatrix=rs0.viewmatrix,
                                           projmatrix=rs0.projmatrix, sh_degree=3, campos=rs0.campos, prefiltered=False,
                                           debug=False)
    wgt = torch.randn((3, H, W), device=gu.DEV, generator=torch.Generator(device=gu.DEV).manual_seed(8))

    def run():
        t = {k: gu.to_dev(v, torch.float32).requires_grad_(True) for k, v in sc.items()}
        r = dgr.GaussianRasterizer(raster_settings=rs)
        m2, rgb, co, radii, depths = r.preprocess_gaussians(t["means3D"], t["scales"], t["rotations"], t["shs"],
                                                            t["opacities"], {})
        m2.retain_grad()
        image, *_ = r.render_gaussians(m2, co, rgb, depths, radii, None, None, {})
        (image * wgt).sum().backward()
        return m2.grad, {k: v.grad for k, v in t.items()}

    m_a, g_a = run()
    m_b, g_b = run()
    assert bits_equal(m_a, m_b)
    for k in g_a:
        assert bits_equal(g_a[k], g_b[k]), k
