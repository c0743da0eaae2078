"""-m gpu: training over a camera set -- pipeline.Trainer over N cameras stepping on the views the caller lists, and the
loss kernels that read each view's resident (3,H,W) ground truth in place (ops.fused_l1_ssim_batched(gt_full=True)).

A step over views [7, 2, 9, 0] of a 12-camera Trainer must be the step of a Trainer built on exactly those four cameras:
the same loss and gradients, bit for bit, under deterministic=True (atomic-free render backward and loss).  Training runs
with changing batches, FusedAdam and a densify/prune must match rebuilding a Trainer for every batch.  The in-place GT
loss must be the strip-copy loss, bit for bit.  Comparisons are of int32 bit patterns."""
import ctypes as C

import numpy as np
import pytest
import torch

from gs_b200 import _lib, densify, ops, pipeline
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TW, TH, N_CAMS, N_GAUSS = 256, 200, 12, 20_000
VIEWS = [7, 2, 9, 0]


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


@pytest.fixture(scope="module")
def camera_set():
    scene = syn.make_scene(N_GAUSS, TW, TH, seed=0)
    cams = [syn.make_camera(TW, TH, yaw_deg=4.0 * k - 20.0, uid=100 + k) for k in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=10 + k)).pin_memory() for k in range(N_CAMS)]
    return scene, cams, gts


def trainer(scene, cams, gts):
    return pipeline.Trainer(scene, cams, gts, DEV, deterministic=True)


def grads_of(tr):
    return [t.grad.detach().clone() for t in tr.params.raw_parameters()]


def assert_same_step(a, b, what):
    for k, (x, y) in enumerate(zip(grads_of(a), grads_of(b))):
        assert same_bits(x, y), f"{what}: gradient of parameter {k} differs"
    assert same_bits(a.means2D.grad, b.means2D.grad), f"{what}: screen-space gradients differ"


# (a) a batch of a camera set is the Trainer of exactly those cameras; a batch of one view runs the per-camera preprocess
@pytest.mark.parametrize("path", ["batched", "one_view"])
@pytest.mark.parametrize("resident", [True, False])
def test_views_equal_trainer_on_those_cameras(camera_set, path, resident):
    scene, cams, gts = camera_set
    views = VIEWS if path == "batched" else VIEWS[:1]
    whole = trainer(scene, cams, gts)
    sub = trainer(scene, [cams[i] for i in views], [gts[i] for i in views])
    la = whole.step(views=views, resident=resident)
    lb = sub.step(resident=resident)
    if not resident:
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (la, lb)
    assert_same_step(whole, sub, f"{path}, resident={resident}")
    # one view after a batch: the per-camera preprocess, too
    one = trainer(scene, [cams[5]], [gts[5]])
    whole.step(views=[5], resident=resident)
    one.step(resident=resident)
    assert_same_step(whole, one, f"{path}, one view")


# (b) views=None: every camera in order, resident in-place GT == strip copies from the host
def test_views_none_is_all_cameras(camera_set):
    scene, cams, gts = camera_set
    a, b, c = (trainer(scene, cams[:4], gts[:4]) for _ in range(3))
    a.step()
    b.step(views=[0, 1, 2, 3])
    lc = c.step(resident=False)
    assert_same_step(a, b, "views=None vs all views listed")
    assert_same_step(a, c, "in-place resident GT vs host strip copies")
    assert a._strip_cache == {} and b._strip_cache == {}
    assert np.isfinite(lc)


# (c) six steps over changing batches + FusedAdam + densify/prune == a Trainer rebuilt for every batch
SCHEDULE = ([7, 2, 9, 0], [3], [11, 3, 4], [7, 2, 9, 0], [0, 0, 5], [10, 1, 6, 8, 2])
DENSIFY_AFTER = 2


def _densify(opt, accum, denom, params, noise):
    extent = float(torch.exp(params._scaling.detach()).max(dim=1).values.median()) / 0.01
    grads = (accum / denom.clamp(min=1))[:, 0]
    return densify.densify_and_prune(opt, accum, denom, float(torch.quantile(grads, 0.8)), 0.005, extent, 0.01, None,
                                     noise=noise)


def test_changing_batches_match_rebuilt_trainers(camera_set):
    scene, cams, gts = camera_set
    noise = torch.randn((2 * N_GAUSS, 3), generator=torch.Generator().manual_seed(3)).to(DEV)
    lr = dict(xyz=1e-3, f_dc=1e-2, f_rest=1e-3, opacity=5e-2, scaling=5e-3, rotation=1e-3)
    # run A: one Trainer over the set
    ta = trainer(scene, cams, gts)
    oa = FusedAdam(ta.optimizer_groups(lr), lr=0.0, eps=1e-15)
    # run B: a Trainer per batch, all sharing one set of parameters and one optimizer
    tb0 = trainer(scene, [cams[0]], [gts[0]])
    ob = FusedAdam(tb0.optimizer_groups(lr), lr=0.0, eps=1e-15)
    shared = {name: getattr(tb0.params, attr) for name, attr in pipeline.Trainer.GROUP_OF.items()}
    stats = {}
    for it, views in enumerate(SCHEDULE):
        la = ta.step(views=views, resident=False)
        tb = trainer(scene, [cams[i] for i in views], [gts[i] for i in views])
        tb.adopt_parameters(shared)
        lb = tb.step(resident=False)
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (it, la, lb)
        assert_same_step(ta, tb, f"step {it} {views}")
        for way, tr in (("a", ta), ("b", tb)):
            P = tr.n_local
            if way not in stats or stats[way][0].shape[0] != P:
                stats[way] = (torch.zeros((P, 1), device=DEV), torch.zeros((P, 1), device=DEV), torch.zeros((P,), device=DEV))
            tr.add_densification_stats(*stats[way])
        assert all(same_bits(x, y) for x, y in zip(stats["a"], stats["b"])), f"step {it}: densification statistics"
        oa.step(grad_scale=1.0 / len(views))
        ob.step(grad_scale=1.0 / len(views))
        if it == DENSIFY_AFTER:
            ra = _densify(oa, stats["a"][0], stats["a"][1], ta.params, noise)
            rb = _densify(ob, stats["b"][0], stats["b"][1], tb.params, noise)
            assert ra["counts"] == rb["counts"] and ra["counts"][1] + ra["counts"][3] > 0, (ra["counts"], rb["counts"])
            ta.adopt_parameters(ra)
            shared = {name: rb[name] for name in pipeline.Trainer.GROUP_OF}
            del stats["a"], stats["b"]
        for name, attr in pipeline.Trainer.GROUP_OF.items():
            assert same_bits(getattr(ta.params, attr), shared[name]), f"step {it}: parameter {name}"


# (d) the in-place GT loss is the strip-copy loss, bit for bit
@pytest.mark.parametrize("det", [True, False])
def test_gt_full_loss_equals_strip_copies(det):
    H, W = 203, 333
    g = torch.Generator().manual_seed(7)
    B = 6
    images = torch.rand((B, 3, H, W), generator=g).to(DEV).requires_grad_(True)
    full = [torch.randint(0, 256, (3, H, W), dtype=torch.uint8, generator=g).to(DEV) for _ in range(B)]
    # strip at row 0, at the last row (one row), the whole image, a view without a local strip, the middle with halo
    # rows that feed the window and are not counted, a one-row strip in the middle
    rows4 = [(0, 64, 0, 64), (H - 1, H, H - 1, H), (0, H, 0, H), (0, 0, 0, 0), (48, 160, 53, 155), (100, 101, 100, 101)]
    strips = [None if r[1] == r[0] else full[k][:, r[0]:r[1]].contiguous() for k, r in enumerate(rows4)]
    g_out = torch.randn((B, 2), generator=g).to(DEV)
    res = {}
    for mode, gts in (("full", full), ("strip", strips)):
        out = ops.fused_l1_ssim_batched(images, gts, rows4, deterministic=det, gt_full=mode == "full")
        (d_img,) = torch.autograd.grad(out, images, g_out)
        res[mode] = (out.detach(), d_img)
    if det:
        assert same_bits(res["full"][0], res["strip"][0])
    else:   # fp64 atomics in either form: the same sums up to their order
        torch.testing.assert_close(res["full"][0], res["strip"][0], rtol=1e-6, atol=0)
    assert same_bits(res["full"][1], res["strip"][1])
    assert bool((res["full"][0][3] == 0).all()) and bool((res["full"][1][3] == 0).all())
    # the single-view loss, window and counted rows as the border exchange passes them
    img = images[4].detach().requires_grad_(True)
    r0, r1, c0, c1 = rows4[4]
    lf = ops.fused_loss(img, full[4], r0, r1, 0.2, c0, c1, deterministic=True, gt_full=True)
    ls = ops.fused_loss(img, strips[4], r0, r1, 0.2, c0, c1, deterministic=True)
    assert same_bits(lf.detach(), ls.detach())
    assert same_bits(torch.autograd.grad(lf, img)[0], torch.autograd.grad(ls, img)[0])


# (e) refusals before any launch leave every output as it was
def test_refusals_leave_outputs_untouched(camera_set):
    scene, cams, gts = camera_set
    H, W = 64, 96
    image = torch.rand((2, 3, H, W), device=DEV)
    buf = torch.zeros((3 * H * W + 16,), dtype=torch.uint8, device=DEV)
    gt, bad = buf[:3 * H * W], buf[1:1 + 3 * H * W]
    assert gt.data_ptr() % 16 == 0 and bad.data_ptr() % 16 == 1
    rows4 = [(0, 32, 0, 32), (32, H, 32, H)]
    tb = _lib.query("gs_loss_temp_bytes_batched_det", 2, (C.c_int32 * 8)(*[v for r in rows4 for v in r]), W)
    temp = torch.full((tb,), 0xA5, dtype=torch.uint8, device=DEV)
    out = torch.full((2, 2), -7.0, device=DEV)
    dimg = torch.full_like(image, -7.0)
    grads = torch.ones((2,), device=DEV)

    def fwd(name, r4, ptrs, nv=2):
        flat = (C.c_int32 * (4 * nv))(*[v for r in r4 for v in r])
        gp = (C.c_void_p * nv)(*ptrs)
        return _lib.query(name, nv, H, W, flat, image.data_ptr(), gp, out.data_ptr(), temp.data_ptr(), tb,
                          torch.cuda.current_stream().cuda_stream)

    def bwd(r4, ptrs):
        flat = (C.c_int32 * 8)(*[v for r in r4 for v in r])
        gp = (C.c_void_p * 2)(*ptrs)
        return _lib.query("gs_loss_backward_batched_gt_full", 2, H, W, flat, image.data_ptr(), gp, temp.data_ptr(),
                          grads.data_ptr(), grads.data_ptr(), dimg.data_ptr(), torch.cuda.current_stream().cuda_stream)

    ok = [gt.data_ptr(), gt.data_ptr()]
    cases = {
        "misaligned gt": (rows4, [gt.data_ptr(), bad.data_ptr()]),
        "null gt": (rows4, [gt.data_ptr(), None]),
        "row1 past the image": ([(0, 32, 0, 32), (32, H + 1, 32, H)], ok),
        "negative row0": ([(-1, 32, 0, 32), (32, H, 32, H)], ok),
        "row1 < row0": ([(0, 32, 0, 32), (40, 32, 40, 32)], ok),
        "count rows outside the window": ([(0, 32, 0, 33), (32, H, 32, H)], ok),
    }
    for name, (r4, ptrs) in cases.items():
        for entry in ("gs_loss_forward_batched_gt_full", "gs_loss_forward_batched_gt_full_det"):
            assert fwd(entry, r4, ptrs) == -1, (entry, name)
        assert bwd(r4, ptrs) == -1, name
    assert fwd("gs_loss_forward_batched_gt_full", [], [], nv=0) == -1
    torch.cuda.synchronize()
    assert bool((out == -7.0).all()) and bool((dimg == -7.0).all()) and bool((temp == 0xA5).all())
    with pytest.raises(ValueError):   # a strip where a whole image is expected
        ops.fused_l1_ssim_batched(image, [gt.view(3, H, W)[:, :32], gt.view(3, H, W)], rows4, gt_full=True)

    # Trainer: a bad view index changes nothing, not even the gradients of the last step
    tr = trainer(scene, cams[:3], gts[:3])
    tr.step(views=[2, 0])
    before = [bits(t).clone() for t in grads_of(tr)]
    for views in ([3], [-1], [], [0] * 65, [0.5], ["0"]):
        with pytest.raises((ValueError, TypeError)):
            tr.step(views=views)
    assert all(torch.equal(bits(t), b) for t, b in zip(grads_of(tr), before))
    # mixed sizes are refused at construction
    with pytest.raises(ValueError, match="one image size"):
        pipeline.Trainer(scene, [cams[0], syn.make_camera(TW + 16, TH, uid=1)], None, DEV)
    with pytest.raises(ValueError, match="one image size"):
        pipeline.Trainer(scene, cams[:2], [gts[0], torch.zeros((3, TH + 16, TW), dtype=torch.uint8)], DEV)
