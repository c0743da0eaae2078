"""-m gpu: the per-view training loss report (Trainer.train_losses) on one GPU.

Each view's recorded [Ll1, ssim] must be ops.fused_l1_ssim_batched recomputed on that step's images and ground truths,
bit for bit, for resident and resident=False steps, batches of 1, 3 and 8 views and local sampling; the resident=False
return value is unchanged; drained bits do not depend on when or whether the records are drained, and neither do the
parameters after FusedAdam; evaluate / image_metrics leave the records alone; border_exchange=True keeps the loss and
gradient bits of its ops.fused_loss arithmetic.  Strips of W = 2 and 3 divisions, rendered separately, sum in rank order
to the whole view's values within W float32 ulps (test_strip_partials_sum_to_the_whole_view states why)."""
import numpy as np
import pytest
import torch

from gs_b200 import ops, pipeline
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TW, TH, N_CAMS, N_GAUSS = 256, 200, 12, 20_000
LAM = 0.2


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def f32(v):
    return np.float32(v).view(np.int32)


@pytest.fixture(scope="module")
def camera_set():
    scene = syn.make_scene(N_GAUSS, TW, TH, seed=0)
    cams = [syn.make_camera(TW, TH, yaw_deg=4.0 * q - 20.0, uid=100 + q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=10 + q)).pin_memory() for q in range(N_CAMS)]
    return scene, cams, gts


def trainer(camera_set, **kw):
    scene, cams, gts = camera_set
    return pipeline.Trainer(scene, cams, gts, DEV, deterministic=True, lambda_dssim=LAM, **kw)


@pytest.fixture
def spy(monkeypatch):
    """The arguments of every ops.fused_l1_ssim_batched call the step makes: (images clone, gts, rows4, gt_full)."""
    calls, orig = [], ops.fused_l1_ssim_batched

    def wrapped(images, gts_u8, rows4, *, deterministic=None, gt_full=False):
        calls.append((images.detach().clone(), list(gts_u8), list(rows4), gt_full))
        return orig(images, gts_u8, rows4, deterministic=deterministic, gt_full=gt_full)

    monkeypatch.setattr(ops, "fused_l1_ssim_batched", wrapped)
    return calls, orig


def assert_entry_is_recomputed(entry, call, orig):
    images, gts, rows4, gt_full = call
    want = orig(images, gts, rows4, deterministic=True, gt_full=gt_full).cpu()
    assert len(entry["views"]) == want.shape[0]
    for q in range(want.shape[0]):
        assert f32(entry["l1"][q]) == bits(want[q, 0]).item(), q
        assert f32(entry["ssim"][q]) == bits(want[q, 1]).item(), q
        l1, ssim = want[q:q + 1, 0], want[q:q + 1, 1]
        assert f32(entry["loss"][q]) == bits((1.0 - LAM) * l1 + LAM * (1.0 - ssim)).item(), q


# 1. the record is the step's own loss kernel output
@pytest.mark.parametrize("views", [[5], [7, 2, 9], [7, 2, 9, 0, 3, 3, 11, 1]])
@pytest.mark.parametrize("resident", [True, False])
def test_record_is_the_steps_loss(camera_set, spy, views, resident):
    calls, orig = spy
    tr = trainer(camera_set)
    assert tr.train_losses() == []
    ret = tr.step(views=views, resident=resident)
    (entry,) = tr.train_losses()
    assert entry["iteration"] == 1 and entry["views"] == views and len(calls) == 1
    assert_entry_is_recomputed(entry, calls[0], orig)
    assert tr.train_losses() == []
    if not resident:   # the return value is loss_sum as the step forms it, and the per-view losses add up to it
        images, gts, rows4, gt_full = calls[0]
        l1_ssim = orig(images, gts, rows4, deterministic=True, gt_full=gt_full)
        coef = torch.tensor([1.0 - LAM, -LAM] * len(views), dtype=torch.float32, device=DEV)
        const = 0.0
        for _ in views:
            const += LAM
        assert f32(ret) == bits(torch.dot(l1_ssim.reshape(-1), coef) + const).item()
        assert sum(entry["loss"]) == pytest.approx(ret, rel=4 * len(views) * np.finfo(np.float32).eps)


def test_local_sampling_record(camera_set, spy):
    calls, orig = spy
    tr = trainer(camera_set, local_sampling=True, local_bsz=2)
    tr.step(views=[4, 0])
    tr.step(views=[1, 1], resident=False)
    entries = tr.train_losses()
    assert [(e["iteration"], e["views"]) for e in entries] == [(1, [4, 0]), (2, [1, 1])]
    for e, c in zip(entries, calls):
        assert_entry_is_recomputed(e, c, orig)


# 2. draining changes nothing, and the bits repeat
SCHEDULE = ([3, 1, 4], [5], [7, 2, 9, 0, 3, 3, 11, 1], [q % N_CAMS for q in range(64)],
            [(5 * q) % N_CAMS for q in range(64)], [q % 5 for q in range(64)], [11 - q % N_CAMS for q in range(64)],
            [2, 8])    # 271 views in all: the record buffer grows past its first 256 slots


def run(camera_set, drain_every):
    tr = trainer(camera_set)
    lr = dict(xyz=1e-3, f_dc=1e-2, f_rest=1e-3, opacity=5e-2, scaling=5e-3, rotation=1e-3)
    opt = FusedAdam(tr.optimizer_groups(lr), lr=0.0, eps=1e-15)
    entries, params = [], []
    for views in SCHEDULE:
        tr.step(views=views)
        opt.step(grad_scale=1.0 / len(views))
        if drain_every:
            entries += tr.train_losses()
        params.append([p.detach().clone() for p in tr.params.raw_parameters()])
    if drain_every is not None:
        entries += tr.train_losses()
    return entries, params


def test_drained_bits_repeat_and_draining_changes_nothing(camera_set):
    every, p_every = run(camera_set, True)
    once, p_once = run(camera_set, False)
    never, p_never = run(camera_set, None)
    assert [e["iteration"] for e in every] == list(range(1, len(SCHEDULE) + 1))
    assert [e["views"] for e in every] == [list(v) for v in SCHEDULE]
    for a, b in zip(every, once):
        assert a == b and all(f32(x) == f32(y) for k in ("l1", "ssim", "loss") for x, y in zip(a[k], b[k]))
    assert never == []
    for s, (a, b, c) in enumerate(zip(p_every, p_once, p_never)):
        assert all(same_bits(x, y) and same_bits(x, z) for x, y, z in zip(a, b, c)), f"step {s}: parameters"


# 3. evaluate and image_metrics leave the records as they were
def test_evaluation_leaves_the_records(camera_set):
    scene, cams, gts = camera_set
    a, b = trainer(camera_set), trainer(camera_set)
    for tr in (a, b):
        tr.step(views=[7, 2, 9])
    a.evaluate([0, 1, 2])
    a.image_metrics([3, 4])
    for tr in (a, b):
        tr.step(views=[1])
    a.evaluate(cams=cams[:2], gts=gts[:2])
    ea, eb = a.train_losses(), b.train_losses()
    assert ea == eb and len(ea) == 2
    a.evaluate([0])
    a.image_metrics([0])
    assert a.train_losses() == []


# 4. border_exchange=True: the record, and the loss and gradient bits of the ops.fused_loss arithmetic
def old_border_step(tr, views):
    """The border path's loss as ops.fused_loss forms it per local strip, summed in view order, and its backward."""
    views = tuple(views)
    strategies, cam_table, span, _ = tr._step_plan(views)
    rs = tr.dcams[views[0]].settings(tr.params.active_sh_degree)
    for t in tr.params.raw_parameters():
        t.grad = None
    tr._trace_on = False   # as _step sets it
    fw = tr._forward(rs, strategies, {}, cam_table, span, training=True)
    loss_sum = None
    for k, st in enumerate(strategies):
        rows = st.local_pixel_rows(tr.H)
        loss = ops.fused_loss(fw.images[k], tr.gts_dev[views[k]], *rows, tr.lambda_dssim, deterministic=True)
        loss_sum = loss if loss_sum is None else loss_sum + loss
    loss_sum.backward()
    return loss_sum, fw.means2D


@pytest.mark.parametrize("views", [[5], [7, 2, 9, 0]])
def test_border_exchange_keeps_its_bits(camera_set, views):
    new, old, plain = trainer(camera_set, border_exchange=True), trainer(camera_set), trainer(camera_set)
    ret = new.step(views=views, resident=False)
    loss, means2D = old_border_step(old, views)
    assert f32(ret) == bits(loss).item()
    for x, y in zip(new.params.raw_parameters(), old.params.raw_parameters()):
        assert same_bits(x.grad, y.grad)
    assert same_bits(new.means2D.grad, means2D.grad)
    plain.step(views=views)   # one rank: each view's pair is the batched loss's, bit for bit
    en, ep = new.train_losses(), plain.train_losses()
    assert en == ep and en[0]["views"] == views


# 5. strip partials summed in rank order against the whole view
def _render(params, dcam, cl=None):
    rs = dcam.settings(params.active_sh_degree)
    with torch.no_grad():
        p = params
        m2, rgb, co, radii, depths = ops.preprocess_gaussians_raw(p._xyz, p._features_dc, p._features_rest, p._scaling,
                                                                  p._rotation, p._opacity, rs)
        return ops.render_gaussians(m2, co, rgb, depths, radii, cl, rs, deterministic=True)[0]


@pytest.mark.parametrize("bounds", [[0, 6, 13], [0, 2, 9, 13], [0, 1, 12, 13]])
def test_strip_partials_sum_to_the_whole_view(camera_set, bounds):
    """The per-pixel terms of a strip are the whole view's (the strip's pixels render the same bits, and with the 5 halo
    rows of its neighbours in the window the SSIM of every counted pixel reads the same inputs).  Only the rounding
    differs: each strip's fp64 sum rounds once to float32 (1/2 ulp), the W - 1 float32 additions in rank order round
    once each (1/2 ulp), and the whole view rounds once (1/2 ulp).  With every partial of one sign that is at most
    W ulps of the whole view's value."""
    scene, cams, gts = camera_set
    params = pipeline.GaussianParams(scene, DEV)
    dcam = pipeline.DeviceCamera(cams[2], DEV)
    gt = gts[2].to(DEV)
    ty, tx = (TH + 15) // 16, (TW + 15) // 16
    whole = ops.fused_l1_ssim_batched(_render(params, dcam).unsqueeze(0), [gt], [(0, TH, 0, TH)], deterministic=True)
    W = len(bounds) - 1
    halo = torch.zeros((2,), dtype=torch.float32, device=DEV)
    plain = torch.zeros((2,), dtype=torch.float32, device=DEV)
    for a, b in zip(bounds, bounds[1:]):   # simulated rank: tile rows [a, b)
        y0, y1 = 16 * a, min(16 * b, TH)
        w0, w1 = max(0, y0 - ops.SSIM_HALO), min(TH, y1 + ops.SSIM_HALO)
        cl = torch.zeros((ty, tx), dtype=torch.bool, device=DEV)
        cl[w0 // 16:(w1 + 15) // 16] = True   # the strip and the tile rows of its halo
        img = _render(params, dcam, cl).unsqueeze(0)
        halo = halo + ops.fused_l1_ssim_batched(img, [gt], [(w0, w1, y0, y1)], deterministic=True, gt_full=True)[0]
        plain = plain + ops.fused_l1_ssim_batched(img, [gt], [(y0, y1, y0, y1)], deterministic=True, gt_full=True)[0]
    whole, halo, plain = whole[0].cpu().numpy(), halo.cpu().numpy(), plain.cpu().numpy()
    bound = W * np.spacing(np.abs(whole))
    assert np.all(np.abs(halo.astype(np.float64) - whole) <= bound), (halo, whole, bound)
    # without the halo the strip's L1 is still its pixels' share; its SSIM sees the strip's edges (the strip step's value)
    assert abs(float(plain[0]) - float(whole[0])) <= bound[0], (plain, whole)
