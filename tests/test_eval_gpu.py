"""-m gpu: held-out view evaluation (ops.eval_sums_batched / eval_finalize, pipeline.Trainer.evaluate).

The slots against the fp64 definitional reference (tests/eval_ref.py); the summed slots of a view rendered as strips of
W = 2, 3, 4 simulated ranks (compute_locally masks, as tests/test_exchange_sim_gpu.py simulates them) equal the whole
view's bit for bit, and so do evaluate's per-view results at every bsz; evaluate against the reference's scoring sequence
on a full render; a training run with an evaluation in it equals the run without, bit for bit; held-out images on the
host (pinned or not) and on the device give the same bits; and a local-sampling Trainer evaluates a held-out set."""
import math

import numpy as np
import pytest
import torch

import eval_ref
from gs_b200 import ops, pipeline
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TW, TH, N_CAMS, N_GAUSS = 251, 200, 7, 20_000     # H not a multiple of 16, odd W


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int64) if t.dtype == torch.float64 else t.view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


@pytest.fixture(scope="module")
def camera_set():
    scene = syn.make_scene(N_GAUSS, TW, TH, seed=0)
    cams = [syn.make_camera(TW, TH, yaw_deg=4.0 * q - 12.0, uid=100 + q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=10 + q)).pin_memory() for q in range(N_CAMS)]
    return scene, cams, gts


def _images(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.rand((B, 3, H, W), generator=g) * 1.6 - 0.3
    img.view(-1)[::7] = 0.0
    img.view(-1)[3::11] = 1.0
    gt = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8)
    gt.view(-1)[::5] = 0
    gt.view(-1)[1::13] = 255
    return img, gt


def _check_slots(got, img, gt, rows):
    got = got.cpu()
    for v in range(img.shape[0]):
        want = torch.from_numpy(eval_ref.slots(img[v].numpy(), gt[v].numpy(), rows[v]))
        live = want != 0
        assert torch.allclose(got[v][live], want[live], rtol=1e-12, atol=0), f"view {v}"
        assert torch.equal(bits(got[v][~live]), torch.zeros_like(bits(got[v][~live]))), f"view {v}: not +0.0 outside"


# 1. slots and finalize against the fp64 reference
@pytest.mark.parametrize("B,H,W", [(1, 200, 251), (3, 64, 33), (64, 40, 17)])
def test_slots_against_the_reference(B, H, W):
    img, gt = _images(B, H, W, seed=B * H)
    rows = [[(0, H), (16, H), (0, 16), (0, 0), (32, 48) if H > 48 else (16, 32)][v % 5] for v in range(B)]
    gts_dev = [gt[v].to(DEV) for v in range(B)]
    slots = ops.eval_sums_batched(img.to(DEV), [g if r[1] > r[0] else None for g, r in zip(gts_dev, rows)], rows,
                                  [0] * B)
    _check_slots(slots, img, gt, rows)
    # strips of the ground truth read at gt_row0 = row0 give the same bits as the whole images read in place
    strips = [g[:, r[0]:r[1]].contiguous() if r[1] > r[0] else None for g, r in zip(gts_dev, rows)]
    s2 = ops.eval_sums_batched(img.to(DEV), strips, rows, [r[0] for r in rows])
    assert same_bits(slots, s2)
    whole = ops.eval_sums_batched(img.to(DEV), gts_dev, [(0, H)] * B, [0] * B)
    out = ops.eval_finalize(whole, H, W).cpu()
    for v in range(B):
        l1, psnr = eval_ref.finalize(eval_ref.slots(img[v].numpy(), gt[v].numpy()), H, W)
        assert out[v, 0].item() == pytest.approx(l1, rel=1e-12) and out[v, 1].item() == pytest.approx(psnr, rel=1e-12)


def test_nan_inf_and_the_per_channel_psnr():
    H, W = 48, 20
    gt = torch.randint(0, 256, (3, 3, H, W), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
    img = (gt.to(DEV) / 255.0).cpu()  # view 0: the reference's gt / 255.0 on the device exactly -> L1 0, PSNR +inf
    img[1, 2, 30, 7] = float("nan")   # view 1: a diverged pixel -> NaN, in its tile row's slot only
    img[2, 0] += 0.02                 # view 2: channel errors of different size
    img[2, 1] -= 0.2
    slots = ops.eval_sums_batched(img.to(DEV), [g.to(DEV) for g in gt], [(0, H)] * 3, [0] * 3)
    out = ops.eval_finalize(slots, H, W).cpu()
    assert out[0, 0].item() == 0.0 and out[0, 1].item() == math.inf
    s1 = slots[1].cpu()
    assert torch.isnan(s1[1, 2]).all() and not torch.isnan(s1[0]).any() and not torch.isnan(s1[2]).any()
    assert math.isnan(out[1, 0].item()) and math.isnan(out[1, 1].item())
    per_channel = eval_ref.finalize(eval_ref.slots(img[2].numpy(), gt[2].numpy()), H, W)[1]
    d = img[2].double() - torch.from_numpy(eval_ref.gt_hat(gt[2].numpy()))
    pooled = 20 * math.log10(1 / math.sqrt(float((d ** 2).mean())))
    assert out[2, 1].item() == pytest.approx(per_channel, rel=1e-12) and abs(out[2, 1].item() - pooled) > 1.0


# 2. the same bits at any strip division and batch size
def _render(params, dcam, cl=None):
    rs = dcam.settings(params.active_sh_degree)
    with torch.no_grad():
        p = params
        m2, rgb, co, radii, depths = ops.preprocess_gaussians_raw(p._xyz, p._features_dc, p._features_rest, p._scaling,
                                                                  p._rotation, p._opacity, rs)
        return ops.render_gaussians(m2, co, rgb, depths, radii, cl, rs)[0]


@pytest.mark.parametrize("bounds", [[0, 6, 13], [0, 2, 9, 13], [0, 1, 5, 12, 13], [0, 12, 13]])
def test_strips_sum_to_the_whole_view_bit_for_bit(camera_set, bounds):
    scene, cams, gts = camera_set
    params = pipeline.GaussianParams(scene, DEV)
    dcam = pipeline.DeviceCamera(cams[2], DEV)
    gt = gts[2].to(DEV)
    ty, tx = (TH + 15) // 16, (TW + 15) // 16
    whole = ops.eval_sums_batched(_render(params, dcam).unsqueeze(0), [gt], [(0, TH)], [0])
    total = torch.zeros_like(whole)
    for a, b in zip(bounds, bounds[1:]):   # simulated rank: tile rows [a, b)
        cl = torch.zeros((ty, tx), dtype=torch.bool, device=DEV)
        cl[a:b] = True
        y0, y1 = 16 * a, min(16 * b, TH)
        strip = gt[:, y0:y1].contiguous()
        total += ops.eval_sums_batched(_render(params, dcam, cl).unsqueeze(0), [strip], [(y0, y1)], [y0])
    assert same_bits(total, whole)
    assert same_bits(ops.eval_finalize(total, TH, TW), ops.eval_finalize(whole, TH, TW))


def test_evaluate_is_the_same_bits_at_every_bsz(camera_set):
    scene, cams, gts = camera_set
    tr = pipeline.Trainer(scene, cams, gts, DEV)
    views = [3, 0, 6, 2, 2, 5, 1]
    res = [tr.evaluate(views, bsz=b) for b in (1, 3, None)]
    for r in res[1:]:
        assert same_bits(r["l1_per_view"], res[0]["l1_per_view"]) and same_bits(r["psnr_per_view"], res[0]["psnr_per_view"])
        assert (r["l1"], r["psnr"]) == (res[0]["l1"], res[0]["psnr"])
    assert res[0]["l1"] == pytest.approx(float(res[0]["l1_per_view"].mean()), rel=1e-15)


# 3. against the reference's scoring sequence on a full render
def test_against_the_reference_sequence(camera_set):
    scene, cams, gts = camera_set
    tr = pipeline.Trainer(scene, cams, gts, DEV, max_sh_degree=3)
    tr.params.active_sh_degree = 1
    bg = torch.tensor([0.3, 0.6, 0.1], device=DEV)
    for c in tr.dcams:
        c.bg = bg
    res = tr.evaluate()
    for v in range(N_CAMS):
        image = _render(tr.params, tr.dcams[v])
        l1, psnr = eval_ref.reference_sequence(image, gts[v].to(DEV), torch.float32)
        assert res["l1_per_view"][v].item() == pytest.approx(l1, rel=2e-5), v
        assert res["psnr_per_view"][v].item() == pytest.approx(psnr, rel=2e-5), v
    # the background and the SH degree are those of the Trainer: a black background scores differently
    tr0 = pipeline.Trainer(scene, cams, gts, DEV, max_sh_degree=3)
    tr0.params.active_sh_degree = 1
    assert tr0.evaluate()["l1"] != res["l1"]


# 4. an evaluation leaves training as it was
def test_training_is_undisturbed(camera_set):
    scene, cams, gts = camera_set
    lr = dict(xyz=1e-3, f_dc=1e-2, f_rest=1e-3, opacity=5e-2, scaling=5e-3, rotation=1e-3)
    runs = []
    for with_eval in (True, False):
        tr = pipeline.Trainer(scene, cams, gts, DEV, deterministic=True)
        opt = FusedAdam(tr.optimizer_groups(lr), lr=0.0, eps=1e-15)
        stats = (torch.zeros((tr.n_local, 1), device=DEV), torch.zeros((tr.n_local, 1), device=DEV),
                 torch.zeros((tr.n_local,), device=DEV))
        losses = [tr.step(views=[1, 4], resident=False)]
        tr.add_densification_stats(*stats)
        opt.step(grad_scale=0.5)
        if with_eval:
            tr.evaluate([0, 6, 2], cams=cams[:3] + cams[3:], gts=gts)
            tr.evaluate(bsz=2)
        losses.append(tr.step(views=[5, 0, 3], resident=False))
        tr.add_densification_stats(*stats)
        grads = [t.grad.clone() for t in tr.params.raw_parameters()]
        opt.step(grad_scale=1 / 3)
        runs.append((tr, losses, grads, stats))
    (a, la, ga, sa), (b, lb, gb, sb) = runs
    assert np.float32(la).view(np.int32).tolist() == np.float32(lb).view(np.int32).tolist()
    assert all(same_bits(x, y) for x, y in zip(ga, gb)), "gradients"
    assert all(same_bits(x, y) for x, y in zip(sa, sb)), "densification statistics"
    for attr in pipeline.Trainer.GROUP_OF.values():
        assert same_bits(getattr(a.params, attr), getattr(b.params, attr)), attr
    assert a.iteration == b.iteration == 2 and a.balance_log == b.balance_log
    assert a.history.history == b.history.history and a.last_info() == b.last_info()


# 5. held-out images wherever they live
def test_held_out_images_give_the_same_bits(camera_set):
    scene, cams, gts = camera_set
    tr = pipeline.Trainer(scene, cams[:2], gts[:2], DEV)
    pageable = [g.clone() for g in gts]
    assert not pageable[0].is_pinned()
    on_dev = [g.to(DEV) for g in gts]
    res = [tr.evaluate([6, 1, 4, 4, 0], cams=cams, gts=g, bsz=b) for g, b in ((gts, None), (pageable, 2), (on_dev, 1))]
    for r in res[1:]:
        assert same_bits(r["l1_per_view"], res[0]["l1_per_view"]) and same_bits(r["psnr_per_view"], res[0]["psnr_per_view"])
    own = pipeline.Trainer(scene, cams, gts, DEV).evaluate([6, 1, 4, 4, 0])   # the same cameras as a Trainer's own set
    assert same_bits(own["l1_per_view"], res[0]["l1_per_view"]) and same_bits(own["psnr_per_view"], res[0]["psnr_per_view"])
    for bad in (dict(views=[7]), dict(views=[]), dict(bsz=0), dict(bsz=65), dict(gts=gts[:6]),
                dict(gts=[g[:, :64] for g in gts]), dict(cams=[syn.make_camera(TW, 64)] * N_CAMS)):
        kw = dict(views=None, cams=cams, gts=gts)
        kw.update(bad)
        with pytest.raises(ValueError):
            tr.evaluate(kw.pop("views"), **kw)


# 6. local sampling
def test_local_sampling_evaluates_a_held_out_set(camera_set):
    scene, cams, gts = camera_set
    held = [g if q % 2 == 0 else None for q, g in enumerate(gts)]
    ls = pipeline.Trainer(scene, cams, held, DEV, local_sampling=True, local_bsz=2)
    ls.step(views=[0, 2])
    with pytest.raises(ValueError, match="local-sampling"):
        ls.evaluate()
    assert ls.iteration == 1
    got = ls.evaluate([5, 3, 0], cams=cams, gts=gts)
    want = pipeline.Trainer(scene, cams, gts, DEV).evaluate([5, 3, 0])
    assert same_bits(got["l1_per_view"], want["l1_per_view"]) and same_bits(got["psnr_per_view"], want["psnr_per_view"])
