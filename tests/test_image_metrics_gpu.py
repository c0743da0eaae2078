"""-m gpu: the image metrics (ops.quantize_u8_batched / image_metric_sums_batched / image_metric_finalize,
pipeline.Trainer.image_metrics).

The quantizer against torch's save_image sequence byte for byte; the slots against the fp64 definitional reference
(tests/metrics_ref.py); the summed slots of a view rendered as strips of W = 2, 3, 4 simulated ranks, each window's halo
cut from the neighbours' quantized strips, equal the whole view's bit for bit, and so do image_metrics' per-view results
at every bsz and on every render path and image source; image_metrics against the reference's render.py + metrics.py
sequence on a full render, and its gathered images; a training run with image_metrics calls in it equals the run
without, bit for bit."""
import math

import numpy as np
import pytest
import torch

import metrics_ref
from gs_b200 import image_halo, ops, pipeline
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


def same_metrics(a, b):
    return same_bits(a["ssim_per_view"], b["ssim_per_view"]) and same_bits(a["psnr_per_view"], b["psnr_per_view"])


@pytest.fixture(scope="module")
def camera_set():
    scene = syn.make_scene(N_GAUSS, TW, TH, seed=0)
    cams = [syn.make_camera(TW, TH, yaw_deg=4.0 * q - 12.0, uid=100 + q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=10 + q)).pin_memory() for q in range(N_CAMS)]
    return scene, cams, gts


def _images(B, H, W, seed, noise=0.05):
    """Renders near their ground truth (an SSIM map that does not cancel to ~0), with exact ties, 0, 1 and values outside
    [0, 1]."""
    g = torch.Generator().manual_seed(seed)
    gt = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8)
    img = gt.float() / 255 + torch.randn((B, 3, H, W), generator=g) * noise
    flat = img.view(-1)
    k = torch.randint(0, 255, (flat.numel() // 13 + 1,), generator=g).float()
    flat[::13] = (k + 0.5) / 255
    flat[5::17] = 0.0
    flat[7::19] = 1.0
    flat[3::23] = -0.4
    flat[11::29] = 1.7
    return img, gt


# 1. the quantizer
def test_quantize_is_torchs_sequence_byte_for_byte():
    B, H, W = 3, 45, 37
    img, _ = _images(B, H, W, seed=1, noise=0.4)
    x = img.to(DEV)
    want = torch.clamp(x, 0, 1).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)
    rows = [(0, H), (16, 45), (3, 30)]
    outs = [torch.full((3, H, W), 7, dtype=torch.uint8, device=DEV), torch.full((3, 29, W), 7, dtype=torch.uint8,
                                                                                 device=DEV),
            torch.full((3, 40, W), 7, dtype=torch.uint8, device=DEV)]
    ops.quantize_u8_batched(x, rows, outs, [0, 16, 1])
    assert torch.equal(outs[0], want[0])
    assert torch.equal(outs[1], want[1, :, 16:45])
    assert torch.equal(outs[2][:, 2:29], want[2, :, 3:30])
    assert (outs[2][:, :2] == 7).all() and (outs[2][:, 29:] == 7).all()   # rows outside [row0, row1) untouched
    nan = torch.tensor([[[float("nan"), 0.5]]] * 3, device=DEV).unsqueeze(0)
    out = torch.full((3, 1, 2), 9, dtype=torch.uint8, device=DEV)
    ops.quantize_u8_batched(nan, [(0, 1)], [out], [0])
    assert out[:, 0].tolist() == [[0, 128]] * 3


def _window(q, g, rows, H):
    a, b = image_halo.window_rows(rows, H)
    return torch.cat([q[:, a:b], g[:, a:b]]).contiguous(), a


# 2. slots and finalize against the fp64 reference
@pytest.mark.parametrize("B,H,W", [(1, 200, 251), (3, 64, 33), (64, 40, 17), (2, 9, 7)])
def test_slots_against_the_reference(B, H, W):
    img, gt = _images(B, H, W, seed=B * H)
    q = torch.from_numpy(metrics_ref.quantize(img.numpy()))
    choices = [(0, H), (16, H), (0, 16), (0, 0), (32, 48) if H > 48 else (16, 32)] if H > 16 else [(0, H), (0, 0)]
    rows = [choices[v % len(choices)] for v in range(B)]
    wins, w0 = [], []
    for v, r in enumerate(rows):
        w, a = _window(q[v].to(DEV), gt[v].to(DEV), r, H) if r[1] > r[0] else (None, 0)
        wins.append(w); w0.append(a)
    slots = ops.image_metric_sums_batched(wins, w0, rows, H).cpu()
    for v in range(B):
        want = torch.from_numpy(metrics_ref.slots(q[v].numpy(), gt[v].numpy(), rows[v]))
        lo, hi = rows[v][0] // 16, -(-rows[v][1] // 16)
        live = torch.zeros(want.shape[0], dtype=torch.bool)
        live[lo:hi] = True
        assert torch.allclose(slots[v][live], want[live], rtol=1e-12, atol=0), f"view {v}"
        assert torch.equal(bits(slots[v][~live]), torch.zeros_like(bits(slots[v][~live]))), f"view {v}: not +0.0"
    # a window larger than the halo (the whole image) gives the same bits
    whole_wins = [None if w is None else torch.cat([q[v], gt[v]]).to(DEV) for v, w in enumerate(wins)]
    assert same_bits(ops.image_metric_sums_batched(whole_wins, [0] * B, rows, H).cpu(), slots)
    # and finalize
    full = ops.image_metric_sums_batched([torch.cat([q[v], gt[v]]).to(DEV) for v in range(B)], [0] * B, [(0, H)] * B, H)
    out = ops.image_metric_finalize(full, H, W).cpu()
    for v in range(B):
        ssim, psnr = metrics_ref.finalize(metrics_ref.slots(q[v].numpy(), gt[v].numpy()), H, W)
        assert out[v, 0].item() == pytest.approx(ssim, rel=1e-12) and out[v, 1].item() == pytest.approx(psnr, rel=1e-12)


def test_perfect_render_and_refused_windows():
    H, W = 40, 21
    gt = torch.randint(0, 256, (3, H, W), generator=torch.Generator().manual_seed(2), dtype=torch.uint8).to(DEV)
    out = ops.image_metric_finalize(ops.image_metric_sums_batched([torch.cat([gt, gt])], [0], [(0, H)], H), H, W)
    assert out[0, 0].item() == pytest.approx(1.0, abs=1e-15) and out[0, 1].item() == math.inf
    short = torch.cat([gt, gt])[:, 12:].contiguous()   # rows [12, 40): misses halo row 11 of rows [16, 40)
    with pytest.raises(RuntimeError, match="halo"):
        ops.image_metric_sums_batched([short], [12], [(16, H)], H)


# 3. the same bits at any strip division
def _render(params, dcam, cl=None):
    rs = dcam.settings(params.active_sh_degree)
    with torch.no_grad():
        p = params
        m2, rgb, co, radii, depths = ops.preprocess_gaussians_raw(p._xyz, p._features_dc, p._features_rest, p._scaling,
                                                                  p._rotation, p._opacity, rs)
        return ops.render_gaussians(m2, co, rgb, depths, radii, cl, rs)[0]


@pytest.mark.parametrize("H,bounds", [(200, [0, 6, 13]), (200, [0, 2, 9, 13]), (200, [0, 1, 5, 12, 13]),
                                      (195, [0, 12, 13]), (195, [0, 4, 12, 13])])
def test_strips_sum_to_the_whole_view_bit_for_bit(camera_set, H, bounds):
    """Simulated ranks own tile rows [a, b) each; a rank's window holds its quantized strip, and its halo rows are cut
    from the neighbours' quantized strips (H = 195: a last strip of 3 rows)."""
    scene, _cams, gts = camera_set
    params = pipeline.GaussianParams(scene, DEV)
    dcam = pipeline.DeviceCamera(syn.make_camera(TW, H, yaw_deg=-4.0, uid=1), DEV)
    gt = gts[2][:, :H].to(DEV)
    ty, tx = (H + 15) // 16, (TW + 15) // 16
    whole = _render(params, dcam).unsqueeze(0)
    q_whole = torch.empty((3, H, TW), dtype=torch.uint8, device=DEV)
    ops.quantize_u8_batched(whole, [(0, H)], [q_whole], [0])
    want = ops.image_metric_sums_batched([torch.cat([q_whole, gt])], [0], [(0, H)], H)
    strips = []
    for a, b in zip(bounds, bounds[1:]):   # each simulated rank renders and quantizes its own strip only
        cl = torch.zeros((ty, tx), dtype=torch.bool, device=DEV)
        cl[a:b] = True
        y0, y1 = 16 * a, min(16 * b, H)
        q = torch.empty((3, y1 - y0, TW), dtype=torch.uint8, device=DEV)
        ops.quantize_u8_batched(_render(params, dcam, cl).unsqueeze(0), [(y0, y1)], [q], [y0])
        strips.append((y0, y1, q))
    total = torch.zeros_like(want)
    for i, (y0, y1, q) in enumerate(strips):
        a, b = image_halo.window_rows((y0, y1), H)
        win = torch.empty((6, b - a, TW), dtype=torch.uint8, device=DEV)
        win[3:] = gt[:, a:b]
        win[:3, y0 - a:y1 - a] = q
        if i > 0:
            p0, p1, pq = strips[i - 1]
            win[:3, :y0 - a] = pq[:, a - p0:]
        if i + 1 < len(strips):
            n0, n1, nq = strips[i + 1]
            win[:3, y1 - a:] = nq[:, :b - y1]
        total += ops.image_metric_sums_batched([win], [a], [(y0, y1)], H)
    assert same_bits(total, want)
    assert same_bits(ops.image_metric_finalize(total, H, TW), ops.image_metric_finalize(want, H, TW))


# 4. image_metrics: every bsz (one-view batches run the per-camera preprocess) and image source
def test_image_metrics_is_the_same_bits_at_every_bsz_and_render_path(camera_set):
    scene, cams, gts = camera_set
    views = [3, 0, 6, 2, 2, 5, 1]
    tr = pipeline.Trainer(scene, cams, gts, DEV)
    res = [tr.image_metrics(views, bsz=b) for b in (1, 3, 4, None)]
    for r in res[1:]:
        assert same_metrics(r, res[0])
        assert (r["ssim"], r["psnr"]) == (res[0]["ssim"], res[0]["psnr"]) and r["images"] is None
    assert res[0]["ssim"] == pytest.approx(float(res[0]["ssim_per_view"].mean()), rel=1e-15)
    assert 0.0 < res[0]["ssim"] < 1.0


def test_held_out_images_give_the_same_bits(camera_set):
    scene, cams, gts = camera_set
    tr = pipeline.Trainer(scene, cams[:2], gts[:2], DEV)
    pageable = [g.clone() for g in gts]
    assert not pageable[0].is_pinned()
    on_dev = [g.to(DEV) for g in gts]
    views = [6, 1, 4, 4, 0]
    res = [tr.image_metrics(views, cams=cams, gts=g, bsz=b) for g, b in ((gts, None), (pageable, 2), (on_dev, 1))]
    for r in res[1:]:
        assert same_metrics(r, res[0])
    assert same_metrics(pipeline.Trainer(scene, cams, gts, DEV).image_metrics(views), res[0])
    held = [g if q % 2 == 0 else None for q, g in enumerate(gts)]
    ls = pipeline.Trainer(scene, cams, held, DEV, local_sampling=True, local_bsz=2)
    ls.step(views=[0, 2])
    with pytest.raises(ValueError, match="local-sampling"):
        ls.image_metrics()
    assert same_metrics(ls.image_metrics(views, cams=cams, gts=gts), res[0]) and ls.iteration == 1


# 5. against render.py + metrics.py on a full render
def test_against_the_reference_sequence_and_the_gathered_images(camera_set):
    scene, cams, gts = camera_set
    tr = pipeline.Trainer(scene, cams, gts, DEV, max_sh_degree=3)
    tr.params.active_sh_degree = 1
    bg = torch.tensor([0.3, 0.6, 0.1], device=DEV)
    for c in tr.dcams:
        c.bg = bg
    res = tr.image_metrics(images=True)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False   # the reference's fp32 convolutions, not TF32 ones
    try:
        for v in range(N_CAMS):
            image = _render(tr.params, tr.dcams[v])
            ssim, psnr = metrics_ref.reference_sequence(image, gts[v].to(DEV), torch.float32)
            # the float32 bounds of tests/test_image_metrics_ref.py, widened for the fp32 means over 50 k pixels; SSIM in
            # absolute terms, as these ground truths are unrelated to the renders and their SSIM is near 0 (0.03)
            assert res["ssim_per_view"][v].item() == pytest.approx(ssim, abs=1e-5), v
            assert res["psnr_per_view"][v].item() == pytest.approx(psnr, rel=2e-5), v
            got = res["images"][v]
            assert got.device.type == "cpu" and got.dtype == torch.uint8
            assert torch.equal(got, metrics_ref.save_image_quantize(image).cpu()), v
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    tr0 = pipeline.Trainer(scene, cams, gts, DEV, max_sh_degree=3)
    tr0.params.active_sh_degree = 1
    assert tr0.image_metrics()["ssim"] != res["ssim"]   # the Trainer's background is the one scored


# 6. image_metrics leaves training as it was
def test_training_is_undisturbed(camera_set):
    scene, cams, gts = camera_set
    lr = dict(xyz=1e-3, f_dc=1e-2, f_rest=1e-3, opacity=5e-2, scaling=5e-3, rotation=1e-3)
    runs = []
    for with_metrics in (True, False):
        tr = pipeline.Trainer(scene, cams, gts, DEV, deterministic=True)
        opt = FusedAdam(tr.optimizer_groups(lr), lr=0.0, eps=1e-15)
        stats = (torch.zeros((tr.n_local, 1), device=DEV), torch.zeros((tr.n_local, 1), device=DEV),
                 torch.zeros((tr.n_local,), device=DEV))
        losses = [tr.step(views=[1, 4], resident=False)]
        tr.add_densification_stats(*stats)
        opt.step(grad_scale=0.5)
        if with_metrics:
            tr.image_metrics([0, 6, 2], cams=cams, gts=gts, images=True)
            tr.image_metrics(bsz=2)
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
