"""CPU pins of the strip loss's fp64 reference (tests/loss_ref.py) and of the case generators (tests/loss_cases.py) that
tests/test_loss_cases_gpu.py holds the kernels to.

loss_ref.strip_terms is the counted-rows contract of csrc/loss.cu written with F.conv2d.  Here it is checked against
tests/torch_ref.ssim_l1_loss (pinned to the reference's loss_utils through the oracle and tests/golden/loss.npz), against
a literal numpy evaluation that sums each pixel's 11x11 window, against its own halo identity, and its autograd gradient
against central differences."""
import numpy as np
import pytest
import torch

import loss_cases as lc
import loss_ref
import torch_ref
from gs_b200 import border


def rand_pair(H, W, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-0.05, 1.3, (3, H, W)), rng.uniform(0, 1, (3, H, W))


@pytest.mark.parametrize("H,W", [(1, 1), (7, 3), (16, 33), (37, 53), (48, 12)])
def test_whole_window_counted_equals_torch_ref_bit_for_bit(H, W):
    img, gt = rand_pair(H, W, H * 100 + W)
    n = (H + 20) * W                      # any normaliser: the strip is a window of a taller image
    x1 = torch.tensor(img, requires_grad=True)
    x2 = torch.tensor(img, requires_grad=True)
    y = torch.tensor(gt)
    _, l1_a, ss_a = torch_ref.ssim_l1_loss(x1, y, n)
    l1_b, ss_b = loss_ref.strip_terms(x2, y, 0, H, n)
    assert l1_a.item() == l1_b.item() and ss_a.item() == ss_b.item()
    for a, b in ((l1_a, l1_b), (ss_a, ss_b)):
        ga, = torch.autograd.grad(a, x1, retain_graph=True)
        gb, = torch.autograd.grad(b, x2, retain_graph=True)
        assert torch.equal(ga, gb)


def literal_terms(xw, yw, c0, c1, n_pixels):
    """Ll1 and ssim of the window (3, rows, W) in numpy fp64: per counted pixel, the sums over its 11x11 window (taps the
    fp64 outer product of the fp32-normalised 1-D taps, zero outside the window)."""
    g = loss_ref.gauss_taps().numpy()
    w2 = np.outer(g, g)
    rows, W = xw.shape[1:]
    pad = ((0, 0), (5, 5), (5, 5))
    xp, yp = np.pad(xw, pad), np.pad(yw, pad)
    l1 = ss = 0.0
    for c in range(3):
        for i in range(c0, c1):
            l1 += np.abs(xw[c, i] - yw[c, i]).sum()
            for j in range(W):
                px, py = xp[c, i:i + 11, j:j + 11], yp[c, i:i + 11, j:j + 11]
                mu1, mu2 = (w2 * px).sum(), (w2 * py).sum()
                s1 = (w2 * px * px).sum() - mu1 * mu1
                s2 = (w2 * py * py).sum() - mu2 * mu2
                s12 = (w2 * px * py).sum() - mu1 * mu2
                ss += ((2 * mu1 * mu2 + loss_ref.C1) * (2 * s12 + loss_ref.C2)
                       / ((mu1 * mu1 + mu2 * mu2 + loss_ref.C1) * (s1 + s2 + loss_ref.C2)))
    return l1 / (3 * n_pixels), ss / (3 * n_pixels)


SIZES = (1, 2, 5, 11, 12, 17)


@pytest.mark.parametrize("H", SIZES)
def test_counted_rows_match_literal_window_sums(H):
    for W in SIZES:
        img, gt = rand_pair(H, W, 7 * H + W)
        gt[:, : (H + 1) // 2, : (W + 1) // 2] = 0.25          # a flat ground-truth corner
        n = 3 * H * W + 5
        for r0, r1 in {(0, H), (H // 3, H), (0, max(1, H - 2)), (H // 4, H // 4 + 1)}:
            for mode in ("all", "halo", "empty"):
                c0, c1 = lc.count_rows(r0, r1, mode)
                xw, yw = img[:, r0:r1], gt[:, r0:r1]
                l1, ss = loss_ref.strip_terms(torch.tensor(xw), torch.tensor(yw), c0 - r0, c1 - r0, n)
                el1, ess = literal_terms(xw, yw, c0 - r0, c1 - r0, n)
                assert abs(float(l1) - el1) <= 1e-13 * abs(el1) + 1e-300, (H, W, r0, r1, mode)
                assert abs(float(ss) - ess) <= 1e-12 * abs(ess) + 1e-300, (H, W, r0, r1, mode)
                if c0 == c1:
                    assert float(l1) == 0.0 and float(ss) == 0.0


@pytest.mark.parametrize("H,W,cuts", [(53, 7, [0, 16, 32, 48, 53]), (70, 32, [0, 5, 11, 16, 32, 37, 64, 70]),
                                      (45, 33, [0, 6, 11, 27, 32, 45])])
def test_halo_strips_sum_to_the_full_image(H, W, cuts):
    """Strips whose windows are widened by HALF_WINDOW rows, each counting only its own rows, add up to the whole-image
    loss and gradient: every counted row's 11-row neighbourhood lies inside its strip's window."""
    img, gt = rand_pair(H, W, H + W)
    img[:, :12, :12] = 0.5                                  # flat x over flat gt: both variances 0
    gt[:, :12, :12] = 0.5
    g_l1, g_ss = 0.7, -1.9
    l1f, ssf, gf = loss_ref.strip_loss(img, gt, 0, H, 0, H, g_l1, g_ss)
    l1s = sss = 0.0
    gs = torch.zeros_like(gf)
    for y0, y1 in zip(cuts, cuts[1:]):
        assert y1 - y0 >= border.HALF_WINDOW
        r0, r1 = max(0, y0 - border.HALF_WINDOW), min(H, y1 + border.HALF_WINDOW)
        l1, ss, g = loss_ref.strip_loss(img, gt[:, r0:r1], r0, r1, y0, y1, g_l1, g_ss)
        l1s, sss, gs = l1s + l1, sss + ss, gs + g
    assert abs(l1s - l1f) <= 1e-12 * abs(l1f) and abs(sss - ssf) <= 1e-12 * abs(ssf)
    gf, gs = gf.numpy(), gs.numpy()
    rms = np.sqrt((gf ** 2).mean())
    assert (np.abs(gs - gf) <= 1e-12 * (np.abs(gf) + rms)).all()


def test_gradient_matches_central_differences():
    """d(g_l1 Ll1 + g_ssim ssim) / dx of a halo window against central differences, at pixels in the counted rows, in the
    halo rows, outside the window and at the centre of a flat window where both variances are 0."""
    H, W, r0, r1, c0, c1 = 30, 24, 4, 26, 9, 21
    img, gt = rand_pair(H, W, 11)
    img[:, 6:22, 3:17] = 0.375                              # both flat, x != y: |x - y| is differentiable
    gt[:, 6:22, 3:17] = 0.625
    g_l1, g_ss = 1.3, -0.8
    _, _, grad = loss_ref.strip_loss(img, gt[:, r0:r1], r0, r1, c0, c1, g_l1, g_ss)

    def f(a):
        l1, ss = loss_ref.strip_terms(torch.tensor(a[:, r0:r1]), torch.tensor(gt[:, r0:r1]), c0 - r0, c1 - r0, H * W)
        return g_l1 * float(l1) + g_ss * float(ss)

    pts = [(0, 14, 10), (1, 12, 20), (2, 20, 5), (0, 5, 9), (1, 24, 1), (2, 2, 7), (0, 27, 3)]
    assert _both_flat(img, gt, 14, 10)
    h = 1e-6
    for c, i, j in pts:
        a, b = img.copy(), img.copy()
        a[c, i, j] += h
        b[c, i, j] -= h
        fd = (f(a) - f(b)) / (2 * h)
        assert abs(float(grad[c, i, j]) - fd) <= 1e-6 * np.abs(grad.numpy()).max(), (c, i, j, float(grad[c, i, j]), fd)
        if not r0 <= i < r1:
            assert float(grad[c, i, j]) == 0.0
    assert float(grad[0, 14, 10]) != 0.0


def _both_flat(img, gt, i, j):
    return all(np.ptp(a[:, i - 5:i + 6, j - 5:j + 6]) == 0 for a in (img, gt))


CASES = ([(H, W, "mixed") for H in (1, 17, 33, 64, 95) for W in (1, 2, 11, 12, 31, 32, 33)]
         + [(56, 64, "checker"), (2, 3, "checker"), (88, 96, "smooth"), (1080, 1920, "smooth")])


def test_case_generators_populate_what_they_claim():
    claimed = set()
    for H, W, kind in CASES:
        img, gt = lc.make_pair(H, W, seed=H + W, kind=kind)
        assert img.dtype == np.float32 and gt.dtype == np.uint8 and img.shape == gt.shape == (3, H, W)
        want = lc.claims(H, W, kind)
        lc.assert_populated(img, gt, want, (H, W, kind))
        claimed |= want
        if "saturated" in want:
            assert 2.0 < img.max() <= 2.5 and img.min() >= -0.05
    assert claimed == set(lc.REGIMES)


def test_windows_cover_the_lengths_and_placements():
    for H in (33, 48, 64, 88, 95, 1080):
        ws = lc.windows(H)
        lengths = {r1 - r0 for r0, r1 in ws}
        assert {n for n in (1, 5, 16, 31, 32, 33, H) if n <= H} == lengths
        assert all(0 <= r0 < r1 <= H for r0, r1 in ws)
        assert any(r0 % 16 == 0 and r0 > 0 for r0, _ in ws) and any(r0 % 16 for r0, _ in ws)
        assert any(r1 == H for _, r1 in ws)
        for r0, r1 in ws:
            for mode in ("all", "halo", "empty"):
                c0, c1 = lc.count_rows(r0, r1, mode)
                assert r0 <= c0 <= c1 <= r1
                if mode == "empty":
                    assert c0 == c1
                if mode == "halo" and r1 - r0 >= 3:
                    assert r0 < c0 < c1 < r1
