"""-m gpu: the fused L1 + SSIM loss kernel (csrc/loss.cu) on tile-row strips with halo windows -- border.py's arithmetic,
which needs no communication to test -- and at the shapes where its 32-pixel tiling goes wrong, against an fp64 autograd
evaluation of tests/torch_ref.ssim_l1_loss and the fp32 oracle.

Shapes: image widths below the 11-pixel window, around the 32-pixel tile and ragged; strips of 5-6 rows; H not a
multiple of 16; images in [-0.05, 1.2]; ground truth with flat 0 and 255 regions (and flat image regions over part of
them), where the SSIM denominators' variances vanish."""
import numpy as np
import pytest
import torch

import gpu_util as gu
import torch_ref
from gs_b200 import border, ops
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

LAMBDA = 0.2
OUTLIER_FRAC = 2e-4   # the outlier allowance of test_gpu_parity.py


@pytest.fixture(scope="module")
def o32():
    return Oracle(np.float32)


def make_pair(H, W, seed):
    rng = np.random.default_rng(seed)
    img = rng.uniform(-0.05, 1.2, (3, H, W)).astype(np.float32)
    gt = rng.integers(0, 256, (3, H, W), dtype=np.uint8)
    gt[:, :H // 3, :(W + 2) // 3] = 0
    gt[:, H // 2:, W // 2:] = 255
    img[:, :H // 4, :(W + 3) // 4] = 0.0          # flat image over flat ground truth: both variances ~0
    img[:, H // 2 + 3:, W // 2 + 2:] = 1.0
    return img, gt


def tile_cuts(H):
    return list(range(0, H, 16)) + [H]


# (H, W, strip boundaries in pixel rows): tile-row strips whose last strip has 5 or 6 rows, and hand cuts into 5-6 row
# strips; every strip has >= border.HALF_WINDOW rows, as add_remote_border_rows requires
SHAPES = [
    (53, 7, tile_cuts(53)),
    (38, 31, tile_cuts(38)),
    (70, 32, [0, 5, 11, 16, 32, 37, 43, 48, 64, 70]),
    (45, 33, [0, 6, 11, 16, 21, 27, 32, 38, 45]),
    (101, 211, tile_cuts(101)),
    (150, 211, [0, 16, 22, 27, 48, 96, 112, 144, 150]),
]


def fp64_reference(img, gt, rows, n_pixels):
    """fp64 autograd of the strip loss on rows [r0, r1) (zero padded there) -> (l1, ssim, d loss / d image)."""
    r0, r1 = rows
    x = torch.tensor(img[:, r0:r1], dtype=torch.float64, requires_grad=True)
    y = torch.tensor(gt[:, r0:r1], dtype=torch.float64) / 255.0
    loss, l1, ss = torch_ref.ssim_l1_loss(x, y, n_pixels, LAMBDA)
    loss.backward()
    g = np.zeros(img.shape, np.float64)
    g[:, r0:r1] = x.grad.numpy()
    return float(l1), float(ss), g


def kernel_loss(img, gt, r0, r1, c0, c1, x=None):
    """ops.fused_l1_ssim on window rows [r0, r1), counting [c0, c1); backward of (1 - lambda) Ll1 + lambda (1 - ssim)
    accumulates into x.grad."""
    if x is None:
        x = gu.to_dev(img).requires_grad_(True)
    l1, ss = ops.fused_l1_ssim(x, gu.to_dev(np.ascontiguousarray(gt[:, r0:r1])), r0, r1, c0, c1)
    ((1 - LAMBDA) * l1 + LAMBDA * (1 - ss)).backward()
    return float(l1), float(ss), x


@pytest.mark.parametrize("H,W,cuts", SHAPES)
def test_loss_halo_strips_add_up_to_the_full_image(o32, H, W, cuts):
    img, gt = make_pair(H, W, seed=H * 1000 + W)
    l1_full, ss_full, xf = kernel_loss(img, gt, 0, H, 0, H)
    g_full = gu.npy(xf.grad)
    # one strip per rank: window widened by the 5 halo rows a neighbour would send, only the strip's own rows counted
    x = gu.to_dev(img).requires_grad_(True)
    l1_sum, ss_sum = 0.0, 0.0
    for s, (y0, y1) in enumerate(zip(cuts, cuts[1:])):
        assert y1 - y0 >= border.HALF_WINDOW
        r0 = y0 - border.HALF_WINDOW if s > 0 else y0
        r1 = min(y1 + border.HALF_WINDOW, H) if y1 < H else y1
        l1, ss, _ = kernel_loss(img, gt, r0, r1, y0, y1, x)
        l1_sum += l1
        ss_sum += ss
    g_sum = gu.npy(x.grad)
    # each strip's sums are exact up to the rounding of its fp32 result
    n = len(cuts) - 1
    assert abs(l1_sum - l1_full) <= 1e-7 * n * abs(l1_full) + 1e-9, (l1_sum, l1_full)
    assert abs(ss_sum - ss_full) <= 1e-7 * n * abs(ss_full) + 1e-9, (ss_sum, ss_full)
    # Per pixel the window sums run in the same order whatever the window origin, and a counted row's 11-row
    # neighbourhood lies inside its strip's window.  So a row whose gradient gathers only SSIM terms of its own strip
    # (rows [y0 + 5, y1 - 5), or up to an image edge) equals the full-image call bit for bit: the other strips' windows
    # do not reach it and contribute exact zeros.  Rows within 5 of a strip boundary sum two strips' partial gradients,
    # which rounds differently from the full-image call's single sum.
    interior = np.zeros(H, bool)
    for y0, y1 in zip(cuts, cuts[1:]):
        a = y0 if y0 == 0 else y0 + border.HALF_WINDOW
        b = y1 if y1 == H else y1 - border.HALF_WINDOW
        interior[a:max(a, b)] = True
    assert np.array_equal(g_sum[:, interior], g_full[:, interior])
    frac, _ = gu.rel_report(f"strips {H}x{W}: summed grad vs full-image call", g_sum, g_full)
    assert frac <= OUTLIER_FRAC
    # both against fp64 and the fp32 oracle of the full image
    gtf = np.clip(gt.astype(np.float32) / np.float32(255), 0, 1)
    ref32 = o32.loss(img, gtf, H * W, LAMBDA)
    ref64 = fp64_reference(img, gt, (0, H), H * W)
    gu.check_vs_fp64(f"strips {H}x{W} full", (l1_full, ss_full, g_full), ref32, ref64)
    gu.check_vs_fp64(f"strips {H}x{W} summed", (l1_sum, ss_sum, g_sum), ref32, ref64)


@pytest.mark.parametrize("H,W,cuts", SHAPES)
def test_loss_edge_shapes_vs_fp64(o32, H, W, cuts):
    """The live path's strip loss (no halo: zero padded at the strip edges, every window row counted) at the edge shapes:
    the whole image, a 5-6 row strip, and a strip ending at H."""
    img, gt = make_pair(H, W, seed=H * 1000 + W + 1)
    small = min(zip(cuts, cuts[1:]), key=lambda r: r[1] - r[0])
    for r0, r1 in {(0, H), small, (cuts[-2], H), (cuts[1], H)}:
        l1, ss, x = kernel_loss(img, gt, r0, r1, r0, r1)
        g = gu.npy(x.grad)
        assert (g[:, :r0] == 0).all() and (g[:, r1:] == 0).all()
        gtf = np.clip(gt[:, r0:r1].astype(np.float32) / np.float32(255), 0, 1)
        ol1, oss, og = o32.loss(img[:, r0:r1], gtf, H * W, LAMBDA)
        og_full = np.zeros(img.shape, np.float32)
        og_full[:, r0:r1] = og
        gu.check_vs_fp64(f"strip [{r0},{r1}) of {H}x{W}", (l1, ss, g), (ol1, oss, og_full),
                         fp64_reference(img, gt, (r0, r1), H * W))
