"""Definitional fp64 reference of the image metrics (csrc/metrics.cu, ops.quantize_u8_batched / image_metric_sums_batched /
image_metric_finalize), and the reference's own render.py + metrics.py sequence restated in torch (render.py:127-138,
torchvision.utils.save_image's quantization, tf.to_tensor, utils/loss_utils.py:26-85, utils/image_utils.py:19-21).

q = uint8(clamp(fl(fl(clamp(x, 0, 1) * 255) + 0.5), 0, 255)), truncated (NaN -> 0); a = fl32(q / 255), b = fl32(g / 255),
promoted to fp64; the SSIM map of _ssim with the separable fp64 window WINDOW, zero padding outside the image,
C1 = 0.01^2, C2 = 0.03^2.  Per tile row: (sum of the map over the row's pixels and channels, S = sum (q - g)^2).
SSIM = the map's sum / (3 H W); PSNR = 20 log10(1 / sqrt(S / (255^2 3 H W))), pooled over the channels."""
import math

import numpy as np
import torch

BLOCK_Y = 16
HALO = 5
# the fp32 taps of gaussian(11, 1.5) as torch builds them on the CPU, as the kernel's c_ssim_w holds them
WINDOW = tuple(float.fromhex(h) for h in (
    "0x1.0d956cp-10", "0x1.f1fe02p-8", "0x1.26eb18p-5", "0x1.bff0fep-4", "0x1.b43c3ep-3", "0x1.10656p-2",
    "0x1.b43c3ep-3", "0x1.bff0fep-4", "0x1.26eb18p-5", "0x1.f1fe02p-8", "0x1.0d956cp-10"))
C1, C2 = 0.01 ** 2, 0.03 ** 2


def quantize(x):
    """float32 array -> uint8: render.py's clamp, then save_image's mul(255).add_(0.5).clamp_(0, 255).to(uint8), each
    fp32 operation rounded on its own; NaN -> 0."""
    x = np.asarray(x, dtype=np.float32)
    c = np.where(np.isnan(x), np.float32(0), np.clip(x, np.float32(0), np.float32(1))).astype(np.float32)
    t = (c * np.float32(255)).astype(np.float32)
    t = (t + np.float32(0.5)).astype(np.float32)
    return np.minimum(t, np.float32(255)).astype(np.uint8)


def unit(u8):
    """tf.to_tensor's fp32 u8 / 255, as float64."""
    return (np.asarray(u8).astype(np.float32) / np.float32(255)).astype(np.float64)


def _filter(z):
    """(3,H,W) fp64 -> the separable WINDOW filter with zero padding, fp64."""
    H, W = z.shape[-2:]
    p = np.pad(z, ((0, 0), (HALO, HALO), (HALO, HALO)))
    h = sum(WINDOW[k] * p[:, :, k:k + W] for k in range(len(WINDOW)))
    return sum(WINDOW[k] * h[:, k:k + H, :] for k in range(len(WINDOW)))


def ssim_map(q, g):
    """(3,H,W) uint8 render and ground truth -> (3,H,W) fp64 SSIM map."""
    a, b = unit(q), unit(g)
    mu1, mu2 = _filter(a), _filter(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s11, s22, s12 = _filter(a * a) - mu1_sq, _filter(b * b) - mu2_sq, _filter(a * b) - mu1_mu2
    return ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s11 + s22 + C2))


def slots(q, g, rows=None):
    """(3,H,W) uint8 q and g, rows (row0, row1) local pixel rows (None = all) -> (TILE_Y, 2) fp64: per tile row (sum of
    the map, S), 0 outside the local rows."""
    q, g = np.asarray(q), np.asarray(g)
    H = q.shape[1]
    row0, row1 = (0, H) if rows is None else rows
    m = ssim_map(q, g)
    d = q.astype(np.int64) - g.astype(np.int64)
    TY = (H + BLOCK_Y - 1) // BLOCK_Y
    out = np.zeros((TY, 2), dtype=np.float64)
    for r in range(TY):
        y0, y1 = r * BLOCK_Y, min((r + 1) * BLOCK_Y, H)
        if y0 < row0 or y1 > row1:
            continue
        out[r, 0] = m[:, y0:y1].sum()
        out[r, 1] = float((d[:, y0:y1] ** 2).sum())
    return out


def slots_torch(q, g, rows=None):
    """slots() in torch float64 on the tensors' device, for images too large for numpy: (3,H,W) uint8 tensors q and g
    on one device -> (TILE_Y, 2) float64 tensor.  a and b come from a table of unit() built on the CPU: on a GPU torch's
    u8 / 255 would multiply by fl32(1/255) instead of dividing."""
    H, W = q.shape[1:]
    row0, row1 = (0, H) if rows is None else rows
    table = torch.from_numpy(unit(np.arange(256, dtype=np.uint8))).to(q.device)
    a, b = table[q.long()], table[g.long()]
    w = torch.tensor(WINDOW, dtype=torch.float64, device=q.device)

    def filt(z):
        p = torch.nn.functional.pad(z, (HALO, HALO, HALO, HALO))
        h = sum(w[k] * p[:, :, k:k + W] for k in range(len(WINDOW)))
        return sum(w[k] * h[:, k:k + H, :] for k in range(len(WINDOW)))

    mu1, mu2 = filt(a), filt(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s11, s22, s12 = filt(a * a) - mu1_sq, filt(b * b) - mu2_sq, filt(a * b) - mu1_mu2
    m = ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s11 + s22 + C2))
    d = (q.long() - g.long()) ** 2
    TY = (H + BLOCK_Y - 1) // BLOCK_Y
    pad = TY * BLOCK_Y - H
    m = torch.nn.functional.pad(m, (0, 0, 0, pad)).view(3, TY, BLOCK_Y * W).sum((0, 2))
    d = torch.nn.functional.pad(d, (0, 0, 0, pad)).view(3, TY, BLOCK_Y * W).sum((0, 2)).double()
    out = torch.stack([m, d], 1)
    y0 = torch.arange(TY, device=q.device) * BLOCK_Y
    out[(y0 < row0) | (torch.clamp(y0 + BLOCK_Y, max=H) > row1)] = 0.0
    return out


def finalize(sl, H, W):
    """(TILE_Y, 2) slots -> (SSIM, PSNR), the rows added in order."""
    s = np.zeros((2,), dtype=np.float64)
    for r in range(sl.shape[0]):
        s = s + sl[r]
    n = 3.0 * H * W
    psnr = math.inf if s[1] == 0 else 20.0 * math.log10(1.0 / math.sqrt(s[1] / (255.0 * 255.0 * n)))
    return float(s[0] / n), float(psnr)


def reference_window():
    """create_window(11, 1) of utils/loss_utils.py:26-42, built on the CPU: (the fp32 1D taps, the fp32 2D window)."""
    g = torch.Tensor([math.exp(-((x - 11 // 2) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    w1 = (g / g.sum()).unsqueeze(1)
    return w1.reshape(-1), w1.mm(w1.t()).float()


def save_image_quantize(image):
    """render.py:127 + torchvision.utils.save_image's quantization of one (3,H,W) fp32 render, on its device."""
    return torch.clamp(image, 0.0, 1.0).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)


def reference_sequence(image, gt_u8, dtype=torch.float32):
    """render.py writes the clamped render and gt / 255 as 8-bit PNGs; metrics.py reads them with tf.to_tensor and scores
    ssim and psnr on (1,3,H,W) tensors -- here in `dtype`, on the tensors' device.  -> (SSIM, PSNR) floats."""
    q = save_image_quantize(torch.as_tensor(image))
    gq = save_image_quantize(torch.as_tensor(gt_u8).to(q.device) / 255.0)
    a = (q.float() / 255).unsqueeze(0).to(dtype)
    b = (gq.float() / 255).unsqueeze(0).to(dtype)
    window = reference_window()[1].expand(3, 1, 11, 11).contiguous().to(a.device).type_as(a)
    conv = lambda z: torch.nn.functional.conv2d(z, window, padding=11 // 2, groups=3)  # noqa: E731
    mu1, mu2 = conv(a), conv(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s11, s22, s12 = conv(a * a) - mu1_sq, conv(b * b) - mu2_sq, conv(a * b) - mu1_mu2
    m = ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s11 + s22 + C2))
    mse = ((a - b) ** 2).view(1, -1).mean(1, keepdim=True)
    psnr = 20 * torch.log10(1.0 / torch.sqrt(mse))
    return float(m.mean()), float(psnr)
