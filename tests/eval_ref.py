"""Definitional fp64 reference of the held-out view metrics (csrc/metrics.cu, ops.eval_sums_batched / eval_finalize), and
the reference's own scoring sequence restated in torch (train_internal.py:471-478, utils/loss_utils.py:18-19,
utils/image_utils.py:19-21).

x^ = clamp(x, 0, 1) (NaN stays NaN), g^ = the reference's gt / 255.0 on the device, fl32(g * fl32(1/255)); per tile row
and channel S1 = sum |x^ - g^| and S2 = sum (x^ - g^)^2 in fp64; L1 = (S1_0 + S1_1 + S1_2) / (3 H W);
PSNR = mean_c 20 log10(1 / sqrt(S2_c / (H W))) -- the per-channel PSNR averaged.

The reference divides a CUDA uint8 tensor by the Python scalar 255.0, which torch evaluates as a multiply by the fp32
reciprocal; that differs from the IEEE quotient fl32(g / 255) by one ulp on 126 of the 256 bytes
(tests/test_image_arith_gpu.py pins both on the device)."""
import numpy as np
import torch

BLOCK_Y = 16
INV255 = np.float32(1.0) / np.float32(255.0)     # fl32(1/255), the reciprocal torch multiplies by on the device


def gt_hat(gt_u8):
    """The reference's gt / 255.0 on a CUDA uint8 image, fl32(g * fl32(1/255)), as float64."""
    return (np.asarray(gt_u8).astype(np.float32) * INV255).astype(np.float64)


def gt_hat_torch(gt_u8):
    """gt_hat as an fp32 tensor on gt_u8's device: bit for bit `gt_u8 / 255.0` on a GPU, and the same product on the CPU,
    where torch's `/ 255.0` would be the IEEE quotient instead."""
    g = torch.as_tensor(gt_u8)
    return g.float() * torch.tensor(INV255, device=g.device)


def slots(image, gt_u8, rows=None):
    """image (3,H,W) float32, gt_u8 (3,H,W) uint8, rows (row0, row1) local pixel rows (None = all)
    -> (TILE_Y, 3, 2) float64: per tile row and channel (S1, S2) over the row's pixels, 0 outside the local rows."""
    image = np.asarray(image, dtype=np.float32)
    H = image.shape[1]
    row0, row1 = (0, H) if rows is None else rows
    x = np.minimum(np.maximum(image.astype(np.float64), 0.0), 1.0)   # np.maximum / np.minimum propagate NaN
    d = x - gt_hat(gt_u8)
    TY = (H + BLOCK_Y - 1) // BLOCK_Y
    out = np.zeros((TY, 3, 2), dtype=np.float64)
    for r in range(TY):
        y0, y1 = r * BLOCK_Y, min((r + 1) * BLOCK_Y, H)
        if y0 < row0 or y1 > row1:
            continue
        blk = d[:, y0:y1, :].reshape(3, -1)
        out[r, :, 0] = np.abs(blk).sum(axis=1)
        out[r, :, 1] = (blk * blk).sum(axis=1)
    return out


def finalize(sl, H, W):
    """(TILE_Y, 3, 2) slots -> (L1, PSNR), the rows added in order."""
    s = np.zeros((3, 2), dtype=np.float64)
    for r in range(sl.shape[0]):
        s = s + sl[r]
    hw = float(H) * float(W)
    with np.errstate(divide="ignore"):
        l1 = (s[0, 0] + s[1, 0] + s[2, 0]) / (3.0 * hw)
        psnr = sum(20.0 * np.log10(1.0 / np.sqrt(s[c, 1] / hw)) for c in range(3)) / 3.0
    return float(l1), float(psnr)


def slots_torch(image, gt_u8, rows=None):
    """slots() in torch float64 on the tensors' device, for images too large for numpy: image (3,H,W) float32 tensor,
    gt_u8 (3,H,W) uint8 tensor on the same device -> (TILE_Y, 3, 2) float64 tensor."""
    H, W = image.shape[1:]
    row0, row1 = (0, H) if rows is None else rows
    TY = (H + BLOCK_Y - 1) // BLOCK_Y
    d = torch.clamp(image.double(), 0.0, 1.0) - gt_hat_torch(gt_u8).double()   # torch.clamp propagates NaN
    d = torch.nn.functional.pad(d, (0, 0, 0, TY * BLOCK_Y - H)).view(3, TY, BLOCK_Y * W)
    out = torch.stack([d.abs().sum(2), (d * d).sum(2)], 2).transpose(0, 1).contiguous()
    y0 = torch.arange(TY, device=image.device) * BLOCK_Y
    live = (y0 >= row0) & (torch.clamp(y0 + BLOCK_Y, max=H) <= row1)
    out[~live] = 0.0
    return out


def reference_sequence(image, gt_u8, dtype=torch.float64):
    """training_report's scoring of one view: torch.clamp -> l1_loss(...).mean() -> psnr(...).mean(), with the images in
    `dtype` after the reference's fp32 gt / 255.0 as the device forms it (gt_hat_torch, on any device).
    -> (L1, PSNR) floats."""
    image = torch.as_tensor(image).to(dtype)
    gt = torch.clamp(gt_hat_torch(gt_u8), 0.0, 1.0).to(dtype)
    image = torch.clamp(image, 0.0, 1.0)
    l1 = torch.abs(image - gt).mean()                                       # l1_loss
    mse = ((image - gt) ** 2).view(image.shape[0], -1).mean(1, keepdim=True)  # psnr
    psnr = 20 * torch.log10(1.0 / torch.sqrt(mse))
    return float(l1.mean().double()), float(psnr.mean().double())
