"""fp64 reference of the strip loss's counted-rows contract (csrc/loss.cu, ops.fused_l1_ssim):

  the maps see the window rows [row0, row1) of the image, zero padded at the window's edges;
  Ll1  = sum over the counted rows [count_row0, count_row1) of |x - y|      / (3 H W)
  ssim = sum over the counted rows of ssim_map(x, y)                        / (3 H W)

normalised by the FULL image's 3 H W.  Written with F.conv2d exactly as tests/torch_ref.ssim_l1_loss (which counts every
window row), so the two agree bit for bit when the counted rows are the window; tests/test_loss_ref.py pins it on CPU.
Works on any device and in fp32 too (the fp32 evaluation is a noise floor for the kernels, not a reference)."""
import numpy as np
import torch
import torch.nn.functional as F

C1, C2 = 0.01 ** 2, 0.03 ** 2


def gauss_taps(dtype=torch.float64, device="cpu"):
    """The 11 window taps of utils/loss_utils.py: fp32 exp values normalised in fp32."""
    g = torch.tensor([np.exp(-((k - 5) ** 2) / (2 * 1.5 ** 2)) for k in range(11)], dtype=torch.float32)
    return (g / g.sum()).to(dtype=dtype, device=device)


def ssim_map(x, y):
    """x, y: (C, rows, W) window -> (1, C, rows, W) SSIM map, zero padding at the window edges."""
    c = x.shape[0]
    g = gauss_taps(x.dtype, x.device)
    w2 = (g[:, None] @ g[None, :]).expand(c, 1, 11, 11).contiguous()
    x, y = x[None], y[None]
    mu1, mu2 = F.conv2d(x, w2, padding=5, groups=c), F.conv2d(y, w2, padding=5, groups=c)
    s1 = F.conv2d(x * x, w2, padding=5, groups=c) - mu1 * mu1
    s2 = F.conv2d(y * y, w2, padding=5, groups=c) - mu2 * mu2
    s12 = F.conv2d(x * y, w2, padding=5, groups=c) - mu1 * mu2
    return ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))


def strip_terms(x, y, c0, c1, n_pixels_total):
    """x, y: (C, rows, W) window (x may require grad); window-relative counted rows [c0, c1).
    -> (Ll1, ssim) 0-dim tensors, both divided by 3 * n_pixels_total."""
    m = ssim_map(x, y)
    ss = m[:, :, c0:c1].sum() / (n_pixels_total * 3)
    l1 = (x - y).abs()[:, c0:c1].sum() / (n_pixels_total * 3)
    return l1, ss


def counted_terms(img, y_win, row0, row1, c0, c1, dtype=torch.float64):
    """The per-element terms the two sums add up, over the counted rows: (|x - y|, ssim map), each (3, c1 - c0, W)."""
    img = torch.as_tensor(img)
    y_win = torch.as_tensor(y_win).to(img.device)
    x, y = img[:, row0:row1].to(dtype), y_win.to(dtype)
    l1, ss = [], []
    for ch in range(3):
        ss.append(ssim_map(x[ch:ch + 1], y[ch:ch + 1])[0, 0, c0 - row0:c1 - row0])
        l1.append((x[ch] - y[ch]).abs()[c0 - row0:c1 - row0])
    return torch.stack(l1), torch.stack(ss)


def strip_loss(img, y_win, row0, row1, c0, c1, g_l1, g_ssim, dtype=torch.float64):
    """The kernel's contract on one view, evaluated in `dtype` on img's device, one channel at a time (the channels are
    independent; this keeps a 3840x2160 fp64 graph near 1 GiB).
    img: (3, H, W) tensor or array; y_win: (3, row1 - row0, W) ground truth as the kernel sees it: the reference's
    gt / 255.0 on the device, fl32(gt * fl32(1/255)) (loss_cases.gt_float);
    rows absolute.  -> (Ll1, ssim, d(g_l1 Ll1 + g_ssim ssim) / d img as a (3, H, W) tensor)."""
    img = torch.as_tensor(img)
    y_win = torch.as_tensor(y_win).to(img.device)
    _, H, W = img.shape
    grad = torch.zeros(img.shape, dtype=dtype, device=img.device)
    l1 = ss = 0.0
    if row1 == row0:
        return l1, ss, grad
    for ch in range(3):
        x = img[ch:ch + 1, row0:row1].to(dtype).clone().requires_grad_(True)
        a, b = strip_terms(x, y_win[ch:ch + 1].to(dtype), c0 - row0, c1 - row0, H * W)
        (g_l1 * a + g_ssim * b).backward()
        grad[ch, row0:row1] = x.grad[0]
        l1 += a.item()
        ss += b.item()
    return l1, ss, grad
