"""-m gpu: the image-space arithmetic the reference performs in torch, against torch on the device and against fp64.

1. The ground truth's unit.  The reference forms `original_image / 255.0` on CUDA uint8 tensors; torch evaluates that
   as a multiply by the fp32 reciprocal, fl32(g * fl32(1/255)), which is one ulp above the IEEE quotient fl32(g / 255)
   on 126 of the 256 byte values (eval_ref.gt_hat).  Pinned here on the device, with the CPU's `div(255)` (metrics.py's
   tf.to_tensor) the IEEE quotient.  Every loss entry point sees a render equal to that ground truth as an exact match
   (L1 gradient +0, Ll1 0) and one ulp either side as a sign; the eval kernel scores it 0 / +inf and sums the ulps
   exactly; render.py's 8-bit round trip of it returns g; and the 8-bit quantizer equals torch's save_image sequence
   on all 2^32 fp32 bit patterns.
2. The eval and image-metric kernels at their limits against the torch-float64 forms of eval_ref.slots and
   metrics_ref.slots (pinned to the numpy forms on the CPU): widths and heights on and beside the 32-column chunk, the
   11-tap window, the 2048-pixel stride and 16-row tiles; 1080p and 4K; 64-view batches with empty views; windows and
   ground-truth strips larger than needed and at odd byte offsets; inf, -0, subnormals, NaN.  Slots within 1e-12
   relative and +0.0 outside the local rows; finalize equal to a host fp64 sum of the slots in row order (PSNR within
   4 ulp: the device log10 is not correctly rounded); strips of uneven simulated ranks summing to the whole view bit
   for bit."""
import math
import time

import numpy as np
import pytest
import torch

import eval_ref
import metrics_ref
from gs_b200 import _lib, image_halo, ops

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BLOCK_Y = 16

G = np.arange(256, dtype=np.uint8)
QUOTIENT = G.astype(np.float32) / np.float32(255)          # IEEE fl32(g / 255)
PRODUCT = G.astype(np.float32) * eval_ref.INV255           # fl32(g * fl32(1/255))
DIFFER = [int(v) for v in np.flatnonzero(PRODUCT != QUOTIENT)]


@pytest.fixture(scope="module", autouse=True)
def report():
    """Reports the file's runtime and peak device memory."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[image arith] {time.perf_counter() - t0:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB on {torch.cuda.get_device_name(0)}")


def u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def u64(t):
    return t.detach().contiguous().view(torch.int64)


def device_gt_hat(gt_dev):
    """The reference's expression, evaluated by torch on the device."""
    return torch.clamp(gt_dev / 255.0, 0.0, 1.0)


# ---- 1a ----------------------------------------------------------------------------------------------------------
def test_device_quotient_is_the_reciprocal_product():
    dev = device_gt_hat(torch.arange(256, dtype=torch.uint8, device=DEV)).cpu().numpy()
    print(f"\n[image arith] fl32(g * fl32(1/255)) != fl32(g / 255) on {len(DIFFER)} byte values: {DIFFER}")
    assert np.array_equal(u32(dev), u32(PRODUCT)), np.flatnonzero(u32(dev) != u32(PRODUCT)).tolist()
    assert not np.array_equal(u32(dev), u32(QUOTIENT))
    assert len(DIFFER) == 126 and np.array_equal(PRODUCT[DIFFER], np.nextafter(QUOTIENT[DIFFER], np.float32(2)))
    assert np.array_equal(u32(eval_ref.gt_hat_torch(torch.arange(256, dtype=torch.uint8, device=DEV)).cpu().numpy()),
                          u32(PRODUCT))
    # metrics.py's tf.to_tensor divides on the CPU: the IEEE quotient, which k_image_metric_sums' table keeps
    cpu = torch.arange(256, dtype=torch.uint8).float().div(255).numpy()
    assert np.array_equal(u32(cpu), u32(QUOTIENT))
    assert np.array_equal(u32(metrics_ref.unit(G).astype(np.float32)), u32(QUOTIENT))


# ---- 1b: every loss entry point on a render equal to the device ground truth, and one ulp either side ---------------
H_L, W_L = 40, 32          # 1280 pixels per channel: each byte value 5 times; tile rows of 16, 16 and 8
# per view (row0, row1, count_row0, count_row1): the image, one 16-row tile, a window with halo rows, no rows
ROWS_L = [(0, H_L, 0, H_L), (16, 32, 16, 32), (3, 40, 8, 35), (0, 0, 0, 0)]
GL1 = np.array([0.8, 1e3, 0.37, 5.0], np.float32)          # positive: a zero sign gives +0, not -0


def every_byte_image(H, W, seed):
    """(3,H,W) uint8 holding every byte value in every channel, each channel a different permutation."""
    rng = np.random.default_rng(seed)
    base = np.tile(G, -(-H * W // 256))[:H * W]
    assert H * W >= 256
    return np.stack([rng.permutation(base) for _ in range(3)]).reshape(3, H, W)


def named(values):
    """A failure's byte values, named when they are the ones where the product and the quotient differ."""
    v = sorted(values)
    return f"the {len(DIFFER)} values where fl32(g * fl32(1/255)) != fl32(g / 255)" if v == DIFFER else v


def moved(y, kind):
    return {"equal": y, "above": torch.nextafter(y, torch.full_like(y, math.inf)),
            "below": torch.nextafter(y, torch.full_like(y, -math.inf))}[kind]


def expected_grad(x, y, rows4, v):
    """fl32(g_l1 * fl32(1/(3HW))) * sgn(x - y) on the counted rows, +0 elsewhere."""
    H, W = x.shape[1:]
    step = np.float32(GL1[v] * np.float32(1.0 / (3.0 * H * W)))
    r0, r1, c0, c1 = rows4
    out = np.zeros(x.shape, np.float32)
    sgn = np.sign(x.astype(np.float64) - y.astype(np.float64)).astype(np.float32)
    out[:, c0:c1] = step * sgn[:, c0:c1]
    return out


def single_view_abi(image, gt_strip, r, det, v):
    """gs_loss_forward[_det] + gs_loss_backward on one view; outputs NaN-filled first -> (out (2,), dimg (3,H,W))."""
    H, W = image.shape[1:]
    r0, r1, c0, c1 = r
    tb = _lib.query("gs_loss_temp_bytes_det" if det else "gs_loss_temp_bytes", r1 - r0, W)
    temp = torch.full((tb,), 0xA5, dtype=torch.uint8, device=DEV)
    out = torch.full((2,), math.nan, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    _lib.call("gs_loss_forward_det" if det else "gs_loss_forward", H, W, r0, r1, c0, c1, image.data_ptr(),
              gt_strip.data_ptr(), out.data_ptr(), temp.data_ptr(), tb, s)
    g = torch.tensor([GL1[v], 0.0], dtype=torch.float32, device=DEV)
    dimg = torch.full_like(image, math.nan)
    _lib.call("gs_loss_backward", H, W, r0, r1, c0, c1, image.data_ptr(), gt_strip.data_ptr(), temp.data_ptr(),
              g.data_ptr(), g.data_ptr() + 4, dimg.data_ptr(), s)
    torch.cuda.synchronize()
    return out.cpu().numpy(), dimg.cpu().numpy()


def batched_ops(images, gt_dev, det, gt_full):
    """ops.fused_l1_ssim_batched forward and backward with output gradients (g_l1[v], 0) -> (out (B,2), dimg)."""
    gts = [None if r[1] == r[0] else (gt_dev if gt_full else gt_dev[:, r[0]:r[1]].contiguous()) for r in ROWS_L]
    x = images.clone().requires_grad_(True)
    out = ops.fused_l1_ssim_batched(x, gts, ROWS_L, deterministic=det, gt_full=gt_full)
    w = torch.from_numpy(np.stack([GL1, np.zeros_like(GL1)], 1)).to(DEV)
    (out * w).sum().backward()
    return out.detach().cpu().numpy(), x.grad.cpu().numpy()


@pytest.mark.parametrize("kind", ["equal", "above", "below"])
def test_every_loss_entry_point_on_the_device_ground_truth(kind):
    """grad_ssim = 0.  equal: dL/dimage is +0 bit for bit everywhere and Ll1 exactly 0.  above / below: dL/dimage is
    +-fl32(g_l1 * fl32(1/(3HW))) bit for bit on the counted rows, with the sign of x - the device ground truth, and +0
    elsewhere.  A failure lists the ground-truth byte values whose elements differ, per entry point."""
    gt = every_byte_image(H_L, W_L, seed=5)
    gt_dev = torch.from_numpy(gt).to(DEV)
    x = moved(device_gt_hat(gt_dev), kind)
    x_np, y_np = x.cpu().numpy(), PRODUCT[gt]
    B = len(ROWS_L)
    images = x.unsqueeze(0).expand(B, -1, -1, -1).contiguous()
    bad = {}

    def judge(name, v, out, dimg):
        want = expected_grad(x_np, y_np, ROWS_L[v], v)
        if kind == "equal":
            assert not u32(want).any()
        diff = u32(dimg) != u32(want)
        if diff.any():
            bad.setdefault(name, set()).update(int(g) for g in np.unique(gt[diff]))
        if kind == "equal" and u32(np.float32(out[0])) != 0:
            bad.setdefault(name + " Ll1", set()).add(float(out[0]))

    for det in (False, True):
        for v, r in enumerate(ROWS_L):
            if r[1] > r[0]:
                out, dimg = single_view_abi(x, gt_dev[:, r[0]:r[1]].contiguous(), r, det, v)
                judge(f"gs_loss_forward{'_det' if det else ''} + gs_loss_backward", v, out, dimg)
        for gt_full in (False, True):
            out, dimg = batched_ops(images, gt_dev, det, gt_full)
            name = f"gs_loss_forward_batched{'_gt_full' if gt_full else ''}{'_det' if det else ''}" \
                   f" + gs_loss_backward_batched{'_gt_full' if gt_full else ''}"
            for v in range(B):
                judge(name, v, out[v], dimg[v])
    assert not bad, {k: named(s) for k, s in bad.items()}


# ---- 1c: the eval kernel on the device ground truth -------------------------------------------------------------
H_E, W_E = 17, 129      # tile row 0: 16 x 129 = 2064 pixels, past one 2048-pixel stride; tile row 1: one row


@pytest.mark.parametrize("kind", ["equal", "above", "below"])
def test_eval_on_the_device_ground_truth(kind):
    """Four batches of 64 views, view v a constant ground truth of byte value 64 b + v.  equal: every slot is +0.0, L1
    +0.0 and PSNR +inf.  above / below: every S1 (S2) is the exact fp64 sum of the ulps |clamp(x) - g^| (their
    squares), and L1 the host's division of their sum.  A failure lists the byte values whose views differ."""
    bad = set()
    for b in range(4):
        vals = torch.arange(64 * b, 64 * b + 64, dtype=torch.uint8, device=DEV)
        gt = vals.view(64, 1, 1, 1).expand(64, 3, H_E, W_E).contiguous()
        x = moved(device_gt_hat(gt), kind)
        slots = ops.eval_sums_batched(x, list(gt.unbind(0)), [(0, H_E)] * 64, [0] * 64)
        out = ops.eval_finalize(slots, H_E, W_E).cpu().numpy()
        slots = slots.cpu().numpy()
        t = np.abs(np.clip(x[:, 0, 0, 0].double().cpu().numpy(), 0, 1) - eval_ref.gt_hat(vals.cpu().numpy()))
        for v in range(64):
            n = np.array([BLOCK_Y * W_E, (H_E - BLOCK_Y) * W_E], np.float64)
            want = np.zeros((2, 3, 2))
            want[:, :, 0] = (n * t[v])[:, None]            # n ulps: exact (n < 2^12, t a power of two)
            want[:, :, 1] = (n * t[v] * t[v])[:, None]
            l1 = (sum(want[:, c, 0].sum() for c in range(3))) / (3.0 * (float(H_E) * W_E))
            ok = np.array_equal(slots[v].view(np.int64), want.view(np.int64)) and same_double(out[v, 0], l1)
            if kind == "equal":
                ok = ok and out[v, 1] == math.inf
            if not ok:
                bad.add(64 * b + v)
    assert not bad, named(bad)


# ---- 1d: render.py's 8-bit round trip of the device ground truth --------------------------------------------------
def test_round_trip_of_the_device_ground_truth():
    """render.py saves clamp(gt / 255.0, 0, 1) through save_image: on the device that returns g for all 256 values, by
    torch's sequence and by the kernel, so the metric kernels may read g itself."""
    g = torch.arange(256, dtype=torch.uint8, device=DEV).view(1, 16, 16).expand(3, 16, 16).contiguous()
    g[1] = g[1].flip(0)
    saved = device_gt_hat(g)
    assert torch.equal(metrics_ref.save_image_quantize(saved), g)
    out = torch.full((3, 16, 16), 7, dtype=torch.uint8, device=DEV)
    ops.quantize_u8_batched(saved.unsqueeze(0), [(0, 16)], [out], [0])
    assert torch.equal(out, g)


# ---- 1e: the quantizer on every fp32 bit pattern -------------------------------------------------------------------
def test_quantizer_on_every_fp32_bit_pattern():
    """All 2^32 patterns through ops.quantize_u8_batched in (1, 3, 8192, 8192) chunks (2^26 pixels per channel: the
    grid-stride loop runs 64 times), against metrics_ref.save_image_quantize on the device byte for byte.  NaNs, whose
    uint8 cast torch leaves undefined, are taken out of that comparison and must give 0."""
    side = 8192
    n = 3 * side * side
    out = torch.empty((3, side, side), dtype=torch.uint8, device=DEV)
    bad, nans = 0, 0
    examples = []
    for start in range(0, 1 << 32, n):
        a = torch.arange(start, start + n, dtype=torch.int64, device=DEV) & 0xFFFFFFFF   # the last chunk wraps
        x = (a - (a >= 1 << 31).long() * (1 << 32)).to(torch.int32).view(torch.float32).view(1, 3, side, side)
        del a
        out.fill_(0xA5)
        ops.quantize_u8_batched(x, [(0, side)], [out], [0])
        want = metrics_ref.save_image_quantize(x[0])
        nan = torch.isnan(x[0])
        nans += int(nan.sum())
        diff = (out != want) & ~nan | nan & (out != 0)
        k = int(diff.sum())
        if k:
            bad += k
            idx = torch.nonzero(diff.view(-1))[:4, 0]
            examples += [(hex(int(x.view(torch.int32).view(-1)[i]) & 0xFFFFFFFF), int(out.view(-1)[i]),
                          int(want.view(-1)[i])) for i in idx]
        del x, want, nan, diff
    assert nans >= 2 * ((1 << 23) - 1)
    assert bad == 0, (bad, examples[:8])


# ---- 2. the eval and image-metric kernels at their limits ---------------------------------------------------------
def host_sum(sl, col):
    s = 0.0
    for r in range(sl.shape[0]):
        s += float(sl[r, col])
    return s


def same_double(a, b):
    return np.float64(a).view(np.int64) == np.float64(b).view(np.int64)


def within_ulp(a, b, k):
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    if math.isinf(a) or math.isinf(b):
        return a == b
    return abs(a - b) <= k * math.ulp(max(abs(a), abs(b)))


def live_rows(H, rows):
    TY = (H + BLOCK_Y - 1) // BLOCK_Y
    y0 = np.arange(TY) * BLOCK_Y
    return (y0 >= rows[0]) & (np.minimum(y0 + BLOCK_Y, H) <= rows[1])


def check_slots(tag, got, want, H, rows):
    """got, want: (TILE_Y, ...) fp64 tensors; want over all rows.  Live rows within 1e-12 (NaN where want is NaN),
    the others +0.0."""
    live = torch.from_numpy(live_rows(H, rows)).to(got.device)
    g, w = got[live], want[live]
    nan = torch.isnan(w)
    assert torch.equal(torch.isnan(g), nan), tag
    assert torch.allclose(g[~nan], w[~nan], rtol=1e-12, atol=0), (tag, float(((g - w).abs() / w.abs()).nan_to_num().max()))
    assert not u64(got[~live]).any(), (tag, "not +0.0 outside the rows")


# image metrics
W_M = [1, 2, 5, 6, 10, 11, 12, 31, 32, 33, 63, 64, 65, 1920, 3840]
H_M = [1, 5, 6, 10, 11, 15, 16, 17, 21, 1080, 2160]
CONTENTS = ["noisy", "checker", "grey", "same", "zero", "full"]


def content(kind, H, W, seed):
    """(q, g) (3,H,W) uint8 on the device.  same: q = g (SSIM exactly 1, PSNR +inf); zero / full: both 0 / 255; grey:
    q = 100, g = 160 (both variances 0 away from the border); checker: q a 0/255 checkerboard, g its inverse; noisy: g
    uniform, q = g + noise in [-12, 12], clamped."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    if kind in ("noisy", "same"):
        g = torch.randint(0, 256, (3, H, W), generator=gen, device=DEV, dtype=torch.uint8)
        if kind == "same":
            return g, g.clone()
        e = torch.randint(-12, 13, (3, H, W), generator=gen, device=DEV)
        return (g.int() + e).clamp(0, 255).to(torch.uint8), g
    if kind == "checker":
        yy, xx = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
        q = ((yy + xx) % 2 * 255).to(torch.uint8).expand(3, H, W).contiguous()
        return q, 255 - q
    val = {"grey": (100, 160), "zero": (0, 0), "full": (255, 255)}[kind]
    return (torch.full((3, H, W), val[0], dtype=torch.uint8, device=DEV),
            torch.full((3, H, W), val[1], dtype=torch.uint8, device=DEV))


def row_choices(H):
    """The whole image, the first tile row, the last, the rows between them, none."""
    TY = (H + BLOCK_Y - 1) // BLOCK_Y
    last = (BLOCK_Y * (TY - 1), H)
    inner = (BLOCK_Y, BLOCK_Y * (TY - 1)) if TY >= 3 else (0, H)
    return [(0, H), (0, min(BLOCK_Y, H)), last, inner, (0, 0)]


def metric_window(q, g, rows, H, how):
    """(window, win_row0): halo = exactly rows [max(0, row0 - 5), min(H, row1 + 5)); whole = the image; odd = the halo
    window at an odd byte offset of a larger buffer."""
    a, b = (0, H) if how == "whole" else image_halo.window_rows(rows, H)
    win = torch.cat([q[:, a:b], g[:, a:b]]).contiguous()
    if how == "odd":
        buf = torch.zeros((win.numel() + 2,), dtype=torch.uint8, device=DEV)
        buf[1:1 + win.numel()] = win.view(-1)
        win = buf[1:1 + win.numel()].view(win.shape)
        assert win.data_ptr() % 2 == 1 and win.is_contiguous()
    return win, a


def check_metric_finalize(tag, slots, out, H, W):
    """finalize = the host fp64 sum of the slots in row order over 3 H W (SSIM bit for bit, PSNR within 4 ulp)."""
    n3hw = 3.0 * H * W
    for v in range(slots.shape[0]):
        sl = slots[v].cpu().numpy()
        ssim, s = host_sum(sl, 0) / n3hw, host_sum(sl, 1)
        psnr = math.inf if s == 0 else 20.0 * math.log10(1.0 / math.sqrt(s / (255.0 * 255.0 * n3hw)))
        assert same_double(float(out[v, 0]), ssim), (tag, v, float(out[v, 0]), ssim)
        assert within_ulp(float(out[v, 1]), psnr, 4), (tag, v, float(out[v, 1]), psnr)


@pytest.mark.parametrize("W", W_M)
def test_image_metric_sums_at_every_shape(W):
    """For each H: six views, one per content, over the row choices in rotation (the first and last tile rows, the
    rows between, the image, none) with halo, whole-image and odd-offset windows; slots against
    metrics_ref.slots_torch, and finalize of the whole views against the host sum of their slots."""
    for i, H in enumerate(H_M):
        tag = f"{H}x{W}"
        pairs = [content(k, H, W, seed=1000 * i + W + j) for j, k in enumerate(CONTENTS)]
        choices = row_choices(H)
        rows = [choices[(i + j) % len(choices)] for j in range(len(CONTENTS))]
        wins, w0 = [], []
        for j, ((q, g), r) in enumerate(zip(pairs, rows)):
            if r[1] == r[0]:
                wins.append(None)
                w0.append(0)
                continue
            w, a = metric_window(q, g, r, H, ("halo", "whole", "odd")[(i + j) % 3])
            wins.append(w)
            w0.append(a)
        slots = ops.image_metric_sums_batched(wins, w0, rows, H)
        for j, ((q, g), r) in enumerate(zip(pairs, rows)):
            check_slots(f"{tag} {CONTENTS[j]} rows {r}", slots[j], metrics_ref.slots_torch(q, g), H, r)
        full = ops.image_metric_sums_batched([torch.cat([q, g]) for q, g in pairs], [0] * len(pairs),
                                             [(0, H)] * len(pairs), H)
        out = ops.image_metric_finalize(full, H, W).cpu()
        check_metric_finalize(tag, full, out, H, W)
        for j, k in enumerate(CONTENTS):
            if k in ("same", "zero", "full"):
                assert out[j, 0].item() == 1.0 and out[j, 1].item() == math.inf, (tag, k, out[j].tolist())
        del pairs, wins, slots, full


def test_image_metric_sums_64_views():
    """B = 64, empty views first, in the middle and last; every view its own content and rows."""
    H, W, B = 53, 45, 64
    choices = row_choices(H)
    rows = [choices[v % 4] for v in range(B)]
    for v in (0, B // 2, B - 1):
        rows[v] = (0, 0)
    pairs = [content(CONTENTS[v % len(CONTENTS)], H, W, seed=v) for v in range(B)]
    wins, w0 = [], []
    for v, ((q, g), r) in enumerate(zip(pairs, rows)):
        w, a = metric_window(q, g, r, H, ("halo", "whole", "odd")[v % 3]) if r[1] > r[0] else (None, 0)
        wins.append(w)
        w0.append(a)
    slots = ops.image_metric_sums_batched(wins, w0, rows, H)
    for v, ((q, g), r) in enumerate(zip(pairs, rows)):
        check_slots(f"view {v} rows {r}", slots[v], metrics_ref.slots_torch(q, g), H, r)


# eval
W_V = [1, 2, 127, 128, 129, 1920, 3840]
H_V = [1, 15, 17, 1080, 2160]


def eval_image(H, W, seed, nan_at=None):
    """(3,H,W) fp32 render on the device: uniform in [-0.3, 1.3] with +-inf, -0, subnormals, values above 1, and x equal
    to and one ulp off the ground truth scattered; optionally one NaN at nan_at = (c, y, x)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randint(0, 256, (3, H, W), generator=gen, device=DEV, dtype=torch.uint8)
    x = torch.rand((3, H, W), generator=gen, device=DEV) * 1.6 - 0.3
    f = x.view(-1)
    special = torch.tensor([math.inf, -math.inf, -0.0, 1e-40, -1e-40, 2.0 ** -149, 1.0 + 2.0 ** -23, 7.5, 0.0, 1.0],
                           device=DEV)
    f[::7] = special.repeat(-(-f[::7].numel() // special.numel()))[:f[::7].numel()]
    y = device_gt_hat(g).view(-1)
    f[3::11] = y[3::11]
    f[5::13] = torch.nextafter(y[5::13], torch.full_like(y[5::13], 2.0))
    if nan_at is not None:
        x[nan_at] = math.nan
    return x, g


def gt_buffer(g, rows, H, how):
    """(gt, gt_row0): whole = the image read in place; strip = rows [row0, row1); wide = rows from 3 above row0 (when
    there are) to 5 below row1 (when there are), at an odd byte offset."""
    if how == "whole":
        return g, 0
    a, b = rows if how == "strip" else (max(0, rows[0] - 3), min(H, rows[1] + 5))
    s = g[:, a:b].contiguous()
    if how == "wide":
        buf = torch.zeros((s.numel() + 2,), dtype=torch.uint8, device=DEV)
        buf[1:1 + s.numel()] = s.view(-1)
        s = buf[1:1 + s.numel()].view(s.shape)
    return s, a


def check_eval_finalize(tag, slots, out, H, W):
    """finalize = the host fp64 sums of the slots in row order: L1 bit for bit, PSNR within 4 ulp."""
    hw = float(H) * W
    for v in range(slots.shape[0]):
        sl = slots[v].cpu().numpy().reshape(-1, 6)
        s = [host_sum(sl, k) for k in range(6)]
        l1 = (s[0] + s[2] + s[4]) / (3.0 * hw)
        with np.errstate(divide="ignore", invalid="ignore"):
            psnr = sum(20.0 * np.log10(1.0 / np.sqrt(np.float64(s[2 * c + 1]) / hw)) for c in range(3)) / 3.0
        got = float(out[v, 0])
        assert (math.isnan(got) and math.isnan(l1)) or same_double(got, l1), (tag, v, got, l1)
        assert within_ulp(float(out[v, 1]), float(psnr), 4), (tag, v, float(out[v, 1]), float(psnr))


@pytest.mark.parametrize("W", W_V)
def test_eval_sums_at_every_shape(W):
    """For each H: four views (the image read in place, a strip, a wider strip at an odd offset with gt_row0 < row0,
    none), one NaN in view 0 reaching its own tile row's slot only; slots against eval_ref.slots_torch, finalize
    against the host sum of the slots."""
    for i, H in enumerate(H_V):
        tag = f"{H}x{W}"
        TY = (H + BLOCK_Y - 1) // BLOCK_Y
        nan_row = TY // 2
        imgs = [eval_image(H, W, seed=100 * i + W + v,
                           nan_at=(1, min(H - 1, BLOCK_Y * nan_row + 3), W // 2) if v == 0 else None)
                for v in range(4)]
        choices = row_choices(H)
        rows = [(0, H), choices[1 + i % 3], choices[2 + i % 2], (0, 0)]
        hows = ["whole", "strip", "wide", None]
        gts, g0 = [], []
        for (x, g), r, how in zip(imgs, rows, hows):
            s, a = gt_buffer(g, r, H, how) if r[1] > r[0] else (None, 0)
            gts.append(s)
            g0.append(a)
        images = torch.stack([x for x, _ in imgs])
        slots = ops.eval_sums_batched(images, gts, rows, g0)
        for v, ((x, g), r) in enumerate(zip(imgs, rows)):
            check_slots(f"{tag} view {v} rows {r}", slots[v], eval_ref.slots_torch(x, g), H, r)
        s0 = slots[0].cpu()
        assert torch.isnan(s0[nan_row, 1]).all() and torch.isnan(s0).sum() == 2, tag
        check_eval_finalize(tag, slots, ops.eval_finalize(slots, H, W).cpu(), H, W)
        del imgs, images, slots


def test_eval_sums_64_views_at_1080p():
    """B = 64 at 1920x1080: every view its own rows and ground-truth buffer, empty views first, middle and last."""
    H, W, B = 1080, 1920, 64
    choices = row_choices(H)
    hows = ["whole", "strip", "wide"]
    rows = [choices[v % 4] for v in range(B)]
    for v in (0, B // 2, B - 1):
        rows[v] = (0, 0)
    images = torch.empty((B, 3, H, W), device=DEV)
    gts, g0, gfull = [], [], []
    for v in range(B):
        x, g = eval_image(H, W, seed=v)
        images[v] = x
        gfull.append(g)
        s, a = gt_buffer(g, rows[v], H, hows[v % 3]) if rows[v][1] > rows[v][0] else (None, 0)
        gts.append(s)
        g0.append(a)
    slots = ops.eval_sums_batched(images, gts, rows, g0)
    for v in range(B):
        check_slots(f"view {v} rows {rows[v]}", slots[v], eval_ref.slots_torch(images[v], gfull[v]), H, rows[v])
    check_eval_finalize("64 views", slots, ops.eval_finalize(slots, H, W).cpu(), H, W)


# strip invariance
STRIPS = [(1080, [0, 30, 68]), (1080, [0, 7, 40, 68]), (1080, [0, 1, 20, 50, 68]), (1073, [0, 33, 67, 68]),
          (1076, [0, 20, 67, 68])]


@pytest.mark.parametrize("H,bounds", STRIPS)
def test_strips_sum_to_the_whole_view(H, bounds):
    """8-bit images and no render, 1920 wide: simulated ranks own tile rows [a, b) (H = 1073 and 1076: a last strip of
    1 and 4 rows); each scores its strip from its halo window (image metrics) and its ground-truth strip (eval).  The
    strips' slots sum to the whole view's bit for bit, and so do the finalized metrics."""
    W = 1920
    q, g = content("noisy", H, W, seed=H)
    x, _ = eval_image(H, W, seed=H)
    whole_m = ops.image_metric_sums_batched([torch.cat([q, g])], [0], [(0, H)], H)
    whole_e = ops.eval_sums_batched(x.unsqueeze(0), [g], [(0, H)], [0])
    tot_m, tot_e = torch.zeros_like(whole_m), torch.zeros_like(whole_e)
    for a, b in zip(bounds, bounds[1:]):
        r = (BLOCK_Y * a, min(BLOCK_Y * b, H))
        w, w0 = metric_window(q, g, r, H, "halo")
        tot_m += ops.image_metric_sums_batched([w], [w0], [r], H)
        tot_e += ops.eval_sums_batched(x.unsqueeze(0), [g[:, r[0]:r[1]].contiguous()], [r], [r[0]])
    assert torch.equal(u64(tot_m), u64(whole_m)) and torch.equal(u64(tot_e), u64(whole_e))
    assert torch.equal(u64(ops.image_metric_finalize(tot_m, H, W)), u64(ops.image_metric_finalize(whole_m, H, W)))
    assert torch.equal(u64(ops.eval_finalize(tot_e, H, W)), u64(ops.eval_finalize(whole_e, H, W)))
