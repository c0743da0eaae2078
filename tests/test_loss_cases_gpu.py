"""-m gpu: the strip loss kernels (csrc/loss.cu) at their limits, against the fp64 reference of their counted-rows
contract (tests/loss_ref.py, pinned on CPU by tests/test_loss_ref.py) on the cases of tests/loss_cases.py.

- The batched entry points equal the single-view ones on every view (dL/dimage bit for bit, (Ll1, ssim) within one fp32
  ulp), at B = 1, 2, 5, 63, 64 with per-view windows, counted rows and output gradients, empty views and gt strips at
  odd byte offsets; and at B = 4 x 1920x1080 cut into the tile-row strips of a 4- and a 3-rank world.
- The L1 branch alone is bit-exact against its closed form, the SSIM branch alone and both together sit within the
  fp32 noise floor of fp64; full-resolution images (1920x1080, 3840x2160) through the autograd operator.
- The batched autograd operator with distinct per-view output gradients, and ops.fused_loss, equal the C ABI calls.
- Workspace: the documented size, sentinel bytes past the maps untouched, one byte short refused with nothing written.

Outputs start NaN-filled and the workspace byte-filled, so an element a kernel leaves unwritten shows.  The fp32 noise
floor is loss_ref in fp32 on the device (TF32 off): the fp32 oracle has neither counted rows nor separate L1 / SSIM
weights."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import gpu_util as gu
import loss_cases as lc
import loss_ref
from gs_b200 import _lib, division, ops

pytestmark = pytest.mark.gpu

HEADER_B = 2 * 8 * 64          # two double accumulators per view, GS_MAX_VIEWS views
SENTINEL = 0xA5
GS_ENOMEM = -3
# per-view (d loss / d Ll1, d loss / d ssim): the training weights, zero, negative, ~1e3, and only one of the two
GRADS = [(0.8, -0.2), (0.0, 0.0), (-1.5, -0.7), (1e3, 2.5e3), (0.6, 0.0), (0.0, -1.1), (-0.3, 0.9)]


@pytest.fixture(scope="module", autouse=True)
def fp32_floor_without_tf32():
    """The fp32 floor must be fp32: TF32 convolutions would put it ~1e-3 off fp64.  Also reports the file's runtime and
    peak device memory."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    torch.backends.cudnn.allow_tf32 = prev
    print(f"\n[loss cases] {time.perf_counter() - t0:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def i32(rows4):
    return (C.c_int32 * max(1, 4 * len(rows4)))(*[int(v) for r in rows4 for v in r])


def gptrs(gts):
    return (C.c_void_p * max(1, len(gts)))(*[None if g is None else g.data_ptr() for g in gts])


def map_bytes(rows4, W):
    return 9 * sum(r[1] - r[0] for r in rows4) * W * 4


def view_grads(B):
    g = [GRADS[v % len(GRADS)] for v in range(B)]
    gl1 = np.array([a * (1 + 0.013 * v) for v, (a, _) in enumerate(g)], np.float32)
    gss = np.array([b * (1 + 0.017 * v) for v, (_, b) in enumerate(g)], np.float32)
    return gl1, gss


def gt_strips(gts_full, rows4):
    """(3, rows, W) uint8 strips: every third view's strip is a slice of one shared buffer at an odd byte offset, the
    others separate allocations; None for empty views."""
    out, shared = [None] * len(rows4), [v for v, r in enumerate(rows4) if r[1] > r[0] and v % 3 == 1]
    sizes = [gts_full[v][:, rows4[v][0]:rows4[v][1]].size for v in shared]
    buf = torch.zeros((sum(sizes) + 2 * len(sizes) + 2,), dtype=torch.uint8, device=gu.DEV)
    off = 1
    for v, n in zip(shared, sizes):
        r0, r1 = rows4[v][:2]
        out[v] = buf[off:off + n].view(3, r1 - r0, -1)
        out[v].copy_(torch.from_numpy(np.ascontiguousarray(gts_full[v][:, r0:r1])))
        assert out[v].data_ptr() % 2 == 1 and out[v].is_contiguous()
        off += n + (2 if n % 2 == 0 else 1)
    for v, r in enumerate(rows4):
        if r[1] > r[0] and out[v] is None:
            out[v] = gu.to_dev(gts_full[v][:, r[0]:r[1]])
    return out


def forward_batched(images, gts, rows4, tb=None):
    """gs_loss_forward_batched with out NaN-filled and temp sentinel-filled -> (rc, out, temp)."""
    B, _, H, W = images.shape
    need = _lib.query("gs_loss_temp_bytes_batched", B, i32(rows4), W)
    temp = torch.full((need if tb is None else tb,), SENTINEL, dtype=torch.uint8, device=gu.DEV)
    out = gu.nan(B, 2)
    rc = _lib.query("gs_loss_forward_batched", B, H, W, i32(rows4), images.data_ptr(), gptrs(gts), out.data_ptr(),
                    temp.data_ptr(), temp.numel(), gu.stream())
    torch.cuda.synchronize()
    return rc, out, temp


def backward_batched(images, gts, rows4, temp, gl1, gss):
    B, _, H, W = images.shape
    dimg = torch.full_like(images, float("nan"))
    gl1_d, gss_d = gu.to_dev(gl1), gu.to_dev(gss)
    _lib.call("gs_loss_backward_batched", B, H, W, i32(rows4), images.data_ptr(), gptrs(gts), temp.data_ptr(),
              gl1_d.data_ptr(), gss_d.data_ptr(), dimg.data_ptr(), gu.stream())
    torch.cuda.synchronize()
    return dimg


def single_view(image, gt, r, gl1, gss):
    """gs_loss_forward / gs_loss_backward on one view -> (out (2,), dimg (3,H,W)), outputs NaN-filled first."""
    _, H, W = image.shape
    r0, r1, c0, c1 = r
    tb = _lib.query("gs_loss_temp_bytes", r1 - r0, W)
    temp = torch.full((tb,), SENTINEL, dtype=torch.uint8, device=gu.DEV)
    out = gu.nan(2)
    _lib.call("gs_loss_forward", H, W, r0, r1, c0, c1, image.data_ptr(), gt.data_ptr(), out.data_ptr(), temp.data_ptr(),
              tb, gu.stream())
    g = gu.to_dev(np.array([gl1, gss], np.float32))
    dimg = gu.nan(3, H, W)
    _lib.call("gs_loss_backward", H, W, r0, r1, c0, c1, image.data_ptr(), gt.data_ptr(), temp.data_ptr(), g.data_ptr(),
              g.data_ptr() + 4, dimg.data_ptr(), gu.stream())
    torch.cuda.synchronize()
    return gu.npy(out), gu.npy(dimg)


def within_ulp(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(float(a) - float(b)) <= float(np.spacing(max(abs(a), abs(b))))


def refs(image, gt_strip, r, gl1, gss):
    """(fp64 reference, fp32 floor, the fp32 floor's summed per-pixel |error| of (Ll1, ssim)) of one view; the first
    two as (Ll1, ssim, grad numpy)."""
    y = gu.to_dev(lc.gt_float(gu.npy(gt_strip)))          # fl32(gt * fl32(1/255)), as the kernel forms it
    out = []
    for dt in (torch.float64, torch.float32):
        l1, ss, g = loss_ref.strip_loss(image, y, *r, float(gl1), float(gss), dtype=dt)
        out.append((l1, ss, gu.npy(g)))
    t64, t32 = (loss_ref.counted_terms(image, y, *r, dtype=dt) for dt in (torch.float64, torch.float32))
    n3 = 3 * image.shape[1] * image.shape[2]
    out.append(tuple(float((a.double() - b).abs().sum()) / n3 for a, b in zip(t32, t64)))
    return out


def check_batch(images, gts, rows4, gl1, gss, fp64=True, tag=""):
    """Forward + backward of the batch through the C ABI against the single-view calls, the zero / NaN rules, the
    workspace sentinel and (fp64=True) the fp64 reference.  -> (out, dimg) as numpy."""
    B, _, H, W = images.shape
    rc, out, temp = forward_batched(images, gts, rows4)
    assert rc == 0, (tag, _lib.load().gs_last_error())
    maps_end = HEADER_B + map_bytes(rows4, W)
    tail = gu.npy(temp[maps_end:])
    assert tail.size == 256 and (tail == SENTINEL).all(), tag
    dimg = backward_batched(images, gts, rows4, temp, gl1, gss)
    assert (gu.npy(temp[maps_end:]) == SENTINEL).all(), tag
    out, dimg = gu.npy(out), gu.npy(dimg)
    assert not np.isnan(out).any() and not np.isnan(dimg).any(), tag
    for v, r in enumerate(rows4):
        r0, r1, c0, c1 = r
        if r1 == r0:
            assert (out[v] == 0).all() and (dimg[v] == 0).all(), (tag, v)
            continue
        assert (dimg[v][:, :r0] == 0).all() and (dimg[v][:, r1:] == 0).all(), (tag, v)
        so, sd = single_view(images[v], gts[v], r, gl1[v], gss[v])
        assert np.array_equal(dimg[v].view(np.uint32), sd.view(np.uint32)), (tag, v, r)
        assert within_ulp(out[v, 0], so[0]) and within_ulp(out[v, 1], so[1]), (tag, v, out[v], so)
        if c0 == c1:
            assert (out[v] == 0).all(), (tag, v)
        if fp64:
            r64, r32, floor = refs(images[v], gts[v], r, gl1[v], gss[v])
            gu.check_vs_fp64(f"{tag} view {v} {r}", (float(out[v, 0]), float(out[v, 1]), dimg[v]), r32, r64, floor)
    return out, dimg


def batch_rows(H, B, seed):
    """B per-view (row0, row1, count_row0, count_row1): windows of every length and placement of loss_cases.windows
    crossed with whole / halo / empty counted rows, shuffled; empty views first, in the middle and last (B >= 3)."""
    table = [(*w, *lc.count_rows(*w, m)) for w in lc.windows(H) for m in ("all", "halo", "empty")]
    order = np.random.default_rng(seed).permutation(len(table))
    rows4 = [table[order[v % len(table)]] for v in range(B)]
    if B >= 3:
        for v in (0, B // 2, B - 1):
            rows4[v] = (0, 0, 0, 0)
    return rows4


BATCHES = [(1, 64, 1), (1, 65, 33), (2, 97, 12), (5, 48, 2), (5, 31, 32), (63, 56, 31), (64, 95, 11), (64, 32, 32)]


@pytest.mark.parametrize("B,H,W", BATCHES)
def test_batched_equals_single_view_and_fp64(B, H, W):
    """H mod 32 in {0, 1, 16, 24, 31}, W in {1, 2, 11, 12, 31, 32, 33}.  B = 1 takes the single-view zeroing path of
    loss_backward_impl (rows outside the window only) and runs six windows in turn; B > 1 the whole-output one."""
    subcases = 6 if B == 1 else 1
    for s in range(subcases):
        rows4 = batch_rows(H, B, seed=B * 1000 + H * 10 + W + 7 * s)
        kinds = ["mixed", "checker", "smooth"]
        pairs = [lc.make_pair(H, W, seed=v + 31 * s, kind=kinds[v % 3] if W > 2 else "mixed") for v in range(B)]
        images = gu.to_dev(np.stack([p[0] for p in pairs]))
        gts = gt_strips([p[1] for p in pairs], rows4)
        gl1, gss = view_grads(B)
        tall = max(r[1] - r[0] for r in rows4)
        assert B == 1 or len({r[1] - r[0] for r in rows4 if r[1] > r[0]}) > 1
        check_batch(images, gts, rows4, gl1, gss, tag=f"B={B} {H}x{W} rows={rows4 if B < 6 else '...'} tall={tall}")


def test_all_views_empty():
    """No window anywhere: no kernel runs, the outputs are still written (zeros), on both zeroing paths."""
    for B in (1, 4):
        H, W = 40, 12
        images = gu.to_dev(np.random.default_rng(B).uniform(0, 1, (B, 3, H, W)).astype(np.float32))
        rows4 = [(0, 0, 0, 0)] * B
        gl1, gss = view_grads(B)
        out, dimg = check_batch(images, [None] * B, rows4, gl1, gss, fp64=False, tag=f"empty B={B}")
        assert (out == 0).all() and (dimg == 0).all()


@pytest.mark.parametrize("world", [4, 3])
def test_c2_views_cut_into_rank_strips(world):
    """B = 4 views of 1920x1080 as division.start_strategy cuts them over `world` ranks; every rank's batch built as
    Trainer builds it (whole counted strips, empty views for cameras it does not render)."""
    H, W, B = 1080, 1920, 4
    uids = list(range(B))
    hist = division.StrategyHistory(uids, (H + 15) // 16, world)
    pairs = [lc.make_pair(H, W, seed=500 + v, kind="smooth") for v in range(B)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gl1, gss = view_grads(B)
    for rank in range(world):
        strategies, _ = division.start_strategy(uids, hist, world, rank)
        rows4 = []
        for st in strategies:
            r = st.local_pixel_rows(H)
            rows4.append((0, 0, 0, 0) if r is None else (r[0], r[1], r[0], r[1]))
        assert any(r[1] > r[0] for r in rows4) and any(r[1] == r[0] for r in rows4)
        gts = gt_strips([p[1] for p in pairs], rows4)
        check_batch(images, gts, rows4, gl1, gss, fp64=(rank == 1), tag=f"c2 world={world} rank={rank}")


L1_SHAPES = [(65, 1), (48, 33), (96, 1920)]


@pytest.mark.parametrize("H,W", L1_SHAPES)
def test_l1_branch_is_exact(H, W):
    """grad_ssim = 0: dL/dimage == fl32(fl32(g_l1 * fl32(1 / (3HW))) * sgn(x - gt_float(gt))) bit for bit, sgn(0) = 0 and
    0 on halo rows and outside the window; Ll1 within 1e-6 of the exact fp64 sum."""
    rows4 = [(0, H, 0, H), (0, 0, 0, 0), (16, H, 21, H - 5), (H - 33, H, H - 33, H), (3, 19, 10, 10)]
    B = len(rows4)
    pairs = [lc.make_pair(H, W, seed=70 + v) for v in range(B)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gts = gt_strips([p[1] for p in pairs], rows4)
    gl1 = np.array([0.8, 5.0, -1.7, 1e3, 0.3], np.float32)
    gss = np.zeros(B, np.float32)
    out, dimg = check_batch(images, gts, rows4, gl1, gss, fp64=False, tag=f"L1 {H}x{W}")
    inv = np.float32(1.0 / (3.0 * H * W))
    counted = np.zeros((3, H, W), np.float32)
    for v, (r0, r1, c0, c1) in enumerate(rows4):
        x, gt = pairs[v]
        y = lc.gt_float(gt)
        sgn = np.zeros((3, H, W), np.float32)
        sgn[:, c0:c1] = np.sign(x[:, c0:c1] - y[:, c0:c1])
        expect = np.float32(gl1[v] * inv) * sgn
        assert np.array_equal(dimg[v], expect), (H, W, v, np.abs(dimg[v] - expect).max())
        exact = np.abs(x[:, c0:c1].astype(np.float64) - y[:, c0:c1].astype(np.float64)).sum() / (3.0 * H * W)
        assert abs(float(out[v, 0]) - exact) <= 1e-6 * exact, (v, float(out[v, 0]), exact)
        if c1 > c0:
            lc.assert_populated(x[:, c0:c1], gt[:, c0:c1], {"equal", "equal_zero", "equal_one", "ulp_above", "ulp_below"},
                                (H, W, v))
            counted[:, c0:c1] = 1
    assert counted.any()


@pytest.mark.parametrize("H,W", L1_SHAPES)
def test_ssim_branch_vs_fp64(H, W):
    """grad_l1 = 0: the SSIM branch alone against fp64, halo and whole windows, flat and checkerboard regions."""
    rows4 = [(0, H, 0, H), (16, H, 21, H - 5), (H - 24, H, H - 24, H)]
    B = len(rows4)
    pairs = [lc.make_pair(H, W, seed=90 + v, kind="checker" if v == 1 and W > 1 else "mixed") for v in range(B)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gts = gt_strips([p[1] for p in pairs], rows4)
    check_batch(images, gts, rows4, np.zeros(B, np.float32), np.array([-0.2, 3.0, -1e3], np.float32),
                tag=f"SSIM {H}x{W}")


@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 3840)])
def test_full_resolution_operator_vs_fp64(H, W):
    """ops.fused_l1_ssim (autograd, single-view entry points) at the resolutions training uses: the whole image and a
    24-row window ending at H, against fp64 autograd on the device."""
    img, gt = lc.make_pair(H, W, seed=H, kind="smooth")
    if H == 1080:
        lc.assert_populated(img, gt, lc.claims(H, W, "smooth"), (H, W))
    x = gu.to_dev(img)
    gl1, gss = np.float32(0.8), np.float32(-0.2)
    for r0, r1 in ((0, H), (H - 24, H)):
        xg = x.clone().requires_grad_(True)
        g_strip = gu.to_dev(gt[:, r0:r1])
        l1, ss = ops.fused_l1_ssim(xg, g_strip, r0, r1)
        (float(gl1) * l1 + float(gss) * ss).backward()
        got = (float(l1), float(ss), gu.npy(xg.grad))
        assert (got[2][:, :r0] == 0).all()
        r64, r32, floor = refs(x, g_strip, (r0, r1, r0, r1), gl1, gss)
        gu.check_vs_fp64(f"{H}x{W} [{r0},{r1})", got, r32, r64, floor)
        del xg, got, r64, r32
        torch.cuda.empty_cache()


def test_batched_operator_and_fused_loss():
    """The autograd operators: ops.fused_l1_ssim_batched (what Trainer runs) with a distinct (d loss / d Ll1,
    d loss / d ssim) per view, which its backward splits out of the (B, 2) output gradient, and ops.fused_loss with its
    cached (1 - lambda, -lambda) weights.  Gradients bit for bit those of the C ABI calls with the same weights, which
    check_batch holds to the single-view calls and fp64; the scalars within one fp32 ulp."""
    H, W = 88, 33
    rows4 = [(0, 0, 0, 0), (0, 48, 0, 48), (16, 88, 21, 83), (40, 41, 40, 41), (3, 60, 30, 30)]
    B = len(rows4)
    kinds = ("mixed", "checker", "smooth")
    pairs = [lc.make_pair(H, W, seed=300 + v, kind=kinds[v % 3]) for v in range(B)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gts = gt_strips([p[1] for p in pairs], rows4)
    gl1 = np.array([0.8, -1.5, 1e3, 0.6, 0.3], np.float32)
    gss = np.array([-0.2, 0.7, 2.5e3, 0.0, -1.1], np.float32)
    out_abi, dimg_abi = check_batch(images, gts, rows4, gl1, gss, tag="operator")
    x = images.clone().requires_grad_(True)
    out = ops.fused_l1_ssim_batched(x, gts, rows4)
    (out * gu.to_dev(np.stack([gl1, gss], 1))).sum().backward()      # output gradient (gl1[v], gss[v]) exactly
    out = gu.npy(out.detach())
    assert all(within_ulp(a, b) for a, b in zip(out.reshape(-1), out_abi.reshape(-1))), (out, out_abi)
    assert np.array_equal(gu.npy(x.grad).view(np.uint32), dimg_abi.view(np.uint32))
    lam = 0.2
    for v in (1, 2, 3):
        r0, r1, c0, c1 = rows4[v]
        xv = images[v].clone().requires_grad_(True)
        loss = ops.fused_loss(xv, gts[v], r0, r1, lam, c0, c1)
        loss.backward()
        so, sd = single_view(images[v], gts[v], rows4[v], np.float32(1 - lam), np.float32(-lam))
        assert np.array_equal(gu.npy(xv.grad).view(np.uint32), sd.view(np.uint32)), v
        expect = (1 - lam) * float(so[0]) + lam * (1 - float(so[1]))
        assert abs(float(loss) - expect) <= 4 * float(np.spacing(np.float32(max(abs(expect), 1.0)))), (v, float(loss), expect)


def test_workspace_size_and_one_byte_short():
    H, W = 70, 33
    rows4 = [(0, 0, 0, 0), (5, 70, 10, 65), (16, 17, 16, 17), (0, 0, 0, 0), (3, 40, 3, 40)]
    B = len(rows4)
    assert _lib.query("gs_loss_temp_bytes_batched", B, i32(rows4), W) == HEADER_B + map_bytes(rows4, W) + 256
    assert _lib.query("gs_loss_temp_bytes_batched", 2, i32([(0, 0, 0, 0)] * 2), W) == HEADER_B + 256
    pairs = [lc.make_pair(H, W, seed=v) for v in range(B)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gts = gt_strips([p[1] for p in pairs], rows4)
    lib = _lib.load()
    short = HEADER_B + map_bytes(rows4, W) - 1
    rc, out, temp = forward_batched(images, gts, rows4, tb=short)
    assert rc == GS_ENOMEM, rc
    assert b"temp" in lib.gs_last_error()
    assert torch.isnan(out).all() and (gu.npy(temp) == SENTINEL).all()
    rc, out, temp = forward_batched(images, gts, rows4, tb=short + 1)     # exactly the maps: no spare needed
    assert rc == 0 and not torch.isnan(out).any()


SECOND_DEVICE = r"""
import json, sys
sys.path[:0] = %(paths)r
import numpy as np, torch
from gs_b200 import ops
import loss_cases as lc
img, gt = lc.make_pair(75, 45, seed=3)
res = {}
for dev in ("cuda:1", "cuda:0"):          # the first loss call of this process runs on the second device
    # the library launches on the current device and stream, so it must be the device the tensors live on
    with torch.cuda.device(dev):
        x = torch.from_numpy(img).to(dev).requires_grad_(True)
        l1, ss = ops.fused_l1_ssim(x, torch.from_numpy(gt[:, 5:70].copy()).to(dev), 5, 70, 9, 66)
        (0.8 * l1 - 0.2 * ss).backward()
        torch.cuda.synchronize(dev)
        res[dev] = [float(l1), float(ss), x.grad.cpu().numpy().view(np.uint32).tobytes().hex()]
print(json.dumps(res["cuda:1"] == res["cuda:0"]))
"""


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second device")
def test_second_device_first_call_matches_device_0():
    """The Gaussian window is uploaded to each device's constant memory on that device's first call (ensure_gauss)."""
    here = os.path.dirname(os.path.abspath(__file__))
    paths = [here, os.path.join(os.path.dirname(here), "grendel-gs_b200")]
    r = subprocess.run([sys.executable, "-c", SECOND_DEVICE % dict(paths=paths)], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert json.loads(r.stdout.strip().splitlines()[-1]) is True
