"""CPU checks of the held-out view metrics: the fp64 definitional reference (tests/eval_ref.py) against the reference's
own formulas restated in torch, the per-tile-row slots under any row partition, and the C-ABI refusals of
gs_eval_sums_batched / gs_eval_finalize in a process that sees no device (a launch there would fail with GS_ECUDA, so a
GS_EINVAL shows nothing was launched)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import eval_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(H=37, W=29, seed=0):
    rng = np.random.default_rng(seed)
    image = rng.uniform(-0.3, 1.3, size=(3, H, W)).astype(np.float32)
    image[0, 0, :5] = [0.0, 1.0, -0.0, 0.5, 2.0]
    gt = rng.integers(0, 256, size=(3, H, W), dtype=np.uint8)
    gt[:, 1, :4] = [0, 255, 0, 255]
    return image, gt


@pytest.mark.parametrize("H,W", [(37, 29), (64, 48), (16, 5), (5, 7)])
def test_reference_matches_the_reference_formulas(H, W):
    image, gt = _case(H, W, seed=H * W)
    got = eval_ref.finalize(eval_ref.slots(image, gt), H, W)
    want = eval_ref.reference_sequence(image, gt)
    assert got[0] == pytest.approx(want[0], rel=1e-12)
    assert got[1] == pytest.approx(want[1], rel=1e-12)


def test_ground_truth_unit_is_the_device_product():
    """gt_hat is fl32(g * fl32(1/255)), which differs from the IEEE quotient, what torch's `/ 255.0` gives on the CPU, on
    126 byte values, always by one ulp upwards; gt_hat_torch is the same bits on the CPU."""
    g = np.arange(256, dtype=np.uint8)
    prod = eval_ref.gt_hat(g).astype(np.float32)
    quot = (torch.from_numpy(g) / 255.0).numpy()
    assert np.array_equal(eval_ref.gt_hat_torch(g).numpy().view(np.uint32), prod.view(np.uint32))
    diff = prod != quot
    assert int(diff.sum()) == 126
    assert np.array_equal(prod[diff], np.nextafter(quot[diff], np.float32(2)))


@pytest.mark.parametrize("H,W", [(1, 1), (5, 2), (16, 7), (17, 33), (37, 29), (40, 129)])
def test_torch_slots_match_numpy(H, W):
    """slots_torch, the large-shape form of slots, against slots at small shapes: NaN, inf, -0, values above 1."""
    rng = np.random.default_rng(7 * H + W)
    image = rng.uniform(-0.3, 1.3, size=(3, H, W)).astype(np.float32)
    gt = rng.integers(0, 256, size=(3, H, W), dtype=np.uint8)
    flat = image.reshape(-1)
    flat[:4] = [np.inf, -np.inf, -0.0, 3.0][:flat.size]
    flat[-1] = np.nan
    for rows in (None, (0, H), (16, H) if H > 16 else (0, 0), (0, 16) if H > 16 else (0, H)):
        want = eval_ref.slots(image, gt, rows)
        got = eval_ref.slots_torch(torch.from_numpy(image), torch.from_numpy(gt), rows).numpy()
        assert got.shape == want.shape
        assert np.allclose(got, want, rtol=1e-13, atol=0, equal_nan=True), rows
        assert np.array_equal(np.signbit(got[want == 0]), np.zeros((want == 0).sum(), bool))


def test_psnr_is_per_channel_then_averaged():
    H, W = 32, 16
    gt = np.full((3, H, W), 128, dtype=np.uint8)
    image = eval_ref.gt_hat(gt).astype(np.float32)
    image[0] += 0.01    # channel errors of different size: the channel PSNRs differ
    image[1] += 0.1
    image[2] -= 0.3
    l1, psnr = eval_ref.finalize(eval_ref.slots(image, gt), H, W)
    d = image.astype(np.float64) - eval_ref.gt_hat(gt)
    per_channel = np.mean([20 * math.log10(1 / math.sqrt((d[c] ** 2).mean())) for c in range(3)])
    pooled = 20 * math.log10(1 / math.sqrt((d ** 2).mean()))
    assert psnr == pytest.approx(per_channel, rel=1e-13)
    assert abs(psnr - pooled) > 1.0
    assert psnr == pytest.approx(eval_ref.reference_sequence(image, gt)[1], rel=1e-12)


def test_clamp_comes_before_the_comparison():
    H, W = 16, 8
    gt = np.zeros((3, H, W), dtype=np.uint8)
    gt[1] = 255
    image = np.empty((3, H, W), dtype=np.float32)
    image[0], image[1], image[2] = -2.0, 3.0, -0.5   # clamped onto the ground truth: no error anywhere
    l1, psnr = eval_ref.finalize(eval_ref.slots(image, gt), H, W)
    assert l1 == 0.0 and psnr == math.inf
    assert eval_ref.reference_sequence(image, gt) == (0.0, math.inf)


def test_perfect_image_scores_inf():
    image, gt = _case(24, 40, seed=3)
    image = eval_ref.gt_hat(gt).astype(np.float32)   # the reference's gt / 255.0 on the device exactly
    assert eval_ref.finalize(eval_ref.slots(image, gt), 24, 40) == (0.0, math.inf)
    assert eval_ref.reference_sequence(image, gt, torch.float32) == (0.0, math.inf)


def test_nan_propagates():
    image, gt = _case(20, 12, seed=4)
    image[2, 17, 3] = np.nan
    sl = eval_ref.slots(image, gt)
    assert np.isnan(sl[1, 2]).all() and not np.isnan(sl[0]).any() and not np.isnan(sl[1, :2]).any()
    l1, psnr = eval_ref.finalize(sl, 20, 12)
    assert math.isnan(l1) and math.isnan(psnr)
    r = eval_ref.reference_sequence(image, gt)
    assert math.isnan(r[0]) and math.isnan(r[1])


@pytest.mark.parametrize("H", [37, 64, 130])
def test_row_partitions_sum_to_the_whole_image_exactly(H):
    W = 23
    image, gt = _case(H, W, seed=H)
    whole = eval_ref.slots(image, gt)
    TY = whole.shape[0]
    rng = np.random.default_rng(H)
    for _ in range(6):
        cuts = sorted(rng.choice(np.arange(1, TY), size=min(TY - 1, rng.integers(0, 4)), replace=False).tolist())
        bounds = [0] + [16 * c for c in cuts] + [H]
        parts = [eval_ref.slots(image, gt, (a, b)) for a, b in zip(bounds, bounds[1:])]
        total = parts[0]
        for p in parts[1:]:
            total = total + p
        assert np.array_equal(total, whole)
        assert all(np.array_equal(p[p != 0], whole[p != 0]) for p in parts)
        assert eval_ref.finalize(total, H, W) == eval_ref.finalize(whole, H, W)


REFUSALS = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from gs_b200 import _lib
lib = _lib.load()
H, W = 40, 24
fake = 1 << 20                     # never dereferenced: every call below is refused first
def i32(*v):
    return (C.c_int32 * len(v))(*v)
def ptrs(*p):
    return (C.c_void_p * len(p))(*p)
ok = dict(n=2, img=fake, gts=ptrs(fake, fake), g0=i32(0, 16), gr=i32(H, 24), r0=i32(0, 16), r1=i32(16, H), slots=fake)
def sums(**kw):
    a = dict(ok, **kw)
    return lib.gs_eval_sums_batched(a["n"], H, W, a["img"], a["gts"], a["g0"], a["gr"], a["r0"], a["r1"], a["slots"], None)
cases = {
    "no views": dict(n=0),
    "too many views": dict(n=65),
    "row0 unaligned": dict(r0=i32(0, 8)),
    "row1 unaligned": dict(r1=i32(16, 39)),
    "inverted": dict(r0=i32(16, 16), r1=i32(0, H)),
    "past H": dict(r1=i32(16, H + 8)),
    "negative": dict(r0=i32(-16, 16)),
    "null gt with rows": dict(gts=ptrs(fake, None)),
    "gt misses rows": dict(g0=i32(0, 32)),
    "gt past H": dict(gr=i32(H, 32)),
    "null image": dict(img=None),
    "null slots": dict(slots=None),
}
for name, kw in cases.items():
    rc = sums(**kw)
    assert rc == -1, (name, rc)
    assert b"invalid argument" in lib.gs_last_error(), name
rc = sums(gts=ptrs(fake, None), r0=i32(0, 16), r1=i32(16, 16))   # a view without rows may have no ground truth ...
assert rc == -2, rc                                                # ... and reaches the launch, which has no device
for n, s, o in ((0, fake, fake), (65, fake, fake), (2, None, fake), (2, fake, None)):
    assert lib.gs_eval_finalize(n, H, W, s, o, None) == -1, (n, s, o)
assert lib.gs_eval_slot_count(3, H) == 3 * 3 * 6 and lib.gs_eval_slot_count(0, H) == 0
print("refused", len(cases))
"""


def test_cabi_refusals_without_a_device():
    from gs_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", REFUSALS, os.path.join(ROOT, "grendel-gs_b200")], capture_output=True,
                       text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "refused 12" in r.stdout


def test_evaluate_refuses_before_any_launch():
    """Trainer.evaluate's refusals come from its arguments alone, before any collective or launch: a Trainer on the CPU
    reaches none."""
    from gs_b200 import pipeline
    from gs_b200 import synthetic as syn
    cams = [syn.make_camera(48, 40, yaw_deg=2.0 * k, uid=k) for k in range(4)]
    gts = [torch.zeros((3, 40, 48), dtype=torch.uint8) for _ in cams]
    tr = pipeline.Trainer(syn.make_scene(8, 48, 40, seed=0), cams, gts, "cpu")
    bad = [dict(views=[4]), dict(views=[-1]), dict(views=[]), dict(bsz=0), dict(bsz=65),
           dict(cams=cams), dict(gts=gts), dict(cams=cams, gts=gts[:3]),
           dict(cams=cams, gts=[g[:, :32] for g in gts]), dict(cams=[syn.make_camera(48, 32)] * 4, gts=gts),
           dict(cams=cams, gts=[g.float() for g in gts]), dict(cams=cams, gts=gts[:3] + [None])]
    for kw in bad:
        with pytest.raises(ValueError):
            tr.evaluate(**kw)
    with pytest.raises(TypeError):
        tr.evaluate([1.0])
    ls = pipeline.Trainer(syn.make_scene(8, 48, 40, seed=0), cams, [gts[0], None, gts[2], None], "cpu",
                          local_sampling=True, local_bsz=1)
    with pytest.raises(ValueError, match="local-sampling"):
        ls.evaluate()
    assert tr.iteration == 0 and tr.history.history == [] and ls.iteration == 0
