"""CPU checks of the image metrics: the fp64 definitional reference (tests/metrics_ref.py) against torchvision's PNG
path and the reference's ssim / psnr restated in torch, exact sums over tile-aligned row partitions, the halo exchange and
image gather (gs_b200.image_halo) over gloo, the C-ABI refusals of gs_quantize_u8_batched / gs_image_metric_* in a
process that sees no device (a launch there would fail with GS_ECUDA, so a GS_EINVAL shows nothing was launched), and
Trainer.image_metrics' refusals."""
import io
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import metrics_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "grendel-gs_b200")


def _png_round_trip(image):
    """render.py's save_image of a (3,H,W) fp32 image, read back as metrics.py reads it -> fp32 (3,H,W) tensor."""
    from PIL import Image
    import torchvision
    import torchvision.transforms.functional as tf
    buf = io.BytesIO()
    torchvision.utils.save_image(image, buf, format="png")
    buf.seek(0)
    return tf.to_tensor(Image.open(buf))[:3]


def _quantizer_inputs():
    k = np.arange(256, dtype=np.float32)
    ties = ((k + np.float32(0.5)) / np.float32(255)).astype(np.float32)   # x * 255 at or next to k + 0.5
    near = np.concatenate([ties, np.nextafter(ties, np.float32(0)), np.nextafter(ties, np.float32(1)),
                           k / np.float32(255), np.nextafter(k / np.float32(255), np.float32(2))])
    special = np.array([0.0, -0.0, 1.0, -1e-8, -0.3, -5.0, 1.0 + 1e-7, 1.3, 7.0, np.inf, -np.inf,
                        np.float32(1) - np.float32(2 ** -24)], dtype=np.float32)
    rnd = np.random.default_rng(0).uniform(-0.2, 1.2, 4096).astype(np.float32)
    x = np.concatenate([near, special, rnd])
    n = -(-x.size // 48) * 48
    return np.pad(x, (0, n - x.size)).reshape(3, -1, 16)


def test_quantizer_equals_the_png_round_trip():
    x = _quantizer_inputs()
    q = metrics_ref.quantize(x)
    assert np.array_equal(q, metrics_ref.save_image_quantize(torch.from_numpy(x)).numpy())
    back = _png_round_trip(torch.from_numpy(x))
    assert torch.equal(back, torch.from_numpy(metrics_ref.unit(q).astype(np.float32)))   # a = fl32(q / 255) exactly
    assert np.array_equal(np.rint(back.numpy() * 255).astype(np.uint8), q)
    # the ties: (k + 0.5) / 255 in fp32, times 255 in fp32, plus 0.5, truncates to k or k + 1 as torch rounds it
    assert q.max() == 255 and q.min() == 0


def test_nan_quantizes_to_zero():
    x = np.array([np.nan, -np.nan, 0.5], dtype=np.float32)
    assert metrics_ref.quantize(x).tolist() == [0, 0, 128]


def test_ground_truth_round_trip_is_exact_for_every_value():
    g = np.arange(256, dtype=np.uint8).reshape(1, 16, 16).repeat(3, 0)
    g[1] = g[1][::-1]
    gt = torch.from_numpy(g)
    saved = torch.clamp(gt / 255.0, 0.0, 1.0)   # render.py:128
    assert np.array_equal(metrics_ref.quantize(saved.numpy()), g)
    back = _png_round_trip(saved)
    assert torch.equal(back, torch.from_numpy(metrics_ref.unit(g).astype(np.float32)))
    # render.py divides on the device, where the quotient is fl32(g * fl32(1/255)): that comes back as g too
    import eval_ref
    assert np.array_equal(metrics_ref.quantize(eval_ref.gt_hat(g).astype(np.float32)), g)


@pytest.mark.parametrize("H,W", [(1, 1), (5, 2), (11, 12), (16, 33), (17, 31), (40, 65)])
def test_torch_slots_match_numpy(H, W):
    """slots_torch, the large-shape form of slots, against slots at small shapes, whole and strip rows."""
    rng = np.random.default_rng(H * 100 + W)
    g = rng.integers(0, 256, (3, H, W), dtype=np.uint8)
    q = np.clip(g.astype(np.int64) + rng.integers(-9, 10, g.shape), 0, 255).astype(np.uint8)
    for rows in (None, (16, H) if H > 16 else (0, 0), (0, 16) if H > 16 else (0, H)):
        want = metrics_ref.slots(q, g, rows)
        got = metrics_ref.slots_torch(torch.from_numpy(q), torch.from_numpy(g), rows).numpy()
        assert got.shape == want.shape and np.allclose(got, want, rtol=1e-13, atol=0), rows
        assert not np.signbit(got[want == 0]).any()


def test_window_is_the_reference_gaussian_bit_for_bit():
    w1, w2 = metrics_ref.reference_window()
    assert w1.dtype == torch.float32 and w2.dtype == torch.float32
    assert w1.tolist() == list(metrics_ref.WINDOW)
    g = torch.Tensor([np.exp(-((x - 5) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    assert g.sum().item() == pytest.approx(3.7592328, abs=5e-8)
    src = open(os.path.join(PKG, "csrc", "metrics.cu")).read()
    body = re.search(r"c_ssim_w\[IM_TAPS\]\s*=\s*\{([^}]*)\}", src).group(1)
    kernel = [float.fromhex(h) for h in re.findall(r"0x[0-9a-fA-F.]+p-?\d+", body)]
    assert kernel == list(metrics_ref.WINDOW)


# (H, W): H or W below 11, H not a multiple of 16, odd W
SIZES = [(37, 29), (64, 48), (16, 5), (5, 7), (9, 10), (130, 77), (33, 16)]
# measured over these cases with seeds 0..2 and noise 0.02 / 0.2 / 1.0: float64 SSIM 4.2e-8 (the fp32 rounding of the
# reference's 2D window), PSNR 8.0e-9 (fl32(q / 255) - fl32(g / 255) against (q - g) / 255); float32 SSIM 3.2e-7, PSNR 1.1e-7
BOUNDS = {torch.float64: (1e-7, 2e-8), torch.float32: (1e-6, 5e-7)}


def _case(H, W, seed, noise):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 256, (3, H, W), dtype=np.uint8)
    x = (g.astype(np.float32) / 255 + rng.normal(0, noise, (3, H, W))).astype(np.float32)
    return x, g


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("H,W", SIZES)
def test_reference_matches_the_reference_ssim_and_psnr(H, W, dtype):
    b_ssim, b_psnr = BOUNDS[dtype]
    for seed, noise in ((H * W, 0.02), (H + W, 0.2), (H, 1.0)):
        x, g = _case(H, W, seed, noise)
        got = metrics_ref.finalize(metrics_ref.slots(metrics_ref.quantize(x), g), H, W)
        want = metrics_ref.reference_sequence(torch.from_numpy(x), torch.from_numpy(g), dtype)
        assert got[0] == pytest.approx(want[0], rel=b_ssim)
        assert got[1] == pytest.approx(want[1], rel=b_psnr)


def test_perfect_render_scores_one_and_inf():
    H, W = 24, 19
    g = np.random.default_rng(3).integers(0, 256, (3, H, W), dtype=np.uint8)
    x = metrics_ref.unit(g).astype(np.float32)
    q = metrics_ref.quantize(x)
    assert np.array_equal(q, g)
    ssim, psnr = metrics_ref.finalize(metrics_ref.slots(q, g), H, W)
    assert ssim == pytest.approx(1.0, abs=1e-15) and psnr == float("inf")


@pytest.mark.parametrize("H", [37, 64, 130])
def test_row_partitions_sum_to_the_whole_image_exactly(H):
    W = 23
    x, g = _case(H, W, H, 0.1)
    q = metrics_ref.quantize(x)
    whole = metrics_ref.slots(q, g)
    TY = whole.shape[0]
    rng = np.random.default_rng(H)
    for _ in range(6):
        cuts = sorted(rng.choice(np.arange(1, TY), size=min(TY - 1, rng.integers(0, 4)), replace=False).tolist())
        bounds = [0] + [16 * c for c in cuts] + [H]
        parts = [metrics_ref.slots(q, g, (a, b)) for a, b in zip(bounds, bounds[1:])]
        total = parts[0]
        for p in parts[1:]:
            total = total + p
        assert np.array_equal(total, whole)
        assert metrics_ref.finalize(total, H, W) == metrics_ref.finalize(whole, H, W)


HALO_WORKER = r"""
import sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from gs_b200 import image_halo
from gs_b200.division import DivisionStrategy
rank, world, store = int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
dist.init_process_group("gloo", init_method="file://" + store, rank=rank, world_size=world)
rng = np.random.default_rng(100 + world)
checked = 0
for trial in range(4):
    W = int(rng.integers(5, 40))
    H = 16 * int(rng.integers(2, 6)) + int(rng.integers(1, 5))    # the last strip: 1-4 rows
    TY = (H + 15) // 16
    strategies, whole = [], []
    for v in range(int(rng.integers(1, 5))):
        n = int(rng.integers(1, min(world, TY) + 1))
        if v == 0:
            n = min(world, TY)
        ids = [int(i) for i in rng.permutation(world)[:n]]
        if v == 1 and world == 3:
            ids = [0, 2] if n >= 2 else [1]           # a view rank 1 (or 0 and 2) does not own
        n = len(ids)
        inner = sorted(rng.choice(np.arange(1, TY - 1), size=n - 2, replace=False).tolist()) if n > 2 else []
        pos = [0] + [int(p) for p in inner] + ([TY - 1] if n > 1 else []) + [TY]   # last strip: the partial tile row
        strategies.append(DivisionStrategy(v, ids, pos, TY, rank))
        whole.append(torch.from_numpy(rng.integers(0, 256, (6, H, W), dtype=np.uint8)))
    wins, win0, strips = [], [], []
    for v, st in enumerate(strategies):
        r = st.local_pixel_rows(H)
        if r is None:
            wins.append(None); win0.append(0); strips.append(None)
            continue
        a, b = image_halo.window_rows(r, H)
        w = torch.full((6, b - a, W), 77, dtype=torch.uint8)
        w[:, r[0] - a:r[1] - a] = whole[v][:, r[0]:r[1]]
        wins.append(w); win0.append(a); strips.append(w[:3, r[0] - a:r[1] - a])
    image_halo.exchange_halos(wins, win0, strategies, H, W, rank, world, None, "cpu")
    for v, w in enumerate(wins):
        if w is not None:
            assert torch.equal(w, whole[v][:, win0[v]:win0[v] + w.shape[1]]), (trial, v)
            checked += 1
    got = image_halo.gather_images(strips, strategies, H, W, rank, world, None, "cpu")
    if rank == 0:
        assert len(got) == len(strategies)
        for v, img in enumerate(got):
            assert img.dtype == torch.uint8 and torch.equal(img, whole[v][:3]), (trial, v)
    else:
        assert got is None
dist.destroy_process_group()
print("ok", checked)
"""


@pytest.mark.parametrize("world", [2, 3])
def test_halo_exchange_and_gather_over_gloo(tmp_path, world):
    store = str(tmp_path / "store")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    procs = [subprocess.Popen([sys.executable, "-c", HALO_WORKER, PKG, str(r), str(world), store], env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(world)]
    outs = [p.communicate(timeout=300) for p in procs]
    for p, (out, err) in zip(procs, outs):
        assert p.returncode == 0, out + err
        assert out.startswith("ok")
    assert sum(int(o.split()[1]) for o, _ in outs) > 0


def test_halo_plan_with_a_short_last_strip():
    from gs_b200 import image_halo
    from gs_b200.division import DivisionStrategy
    H = 16 * 3 + 3   # tile rows [0, 3) on rank 1, the 3-row last tile row on rank 0
    st = DivisionStrategy(0, [1, 0], [0, 3, 4], 4, 0)
    assert image_halo.halo_plan([st], H) == [(0, 1, 0, 43, 48), (0, 0, 1, 48, 51)]
    assert image_halo.window_rows((48, 51), H) == (43, 51) and image_halo.window_rows((0, 48), H) == (0, 51)


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
ok = dict(n=2, img=fake, r0=i32(0, 16), r1=i32(16, H), outs=ptrs(fake, fake), o0=i32(0, 11), orows=i32(21, 29))
def quant(**kw):
    a = dict(ok, **kw)
    return lib.gs_quantize_u8_batched(a["n"], H, W, a["img"], a["r0"], a["r1"], a["outs"], a["o0"], a["orows"], None)
qcases = {
    "no views": dict(n=0), "too many views": dict(n=65), "inverted": dict(r0=i32(16, 16), r1=i32(0, H)),
    "past H": dict(r1=i32(16, H + 1)), "negative": dict(r0=i32(-1, 16)), "null out with rows": dict(outs=ptrs(fake, None)),
    "out misses rows": dict(o0=i32(1, 11)), "out past H": dict(orows=i32(21, 30)), "null image": dict(img=None),
}
ok2 = dict(n=2, wins=ptrs(fake, fake), w0=i32(0, 11), wr=i32(21, 29), r0=i32(0, 16), r1=i32(16, H), slots=fake)
def sums(**kw):
    a = dict(ok2, **kw)
    return lib.gs_image_metric_sums_batched(a["n"], H, W, a["wins"], a["w0"], a["wr"], a["r0"], a["r1"], a["slots"], None)
scases = {
    "no views": dict(n=0), "too many views": dict(n=65), "row0 unaligned": dict(r0=i32(0, 8)),
    "row1 unaligned": dict(r1=i32(16, 39)), "inverted": dict(r0=i32(16, 16), r1=i32(0, H)), "past H": dict(r1=i32(16, 48)),
    "null window with rows": dict(wins=ptrs(fake, None)), "halo above missing": dict(w0=i32(0, 12), wr=i32(21, 28)),
    "halo below missing": dict(wr=i32(20, 29)), "window past H": dict(wr=i32(21, 30)), "null slots": dict(slots=None),
}
for table, call in ((qcases, quant), (scases, sums)):
    for name, kw in table.items():
        rc = call(**kw)
        assert rc == -1, (name, rc)
        assert b"invalid argument" in lib.gs_last_error(), name
# views without rows need no buffers: the quantizer then has nothing to launch, the sums launch (and find no device)
assert quant(outs=ptrs(None, None), r0=i32(0, 16), r1=i32(0, 16)) == 0
assert sums(wins=ptrs(fake, None), r0=i32(0, 16), r1=i32(16, 16)) == -2
assert quant() == -2
for n, s, o in ((0, fake, fake), (65, fake, fake), (2, None, fake), (2, fake, None)):
    assert lib.gs_image_metric_finalize(n, H, W, s, o, None) == -1, (n, s, o)
print("refused", len(qcases) + len(scases))
"""


def test_cabi_refusals_without_a_device():
    from gs_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", REFUSALS, PKG], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "refused 20" in r.stdout


def test_image_metrics_refuses_before_any_launch():
    """Trainer.image_metrics' refusals come from its arguments alone, before any collective or launch: a Trainer on the
    CPU reaches none."""
    from gs_b200 import pipeline
    from gs_b200 import synthetic as syn
    cams = [syn.make_camera(48, 40, yaw_deg=2.0 * k, uid=k) for k in range(4)]
    gts = [torch.zeros((3, 40, 48), dtype=torch.uint8) for _ in cams]
    tr = pipeline.Trainer(syn.make_scene(8, 48, 40, seed=0), cams, gts, "cpu")
    bad = [dict(views=[4]), dict(views=[-1]), dict(views=[]), dict(bsz=0), dict(bsz=65),
           dict(cams=cams), dict(gts=gts), dict(cams=cams, gts=gts[:3]),
           dict(cams=cams, gts=[g[:, :32] for g in gts]), dict(cams=[syn.make_camera(48, 32)] * 4, gts=gts),
           dict(cams=cams, gts=[g.float() for g in gts]), dict(cams=cams, gts=gts[:3] + [None]),
           dict(images=True, views=[9])]
    for kw in bad:
        with pytest.raises(ValueError, match="image_metrics"):
            tr.image_metrics(**kw)
    with pytest.raises(TypeError):
        tr.image_metrics([1.0])
    ls = pipeline.Trainer(syn.make_scene(8, 48, 40, seed=0), cams, [gts[0], None, gts[2], None], "cpu",
                          local_sampling=True, local_bsz=1)
    with pytest.raises(ValueError, match="local-sampling"):
        ls.image_metrics()
    assert tr.iteration == 0 and tr.history.history == [] and ls.iteration == 0
