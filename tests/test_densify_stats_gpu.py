"""-m gpu: gs_densify_stats (gs_b200.densify.add_densification_stats, pipeline.Trainer.add_densification_stats) against
the reference's densification statistics, bit for bit.

The reference here is the literal torch chain of the reference's densification.py:15-24 with
GaussianModel.add_densification_stats (scene/gaussian_model.py:1046-1052), run camera by camera on copies of the same
statistics on the same device (`reference_chain`).  Outputs are compared as int32 bit patterns, so NaN payloads,
signed zeros and infinities count."""
import warnings

import numpy as np
import pytest
import torch

from gs_b200 import _lib, densify, pipeline
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32_BITS = {"nan_a": 0x7FC0_1234, "nan_b": 0xFFC0_0777, "snan": 0x7F80_DEAD, "neg0": 0x8000_0000}
# never-visible rows start at these patterns; the kernel must leave them exactly so
SENTINEL = (0x7FA5_A5A5, 0x8000_0000, 0xFF80_0001)   # accum: NaN payload, denom: -0.0, max: signalling NaN


def reference_chain(accum, denom, max_radii2D, grads, radii):
    """densification.py:15-24 + gaussian_model.py:1046-1052, transcribed (means2D.grad is (P, 2) here)."""
    for g, r in zip(grads, radii):
        visibility_filter = r > 0
        max_radii2D[visibility_filter] = torch.max(max_radii2D[visibility_filter], r[visibility_filter])
        accum[visibility_filter] += torch.norm(g[visibility_filter, :2], dim=-1, keepdim=True)
        denom[visibility_filter] += 1


def i32(b):
    """A 32-bit pattern as the int32 value torch stores for it."""
    return b - (1 << 32) if b >= 1 << 31 else b


def f32(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


def bits(t):
    return t.contiguous().view(torch.int32).cpu()


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def run_both(stats, grads, radii, form):
    """-> (kernel result, reference result), each a tuple of (accum, denom, max) run on its own copy of `stats`."""
    got = tuple(t.clone() for t in stats)
    ref = tuple(t.clone() for t in stats)
    g = grads if form == "stacked" else [x.clone() for x in grads.unbind(0)]      # separate allocations
    r = radii if form == "stacked" else [x.clone() for x in radii.unbind(0)]
    densify.add_densification_stats(*got, g, r)
    reference_chain(*ref, grads.unbind(0), radii.unbind(0))
    torch.cuda.synchronize()
    return got, ref


def assert_equal_stats(got, ref, what):
    for name, a, b in zip(("xyz_gradient_accum", "denom", "max_radii2D"), got, ref):
        if not same_bits(a, b):
            d = (bits(a) != bits(b)).reshape(-1).nonzero()[:5, 0].tolist()
            raise AssertionError(f"{what}: {name} differs at rows {d}: kernel {bits(a).reshape(-1)[d].tolist()} "
                                 f"reference {bits(b).reshape(-1)[d].tolist()}")


def random_batch(B, P, seed, hidden_every=7):
    """Radii in [-3, 40] (about 40 % not visible per view), normal gradients, positive statistics; every
    `hidden_every`-th Gaussian is visible in no view and holds the sentinels."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    radii = torch.randint(-3, 41, (B, P), generator=g, device=DEV, dtype=torch.int32)
    radii[radii > 24] = 0
    hidden = torch.zeros((P,), dtype=torch.bool, device=DEV)
    hidden[::hidden_every] = True
    radii[:, hidden] = torch.randint(-2, 1, (B, int(hidden.sum())), generator=g, device=DEV, dtype=torch.int32)
    grads = torch.randn((B, P, 2), generator=g, device=DEV) * 1e-3
    accum = torch.rand((P, 1), generator=g, device=DEV)
    denom = torch.randint(0, 50, (P, 1), generator=g, device=DEV).float()
    maxr = torch.randint(0, 30, (P,), generator=g, device=DEV).float()
    for t, s in zip((accum, denom, maxr), SENTINEL):
        t.view(torch.int32).reshape(-1)[hidden] = i32(s)
    return (accum, denom, maxr), grads, radii, hidden


def assert_sentinels(stats, hidden):
    for t, s in zip(stats, SENTINEL):
        b = bits(t).reshape(-1)[hidden.cpu()]
        assert b.numel() and bool((b == i32(s)).all()), s


# (a) both input forms over batch sizes and sizes around the CTA boundary
@pytest.mark.parametrize("P", [1, 255, 256, 257, (1 << 21) + 5])
@pytest.mark.parametrize("B", [1, 2, 4, 17, 64])
def test_matches_reference_chain(B, P):
    stats, grads, radii, hidden = random_batch(B, P, seed=1000 * B + P % 997, hidden_every=7 if P > 1 else 2)
    for form in ("stacked", "list"):
        got, ref = run_both(stats, grads, radii, form)
        assert_equal_stats(got, ref, f"B={B} P={P} {form}")
        if hidden.any():   # (c) never-visible rows keep their sentinels
            assert_sentinels(got, hidden)
    assert P == 1 or not torch.equal(bits(got[1]), bits(stats[1]))    # something was visible


# (b) constructed populations: every regime present, asserted
RADII = np.array([0, -1, 1, (1 << 24) + 1, (1 << 24) + 3, (1 << 31) - 1, 7, 12], dtype=np.int64)
SUB = float(f32(0x0000_0101))          # a subnormal


def regime_population(B=8, P=8192, seed=3):
    rng = np.random.default_rng(seed)
    radii = RADII[rng.integers(0, RADII.size, (B, P))].astype(np.int32)
    comp = np.array([0.0, -0.0, SUB, -SUB, 1.5e19, -3e19, 1.1e-19, -7e-20, 3e-23, np.inf, -np.inf, np.nan,
                     0.25, -1.75], dtype=np.float32)
    grads = comp[rng.integers(0, comp.size, (B, P, 2))]
    normal = rng.random((B, P, 2)) < 0.4
    grads[normal] = rng.normal(size=int(normal.sum())).astype(np.float32)
    vals = np.array([0.0, 1.0, 3e38, np.inf, float(f32(F32_BITS["nan_a"])), float(f32(F32_BITS["nan_b"])), 2.5],
                    dtype=np.float32)
    accum = vals[rng.integers(0, vals.size, (P, 1))]
    denom = np.array([0.0, 1.0, 16777216.0, np.inf, np.nan, 3.0], np.float32)[rng.integers(0, 6, (P, 1))]
    maxr = np.array([0.0, 5.0, 2147483648.0, np.inf, float(f32(F32_BITS["nan_b"])), float(f32(F32_BITS["snan"])),
                     16777216.0], np.float32)[rng.integers(0, 7, (P,))]
    # reinsert the NaN payloads bit-exactly (numpy may quieten them through float())
    for arr, pick in ((accum, rng.random(accum.shape) < 0.05), (maxr, rng.random(maxr.shape) < 0.05)):
        arr.view(np.uint32)[pick] = F32_BITS["nan_a"]
    maxr.view(np.uint32)[rng.random(maxr.shape) < 0.05] = F32_BITS["snan"]
    return accum, denom, maxr, grads, radii


def test_regime_population_is_populated():
    accum, denom, maxr, grads, radii = regime_population()
    vis = radii > 0
    g = grads[vis]
    a = np.abs(g.astype(np.float64))
    regimes = {
        "x^2 overflows": ((a > 1.8446744e19) & np.isfinite(a)).any(axis=1),
        "x^2 underflows": ((a > 0) & (a < 1.0842022e-19)).any(axis=1),
        "subnormal": ((a > 0) & (a < 1.1754944e-38)).any(axis=1),
        "+0": (~np.signbit(g) & (g == 0)).any(axis=1),
        "-0": (np.signbit(g) & (g == 0)).any(axis=1),
        "inf": np.isinf(g).any(axis=1), "nan": np.isnan(g).any(axis=1),
    }
    for k, v in regimes.items():
        assert v.sum() > 10, k
    for r in RADII:
        assert (radii == r).sum() > 10, r
    seen = vis.any(axis=0)
    for name, arr in (("accum", accum[:, 0]), ("denom", denom[:, 0]), ("max", maxr)):
        s = arr[seen]
        assert np.isnan(s).sum() > 10 and np.isinf(s).sum() > 10 and ((s != 0) & np.isfinite(s)).sum() > 10, name
    assert (maxr.view(np.uint32)[seen] == F32_BITS["snan"]).sum() > 10


@pytest.mark.parametrize("form", ["stacked", "list"])
def test_regimes_match_reference_chain(form):
    accum, denom, maxr, grads, radii = regime_population()
    stats = tuple(torch.from_numpy(x).to(DEV) for x in (accum, denom, maxr))
    got, ref = run_both(stats, torch.from_numpy(grads).to(DEV), torch.from_numpy(radii).to(DEV), form)
    assert_equal_stats(got, ref, form)
    # every regime reaches the outputs: inf and NaN accumulations, rounded radii, denom stuck at 2^24
    out_a, out_d, out_m = (bits(t).reshape(-1).numpy().view(np.float32) for t in got)
    assert np.isnan(out_a).sum() > 10 and np.isinf(out_a).sum() > 10
    assert (out_m == 2147483648.0).sum() > 10 and (out_m == 16777220.0).sum() > 0
    assert (out_d == 16777216.0).sum() > 0


def _order_sums(init, n):
    """fp32 sums of init + n[0] + ... + n[63]: batch order, reversed, pairwise tree (numpy, one rounding each)."""
    seq = init.copy()
    for k in range(n.shape[0]):
        seq = (seq + n[k]).astype(np.float32)
    rev = init.copy()
    for k in range(n.shape[0] - 1, -1, -1):
        rev = (rev + n[k]).astype(np.float32)
    t = n.copy()
    while t.shape[0] > 1:
        t = (t[0::2] + t[1::2]).astype(np.float32)
    pair = (init + t[0]).astype(np.float32)
    return seq, rev, pair


def test_summation_order_over_64_views():
    """Gaussians visible in all 64 views, with norms spread over 2^-30 .. 2^10 so that the order of the sum shows."""
    B, P = 64, 97
    rng = np.random.default_rng(11)
    mag = np.exp2(rng.uniform(-30, 10, (B, P))).astype(np.float32)
    ang = rng.uniform(0, 2 * np.pi, (B, P))
    grads = np.stack([mag * np.cos(ang), mag * np.sin(ang)], axis=-1).astype(np.float32)
    radii = np.full((B, P), 3, np.int32)
    accum = rng.uniform(0, 1, (P, 1)).astype(np.float32)
    g = torch.from_numpy(grads).to(DEV)
    norms = torch.norm(g, dim=-1).cpu().numpy()          # the device's own norms: the sums below differ only by order
    seq, rev, pair = _order_sums(accum[:, 0], norms)
    assert (seq != rev).sum() > P // 4 and (seq != pair).sum() > P // 4, ((seq != rev).sum(), (seq != pair).sum())
    stats = (torch.from_numpy(accum).to(DEV), torch.zeros((P, 1), device=DEV), torch.zeros((P,), device=DEV))
    got, ref = run_both(stats, g, torch.from_numpy(radii).to(DEV), "stacked")
    assert_equal_stats(got, ref, "64 views")
    assert np.array_equal(got[0].cpu().numpy()[:, 0].view(np.uint32), seq.view(np.uint32))
    assert bool((got[1] == 64).all())


# (d) which fp32 form torch.norm takes for a 2-vector on this device
def _rn_sum_f32(a, b):
    """Correctly rounded fp32 of a + b for float64 a, b whose exact sum needs more than 53 bits: TwoSum, then fix the
    one case where rounding the float64 sum to fp32 lands on a tie that the error term breaks."""
    s = a + b
    bb = s - a
    e = (a - (s - bb)) + (b - bb)
    r = s.astype(np.float32)
    up = np.nextafter(r, np.float32(np.inf))
    dn = np.nextafter(r, np.float32(-np.inf))
    r64 = r.astype(np.float64)
    tie_hi = (r64 > s) & ((r64 - s) == (r64 - dn.astype(np.float64)) / 2)     # s is the midpoint below r
    tie_lo = (r64 < s) & ((s - r64) == (up.astype(np.float64) - r64) / 2)     # s is the midpoint above r
    r = np.where(tie_hi & (e < 0), dn, r)
    r = np.where(tie_lo & (e > 0), up, r)
    return r


def norm_candidates(x, y):
    """The three fp32 forms of sqrt(x^2 + y^2): rn(rn(x^2) + rn(y^2)), fma(y, y, rn(x^2)), fma(x, x, rn(y^2))."""
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    x2, y2 = (x64 * x64).astype(np.float32), (y64 * y64).astype(np.float32)
    s_add = (x2.astype(np.float64) + y2.astype(np.float64)).astype(np.float32)
    s_fy = _rn_sum_f32(y64 * y64, x2.astype(np.float64))
    s_fx = _rn_sum_f32(x64 * x64, y2.astype(np.float64))
    return {"rn(rn(x2)+rn(y2))": np.sqrt(s_add), "fma(y,y,rn(x2))": np.sqrt(s_fy), "fma(x,x,rn(y2))": np.sqrt(s_fx)}


def test_norm_form():
    rng = np.random.default_rng(7)
    n = 1 << 20
    x = (rng.normal(size=n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    y = (rng.normal(size=n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    c = norm_candidates(x, y)
    a, b, d = (v.view(np.uint32) for v in c.values())
    # after the square root at most two of the three differ on one input; every pair must differ somewhere
    assert min((a != b).sum(), (a != d).sum(), (b != d).sum()) > 100
    keep = (a != b) | (a != d) | (b != d)
    x, y = x[keep], y[keep]
    c = {k: v[keep] for k, v in c.items()}
    g = torch.from_numpy(np.stack([x, y], axis=-1)).to(DEV)
    tn = torch.norm(g, dim=-1).cpu().numpy()
    match = {k: int((v.view(np.uint32) == tn.view(np.uint32)).sum()) for k, v in c.items()}
    print(f"[densify_stats] torch.norm on {torch.cuda.get_device_name()} ({x.size} pairs where the forms differ): "
          f"{match}")
    assert max(match.values()) == x.size, match            # torch takes exactly one of the forms
    P = x.size
    st = (torch.zeros((P, 1), device=DEV), torch.zeros((P, 1), device=DEV), torch.zeros((P,), device=DEV))
    densify.add_densification_stats(*st, g.unsqueeze(0), torch.ones((1, P), dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    assert np.array_equal(st[0].cpu().numpy()[:, 0].view(np.uint32), tn.view(np.uint32))


# (e) no host synchronisation
def test_no_host_sync():
    B, P = 4, 100_000
    stats, grads, radii, _ = random_batch(B, P, seed=5)
    got = tuple(t.clone() for t in stats)
    ref = tuple(t.clone() for t in stats)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        densify.add_densification_stats(*got, grads, radii)
        densify.add_densification_stats(*got, list(grads.unbind(0)), list(radii.unbind(0)))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            reference_chain(*ref, grads.unbind(0), radii.unbind(0))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    n = sum("synchroniz" in str(x.message) for x in w)
    print(f"[densify_stats] reference chain: {n} synchronising calls for {B} cameras ({n / B:g} per camera)")
    assert n >= B


# (f) end to end: Trainer steps, then densify_and_prune; "one_view" steps through the views one at a time, which runs the
# per-camera preprocess
@pytest.mark.parametrize("path", ["batched", "one_view"])
def test_trainer_statistics_and_densification(path):
    cfg = syn.CONFIGS["c1"]
    W, H, N, B = cfg["width"], cfg["height"], cfg["n"], 4
    scene = syn.make_scene(N, W, H, seed=0)
    cams = syn.make_batch_cameras(W, H, B)
    gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=1 + k)).pin_memory() for k in range(B)]
    batches = [None] * 4 if path == "batched" else [[k] for k in range(B)] * 4
    runs = {}
    for way in ("kernel", "reference"):
        tr = pipeline.Trainer(scene, cams, gts, torch.device("cuda", 0), deterministic=True)
        opt = FusedAdam(tr.optimizer_groups(), lr=0.0, eps=1e-15)
        P = tr.n_local
        st = (torch.zeros((P, 1), device=DEV), torch.zeros((P, 1), device=DEV), torch.zeros((P,), device=DEV))
        for views in batches:
            tr.step(views=views, resident=True)
            nv = B if views is None else len(views)
            assert isinstance(tr.means2D, torch.Tensor) and tuple(tr.means2D.shape) == (nv, P, 2)
            if way == "kernel":
                tr.add_densification_stats(*st)
            else:
                reference_chain(*st, tr.means2D.grad.unbind(0), tr._radii_local.unbind(0))
            opt.step(grad_scale=1.0 / nv)
        runs[way] = (tr, opt, st)
    assert_equal_stats(runs["kernel"][2], runs["reference"][2], path)
    accum, denom, maxr = runs["kernel"][2]
    vis = denom[:, 0] > 0
    assert int(vis.sum()) > N // 2 and float(denom.max()) == 4 * B and float(maxr.max()) > 0
    grads = (accum / denom)[vis]
    max_grad = float(torch.quantile(grads, 0.8))
    p = runs["kernel"][0].params
    extent = float(torch.exp(p._scaling.detach()).max(dim=1).values.median()) / 0.01
    noise = torch.randn((2 * N, 3), generator=torch.Generator().manual_seed(3)).to(DEV)
    res = {}
    for way, (tr, opt, (a, d, _m)) in runs.items():
        res[way] = densify.densify_and_prune(opt, a, d, max_grad, 0.005, extent, 0.01, None, noise=noise)
    torch.cuda.synchronize()
    counts = res["kernel"]["counts"]
    print(f"[densify_stats] {path}: counts {counts}")
    assert counts == res["reference"]["counts"] and counts[1] > 0 and counts[3] > 0
    for k in densify.NAMES:
        assert same_bits(res["kernel"][k].detach(), res["reference"][k].detach()), k


# (g) refusals before any launch, outputs left at their sentinels
def test_refusals_leave_outputs_untouched():
    B, P = 3, 1000
    stats, grads, radii, _ = random_batch(B, P, seed=9)
    out = tuple(torch.empty_like(t).view(torch.int32).fill_(i32(s)).view(torch.float32)
                for t, s in zip(stats, (0x7FA5_A5A5, 0x0BAD_F00D, 0xFF80_0001)))
    before = [bits(t) for t in out]
    bad_view = torch.empty(2 * P + 1, device=DEV)[1:].view(P, 2)          # 4 bytes past an 8-byte boundary
    assert bad_view.data_ptr() % 8 == 4
    cases = {
        "B = 0, list": (ValueError, [], []),
        "B = 0, tensor": (ValueError, grads[:0], radii[:0]),
        "B = 65": (ValueError, grads[[0] * 65], radii[[0] * 65]),
        "P mismatch between views": (ValueError, [grads[0], grads[1][:-1]], [radii[0], radii[1]]),
        "P mismatch with the statistics": (ValueError, grads[:, :-1], radii[:, :-1]),
        "float64 gradients": (TypeError, grads.double(), radii),
        "int64 radii": (TypeError, grads, radii.long()),
        "CPU gradients": (TypeError, grads.cpu(), radii),
        "CPU radii": (TypeError, grads, [radii[0].cpu(), radii[1], radii[2]]),
        "None gradient": (TypeError, [grads[0], None, grads[2]], radii),
        "non-contiguous gradients": (ValueError, grads.transpose(1, 2).contiguous().transpose(1, 2), radii),
        "misaligned gradient view": (_lib.GsError, [grads[0], bad_view, grads[2]], radii),
    }
    for name, (exc, g, r) in cases.items():
        with pytest.raises(exc):
            densify.add_densification_stats(*out, g, r)
    with pytest.raises(TypeError):
        densify.add_densification_stats(out[0].cpu(), out[1], out[2], grads, radii)
    with pytest.raises(ValueError):
        densify.add_densification_stats(out[0].reshape(-1), out[1], out[2], grads, radii)
    torch.cuda.synchronize()
    for t, b in zip(out, before):
        assert torch.equal(bits(t), b)
