"""Helpers for the -m gpu parity tests: call the C ABI with torch-owned device buffers and bring
every intermediate back as numpy for comparison with the oracle."""
import ctypes as C

import numpy as np
import torch

from gs_b200 import _lib

DEV = "cuda:0"


def to_dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(DEV)


def stream():
    return torch.cuda.current_stream().cuda_stream


def cam_dev(cam):
    return dict(V=to_dev(cam["viewmatrix"], torch.float32), PM=to_dev(cam["projmatrix"], torch.float32),
                cp=to_dev(cam["campos"], torch.float32))


def nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def preprocess_forward(sc, cam, scale_modifier=1.0):
    """Outputs start as NaN / -7 / 0xAB: the kernel promises to write every one of them for every splat."""
    P = sc["means3D"].shape[0]
    d = {k: to_dev(v, torch.float32) for k, v in sc.items()}
    c = cam_dev(cam)
    out = dict(means2D=nan(P, 2), depths=nan(P), radii=torch.full((P,), -7, dtype=torch.int32, device=DEV),
               conic_opacity=nan(P, 4), rgb=nan(P, 3), clamped=torch.full((P,), 0xAB, dtype=torch.uint8, device=DEV))
    _lib.call("gs_preprocess_forward", P, cam["sh_degree"], d["means3D"].data_ptr(), d["scales"].data_ptr(),
              float(scale_modifier), d["rotations"].data_ptr(), d["opacities"].data_ptr(), d["shs"].data_ptr(),
              c["V"].data_ptr(), c["PM"].data_ptr(), c["cp"].data_ptr(), cam["image_width"], cam["image_height"],
              float(cam["tanfovx"]), float(cam["tanfovy"]), out["means2D"].data_ptr(), out["depths"].data_ptr(),
              out["radii"].data_ptr(), out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(),
              out["clamped"].data_ptr(), stream())
    torch.cuda.synchronize()
    return out, d, c


def preprocess_backward(d, c, cam, pre, g_means2D, g_conic, g_rgb, scale_modifier=1.0):
    P = d["means3D"].shape[0]
    out = dict(means3D=nan(P, 3), scales=nan(P, 3), rotations=nan(P, 4), opacities=nan(P, 1), shs=nan(P, 16, 3))
    _lib.call("gs_preprocess_backward", P, cam["sh_degree"], d["means3D"].data_ptr(), d["scales"].data_ptr(),
              float(scale_modifier), d["rotations"].data_ptr(), d["shs"].data_ptr(), c["V"].data_ptr(),
              c["PM"].data_ptr(), c["cp"].data_ptr(), cam["image_width"], cam["image_height"], float(cam["tanfovx"]),
              float(cam["tanfovy"]), pre["radii"].data_ptr(), pre["clamped"].data_ptr(), g_means2D.data_ptr(),
              g_conic.data_ptr(), g_rgb.data_ptr(), out["means3D"].data_ptr(), out["scales"].data_ptr(),
              out["rotations"].data_ptr(), out["opacities"].data_ptr(), out["shs"].data_ptr(), stream())
    torch.cuda.synchronize()
    return out


def raw_parameters(sc):
    """The six raw GaussianModel parameters of an activated scene (pipeline.GaussianParams) as plain device tensors."""
    from gs_b200 import pipeline
    p = pipeline.GaussianParams(sc, DEV)
    return [t.detach() for t in p.raw_parameters()]


def preprocess_forward_raw(raw, cam, scale_modifier=1.0):
    """gs_preprocess_forward_raw on raw = raw_parameters(...); outputs pre-filled like preprocess_forward's."""
    P = raw[0].shape[0]
    c = cam_dev(cam)
    out = dict(means2D=nan(P, 2), depths=nan(P), radii=torch.full((P,), -7, dtype=torch.int32, device=DEV),
               conic_opacity=nan(P, 4), rgb=nan(P, 3), clamped=torch.full((P,), 0xAB, dtype=torch.uint8, device=DEV))
    _lib.call("gs_preprocess_forward_raw", P, cam["sh_degree"], *(t.data_ptr() for t in raw[:4]), float(scale_modifier),
              raw[4].data_ptr(), raw[5].data_ptr(), c["V"].data_ptr(), c["PM"].data_ptr(), c["cp"].data_ptr(),
              cam["image_width"], cam["image_height"], float(cam["tanfovx"]), float(cam["tanfovy"]),
              out["means2D"].data_ptr(), out["depths"].data_ptr(), out["radii"].data_ptr(),
              out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(), out["clamped"].data_ptr(), stream())
    torch.cuda.synchronize()
    return out


def preprocess_backward_raw(raw, cam, pre, g_means2D, g_conic, g_rgb, scale_modifier=1.0):
    """gs_preprocess_backward_raw -> [d_xyz, d_features_dc, d_features_rest, d_scaling, d_rotation, d_opacity]."""
    P = raw[0].shape[0]
    c = cam_dev(cam)
    out = [torch.full_like(t, float("nan")) for t in raw]
    _lib.call("gs_preprocess_backward_raw", P, cam["sh_degree"], *(t.data_ptr() for t in raw[:4]), float(scale_modifier),
              raw[4].data_ptr(), raw[5].data_ptr(), c["V"].data_ptr(), c["PM"].data_ptr(), c["cp"].data_ptr(),
              cam["image_width"], cam["image_height"], float(cam["tanfovx"]), float(cam["tanfovy"]),
              pre["radii"].data_ptr(), pre["clamped"].data_ptr(), g_means2D.data_ptr(), g_conic.data_ptr(),
              g_rgb.data_ptr(), *(t.data_ptr() for t in out), stream())
    torch.cuda.synchronize()
    return out


def render_forward(H, W, means2D, conic_opacity, rgb, depths, radii, compute_locally, bg, seg=True, stats=True):
    """All tensors on the device. Returns a dict holding every intermediate of the binning + blend.
    seg=False: forward-only call (no segment workspace; a backward then runs the tile-parallel kernel).
    stats=False: no statistics pointer (the forward's non-statistics instantiation)."""
    P = means2D.shape[0]
    T = ((H + 15) // 16) * ((W + 15) // 16)
    cl = compute_locally.to(torch.uint8).contiguous()
    bg_t = to_dev(np.asarray(bg, np.float32))
    offsets = torch.empty((max(P, 1),), dtype=torch.int32, device=DEV)
    order = torch.empty((max(P, 1),), dtype=torch.int32, device=DEV)
    rec = torch.empty((max(P, 1), 12), dtype=torch.float32, device=DEV)
    tb = _lib.query("gs_render_count_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=DEV)
    R = C.c_int64(0)
    _lib.call("gs_render_count", P, H, W, means2D.data_ptr(), conic_opacity.data_ptr(), rgb.data_ptr(),
              depths.data_ptr(), radii.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(),
              temp.data_ptr(), tb, C.byref(R), stream())
    R = int(R.value)
    Ra = max(R, 1)
    tiles = torch.zeros((2, Ra), dtype=torch.int32, device=DEV)
    ids = torch.zeros((2, Ra), dtype=torch.int32, device=DEV)
    sb = _lib.query("gs_render_sort_temp_bytes", R)
    sort_temp = torch.empty((sb,), dtype=torch.uint8, device=DEV)
    ranges = torch.empty((T, 2), dtype=torch.int32, device=DEV)
    image = torch.full((3, H, W), float("nan"), device=DEV)
    final_T = torch.zeros((H, W), device=DEV)
    n_contrib = torch.zeros((H, W), dtype=torch.int32, device=DEV)
    stats = torch.zeros((3,), dtype=torch.int64, device=DEV) if stats else None
    segb = _lib.query("gs_render_seg_bytes", R, T) if seg else 0
    # NaN-filled: the backward must only read checkpoints the forward wrote
    seg_ws = torch.full((segb // 4,), float("nan"), device=DEV).view(torch.uint8) if seg else None
    _lib.call("gs_render_forward", P, R, H, W, means2D.data_ptr(), radii.data_ptr(), cl.data_ptr(), order.data_ptr(),
              offsets.data_ptr(), rec.data_ptr(), bg_t.data_ptr(), tiles[0].data_ptr(), ids[0].data_ptr(),
              tiles[1].data_ptr(), ids[1].data_ptr(), sort_temp.data_ptr(), sb, ranges.data_ptr(), image.data_ptr(),
              final_T.data_ptr(), n_contrib.data_ptr(), _lib.ptr(stats), _lib.ptr(seg_ws), segb, stream())
    torch.cuda.synchronize()
    # the 64-bit keys of the published algorithm, rebuilt from the sorted (tile, splat id) pairs
    ids_s, tiles_s = ids[1][:R].to(torch.int64) & 0xffffffff, tiles[1][:R].to(torch.int64) & 0xffffffff
    dbits = depths.view(torch.int32).to(torch.int64) & 0xffffffff
    keys = (tiles_s << 32) | dbits[ids_s] if R > 0 else torch.zeros((0,), dtype=torch.int64, device=DEV)
    return dict(R=R, offsets=offsets, order=order, rec=rec, keys=keys, ids=ids[1][:R], ids_buf=ids[1], ranges=ranges,
                image=image, final_T=final_T, n_contrib=n_contrib, stats=stats, cl=cl, bg=bg_t, P=P, H=H, W=W,
                seg_ws=seg_ws, seg_bytes=segb)


def render_backward(f, dL_dimage):
    P = f["P"]
    out = dict(means2D=torch.full((P, 2), float("nan"), device=DEV), conic_opacity=torch.full((P, 4), float("nan"), device=DEV),
               rgb=torch.full((P, 3), float("nan"), device=DEV))
    _lib.call("gs_render_backward", P, f["R"], f["H"], f["W"], f["rec"].data_ptr(), f["bg"].data_ptr(),
              f["cl"].data_ptr(), f["ranges"].data_ptr(), f["ids_buf"].data_ptr(), f["final_T"].data_ptr(),
              f["n_contrib"].data_ptr(), dL_dimage.data_ptr(), _lib.ptr(f["seg_ws"]), f["seg_bytes"], out["means2D"].data_ptr(),
              out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(), stream())
    torch.cuda.synchronize()
    return out


def render_forward_batched(H, W, views, bg):
    """gs_render_count_batched + gs_render_forward_batched over views = [(means2D, conic_opacity, rgb, depths, radii,
    compute_locally)] (device tensors; a view may hold no splat).  Outputs start filled like render_forward's."""
    B = len(views)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    cat = [torch.cat([v[q] for v in views]).contiguous() for q in range(5)]
    cl = torch.cat([v[5].to(torch.uint8).reshape(-1) for v in views]).contiguous()
    counts = [int(v[0].shape[0]) for v in views]
    vs = (C.c_int32 * (B + 1))(*np.concatenate([[0], np.cumsum(counts)]).astype(int).tolist())
    P = int(sum(counts))
    bg_t = to_dev(np.asarray(bg, np.float32))
    offsets = torch.empty((max(P, 1),), dtype=torch.int32, device=DEV)
    order = torch.empty((max(P, 1),), dtype=torch.int32, device=DEV)
    rec = torch.empty((max(P, 1), 12), dtype=torch.float32, device=DEV)
    tb = _lib.query("gs_render_count_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=DEV)
    R = C.c_int64(0)
    _lib.call("gs_render_count_batched", B, vs, H, W, *(t.data_ptr() for t in cat[:4]), cat[4].data_ptr(), cl.data_ptr(),
              order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), temp.data_ptr(), tb, C.byref(R), stream())
    R = int(R.value)
    Ra = max(R, 1)
    tiles = torch.zeros((2, Ra), dtype=torch.int32, device=DEV)
    ids = torch.zeros((2, Ra), dtype=torch.int32, device=DEV)
    sb = _lib.query("gs_render_sort_temp_bytes", R)
    sort_temp = torch.empty((sb,), dtype=torch.uint8, device=DEV)
    ranges = torch.empty((B * T, 2), dtype=torch.int32, device=DEV)
    image = torch.full((B, 3, H, W), float("nan"), device=DEV)
    final_T = torch.zeros((B, H, W), device=DEV)
    n_contrib = torch.zeros((B, H, W), dtype=torch.int32, device=DEV)
    stats = torch.zeros((B, 3), dtype=torch.int64, device=DEV)
    segb = _lib.query("gs_render_seg_bytes", R, B * T)
    seg_ws = torch.full((segb // 4,), float("nan"), device=DEV).view(torch.uint8)
    _lib.call("gs_render_forward_batched", B, vs, R, H, W, cat[0].data_ptr(), cat[4].data_ptr(), cl.data_ptr(),
              order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), bg_t.data_ptr(), tiles[0].data_ptr(), ids[0].data_ptr(),
              tiles[1].data_ptr(), ids[1].data_ptr(), sort_temp.data_ptr(), sb, ranges.data_ptr(), image.data_ptr(),
              final_T.data_ptr(), n_contrib.data_ptr(), stats.data_ptr(), seg_ws.data_ptr(), segb, stream())
    torch.cuda.synchronize()
    return dict(B=B, P=P, R=R, H=H, W=W, rec=rec, bg=bg_t, cl=cl, ranges=ranges, ids_buf=ids[1], image=image,
                final_T=final_T, n_contrib=n_contrib, stats=stats, seg_ws=seg_ws, seg_bytes=segb, counts=counts)


def render_backward_batched(f, dL_dimage):
    P = f["P"]
    out = dict(means2D=torch.full((P, 2), float("nan"), device=DEV), conic_opacity=torch.full((P, 4), float("nan"), device=DEV),
               rgb=torch.full((P, 3), float("nan"), device=DEV))
    _lib.call("gs_render_backward_batched", f["B"], P, f["R"], f["H"], f["W"], f["rec"].data_ptr(), f["bg"].data_ptr(),
              f["cl"].data_ptr(), f["ranges"].data_ptr(), f["ids_buf"].data_ptr(), f["final_T"].data_ptr(),
              f["n_contrib"].data_ptr(), dL_dimage.data_ptr(), f["seg_ws"].data_ptr(), f["seg_bytes"],
              out["means2D"].data_ptr(), out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(), stream())
    torch.cuda.synchronize()
    return out


def npy(t):
    return t.detach().cpu().numpy()


def outside(got, ref, rtol=1e-4, atol_scale=1e-4):
    """Fraction of entries with |got-ref| > rtol*|ref| + atol_scale*rms(ref), and the worst |err| / (|ref| + rms)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if not ref.size:
        return 0.0, 0.0
    rms = float(np.sqrt(np.mean(ref ** 2)))
    err = np.abs(got - ref)
    return float((err > rtol * np.abs(ref) + atol_scale * rms).mean()), float((err / (np.abs(ref) + rms + 1e-30)).max())


def floor_report(name, got, ref32, ref64, rtol=1e-4, atol_scale=1e-4):
    """The fp32 noise floor of a quantity: how far the ORACLE's own fp32 evaluation is from its fp64 evaluation of the
    same algorithm, under the same bar as the kernel.  Two fp32 implementations that order their sums differently
    (oracle: pixel-major; kernels: segment / lane-major, FMA-contracted) cannot agree with each other better than each
    agrees with the fp64 value, and hard thresholds (alpha >= 1/255, T < 1e-4, the integer radius) make a few entries flip
    discretely in ANY fp32 evaluation.  -> (outside fraction of got vs fp64, outside fraction of the fp32 oracle vs fp64)."""
    g, wg = outside(got, ref64, rtol, atol_scale)
    o, wo = outside(ref32, ref64, rtol, atol_scale)
    print(f"[parity] {name}: vs the fp64 oracle: kernel outside_tol={g:.2e} worst_rel={wg:.2e} | fp32 oracle outside_tol={o:.2e} "
          f"worst_rel={wo:.2e}   (the fp32 noise floor of this quantity)")
    return g, o


def check_vs_fp64(tag, got, ref32, ref64, scalar_floor=(0.0, 0.0)):
    """The strip loss's bar: (Ll1, ssim, d loss / d image) of a kernel no farther from fp64 than an fp32 evaluation of
    the same loss (the fp32 oracle, or the fp32 form of the fp64 reference).

    A scalar's fp32 error is a sum of per-pixel errors, and one fp32 evaluation's total is one sample of it: where the
    variances cancel (a smooth field over a few hundred pixels) two fp32 evaluations can land 1e-5 relative off fp64
    on either side.  scalar_floor = (Ll1, ssim) sums of the fp32 evaluation's per-pixel |error| bound that sample from
    above; the bar takes the larger of the two.

    The gradient is judged by its worst error, err / (|ref| + rms(ref)), not by the count of entries past the 1e-4 bar.
    Near-flat windows (the flat ground-truth and image regions) make sigma^2 = E[x^2] - mu^2 a cancellation of two
    numbers ~1 down to ~1e-7 next to C2 = 9e-4, so EVERY fp32 evaluation's gradient there is ~1e-4 relative off fp64:
    right at the bar, and how many entries land past it depends on the summation order (the kernel's separable row /
    column passes vs the oracle's), not on correctness.  Measured on an H100: kernel worst 2.4e-4 against the oracle's
    1.8e-4, with up to 0.9 % of the kernel's entries past 1e-4 (0.07 % of the oracle's).  A wrong weight, row or tile
    edge moves the worst error by orders of magnitude."""
    (gl1, gss, gg), (ol1, oss, og), (rl1, rss, rg) = got, ref32, ref64
    for name, k, o, r, f in (("Ll1", gl1, ol1, rl1, scalar_floor[0]), ("ssim", gss, oss, rss, scalar_floor[1])):
        bar = 2 * max(abs(o - r), f) + 1e-6 * abs(r) + 1e-9
        print(f"[parity] {tag}.{name}: rel err kernel {abs(k - r) / (abs(r) + 1e-30):.2e} fp32 {abs(o - r) / (abs(r) + 1e-30):.2e}"
              f" per-pixel floor {f / (abs(r) + 1e-30):.2e} bar {bar / (abs(r) + 1e-30):.2e}")
        assert abs(k - r) <= bar, (tag, name, k, o, r, f)
    floor_report(tag + ".grad", gg, og, rg)
    _, mine = outside(gg, rg)
    _, floor = outside(og, rg)
    assert mine <= 2.0 * floor + 1e-6, (tag, mine, floor)


def rel_report(name, got, ref, rtol=1e-4, atol_scale=1e-4):
    """Fraction of entries outside |got-ref| <= rtol*|ref| + atol_scale*rms(ref).

    The bar: 1e-4 relative (BASELINE.json north_star) plus an absolute floor of 1e-4 x the tensor's RMS.  The floor is
    there because a gradient entry is a signed sum of up to ~1e3 per-pixel terms of magnitude ~RMS: reordering that sum
    perturbs it by ~1e-7 x sum|terms|, which is NOT small relative to an entry that cancels to near zero, and says nothing
    about the entry's own size.  floor_report() measures what that floor has to be (the oracle's fp32-vs-fp64 distance)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    rms = float(np.sqrt(np.mean(ref ** 2))) if ref.size else 0.0
    err = np.abs(got - ref)
    tol = rtol * np.abs(ref) + atol_scale * rms
    bad = err > tol
    frac = float(bad.mean()) if ref.size else 0.0
    worst = float((err / (np.abs(ref) + rms + 1e-30)).max()) if ref.size else 0.0
    print(f"[parity] {name}: n={ref.size} rms={rms:.3e} max_abs_err={err.max() if ref.size else 0:.3e} "
          f"worst_rel={worst:.3e} outside_tol={frac:.2e}")
    return frac, worst
