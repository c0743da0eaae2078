"""-m gpu: the blend kernels on the constructed scenes of tests/blend_cases.py, against the fp32 and fp64 oracles.

Every case runs through both forwards (packed k_blend_fwd2 and half-warp k_blend_fwd), with and without checkpoints and
statistics, the segment backward on each forward's checkpoints, the tile backward (no workspace, and
GS_DEBUG_BWD_TILE), GS_DEBUG_NO_BLOCK_CULL, and the batched forms.  Per-pixel comparisons run on decision-safe pixels
(blend_cases.decision_walk); ambiguous pixels get a zero dL/dimage.  Bars:
  * ids, ranges, keys bit-exact; n_contrib equal to both oracles; statistics exact when no pixel is ambiguous;
  * image and final_T: worst |err| against fp64 <= 2 x the fp32 oracle's + IMG_FLOOR;
  * gradients: worst |err| / (|ref| + rms(ref)) against fp64 <= 2 x the fp32 oracle's + GRAD_FLOOR;
  * splats on no list, culled or below the alpha floor: exactly zero gradient.
"""
import numpy as np
import pytest
import torch

import blend_cases as bc
import gpu_util as gu
from gs_b200 import _lib
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

IMG_FLOOR = 1e-6
GRAD_FLOOR = 1e-5
ATOMICS = 1e-5       # same (splat, tile) sums, different order of the global adds
AMBIGUOUS_MAX = 1e-2  # share of a case's pixels the decision walk may leave out

CASES = {c["name"]: c for c in bc.all_cases()}
_REFS = {}


@pytest.fixture(scope="module")
def oracles():
    import os
    n = max(1, (os.cpu_count() or 8) // 2)
    return Oracle(np.float32, threads=n), Oracle(np.float64, threads=n)


def refs(c, oracles):
    """fp32 / fp64 oracle forward and backward (with the ambiguous pixels' dL/dimage zeroed) and the decision walk."""
    if c["name"] in _REFS:
        return _REFS[c["name"]]
    o32, o64 = oracles
    H, W = c["H"], c["W"]
    f32 = o32.render_forward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["depths"], c["radii"], c["cl"], c["bg"])
    m, co, rgb = bc.upcast(c)
    f64 = o64.render_forward(H, W, m, co, rgb, c["depths"], c["radii"], c["cl"], c["bg"])
    walk = bc.decision_walk(c, f32)
    g = bc.masked_dl(c, walk)
    b32 = o32.render_backward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["bg"], f32, g)
    b64 = o64.render_backward(H, W, m, co, rgb, c["bg"], f64, g.astype(np.float64))
    r = dict(f32=f32, f64=f64, walk=walk, g=g, b32=b32, b64=b64)
    _REFS[c["name"]] = r
    return r


def dev_inputs(c):
    return [gu.to_dev(c[k]) for k in ("means2D", "conic_opacity", "rgb", "depths", "radii")]


def forward(c, bg=None, **kw):
    return gu.render_forward(c["H"], c["W"], *dev_inputs(c), gu.to_dev(c["cl"]), c["bg"] if bg is None else bg, **kw)


def with_flags(flags, fn, *a, **kw):
    old = _lib.debug_set(flags)
    try:
        return fn(*a, **kw)
    finally:
        _lib.debug_set(old)


def worst(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if not ref.size:
        return 0.0
    rms = float(np.sqrt(np.mean(ref ** 2)))
    return float((np.abs(got - ref) / (np.abs(ref) + rms + 1e-30)).max())


def check_grads(tag, got, r):
    for k in ("means2D", "conic_opacity", "rgb"):
        a = gu.npy(got[k])
        assert np.isfinite(a).all(), (tag, k)
        wk, wo = worst(a, r["b64"][k]), worst(r["b32"][k], r["b64"][k])
        print(f"[blend] {tag}.{k}: worst vs fp64 kernel={wk:.2e} fp32 oracle={wo:.2e}")
        assert wk <= 2.0 * wo + GRAD_FLOOR, (tag, k, wk, wo)


def close_atomics(a, b, what):
    for k in ("means2D", "conic_opacity", "rgb"):
        w = worst(gu.npy(a[k]), gu.npy(b[k]))
        assert w <= ATOMICS, (what, k, w)


def seg_layout(f, T):
    """Byte offsets of the segment workspace (blend.cu seg_carve): n_units, tile_last, units, ckpt, cull."""
    al = lambda v: (v + 255) // 256 * 256
    slots = f["R"] // bc.SEG_K + T + 1
    o_tl = 256
    o_units = o_tl + al(T * 4)
    o_ck = o_units + al(slots * 8)
    o_cull = o_ck + slots * 256 * 16
    return dict(o_tl=o_tl, o_units=o_units, o_ck=o_ck, o_cull=o_cull, slots=slots)


def read_checkpoints(f, c, nc):
    """The checkpoint float4s the segment backward reads: pixel p of tile t, boundary s with n_contrib[p] > (s+1) SEG_K,
    as int32 bits -> (keys, values)."""
    H, W = c["H"], c["W"]
    gx, gy = bc.tiles_of(W, H)
    L = seg_layout(f, gx * gy)
    ws = f["seg_ws"]
    ck = ws[L["o_ck"]:L["o_cull"]].view(torch.int32).reshape(-1, 4)
    ranges = gu.npy(f["ranges"]).view(np.uint32)
    keys = []
    ys, xs = np.nonzero(nc > bc.SEG_K)
    for y, x in zip(ys, xs):
        t = (y // 16) * gx + x // 16
        ly, lx = y % 16, x % 16
        idx = ((ly // 4) * 2 + lx // 8) * 32 + (ly % 4) * 8 + lx % 8
        for s in range((int(nc[y, x]) - 1) // bc.SEG_K):
            keys.append((int(ranges[t, 0]) // bc.SEG_K + t + s) * 256 + idx)
    keys = np.array(keys, np.int64)
    return keys, (gu.npy(ck[torch.as_tensor(keys, device=gu.DEV)]) if keys.size else np.zeros((0, 4), np.int32))


def seg_state(f, c):
    gx, gy = bc.tiles_of(c["W"], c["H"])
    L = seg_layout(f, gx * gy)
    ws = f["seg_ws"]
    n_units = int(ws[0:4].view(torch.int32)[0])
    tl = gu.npy(ws[L["o_tl"]:L["o_tl"] + 4 * gx * gy].view(torch.int32))
    units = gu.npy(ws[L["o_units"]:L["o_units"] + 8 * n_units].view(torch.int32)).reshape(-1, 2)
    cull = gu.npy(ws[L["o_cull"]:L["o_cull"] + 2 * f["R"]].view(torch.int16))
    return n_units, tl, units[np.lexsort(units.T[::-1])], cull


@pytest.mark.parametrize("name", list(CASES))
def test_blend_case(oracles, name):
    c = CASES[name]
    r = refs(c, oracles)
    H, W = c["H"], c["W"]
    f32, f64, walk = r["f32"], r["f64"], r["walk"]
    amb = walk["ambiguous"]
    safe = ~amb
    print(f"[blend] {name}: R={f32['R']} ambiguous pixels {int(amb.sum())} of {H * W}")
    assert amb.mean() <= AMBIGUOUS_MAX
    f = forward(c)
    assert f["R"] == f32["R"]
    assert np.array_equal(gu.npy(f["ids"]).view(np.uint32), f32["ids"])
    assert np.array_equal(gu.npy(f["ranges"]).view(np.uint32), f32["ranges"])
    assert np.array_equal(gu.npy(f["keys"]).view(np.uint64), f32["keys"])
    img, fT, nc = gu.npy(f["image"]), gu.npy(f["final_T"]), gu.npy(f["n_contrib"]).astype(np.int64)
    assert np.isfinite(img).all()
    assert np.array_equal(nc[safe], f32["n_contrib"][safe].astype(np.int64))
    assert np.array_equal(nc[safe], f64["n_contrib"][safe].astype(np.int64))
    gx, gy = bc.tiles_of(W, H)
    local = np.repeat(np.repeat(c["cl"].reshape(gy, gx), 16, 0), 16, 1)[:H, :W].astype(bool)
    assert (img[:, ~local] == 0).all()
    for what, got, o32v, o64v in (("image", img[:, safe], f32["image"][:, safe], f64["image"][:, safe]),
                                  ("final_T", fT[safe & local], f32["final_T"][safe & local], f64["final_T"][safe & local])):
        ek = float(np.abs(got - o64v).max()) if got.size else 0.0
        eo = float(np.abs(o32v - o64v).max()) if got.size else 0.0
        print(f"[blend] {name}.{what}: worst |err| vs fp64 kernel={ek:.2e} fp32 oracle={eo:.2e}")
        assert ek <= 2.0 * eo + IMG_FLOOR, (what, ek, eo)
    st = gu.npy(f["stats"])
    assert st[0] == f32["stats"][0]
    if not amb.any():
        assert np.array_equal(st, f32["stats"])

    # ---- forwards: half-warp kernel, no statistics, no checkpoints, no block cull -----------------------------------
    f1 = with_flags(_lib.DEBUG_FWD_HALFWARP, forward, c)
    for k in ("image", "final_T", "n_contrib", "stats"):
        assert torch.equal(f[k], f1[k]), k
    if f["R"]:
        k2, v2 = read_checkpoints(f, c, nc)
        k1, v1 = read_checkpoints(f1, c, nc)
        assert np.array_equal(k1, k2) and np.array_equal(v1, v2), "checkpoints"
        assert not np.isnan(v2.view(np.float32)).any()
        s2, s1 = seg_state(f, c), seg_state(f1, c)
        assert s2[0] == s1[0] and all(np.array_equal(a, b) for a, b in zip(s2[1:], s1[1:])), "segment bookkeeping"
        assert s2[0] == int(((s2[1].astype(np.int64) + bc.SEG_K - 1) // bc.SEG_K).sum())
        assert np.array_equal(s2[1], (np.maximum(walk_tile_max(nc, gx, gy), 0) * c["cl"]).astype(np.int32))
    for flags in (0, _lib.DEBUG_FWD_HALFWARP):
        fs = with_flags(flags, forward, c, stats=False)
        fn = with_flags(flags, forward, c, seg=False)
        for k in ("image", "final_T", "n_contrib"):
            assert torch.equal(fs[k], f[k]) and torch.equal(fn[k], f[k]), (flags, k)
    fc = with_flags(_lib.DEBUG_NO_BLOCK_CULL, forward, c)
    for k in ("image", "final_T", "n_contrib", "stats"):
        assert torch.equal(fc[k], f[k]), ("no block cull", k)

    # ---- backwards ----------------------------------------------------------------------------------------------------
    g = gu.to_dev(r["g"])
    b_seg = gu.render_backward(f, g)
    check_grads(f"{name}.seg", b_seg, r)
    check_grads(f"{name}.seg_on_halfwarp", gu.render_backward(f1, g), r)
    check_grads(f"{name}.tile_flag", with_flags(_lib.DEBUG_BWD_TILE, gu.render_backward, f, g), r)
    check_grads(f"{name}.tile_noseg", gu.render_backward(fn, g), r)
    close_atomics(gu.render_backward(fc, g), b_seg, "no block cull")
    close_atomics(with_flags(_lib.DEBUG_NO_BLOCK_CULL | _lib.DEBUG_BWD_TILE, gu.render_backward, fc, g),
                  with_flags(_lib.DEBUG_BWD_TILE, gu.render_backward, f, g), "no block cull, tile backward")

    # ---- exact zeros ---------------------------------------------------------------------------------------------------
    P = c["means2D"].shape[0]
    off_list = ~np.isin(np.arange(P), f32["ids"])
    below = c["conic_opacity"][:, 3] < bc.INV255
    for k in ("means2D", "conic_opacity", "rgb"):
        a = gu.npy(b_seg[k])
        assert (a[off_list | below] == 0).all(), k


def walk_tile_max(nc, gx, gy):
    H, W = nc.shape
    pad = np.zeros((gy * 16, gx * 16), np.int64)
    pad[:H, :W] = nc
    return pad.reshape(gy, 16, gx, 16).max((1, 3)).reshape(-1)


@pytest.mark.parametrize("name", ["saturation_bg1", "lengths_mask_all", "clamp", "floor", "degenerate", "ragged_17x33"])
def test_single_pixel_gradient(oracles, name):
    """dL/dimage non-zero at ONE pixel: only the splats of that pixel's list up to its n_contrib may get a gradient,
    and those match the fp64 oracle."""
    base = CASES[name]
    rb = refs(base, oracles)
    nc = rb["f32"]["n_contrib"].astype(np.int64)
    cand = np.where(rb["walk"]["ambiguous"], -1, nc)
    y, x = np.unravel_index(int(np.argmax(cand)), cand.shape)
    c = bc.single_pixel_dl(base, y, x)
    r = refs(c, oracles)
    f = forward(c)
    gx, _ = bc.tiles_of(c["W"], c["H"])
    t = (y // 16) * gx + x // 16
    beg = int(r["f32"]["ranges"][t, 0])
    allowed = np.zeros(c["means2D"].shape[0], bool)
    allowed[r["f32"]["ids"][beg:beg + nc[y, x]]] = True
    assert allowed.sum() == nc[y, x] > 0
    g = gu.to_dev(r["g"])
    for tag, b in (("seg", gu.render_backward(f, g)), ("tile", with_flags(_lib.DEBUG_BWD_TILE, gu.render_backward, f, g))):
        for k in ("means2D", "conic_opacity", "rgb"):
            a = gu.npy(b[k])
            assert (a[~allowed] == 0).all(), (tag, k)
            assert (np.abs(a[allowed]).sum(1) > 0).any(), (tag, k)
        check_grads(f"{c['name']}.{tag}", b, r)


def _views_of(cs):
    return [(*dev_inputs(c), gu.to_dev(c["cl"])) for c in cs]


def _empty_view(c):
    z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=gu.DEV)
    return (z(0, 2), z(0, 4), z(0, 3), z(0), z(0, dt=torch.int32), gu.to_dev(np.ones_like(c["cl"])))


def _check_batched(cs, bg):
    """cs: cases of one image size, None = an empty view.  Each slice == the single-view call bit for bit; gradients
    equal up to the order of the atomics."""
    real = [c for c in cs if c is not None]
    H, W = real[0]["H"], real[0]["W"]
    views = [(_empty_view(real[0]) if c is None else _views_of([c])[0]) for c in cs]
    fb = gu.render_forward_batched(H, W, views, bg)
    dl = torch.stack([gu.to_dev(np.zeros((3, H, W), np.float32) if c is None else c["dL"]) for c in cs])
    bb = gu.render_backward_batched(fb, dl.contiguous())
    vs = np.concatenate([[0], np.cumsum(fb["counts"])])
    for k, c in enumerate(cs):
        if c is None:
            assert fb["counts"][k] == 0 and int(fb["stats"][k, 0]) == 0
            assert (fb["image"][k] == torch.tensor(bg, device=gu.DEV)[:, None, None]).all()
            continue
        f = forward(c, bg=bg)
        for q in ("image", "final_T", "n_contrib"):
            assert torch.equal(fb[q][k], f[q]), (c["name"], k, q)
        assert torch.equal(fb["stats"][k], f["stats"]), (c["name"], k)
        b = gu.render_backward(f, gu.to_dev(c["dL"]))
        close_atomics({q: bb[q][vs[k]:vs[k + 1]] for q in b}, b, f"batched view {k} ({c['name']})")


def test_batched_views_equal_single_view_calls():
    """The 64x48 cases as the views of one batched call (ragged view_start, one empty view), then 64 views."""
    group = [c for c in CASES.values() if (c["W"], c["H"]) == (64, 48)]
    assert len(group) >= 6
    bg = (0.3, 0.6, 0.9)
    _check_batched([group[0], None] + group[1:], bg)
    cs = [group[k % len(group)] for k in range(63)]
    _check_batched(cs[:20] + [None] + cs[20:], bg)
    small = [CASES[n] for n in ("ties", "degenerate")]
    _check_batched(small + [None], (0.0, 0.0, 0.0))
