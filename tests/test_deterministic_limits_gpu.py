"""-m gpu: the deterministic render and loss at their limits, against the orders tests/det_ref.py states (pinned on CPU
by tests/test_det_ref.py) and the fp64 oracle.

  * order pinned: after gs_render_backward_det the workspace still holds the instance rows, rank, n_long and long_g;
    rank inverts order, the long list is the set of ranges longer than 16 rows, and every splat's 9 outputs are
    det_ref.reduce_splat of its rows bit for bit -- on ranges of exactly 0, 1, 15, 16, 17, 255, 256, 257, 4097 and
    8224 rows (plus a checkerboard-masked second view), 3200 long ranges (three rounds of the 1056 persistent CTAs),
    the whole-image splat and c2;
  * instance rows: on the 64x48 blend cases each stored row is its tile's share, against the fp64 oracle run on that
    tile alone; rows past the tile's n_contrib or block-culled are exactly 0;
  * every blend case against fp64 with test_blend_gpu's bars, on the packed and the half-warp forward's checkpoints
    (the same bits), splats on no list +0.0, and the single-pixel allowed-splat check;
  * batched == single-view calls bit for bit, at ragged view_start with empty views and at B = 64; B = 65 refused;
  * the deterministic forward == the default on the binning populations (depth kinds, 64 x 1080p, 2 M at 4K);
  * the loss: CTA partials at their documented slots (unused ones 0.0), each output finalize_view of its slots bit for
    bit, within 1 ulp of the atomic form and within the loss suite's fp64 bar, on loss_cases windows, halo rows,
    unequal and empty views and 4K;
  * refusals with every output still holding its sentinel.
Each call runs once; nothing is repeated to look for a difference."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import binning_cases as bic
import blend_cases as bc
import det_ref as dr
import gpu_util as gu
import loss_cases as lc
from det_util import (assert_forward_unchanged, backward, binning_views, bits_equal, case_view, dl_like, empty_view,
                      forward, grad_rows, projected_view, read_det_ws, whole_image_scene)
from gs_b200 import _lib
from gs_b200 import synthetic as syn
from test_blend_gpu import CASES, GRAD_FLOOR, check_grads, oracles, refs, seg_layout, with_flags, worst  # noqa: F401
from test_loss_cases_gpu import batch_rows, gptrs, gt_strips, i32, view_grads, within_ulp
from test_loss_cases_gpu import refs as loss_refs

pytestmark = pytest.mark.gpu

GS_EINVAL, GS_ENOMEM = -1, -3
SMALL = [n for n, c in CASES.items() if (c["W"], c["H"]) == (64, 48)]


@pytest.fixture(scope="module", autouse=True)
def file_time():
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[det limits] {time.perf_counter() - t0:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ---------------------------------------------------------------------------------------------------------------------
# the reduce order, read back out of the workspace
# ---------------------------------------------------------------------------------------------------------------------
def check_order(f, g, ws, tag):
    """-> (range lengths per depth position, n_long)."""
    P, R = f["P"], f["R"]
    order = gu.npy(f["order"][:P]).view(np.uint32).astype(np.int64)
    offsets = gu.npy(f["offsets"][:P]).view(np.uint32)
    n_long, inst, rank, long_g = read_det_ws(ws, R, P)
    assert np.array_equal(rank[order], np.arange(P)), tag                      # rank inverts order
    want = dr.long_set(offsets, order)
    assert n_long == want.size and np.array_equal(np.sort(long_g.astype(np.int64)), want), (tag, n_long, want.size)
    exp = dr.reduce_all(inst, offsets, order)
    got = grad_rows(g)
    bad = np.nonzero((got.view(np.uint32) != exp.view(np.uint32)).any(1))[0]
    lens = dr.range_lengths(offsets)
    assert bad.size == 0, (tag, bad[:8], lens[np.argsort(order)][bad[:8]])
    return lens, n_long


def order_scene(name):
    if name == "range_lengths":
        c, _ = dr.range_length_scene()
        return c["H"], c["W"], binning_views(c), (0.1, 0.2, 0.3)
    if name == "long_population":
        c, _ = dr.long_population()
        return c["H"], c["W"], binning_views(c), (0.0, 0.0, 0.0)
    if name == "whole_image":
        c = whole_image_scene()
        return c["H"], c["W"], [case_view(c)], c["bg"]
    cfg = syn.CONFIGS["c2"]
    W, H = cfg["width"], cfg["height"]
    sc = syn.make_scene(cfg["n"], W, H, seed=0)
    return H, W, [projected_view(sc, syn.make_camera(W, H, yaw_deg=0.0))], (0.0, 0.0, 0.0)


@pytest.mark.parametrize("name", ["range_lengths", "long_population", "whole_image", "c2"])
def test_reduce_order_pinned(name):
    H, W, views, bg = order_scene(name)
    f = forward(views, H, W, bg, det=True)
    g, ws = backward(f, dl_like(f, 11), det=True, return_ws=True)
    lens, n_long = check_order(f, g, ws, name)
    hist = {int(k): int(v) for k, v in zip(*np.unique(lens, return_counts=True))}
    shown = {k: v for k, v in hist.items() if k <= 20 or k in (255, 256, 257) or k > 4000}
    print(f"[det limits] {name}: P={f['P']} R={f['R']} n_long={n_long} range lengths (rows: splats) {shown}")
    if name == "range_lengths":
        for n in (0, 1, 15, 16, 17, 255, 256, 257, 4097, 257 * 32):
            assert hist.get(n, 0) > 0, n
    if name == "long_population":
        assert n_long > dr.DR_LONG_CTAS * 2
    if name == "whole_image":
        assert max(hist) >= 1200


# ---------------------------------------------------------------------------------------------------------------------
# instance rows: each one its tile's share
# ---------------------------------------------------------------------------------------------------------------------
def tile_refs(c, g, oracles):
    """Per tile t with a list: the fp32 / fp64 oracle backward of the case with only tile t local -> {t: (b32, b64)}."""
    o32, o64 = oracles
    H, W = c["H"], c["W"]
    m, co, rgb = bc.upcast(c)
    out = {}
    for t in np.nonzero(c["cl"])[0]:
        cl = np.zeros_like(c["cl"])
        cl[t] = 1
        f32 = o32.render_forward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["depths"], c["radii"], cl, c["bg"])
        if f32["R"] == 0:
            continue
        f64 = o64.render_forward(H, W, m, co, rgb, c["depths"], c["radii"], cl, c["bg"])
        b32 = o32.render_backward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["bg"], f32, g)
        b64 = o64.render_backward(H, W, m, co, rgb, c["bg"], f64, g.astype(np.float64))
        out[int(t)] = tuple(np.concatenate([b[k] for k in ("means2D", "conic_opacity", "rgb")], 1) for b in (b32, b64))
    return out


@pytest.mark.parametrize("name", SMALL)
def test_instance_rows_vs_fp64_per_tile(oracles, name):
    c = CASES[name]
    r = refs(c, oracles)
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True)
    g, ws = backward(f, gu.to_dev(r["g"])[None].contiguous(), det=True, return_ws=True)
    R, P = f["R"], f["P"]
    _, inst, _, _ = read_det_ws(ws, R, P)
    if R == 0:
        assert (grad_rows(g).view(np.uint32) == 0).all()
        return
    slot_tile = gu.npy(f["tiles_unsorted"][:R]).astype(np.int64)
    slot_id = gu.npy(f["ids_unsorted"][:R]).astype(np.int64)
    per_tile = tile_refs(c, r["g"], oracles)
    assert set(np.unique(slot_tile)) == set(per_tile)
    r32, r64 = np.zeros((R, 9)), np.zeros((R, 9))
    for s in range(R):
        b32, b64 = per_tile[slot_tile[s]]
        r32[s], r64[s] = b32[slot_id[s]], b64[slot_id[s]]
    for k, cols in (("means2D", slice(0, 2)), ("conic_opacity", slice(2, 6)), ("rgb", slice(6, 9))):
        wk, wo = worst(inst[:, cols], r64[:, cols]), worst(r32[:, cols], r64[:, cols])
        print(f"[det limits] {name}.instance_rows.{k}: worst vs fp64 det={wk:.2e} fp32 oracle={wo:.2e}")
        assert wk <= 2.0 * wo + GRAD_FLOOR, (name, k, wk, wo)
    # rows the walk never reaches: past the tile's deepest contributing entry, or culled in every 4x4 block
    nc = gu.npy(f["n_contrib"][0]).astype(np.int64)
    gx, gy = bc.tiles_of(c["W"], c["H"])
    pad = np.zeros((gy * 16, gx * 16), np.int64)
    pad[:c["H"], :c["W"]] = nc
    tile_last = pad.reshape(gy, 16, gx, 16).max((1, 3)).reshape(-1)
    ranges = gu.npy(f["ranges"]).astype(np.int64)
    su = gu.npy(f["sorted_u"][:R]).astype(np.int64)
    pos = np.empty(R, np.int64)
    pos[su] = np.arange(R) - ranges[slot_tile[su], 0]               # list position of every slot in its tile
    o_cull = seg_layout(f, gx * gy)["o_cull"]
    cull = np.empty(R, np.int64)
    cull[su] = gu.npy(f["seg_ws"][o_cull:o_cull + 2 * R].view(torch.int16)).astype(np.int64)
    unreached = pos >= tile_last[slot_tile]
    culled = ~unreached & (cull == 0)
    assert (inst[unreached | culled] == 0).all(), name
    print(f"[det limits] {name}: {R} instance rows, {int(unreached.sum())} past n_contrib, {int(culled.sum())} culled")


# ---------------------------------------------------------------------------------------------------------------------
# every blend case against fp64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_blend_case_deterministic(oracles, name):
    c = CASES[name]
    r = refs(c, oracles)
    g = gu.to_dev(r["g"])[None].contiguous()
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True)
    b = backward(f, g, det=True)
    check_grads(f"{name}.det", b, r)
    f1 = with_flags(_lib.DEBUG_FWD_HALFWARP, forward, [case_view(c)], c["H"], c["W"], c["bg"], det=True)
    b1 = backward(f1, g, det=True)
    for k in b:
        assert bits_equal(b[k], b1[k]), (name, "half-warp checkpoints", k)
    P = c["means2D"].shape[0]
    off_list = ~np.isin(np.arange(P), r["f32"]["ids"])
    below = c["conic_opacity"][:, 3] < bc.INV255
    rows = grad_rows(b)
    assert (rows[off_list].view(np.uint32) == 0).all(), name       # no rows: the sum's own +0.0
    assert (rows[below] == 0).all(), name                          # rows of zeros, each times a signed scale


@pytest.mark.parametrize("name", ["saturation_bg1", "lengths_mask_all", "clamp", "floor", "degenerate", "ragged_17x33"])
def test_single_pixel_gradient_deterministic(oracles, name):
    base = CASES[name]
    rb = refs(base, oracles)
    nc = rb["f32"]["n_contrib"].astype(np.int64)
    y, x = np.unravel_index(int(np.argmax(np.where(rb["walk"]["ambiguous"], -1, nc))), nc.shape)
    c = bc.single_pixel_dl(base, y, x)
    r = refs(c, oracles)
    gx, _ = bc.tiles_of(c["W"], c["H"])
    beg = int(r["f32"]["ranges"][(y // 16) * gx + x // 16, 0])
    allowed = np.zeros(c["means2D"].shape[0], bool)
    allowed[r["f32"]["ids"][beg:beg + nc[y, x]]] = True
    assert allowed.sum() == nc[y, x] > 0
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True)
    b = backward(f, gu.to_dev(r["g"])[None].contiguous(), det=True)
    rows = grad_rows(b)
    assert (rows[~allowed] == 0).all() and (np.abs(rows[allowed]).sum(1) > 0).any()
    check_grads(f"{c['name']}.det", b, r)


# ---------------------------------------------------------------------------------------------------------------------
# batched == single-view, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def check_batched_equals_single(cs, bg):
    """cs: cases of one size, None = an empty view."""
    real = [c for c in cs if c is not None]
    H, W = real[0]["H"], real[0]["W"]
    views = [empty_view(H, W) if c is None else case_view(c) for c in cs]
    fb = forward(views, H, W, bg, det=True)
    dl = torch.stack([torch.zeros((3, H, W), device=gu.DEV) if c is None else gu.to_dev(c["dL"]) for c in cs])
    gb = backward(fb, dl.contiguous(), det=True)
    vs = np.concatenate([[0], np.cumsum([0 if c is None else c["means2D"].shape[0] for c in cs])])
    single = {}
    for k, c in enumerate(cs):
        if c is None:
            assert vs[k + 1] == vs[k] and bool((fb["n_contrib"][k] == 0).all())
            continue
        if c["name"] not in single:
            f = forward([case_view(c)], H, W, bg, det=True)
            single[c["name"]] = (f, backward(f, gu.to_dev(c["dL"])[None].contiguous(), det=True))
        f, g = single[c["name"]]
        for q in ("image", "final_T", "n_contrib"):
            assert bits_equal(fb[q][k], f[q][0]), (c["name"], k, q)
        for q in g:
            assert bits_equal(gb[q][vs[k]:vs[k + 1]], g[q]), (c["name"], k, q)
    return fb["B"]


def test_batched_equals_single_view_calls_bit_for_bit():
    group = [CASES[n] for n in SMALL]
    assert len(group) >= 6
    bg = (0.3, 0.6, 0.9)
    check_batched_equals_single([group[0], None] + group[1:] + [None], bg)
    cs = [group[k % len(group)] for k in range(63)]
    B = check_batched_equals_single(cs[:20] + [None] + cs[20:], bg)
    assert B == 64
    print(f"[det limits] batched == single bit for bit, largest batch {B} views")


def test_65_views_refused_before_any_launch():
    c = CASES[SMALL[0]]
    H, W = c["H"], c["W"]
    T = int(np.prod(bc.tiles_of(W, H)))
    lib = _lib.load()
    B = 65
    vs = (C.c_int32 * (B + 1))(*([0] + [1] * B))
    P, R = 1, 4
    buf = {k: torch.full((n,), -7, dtype=torch.int32, device=gu.DEV)
           for k, n in (("order", P), ("offsets", P), ("t0", R), ("i0", R), ("t1", R), ("i1", R), ("su", R),
                        ("ranges", 2 * B * T), ("nc", B * H * W))}
    fl = {k: gu.nan(n) for k, n in (("m", 2 * P), ("rec", 12 * P), ("bg", 3), ("img", 3 * B * H * W),
                                     ("fT", B * H * W))}
    rad = torch.ones((P,), dtype=torch.int32, device=gu.DEV)
    cl = torch.ones((B * T,), dtype=torch.uint8, device=gu.DEV)
    stats = torch.full((B, 3), -7, dtype=torch.int64, device=gu.DEV)
    ts = torch.full((B * T, 3), -7, dtype=torch.int64, device=gu.DEV)
    st = torch.empty((1 << 16,), dtype=torch.uint8, device=gu.DEV)
    torch.cuda.synchronize()
    rc = lib.gs_render_forward_det(B, vs, P, R, H, W, fl["m"].data_ptr(), rad.data_ptr(), cl.data_ptr(),
                                   buf["order"].data_ptr(), buf["offsets"].data_ptr(), fl["rec"].data_ptr(),
                                   fl["bg"].data_ptr(), *(buf[k].data_ptr() for k in ("t0", "i0", "t1", "i1", "su")),
                                   st.data_ptr(), st.numel(), buf["ranges"].data_ptr(), fl["img"].data_ptr(),
                                   fl["fT"].data_ptr(), buf["nc"].data_ptr(), stats.data_ptr(), ts.data_ptr(), None, 0,
                                   gu.stream())
    assert rc == GS_EINVAL and b"GS_MAX_VIEWS" in lib.gs_last_error()
    grads = [gu.nan(2 * P), gu.nan(4 * P), gu.nan(3 * P)]
    nb = _lib.query("gs_render_det_bytes", R, P)
    ws = torch.full((nb,), 0x5A, dtype=torch.uint8, device=gu.DEV)
    rc = lib.gs_render_backward_det(B, P, R, H, W, fl["rec"].data_ptr(), fl["bg"].data_ptr(), cl.data_ptr(),
                                    buf["ranges"].data_ptr(), buf["i1"].data_ptr(), buf["su"].data_ptr(),
                                    buf["order"].data_ptr(), buf["offsets"].data_ptr(), fl["fT"].data_ptr(),
                                    buf["nc"].data_ptr(), fl["img"].data_ptr(), st.data_ptr(), st.numel(),
                                    ws.data_ptr(), nb, *(t.data_ptr() for t in grads), gu.stream())
    assert rc == GS_EINVAL and b"GS_MAX_VIEWS" in lib.gs_last_error()
    torch.cuda.synchronize()
    assert all(bool((t == -7).all()) for t in buf.values()) and bool((stats == -7).all()) and bool((ts == -7).all())
    assert all(bool(torch.isnan(t).all()) for t in list(fl.values()) + grads) and bool((ws == 0x5A).all())


# ---------------------------------------------------------------------------------------------------------------------
# the deterministic forward on the binning populations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["equal", "runs", "ulp", "loguniform", "special"])
def test_forward_unchanged_depth_kinds(kind):
    c = bic.depth_case(kind)
    assert_forward_unchanged(binning_views(c), c["H"], c["W"], (0.1, 0.2, 0.3), c["name"])


@pytest.mark.parametrize("which", ["views_1080p", "p_2m_4k"])
def test_forward_unchanged_large(which):
    c = bic.views_1080p() if which == "views_1080p" else bic.size_case(2 ** 21 + 5, 3840, 2160, rmax=12)
    _, b = assert_forward_unchanged(binning_views(c), c["H"], c["W"], (0.0, 0.0, 0.0), c["name"])
    print(f"[det limits] {which}: B={b['B']} P={b['P']} R={b['R']} forward bit-identical")
    del b
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# loss
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_tf32():
    """The fp32 floor of the loss bar must be fp32 (TF32 convolutions sit ~1e-3 off fp64)."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def loss_det(images, gts, rows4, single=False, short=0):
    """The _det loss forward (batched entry point, or the single-view one for one view) with out NaN-filled and temp
    0xA5-filled; short: bytes less than it needs -> (rc, out, temp, header)."""
    B, _, H, W = images.shape
    header = dr.LOSS_HEADER_1 if single else dr.LOSS_HEADER_B
    tb = (_lib.query("gs_loss_temp_bytes_det", rows4[0][1] - rows4[0][0], W) if single else
          _lib.query("gs_loss_temp_bytes_batched_det", B, i32(rows4), W))
    assert tb == dr.loss_need(header, rows4, W) + 256
    if short:
        tb = dr.loss_need(header, rows4, W) - short
    temp = torch.full((tb,), 0xA5, dtype=torch.uint8, device=gu.DEV)
    out = gu.nan(B, 2)
    if single:
        rc = _lib.query("gs_loss_forward_det", H, W, *rows4[0], images[0].data_ptr(), gts[0].data_ptr(), out.data_ptr(),
                        temp.data_ptr(), tb, gu.stream())
    else:
        rc = _lib.query("gs_loss_forward_batched_det", B, H, W, i32(rows4), images.data_ptr(), gptrs(gts),
                        out.data_ptr(), temp.data_ptr(), tb, gu.stream())
    torch.cuda.synchronize()
    return rc, out, temp, header


def loss_atomic(images, gts, rows4, gl1, gss):
    """The atomic batched forward + backward -> (out, dimg) numpy."""
    B, _, H, W = images.shape
    tb = _lib.query("gs_loss_temp_bytes_batched", B, i32(rows4), W)
    temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
    out = gu.nan(B, 2)
    _lib.call("gs_loss_forward_batched", B, H, W, i32(rows4), images.data_ptr(), gptrs(gts), out.data_ptr(),
              temp.data_ptr(), tb, gu.stream())
    return gu.npy(out), loss_backward(images, gts, rows4, temp, gl1, gss, False)


def loss_backward(images, gts, rows4, temp, gl1, gss, single):
    B, _, H, W = images.shape
    dimg = torch.full_like(images, float("nan"))
    g1, g2 = gu.to_dev(gl1), gu.to_dev(gss)
    if single:
        _lib.call("gs_loss_backward", H, W, *rows4[0], images[0].data_ptr(), gts[0].data_ptr(), temp.data_ptr(),
                  g1.data_ptr(), g2.data_ptr(), dimg.data_ptr(), gu.stream())
    else:
        _lib.call("gs_loss_backward_batched", B, H, W, i32(rows4), images.data_ptr(), gptrs(gts), temp.data_ptr(),
                  g1.data_ptr(), g2.data_ptr(), dimg.data_ptr(), gu.stream())
    torch.cuda.synchronize()
    return gu.npy(dimg)


def check_loss(images, gts, rows4, tag, single=False, fp64_views=None):
    B, _, H, W = images.shape
    rc, out, temp, header = loss_det(images, gts, rows4, single)
    assert rc == 0, (tag, _lib.load().gs_last_error())
    out = gu.npy(out)
    off, slots = dr.loss_slots(header, rows4, W)
    part = gu.npy(temp[off:off + 16 * B * slots].view(torch.float64)).reshape(B, slots, 2)
    assert (gu.npy(temp[off + 16 * B * slots:]) == 0xA5).all(), tag          # nothing past the last slot
    gxl = -(-W // dr.LS_TILE)
    inv = dr.loss_inv_norm(H, W)
    gl1, gss = view_grads(B)
    ref_out, ref_dimg = loss_atomic(images, gts, rows4, gl1, gss)
    dimg = loss_backward(images, gts, rows4, temp, gl1, gss, single)
    assert np.array_equal(dimg.view(np.uint32), ref_dimg.view(np.uint32)), tag   # the maps are the atomic form's
    for v, r in enumerate(rows4):
        used = -(-(r[1] - r[0]) // dr.LS_TILE) * gxl
        assert (part[v, used:] == 0).all() and not (part[v, used:].view(np.uint64) >> 63).any(), (tag, v)
        for q in range(2):
            want = dr.finalize_view(part[v, :, q], inv)
            assert out[v, q].view(np.uint32) == want.view(np.uint32), (tag, v, q, out[v, q], want)
            assert within_ulp(out[v, q], ref_out[v, q]), (tag, v, q, out[v, q], ref_out[v, q])
        if fp64_views is not None and v in fp64_views and r[1] > r[0]:
            # the loss suite's scalar bar (gu.check_vs_fp64); the gradient is the atomic form's, bit for bit (above)
            r64, r32, floor = loss_refs(images[v], gts[v], r, gl1[v], gss[v])
            for q in range(2):
                bar = 2 * max(abs(r32[q] - r64[q]), floor[q]) + 1e-6 * abs(r64[q]) + 1e-9
                assert abs(float(out[v, q]) - r64[q]) <= bar, (tag, v, q, float(out[v, q]), r32[q], r64[q], floor[q])
    return slots


@pytest.mark.parametrize("B,H,W", [(5, 48, 33), (7, 97, 12), (64, 95, 11), (64, 32, 32)])
def test_loss_windows_halo_and_unequal_views(no_tf32, B, H, W):
    """loss_cases windows crossed with whole / halo / empty counted rows (batch_rows): unequal heights, empty views first,
    in the middle and last, so the CTAs below a short strip write zeros."""
    rows4 = batch_rows(H, B, seed=B * 7 + H + W)
    assert len({r[1] - r[0] for r in rows4}) > 2
    pairs = [lc.make_pair(H, W, seed=600 + v, kind=("mixed", "checker", "smooth")[v % 3] if W > 2 else "mixed")
             for v in range(B)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gts = gt_strips([p[1] for p in pairs], rows4)
    check_loss(images, gts, rows4, f"B={B} {H}x{W}", fp64_views=set(range(0, B, 5)))


def test_loss_4k(no_tf32):
    """3840x2160: the single-view entry point on the whole image (8160 slots: 255 per lane), then two views of it and an
    empty one through the batched entry point, one a 24-row halo window."""
    H, W = 2160, 3840
    img, gt = lc.make_pair(H, W, seed=H, kind="smooth")
    x = gu.to_dev(img)[None].contiguous()
    slots = check_loss(x, [gu.to_dev(gt)], [(0, H, 0, H)], "4K single", single=True, fp64_views={0})
    assert slots == 120 * 68
    rows4 = [(0, H, 0, H), (0, 0, 0, 0), (H - 40, H, H - 35, H - 5)]
    images = x.expand(3, 3, H, W).contiguous()
    gts = [gu.to_dev(gt), None, gu.to_dev(gt[:, H - 40:])]
    check_loss(images, gts, rows4, "4K batched")


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_outputs_untouched():
    c = CASES[SMALL[0]]
    f = forward([case_view(c)], c["H"], c["W"], c["bg"], det=True)
    dL = dl_like(f, 2)
    P, R = f["P"], f["R"]
    assert R > 0
    nb = _lib.query("gs_render_det_bytes", R, P)
    assert nb == dr.det_carve(R, P)["total"]
    lib = _lib.load()
    ws = torch.full((nb + 512,), 0x5A, dtype=torch.uint8, device=gu.DEV)
    base = (ws.data_ptr() + 255) // 256 * 256

    def call(R_, seg_bytes, ws_ptr, ws_bytes):
        grads = [gu.nan(P, 2), gu.nan(P, 4), gu.nan(P, 3)]
        rc = lib.gs_render_backward_det(1, P, R_, f["H"], f["W"], f["rec"].data_ptr(), f["bg"].data_ptr(),
                                        f["cl"].data_ptr(), f["ranges"].data_ptr(), f["ids"].data_ptr(),
                                        f["sorted_u"].data_ptr(), f["order"].data_ptr(), f["offsets"].data_ptr(),
                                        f["final_T"].data_ptr(), f["n_contrib"].data_ptr(), dL.data_ptr(),
                                        f["seg_ws"].data_ptr(), seg_bytes, ws_ptr, ws_bytes,
                                        *(t.data_ptr() for t in grads), gu.stream())
        torch.cuda.synchronize()
        return rc, lib.gs_last_error(), grads

    for what, args, code, msg in (
            ("det_ws one byte short", (R, f["seg_bytes"], base, nb - 1), GS_ENOMEM, b"det_ws too small"),
            ("det_ws misaligned", (R, f["seg_bytes"], base + 4, nb), GS_EINVAL, b"256-byte aligned"),
            ("segment workspace one byte short", (R, f["seg_bytes"] - 1, base, nb), GS_ENOMEM, b"segment workspace"),
            ("R = 2^31", (2 ** 31, f["seg_bytes"], base, nb), GS_EINVAL, b"sizes")):
        rc, err, grads = call(*args)
        assert rc == code and msg in err, (what, rc, err)
        assert all(bool(torch.isnan(t).all()) for t in grads), what
        assert bool((ws == 0x5A).all()), what
    rc, _, grads = call(R, f["seg_bytes"], base, nb)           # the same buffers at their sizes: accepted
    assert rc == 0 and all(bool(torch.isfinite(t).all()) for t in grads)

    H, W = 70, 33
    rows4 = [(5, 70, 10, 65), (0, 0, 0, 0), (3, 40, 3, 40)]
    pairs = [lc.make_pair(H, W, seed=v) for v in range(3)]
    images = gu.to_dev(np.stack([p[0] for p in pairs]))
    gts = gt_strips([p[1] for p in pairs], rows4)
    for single, r4, im, gg in ((False, rows4, images, gts), (True, rows4[:1], images[:1].contiguous(), gts[:1])):
        rc, out, temp, _ = loss_det(im, gg, r4, single=single, short=1)
        assert rc == GS_ENOMEM and b"temp too small" in lib.gs_last_error(), (single, rc)
        assert bool(torch.isnan(out).all()) and bool((temp == 0xA5).all()), single
        rc, out, _, _ = loss_det(im, gg, r4, single=single, short=0)
        assert rc == 0 and not bool(torch.isnan(out).any()), single
