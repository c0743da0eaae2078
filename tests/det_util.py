"""C-ABI harness of the deterministic render tests (test_deterministic_gpu.py, test_deterministic_limits_gpu.py):
count + forward (default or deterministic) + backward over B views, with every output sentinel-filled first, and the
readers of what the deterministic backward leaves in its workspace."""
import ctypes as C

import numpy as np
import torch

import blend_cases as bc
import det_ref as dr
import gpu_util as gu
from gs_b200 import _lib

FWD_KEYS = ("image", "final_T", "n_contrib", "ranges", "ids", "stats", "tile_stats")


def bits_equal(a, b):
    if a.shape != b.shape:
        return False
    if a.dtype == torch.float32:
        a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    return torch.equal(a, b)


def forward(views, H, W, bg, det, seg=True):
    """views: [(means2D, conic_opacity, rgb, depths, radii, compute_locally)] device tensors.  Every output is filled with
    a sentinel first; tile statistics are always requested."""
    B = len(views)
    T = ((H + 15) // 16) * ((W + 15) // 16)
    cat = [torch.cat([v[q] for v in views]).contiguous() for q in range(5)]
    cl = torch.cat([v[5].to(torch.uint8).reshape(-1) for v in views]).contiguous()
    counts = [int(v[0].shape[0]) for v in views]
    vs = (C.c_int32 * (B + 1))(*np.concatenate([[0], np.cumsum(counts)]).astype(int).tolist())
    P = int(sum(counts))
    bg_t = gu.to_dev(np.asarray(bg, np.float32))
    offsets = torch.empty((max(P, 1),), dtype=torch.int32, device=gu.DEV)
    order = torch.empty((max(P, 1),), dtype=torch.int32, device=gu.DEV)
    rec = torch.empty((max(P, 1), 12), dtype=torch.float32, device=gu.DEV)
    tb = _lib.query("gs_render_count_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
    R = C.c_int64(0)
    _lib.call("gs_render_count_batched", B, vs, H, W, *(t.data_ptr() for t in cat[:4]), cat[4].data_ptr(), cl.data_ptr(),
              order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), temp.data_ptr(), tb, C.byref(R), gu.stream())
    R = int(R.value)
    Ra = max(R, 1)
    tiles = torch.full((2, Ra), -1, dtype=torch.int32, device=gu.DEV)
    ids = torch.full((2, Ra), -1, dtype=torch.int32, device=gu.DEV)
    sorted_u = torch.full((Ra,), -1, dtype=torch.int32, device=gu.DEV)
    sb = _lib.query("gs_render_sort_temp_bytes", R)
    sort_temp = torch.empty((sb,), dtype=torch.uint8, device=gu.DEV)
    ranges = torch.full((B * T, 2), -1, dtype=torch.int32, device=gu.DEV)
    image = gu.nan(B, 3, H, W)
    final_T = gu.nan(B, H, W)
    n_contrib = torch.full((B, H, W), -1, dtype=torch.int32, device=gu.DEV)
    stats = torch.zeros((B, 3), dtype=torch.int64, device=gu.DEV)
    ts = torch.full((B * T, 3), -1, dtype=torch.int64, device=gu.DEV)
    segb = _lib.query("gs_render_seg_bytes", R, B * T) if seg else 0
    seg_ws = torch.full((segb // 4,), float("nan"), device=gu.DEV).view(torch.uint8) if seg else None
    args = (cat[0].data_ptr(), cat[4].data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(),
            bg_t.data_ptr(), tiles[0].data_ptr(), ids[0].data_ptr(), tiles[1].data_ptr(), ids[1].data_ptr())
    tail = (sort_temp.data_ptr(), sb, ranges.data_ptr(), image.data_ptr(), final_T.data_ptr(), n_contrib.data_ptr(),
            stats.data_ptr(), ts.data_ptr(), _lib.ptr(seg_ws), segb, gu.stream())
    if det:
        _lib.call("gs_render_forward_det", B, vs, P, R, H, W, *args, sorted_u.data_ptr(), *tail)
    else:
        _lib.call("gs_render_forward_batched_ts", B, vs, R, H, W, *args, *tail)
    torch.cuda.synchronize()
    return dict(B=B, P=P, R=R, H=H, W=W, rec=rec, bg=bg_t, cl=cl, order=order, offsets=offsets, ranges=ranges,
                ids=ids[1], ids_unsorted=ids[0], tiles_unsorted=tiles[0], sorted_u=sorted_u, image=image,
                final_T=final_T, n_contrib=n_contrib, stats=stats, tile_stats=ts, seg_ws=seg_ws, seg_bytes=segb)


def backward(f, dL, det, return_ws=False):
    """Gradients start NaN-filled: the deterministic backward must write every row itself.  return_ws: also return the
    deterministic backward's workspace (NaN-filled before the call)."""
    P = f["P"]
    out = dict(means2D=gu.nan(P, 2), conic_opacity=gu.nan(P, 4), rgb=gu.nan(P, 3))
    ws = None
    if det:
        nb = _lib.query("gs_render_det_bytes", f["R"], P)
        ws = torch.full((nb // 4,), float("nan"), device=gu.DEV).view(torch.uint8)   # stale rows must not leak
        _lib.call("gs_render_backward_det", f["B"], P, f["R"], f["H"], f["W"], f["rec"].data_ptr(), f["bg"].data_ptr(),
                  f["cl"].data_ptr(), f["ranges"].data_ptr(), f["ids"].data_ptr(), f["sorted_u"].data_ptr(),
                  f["order"].data_ptr(), f["offsets"].data_ptr(), f["final_T"].data_ptr(), f["n_contrib"].data_ptr(),
                  dL.data_ptr(), _lib.ptr(f["seg_ws"]), f["seg_bytes"], ws.data_ptr(), nb, out["means2D"].data_ptr(),
                  out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(), gu.stream())
    else:
        for t in out.values():
            t.zero_()
        _lib.call("gs_render_backward_batched", f["B"], P, f["R"], f["H"], f["W"], f["rec"].data_ptr(), f["bg"].data_ptr(),
                  f["cl"].data_ptr(), f["ranges"].data_ptr(), f["ids"].data_ptr(), f["final_T"].data_ptr(),
                  f["n_contrib"].data_ptr(), dL.data_ptr(), _lib.ptr(f["seg_ws"]), f["seg_bytes"],
                  out["means2D"].data_ptr(), out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(), gu.stream())
    torch.cuda.synchronize()
    return (out, ws) if return_ws else out


def grad_rows(g):
    """The three gradient outputs as one (P, 9) array in the instance rows' column order."""
    return np.concatenate([gu.npy(g["means2D"]), gu.npy(g["conic_opacity"]), gu.npy(g["rgb"])], 1)


def read_det_ws(ws, R, P):
    """-> n_long, inst (R, 9) fp32, rank (P) and long_g (n_long) uint32, as numpy (det_ref.det_carve's layout)."""
    w = dr.det_carve(R, P)
    u = lambda a, n: gu.npy(ws[a:a + 4 * n].view(torch.int32)).view(np.uint32)   # noqa: E731
    n_long = int(u(w["n_long"], 1)[0])
    inst = gu.npy(ws[w["inst"]:w["inst"] + 36 * R].view(torch.float32)).reshape(R, 9)
    return n_long, inst, u(w["rank"], P), u(w["long_g"], n_long)


def case_view(c):
    return tuple(gu.to_dev(c[k]) for k in ("means2D", "conic_opacity", "rgb", "depths", "radii", "cl"))


def binning_views(c):
    """A binning_cases-style case (view_start vs, one mask per view) as forward()'s views."""
    vs = c["vs"]
    B = len(vs) - 1
    cl = c["cl"].reshape(B, -1)
    return [tuple(gu.to_dev(c[k][vs[v]:vs[v + 1]]) for k in ("means2D", "conic_opacity", "rgb", "depths", "radii")) +
            (gu.to_dev(cl[v]),) for v in range(B)]


def projected_view(sc, cam):
    pre, _, _ = gu.preprocess_forward(sc, cam)
    T = ((cam["image_height"] + 15) // 16) * ((cam["image_width"] + 15) // 16)
    return (pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
            torch.ones((T,), dtype=torch.uint8, device=gu.DEV))


def empty_view(H, W):
    T = ((H + 15) // 16) * ((W + 15) // 16)
    z = lambda *s: torch.zeros(s, device=gu.DEV)   # noqa: E731
    return (z(0, 2), z(0, 4), z(0, 3), z(0), torch.zeros((0,), dtype=torch.int32, device=gu.DEV),
            torch.ones((T,), dtype=torch.uint8, device=gu.DEV))


def dl_like(f, seed):
    g = torch.Generator(device=gu.DEV).manual_seed(seed)
    return torch.randn((f["B"], 3, f["H"], f["W"]), device=gu.DEV, generator=g)


def whole_image_scene(W=640, H=480, n_small=300, seed=9):
    """One splat whose ellipse covers the whole image (its rows sum over every tile: the warp-wide reduce path), many
    small ones on top, and culled splats (radius 0) that must read exactly 0."""
    rng = np.random.default_rng(seed)
    sc = bc._Scene(W, H, rng)
    sc.iso(W / 2, H / 2, 400.0, 0.9, 50.0, 1200, "whole")
    for k in range(n_small):
        sc.iso(rng.uniform(0, W), rng.uniform(0, H), rng.uniform(1.0, 6.0), rng.uniform(0.05, 0.9),
               1.0 + k * 0.01, 20, "small")
    for k in range(40):
        sc.iso(rng.uniform(0, W), rng.uniform(0, H), 3.0, 0.5, 2.0 + k, 0, "culled")
    return bc._finish(sc, "whole_image", "det", (0.2, 0.4, 0.6))


def assert_forward_unchanged(views, H, W, bg, tag):
    """The deterministic forward equals the default one in every output; sorted_u is a permutation of [0, R) and
    ids_sorted = ids_unsorted[sorted_u]."""
    a, b = forward(views, H, W, bg, det=False), forward(views, H, W, bg, det=True)
    assert a["R"] == b["R"]
    R = a["R"]
    for k in FWD_KEYS:
        x, y = (a[k][:R], b[k][:R]) if k == "ids" else (a[k], b[k])
        assert bits_equal(x, y), (tag, k)
    if R:
        su = b["sorted_u"][:R].long()
        assert torch.equal(torch.sort(su).values, torch.arange(R, device=gu.DEV))
        assert torch.equal(b["ids_unsorted"][:R][su], b["ids"][:R])
    return a, b
