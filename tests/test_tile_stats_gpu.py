"""-m gpu: per-tile blend statistics (gs_render_forward_ts, ops.render_gaussians(tile_stats=True)) and the drop-in's
--zhx_time / --zhx_debug logs.

  * tile_stats against a per-tile reference summed from an fp64 walk of every pixel over the fp32 oracle's tile lists:
    exact on every tile without an ambiguous pixel (blend_cases.decision_walk, the rule of test_blend_gpu.py), list
    lengths exact everywhere; on every scene of tests/blend_cases.py and on a projected c1 scene;
  * columns 1-2 summed per view == stats[1:], column 0 weighted by in-image pixels == stats[0], bit for bit;
  * both forwards (packed, half-warp) agree; with and without statistics / checkpoints;
  * non-local tiles and empty lists read 0, and nothing past the B*T rows is written;
  * tile_stats = NULL: image, final_T, n_contrib, stats and checkpoints bit-identical to gs_render_forward;
  * batched slices == single-view calls (ragged view_start, an empty view, 64 views);
  * the drop-in writes the two logs on a logging iteration, with tile lines equal to tile_stats, and nothing otherwise.
"""
import ctypes as C
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import blend_cases as bc
import gpu_util as gu
import test_blend_gpu as tb
from gs_b200 import _lib, ops, pipeline, statlog
from gs_b200 import synthetic as syn
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

SENTINEL = -0x5A5A5A5A5A5A5A5B
EXTRA_ROWS = 5


@pytest.fixture(scope="module")
def o32():
    n = max(1, (os.cpu_count() or 8) // 2)
    return Oracle(np.float32, threads=n)


def forward_ts(c, ts=True, stats=True, seg=True):
    """gs_render_forward_ts on case c; tile_stats (T + EXTRA_ROWS, 3) starts as SENTINEL (ts=False: NULL)."""
    H, W = c["H"], c["W"]
    means2D, conic_opacity, rgb, depths, radii = tb.dev_inputs(c)
    P = means2D.shape[0]
    T = ((H + 15) // 16) * ((W + 15) // 16)
    cl = gu.to_dev(c["cl"]).to(torch.uint8).contiguous()
    bg_t = gu.to_dev(np.asarray(c["bg"], np.float32))
    offsets = torch.empty((max(P, 1),), dtype=torch.int32, device=gu.DEV)
    order = torch.empty((max(P, 1),), dtype=torch.int32, device=gu.DEV)
    rec = torch.empty((max(P, 1), 12), dtype=torch.float32, device=gu.DEV)
    tbytes = _lib.query("gs_render_count_temp_bytes", P)
    temp = torch.empty((tbytes,), dtype=torch.uint8, device=gu.DEV)
    R = C.c_int64(0)
    _lib.call("gs_render_count", P, H, W, means2D.data_ptr(), conic_opacity.data_ptr(), rgb.data_ptr(),
              depths.data_ptr(), radii.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(),
              temp.data_ptr(), tbytes, C.byref(R), gu.stream())
    R = int(R.value)
    tiles = torch.zeros((2, max(R, 1)), dtype=torch.int32, device=gu.DEV)
    ids = torch.zeros((2, max(R, 1)), dtype=torch.int32, device=gu.DEV)
    sb = _lib.query("gs_render_sort_temp_bytes", R)
    sort_temp = torch.empty((sb,), dtype=torch.uint8, device=gu.DEV)
    ranges = torch.empty((T, 2), dtype=torch.int32, device=gu.DEV)
    image = torch.full((3, H, W), float("nan"), device=gu.DEV)
    final_T = torch.zeros((H, W), device=gu.DEV)
    n_contrib = torch.zeros((H, W), dtype=torch.int32, device=gu.DEV)
    st = torch.zeros((3,), dtype=torch.int64, device=gu.DEV) if stats else None
    tsb = torch.full((T + EXTRA_ROWS, 3), SENTINEL, dtype=torch.int64, device=gu.DEV) if ts else None
    segb = _lib.query("gs_render_seg_bytes", R, T) if seg else 0
    seg_ws = torch.full((segb // 4,), float("nan"), device=gu.DEV).view(torch.uint8) if seg else None
    _lib.call("gs_render_forward_ts", P, R, H, W, means2D.data_ptr(), radii.data_ptr(), cl.data_ptr(), order.data_ptr(),
              offsets.data_ptr(), rec.data_ptr(), bg_t.data_ptr(), tiles[0].data_ptr(), ids[0].data_ptr(),
              tiles[1].data_ptr(), ids[1].data_ptr(), sort_temp.data_ptr(), sb, ranges.data_ptr(), image.data_ptr(),
              final_T.data_ptr(), n_contrib.data_ptr(), _lib.ptr(st), _lib.ptr(tsb), _lib.ptr(seg_ws), segb, gu.stream())
    torch.cuda.synchronize()
    return dict(R=R, ranges=ranges, ids=ids[1][:R], image=image, final_T=final_T, n_contrib=n_contrib, stats=st,
                ts=None if tsb is None else gu.npy(tsb), seg_ws=seg_ws, seg_bytes=segb, P=P, H=H, W=W)


def tile_reference(c, f32):
    """Per tile: (list length, sum of entries walked, sum of entries blended) over the in-image pixels, from an fp64 walk
    of the oracle's tile lists with the kernels' decision rules, and whether any pixel of the tile is ambiguous."""
    H, W = c["H"], c["W"]
    gx, gy = bc.tiles_of(W, H)
    walk = bc.decision_walk(c, f32)
    m, co, _ = bc.upcast(c)
    ref = np.zeros((gx * gy, 3), np.int64)
    amb = np.zeros(gx * gy, bool)
    for t in range(gx * gy):
        if not c["cl"][t]:
            continue
        beg, end = int(f32["ranges"][t, 0]), int(f32["ranges"][t, 1])
        L = end - beg
        ref[t, 0] = L
        ty, tx = divmod(t, gx)
        ys, xs = np.mgrid[ty * 16:min(H, ty * 16 + 16), tx * 16:min(W, tx * 16 + 16)]
        amb[t] = walk["ambiguous"][ys, xs].any()
        if L == 0:
            continue
        ids = f32["ids"][beg:end].astype(np.int64)
        A, B, Cc, o = (co[ids, q][None, :] for q in range(4))
        dx, dy = m[ids, 0][None, :] - xs.reshape(-1, 1), m[ids, 1][None, :] - ys.reshape(-1, 1)
        tA, tB, tC = -0.5 * A * dx * dx, -B * dx * dy, -0.5 * Cc * dy * dy
        power = tA + tC + tB
        exact = (np.abs(tA) + np.abs(tB) + np.abs(tC)) == 0.0        # the walk's rules (blend_cases.decision_walk)
        live = np.where(exact, o > 1.0 / 255.0, power + np.log(255.0 * o) >= 0.0) & (power <= 0.0)
        alpha = np.minimum(bc.ALPHA_MAX, o * np.exp(np.minimum(power, 0.0)))
        a_eff = np.where(live, alpha, 0.0)
        Tb = np.cumprod(np.concatenate([np.ones((dx.shape[0], 1)), 1.0 - a_eff[:, :-1]], 1), 1)
        ends = live & (Tb * (1.0 - alpha) < bc.T_EPS)
        first = np.where(ends.any(1), ends.argmax(1), L)
        walked = np.where(first < L, first + 1, L)
        blended = (live & (np.arange(L)[None, :] < first[:, None])).sum(1)
        ref[t, 1], ref[t, 2] = int(walked.sum()), int(blended.sum())
    return ref, amb


def in_image_pixels(H, W):
    gx, gy = bc.tiles_of(W, H)
    px = np.minimum(16, W - 16 * np.arange(gx))
    py = np.minimum(16, H - 16 * np.arange(gy))
    return (py[:, None] * px[None, :]).reshape(-1)


def check_case(c, o32):
    H, W = c["H"], c["W"]
    gx, gy = bc.tiles_of(W, H)
    T = gx * gy
    f32 = o32.render_forward(H, W, c["means2D"], c["conic_opacity"], c["rgb"], c["depths"], c["radii"], c["cl"], c["bg"])
    ref, amb = tile_reference(c, f32)
    base = tb.forward(c)                                      # gs_render_forward, the existing entry point
    f = forward_ts(c)
    ts = f["ts"]
    assert (ts[T:] == SENTINEL).all(), "rows past B*T"
    ts = ts[:T]
    cl = c["cl"].astype(bool)
    assert (ts[~cl] == 0).all() and (ts[ref[:, 0] == 0] == 0).all(), "non-local / empty tiles"
    assert np.array_equal(ts[:, 0], ref[:, 0]), "list lengths"
    safe = ~amb
    assert np.array_equal(ts[safe], ref[safe]), "walked / blended on tiles without an ambiguous pixel"
    st = gu.npy(f["stats"])
    assert st[0] == int((ts[:, 0] * in_image_pixels(H, W)).sum()) and np.array_equal(st[1:], ts[:, 1:].sum(0))
    for k in ("image", "final_T", "n_contrib", "stats", "ranges", "ids"):
        assert torch.equal(f[k], base[k]), k
    # the other forms: half-warp kernel, no statistics pointer, no checkpoints, tile_stats NULL
    for flags in (0, _lib.DEBUG_FWD_HALFWARP):
        for kw in (dict(), dict(stats=False), dict(seg=False), dict(stats=False, seg=False)):
            g = tb.with_flags(flags, forward_ts, c, **kw)
            assert np.array_equal(g["ts"], f["ts"]), (flags, kw)
            for k in ("image", "final_T", "n_contrib"):
                assert torch.equal(g[k], base[k]), (flags, kw, k)
        g = tb.with_flags(flags, forward_ts, c, ts=False)
        b = tb.with_flags(flags, tb.forward, c)
        for k in ("image", "final_T", "n_contrib", "stats"):
            assert torch.equal(g[k], b[k]), (flags, "NULL", k)
        if f["R"]:
            nc = gu.npy(b["n_contrib"]).astype(np.int64)
            k1, v1 = tb.read_checkpoints(g, c, nc)
            k2, v2 = tb.read_checkpoints(b, c, nc)
            assert np.array_equal(k1, k2) and np.array_equal(v1, v2), (flags, "checkpoints")
            s1, s2 = tb.seg_state(g, c), tb.seg_state(b, c)
            assert s1[0] == s2[0] and all(np.array_equal(x, y) for x, y in zip(s1[1:], s2[1:])), (flags, "segments")
    print(f"[tile_stats] {c['name']}: {T} tiles, {int(amb.sum())} with an ambiguous pixel, R={f['R']}")
    return ts


@pytest.mark.parametrize("name", list(tb.CASES))
def test_tile_stats_case(o32, name):
    check_case(tb.CASES[name], o32)


def c1_case():
    cfg = syn.CONFIGS["c1"]
    W, H = cfg["width"], cfg["height"]
    cam = syn.make_camera(W, H, yaw_deg=4.0)
    pre, _, _ = gu.preprocess_forward(syn.make_scene(cfg["n"], W, H, seed=7), cam)
    gx, gy = bc.tiles_of(W, H)
    cl = np.ones(gx * gy, np.uint8)
    cl[(np.arange(gx * gy) * 7) % 5 == 0] = 0                 # a partial mask
    c = {k: gu.npy(pre[k]) for k in ("means2D", "conic_opacity", "rgb", "depths", "radii")}
    c.update(name="c1", H=H, W=W, cl=cl, bg=(0.1, 0.2, 0.3))
    return c


def test_tile_stats_projected_c1(o32):
    c = c1_case()
    ts = check_case(c, o32)
    assert ts[:, 0].sum() > 100_000 and (ts[:, 2] > 0).sum() > 200


def _rs(H, W, bg):
    return SimpleNamespace(image_height=H, image_width=W, bg=torch.tensor(bg, dtype=torch.float32, device=gu.DEV))


def _check_batched(cs, bg):
    real = [c for c in cs if c is not None]
    H, W = real[0]["H"], real[0]["W"]
    gx, gy = bc.tiles_of(W, H)
    views = [(tb._empty_view(real[0]) if c is None else tb._views_of([c])[0]) for c in cs]
    cat = [torch.cat([v[q] for v in views]).contiguous() for q in range(5)]
    cl = torch.stack([v[5].to(torch.uint8).reshape(-1) for v in views])
    vs = np.concatenate([[0], np.cumsum([v[0].shape[0] for v in views])]).astype(int).tolist()
    rs = _rs(H, W, bg)
    img, st, ts = ops.render_gaussians_batched(*cat, cl, vs, rs, tile_stats=True)
    img0, st0 = ops.render_gaussians_batched(*cat, cl, vs, rs)
    assert torch.equal(img, img0) and torch.equal(st, st0)
    assert tuple(ts.shape) == (len(cs), gy, gx, 3) and ts.dtype == torch.int64
    for k, c in enumerate(cs):
        if c is None:
            assert (ts[k] == 0).all()
            continue
        one = ops.render_gaussians(*tb.dev_inputs(c), gu.to_dev(c["cl"]), rs, tile_stats=True)
        assert len(one) == 5 and torch.equal(img[k], one[0])
        assert torch.equal(ts[k], one[4]), (k, c["name"])
        assert torch.equal(st[k, 1:], ts[k].reshape(-1, 3)[:, 1:].sum(0))
    assert len(ops.render_gaussians(*tb.dev_inputs(real[0]), gu.to_dev(real[0]["cl"]), rs)) == 4


def test_batched_tile_stats_equal_single_view_calls():
    group = [c for c in tb.CASES.values() if (c["W"], c["H"]) == (64, 48)]
    bg = (0.3, 0.6, 0.9)
    _check_batched([group[0], None] + group[1:], bg)
    cs = [group[k % len(group)] for k in range(63)]
    _check_batched(cs[:20] + [None] + cs[20:], bg)


def test_dropin_writes_the_logs(tmp_path):
    """Forward + backward through the drop-in with zhx_time / zhx_debug at iteration 1 and a partial compute_locally:
    both files, every stage key >= 0, one tile line per local tile equal to tile_stats; iteration 2, mode test and the
    flags off write nothing and leave the profiler off."""
    import diff_gaussian_rasterization as dgr
    W, H = 160, 96
    cam = syn.make_camera(W, H)
    sc = syn.make_scene(3000, W, H, seed=5)
    rs = pipeline.DeviceCamera(cam, gu.DEV).settings(3)
    gx, gy = bc.tiles_of(W, H)
    cl = torch.tensor([(t % gx) >= 3 for t in range(gx * gy)], device=gu.DEV).reshape(gy, gx)

    def run(**kw):
        args = dict(mode="train", world_size="1", global_rank="0", local_rank="0", log_folder=str(tmp_path),
                    log_interval="250", iteration="1", zhx_debug="True", zhx_time="True", avoid_pixel_all2all=False,
                    stats_collector={})
        args.update(kw)
        t = {k: gu.to_dev(v, torch.float32).requires_grad_(True) for k, v in sc.items()}
        r = dgr.GaussianRasterizer(raster_settings=rs)
        m2, rgb, co, radii, depths = r.preprocess_gaussians(t["means3D"], t["scales"], t["rotations"], t["shs"],
                                                            t["opacities"], args)
        image, *_ = r.render_gaussians(m2, co, rgb, depths, radii, cl, None, args)
        (image * image).sum().backward()
        torch.cuda.synchronize()
        return m2.detach(), co.detach(), rgb.detach(), depths, radii, image.detach()

    files = [tmp_path / "gpu_time_ws=1_rk=0.log", tmp_path / "n_contrib_ws=1_rk=0.log"]
    for kw in (dict(iteration="2"), dict(mode="test", iteration="-1"), dict(zhx_time="False", zhx_debug="False")):
        run(**kw)
        assert not any(f.exists() for f in files), kw
        assert not _lib.PROFILE_ON
    m2, co, rgb, depths, radii, image = run()
    assert not _lib.PROFILE_ON
    assert all(f.exists() for f in files)
    times = {}
    for line in files[0].read_text().splitlines():
        if line.startswith("it="):
            assert line.startswith("it=1,")
            continue
        k, v = line.split(":")
        assert v.endswith(" ms")
        times[k] = float(v[:-3])
    keys = [k for call in ops.REFERENCE_STAGE_KEYS.values() for k, _ in call]
    assert sorted(times) == sorted(keys) and all(v >= 0.0 for v in times.values())
    assert times["70 render time"] > 0 and times["b10 render time"] > 0 and times["10 preprocess time"] > 0
    # the tile lines: the same render with tile_stats=True (the image is bit-identical)
    out = ops.render_gaussians(m2, co, rgb, depths, radii, cl, rs, tile_stats=True)
    assert torch.equal(out[0], image)
    ts = gu.npy(out[4]).reshape(-1, 3)
    local = np.nonzero(gu.npy(cl).reshape(-1))[0]
    lines = files[1].read_text().splitlines()
    assert len(lines) == local.size + 1 and "world_size: 1" in lines[-1]
    pat = re.compile(r"iteration: 1, tile: \((\d+), (\d+)\), range: \((\d+), (\d+)\), num_rendered_this_tile: (\d+), "
                     r"n_considered_per_pixel: ([\d.]+), n_contrib2loss_per_pixel: ([\d.]+), contrib2loss_ratio: [\d.]+")
    for line, t in zip(lines, local):
        m = pat.fullmatch(line)
        assert m, line
        assert (int(m[1]), int(m[2])) == (t // gx, t % gx) and int(m[3]) - int(m[4]) == ts[t, 0] == int(m[5])
        assert m[6] == f"{ts[t, 1] / 256:.6f}" and m[7] == f"{ts[t, 2] / 256:.6f}"
    assert f"num_tiles: {local.size}," in lines[-1] and f"num_rendered: {int(ts[local, 0].sum())}," in lines[-1]
