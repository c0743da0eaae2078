"""-m gpu: tile binning (csrc/binning.cu) against tests/binning_ref.py on the populations of tests/binning_cases.py.

  * exact: R, order, offsets, the sorted tile keys and ids, ranges, bit for bit, single-view and batched, with every
    output pre-filled with a sentinel and guard entries past R that must stay untouched;
  * large R (~5e7): the list checked on the device with int64 torch ops -- ranges partition [0, R) in tile order, each
    id appears touched[i] times, every (tile, id) lies in that splat's rect, view and mask, and inside a tile
    (depth bits, id) strictly increases; together these determine the list;
  * record: pass-through fields bit-exact, thr within 2 ulp of the fp64 -log of the product the kernel forms (exactly
    -0 where it is 1), ex / ey conservative against the fp64 half extents and tight for well-conditioned conics;
  * limits: totals of 2^31 - 1, 2^31, 2^32 and 2^32 + 5 through the count alone; the operator's GsError and a clean
    state after it;
  * operator host side: instance-buffer hints across R jumping by 10x and to 0, two forwards alive at once, and 64
    count tickets outstanding on 64 streams.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import binning_cases as bc
import binning_ref as br
import gpu_util as gu
from gs_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = gu.DEV
SENTINEL = 0x5A5A5A5A
GUARD = 64
F32 = np.float32


def dev_inputs(c):
    return [gu.to_dev(c[k]) for k in ("means2D", "conic_opacity", "rgb", "depths", "radii")]


def filled(n, value, dtype=torch.int32):
    return torch.full((n,), value, dtype=dtype, device=DEV)


def run(c, batched):
    """count + forward (forward-only blend) through the single-view or batched entry points; every output starts as a
    sentinel and the instance buffers carry GUARD entries past R."""
    H, W, vs = c["H"], c["W"], c["vs"]
    B, P = len(vs) - 1, vs[-1]
    T = int(np.prod(br.tiles_of(W, H)))
    m2, co, rgb, d, rad = dev_inputs(c)
    cl = gu.to_dev(c["cl"])
    Pa = max(P, 1)
    order, offsets = filled(Pa, SENTINEL), filled(Pa, SENTINEL)
    rec = torch.full((Pa, 12), float("nan"), device=DEV)
    tb = _lib.query("gs_render_count_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=DEV)
    vsa = (C.c_int32 * (B + 1))(*vs)
    R = C.c_int64(-1)
    if batched:
        _lib.call("gs_render_count_batched", B, vsa, H, W, m2.data_ptr(), co.data_ptr(), rgb.data_ptr(), d.data_ptr(),
                  rad.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), temp.data_ptr(),
                  tb, C.byref(R), gu.stream())
    else:
        assert B == 1
        _lib.call("gs_render_count", P, H, W, m2.data_ptr(), co.data_ptr(), rgb.data_ptr(), d.data_ptr(),
                  rad.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(), temp.data_ptr(),
                  tb, C.byref(R), gu.stream())
    R = int(R.value)
    bufs = [filled(R + GUARD, SENTINEL) for _ in range(4)]   # tiles, ids unsorted; tiles, ids sorted
    sb = _lib.query("gs_render_sort_temp_bytes", R)
    sort_temp = torch.empty((sb,), dtype=torch.uint8, device=DEV)
    ranges = filled(2 * B * T, SENTINEL)
    bg = torch.zeros(3, device=DEV)
    image = torch.empty((B, 3, H, W), device=DEV)
    final_T = torch.empty((B, H, W), device=DEV)
    n_contrib = torch.empty((B, H, W), dtype=torch.int32, device=DEV)
    args = (R, H, W, m2.data_ptr(), rad.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(),
            bg.data_ptr(), *(b.data_ptr() for b in bufs), sort_temp.data_ptr(), sb, ranges.data_ptr(), image.data_ptr(),
            final_T.data_ptr(), n_contrib.data_ptr(), None, None, 0, gu.stream())
    if batched:
        _lib.call("gs_render_forward_batched", B, vsa, *args)
    else:
        _lib.call("gs_render_forward", P, *args)
    torch.cuda.synchronize()
    for b in bufs:
        assert bool((b[R:] == SENTINEL).all()), "write past R"
    return dict(R=R, order=order[:P], offsets=offsets[:P], rec=rec[:P], tiles=bufs[2][:R], ids=bufs[3][:R],
                ranges=ranges.view(B * T, 2), image=image)


def u32(t):
    return gu.npy(t).view(np.uint32)


def check_record(c, rec, touched):
    """rec: (P, 12) kernel record (numpy fp32)."""
    ref = br.record(c["means2D"], c["conic_opacity"], c["rgb"], touched)
    got = np.asarray(rec, F32)
    dfn = ref["defined"]
    assert np.array_equal(got.view(np.uint32)[dfn], ref["rec"].view(np.uint32)[dfn]), "record fields"
    live = touched > 0
    thr = got[:, 6].astype(np.float64)
    one = live & (ref["prod"] == F32(1))
    assert (got[one, 6].view(np.uint32) == 0x80000000).all(), "thr is -0 where 255 o rounds to 1"
    rest = live & ~one
    tol = 2.0 * np.spacing(np.abs(ref["thr64"][rest]).astype(F32)).astype(np.float64)
    assert (np.abs(thr[rest] - ref["thr64"][rest]) <= tol).all(), "thr within 2 ulp"
    box = ref["kind"] == br.BOX
    hx, hy, cond = br.true_half_extents(got)
    ex, ey = got[:, 10].astype(np.float64), got[:, 11].astype(np.float64)
    fin = box & np.isfinite(hx) & np.isfinite(hy)
    assert fin.sum() >= 0.99 * box.sum()
    assert (ex[fin] >= hx[fin]).all() and (ey[fin] >= hy[fin]).all(), "box not conservative"
    tight = fin & (cond <= 1e4)
    assert (ex[tight] <= 1.03 * hx[tight] + 0.5 + 1e-3).all() and (ey[tight] <= 1.03 * hy[tight] + 0.5 + 1e-3).all()
    return dict(box=int(box.sum()), dead=int((ref["kind"] == br.DEAD).sum()),
                degenerate=int((ref["kind"] == br.DEGENERATE).sum()))


def check_exact(c, f, ref):
    assert f["R"] == ref["R"]
    assert np.array_equal(u32(f["order"]), ref["order"])
    assert np.array_equal(u32(f["offsets"]), ref["offsets"])
    assert np.array_equal(u32(f["tiles"]), ref["tiles"])
    assert np.array_equal(u32(f["ids"]), ref["ids"])
    assert np.array_equal(u32(f["ranges"]), ref["ranges"])
    return check_record(c, gu.npy(f["rec"]), ref["touched"])


def exact(c, batched):
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], c["vs"])
    return check_exact(c, run(c, batched), ref)


SINGLE = [bc.rect_case(), bc.record_case()] + [bc.size_case(P) for P in (0, 1, 255, 256, 257)]


@pytest.mark.parametrize("batched", [False, True], ids=["single", "batched"])
@pytest.mark.parametrize("c", SINGLE, ids=lambda c: c["name"])
def test_single_view_populations_bit_exact(c, batched):
    kinds = exact(c, batched)
    if c["name"] == "record":
        assert min(kinds.values()) >= 10, kinds


@pytest.mark.parametrize("W,H", bc.SHAPES, ids=lambda v: str(v))
def test_image_shapes_and_masks_bit_exact(W, H):
    for m in ("all", "none", "checkerboard", "single", "last"):
        exact(bc.shape_case(W, H, m), batched=False)


@pytest.mark.parametrize("kind", ["equal", "runs", "ulp", "loguniform", "special"])
def test_depth_orders_bit_exact(kind):
    """Three views with per-view masks; the special depths (+-0, negative, subnormal, +inf) order by raw bits."""
    exact(bc.depth_case(kind), batched=True)


@pytest.mark.parametrize("c", bc.view_cases(), ids=lambda c: c["name"])
def test_view_counts_and_view_start_bit_exact(c):
    exact(c, batched=True)


@pytest.fixture(scope="module")
def big_cases():
    return dict(views_1080p=bc.views_1080p(), p_2m=bc.size_case(2 ** 21 + 5, 3840, 2160, rmax=12))


def test_64_views_of_1080p_bit_exact(big_cases):
    exact(big_cases["views_1080p"], batched=True)


def test_two_million_splats_at_4k_bit_exact(big_cases):
    exact(big_cases["p_2m"], batched=False)


def test_large_instance_list_on_the_device():
    """R ~ 5e7 at 1080p: checked with int64 device ops instead of a host sort."""
    c = bc.size_case(2 ** 21 + 5, 1920, 1080, rmax=60)
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], with_list=False)
    f = run(c, batched=False)
    R, P = f["R"], len(c["radii"])
    assert R == ref["R"] > 3 * 10 ** 7
    assert np.array_equal(u32(f["order"]), ref["order"]) and np.array_equal(u32(f["offsets"]), ref["offsets"])
    gx, gy = br.tiles_of(c["W"], c["H"])
    T = gx * gy
    tiles = f["tiles"].to(torch.int64)
    assert bool((tiles[1:] >= tiles[:-1]).all()) and int(tiles[0]) >= 0 and int(tiles[-1]) < T
    counts = torch.bincount(tiles, minlength=T)
    ends = torch.cumsum(counts, 0)
    rg = f["ranges"].to(torch.int64)
    nz = counts > 0
    assert bool((rg[nz, 0] == (ends - counts)[nz]).all()) and bool((rg[nz, 1] == ends[nz]).all())
    assert bool((rg[~nz] == 0).all())
    ids = f["ids"].to(torch.int64)
    assert bool((ids >= 0).all()) and bool((ids < P).all())
    assert torch.equal(torch.bincount(ids, minlength=P).cpu(), torch.from_numpy(ref["touched"]))
    x0, y0, x1, y1 = (torch.from_numpy(q).to(DEV)[ids] for q in ref["rect"])
    ty, tx = tiles // gx, tiles % gx
    assert bool(((tx >= x0) & (tx < x1) & (ty >= y0) & (ty < y1)).all())
    del x0, y0, x1, y1, tx, ty
    assert bool((gu.to_dev(c["cl"]).to(torch.bool)[tiles]).all())
    dk = gu.to_dev(c["depths"].view(np.uint32).astype(np.int64))[ids]
    same = tiles[1:] == tiles[:-1]
    inc = (dk[1:] > dk[:-1]) | ((dk[1:] == dk[:-1]) & (ids[1:] > ids[:-1]))
    assert bool((inc | ~same).all()), "(depth bits, id) must strictly increase inside a tile (no repeated pair)"
    print(f"[binning] large R = {R}, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ---- limits ---------------------------------------------------------------------------------------------------------

LIMIT_SIZE = 16384           # one full-image splat is 2^20 local tiles


def limit_scene(full0, full1, hole_in_view1, small0=0):
    """Two views of 16384^2: full0 + small0 splats in view 0 (the small ones cover one tile each), full1 in view 1,
    whose mask misses one tile when hole_in_view1."""
    P0 = full0 + small0
    P = P0 + full1
    m = np.full((P, 2), LIMIT_SIZE / 2, F32)
    r = np.full(P, 20000, np.int32)
    m[full0:P0] = 8.0
    r[full0:P0] = 1
    T = (LIMIT_SIZE // 16) ** 2
    cl = np.ones(2 * T, np.uint8)
    if hole_in_view1:
        cl[T + 12345] = 0
    co = np.tile(np.array([0.01, 0.0, 0.01, 0.5], F32), (P, 1))
    return dict(W=LIMIT_SIZE, H=LIMIT_SIZE, vs=[0, P0, P], means2D=m, radii=r, cl=cl, conic_opacity=co,
                rgb=np.full((P, 3), 0.5, F32), depths=np.linspace(1, 2, P, dtype=F32))


def count_only(c):
    """gs_render_count_launch + gs_render_count_read -> (rc, R, message, offsets)."""
    m2, co, rgb, d, rad = dev_inputs(c)
    cl = gu.to_dev(c["cl"])
    P = c["vs"][-1]
    order, offsets = filled(P, SENTINEL), filled(P, SENTINEL)
    rec = torch.empty((P, 12), device=DEV)
    tb = _lib.query("gs_render_count_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=DEV)
    vs = (C.c_int32 * 3)(*c["vs"])
    ticket = C.c_void_p()
    lib = _lib.load()
    rc = lib.gs_render_count_launch(2, vs, P, c["H"], c["W"], m2.data_ptr(), co.data_ptr(), rgb.data_ptr(), d.data_ptr(),
                                    rad.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(),
                                    temp.data_ptr(), tb, C.byref(ticket), gu.stream())
    assert rc == 0
    R = C.c_int64(-1)
    rc = lib.gs_render_count_read(ticket, C.byref(R), gu.stream())
    msg = lib.gs_last_error().decode() if rc else ""
    torch.cuda.synchronize()
    return rc, int(R.value), msg, u32(offsets)


@pytest.mark.parametrize("name,full0,full1,hole,small0", [
    ("2^31-1", 2047, 1, True, 0), ("2^31", 2048, 0, False, 0), ("2^32", 4096, 0, False, 0),
    ("2^32+5", 4096, 0, False, 5)])
def test_instance_count_limit(name, full0, full1, hole, small0):
    c = limit_scene(full0, full1, hole, small0)
    ref = br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], c["W"], c["H"], c["vs"], with_list=False)
    assert ref["R"] == {"2^31-1": 2 ** 31 - 1, "2^31": 2 ** 31, "2^32": 2 ** 32, "2^32+5": 2 ** 32 + 5}[name]
    rc, R, msg, offsets = count_only(c)
    if ref["R"] < 2 ** 31:
        assert rc == 0 and R == ref["R"]
        assert np.array_equal(offsets, ref["offsets"])
    else:
        assert rc == -1 and R == 0, (rc, R)            # GS_EINVAL; 2^32 + 5 must not come back as 5
        assert "limit 2^31 - 1" in msg and str(ref["R"]) in msg, msg


def test_forward_rejects_2_to_the_31_instances_before_any_launch():
    T = (LIMIT_SIZE // 16) ** 2
    vs = (C.c_int32 * 3)(0, 1, 2)
    lib = _lib.load()
    rc = lib.gs_render_forward_batched(2, vs, 2 ** 31, LIMIT_SIZE, LIMIT_SIZE, *([None] * 12), 0, *([None] * 6), 0,
                                       gu.stream())
    assert rc == -1 and "2^31" in lib.gs_last_error().decode()
    torch.cuda.synchronize()
    assert T * 2 < 2 ** 31


def settings(W, H, bg=(0.1, 0.2, 0.3)):
    return SimpleNamespace(image_height=H, image_width=W, bg=torch.tensor(bg, device=DEV))


def op_inputs(c, grad=False):
    m2, co, rgb, d, rad = dev_inputs(c)
    for t in (m2, co, rgb):
        t.requires_grad_(grad)
    return m2, co, rgb, d, rad


def test_operator_raises_on_the_limit_and_recovers():
    from gs_b200 import ops
    W, H = 1920, 1080
    small = bc.size_case(3000, W, H, seed=5)
    rs = settings(W, H)
    before, *_ = ops.render_gaussians(*op_inputs(small), None, rs)
    n = 270000                                          # 270 000 x 8160 tiles > 2^31
    p = bc.Pop(W, H, seed=3)
    p.add(np.full(n, W / 2), H / 2, 3000)
    huge = p.finish("huge")
    with pytest.raises(_lib.GsError, match=r"limit 2\^31 - 1"):
        ops.render_gaussians(*op_inputs(huge), None, rs)
    after, *_ = ops.render_gaussians(*op_inputs(small), None, rs)
    torch.cuda.synchronize()
    assert torch.equal(before, after)


# ---- operator host side -------------------------------------------------------------------------------------------

def _grad_close(a, b, what):
    a, b = a.double(), b.double()
    tol = 2e-5 * b.abs() + 2e-5 * b.abs().mean()      # same pairs, different atomics order
    frac = float(((a - b).abs() > tol).double().mean())
    assert frac <= 1e-4, (what, frac)


def sequence_scenes(W=1920, H=1080):
    """R of about 1e4, 1e6, 0, 1e5, 1e6."""
    out = []
    for n, rmax, zero in ((1500, 12, False), (90000, 40, False), (700, 12, True), (12000, 30, False),
                          (90000, 40, False)):
        c = bc.size_case(n, W, H, seed=n + rmax, rmax=rmax)
        if zero:
            c["radii"][:] = 0
        out.append(c)
    return out


def op_render(c, batched, grad, g_seed=0, cuda_args=None):
    from gs_b200 import ops
    W, H = c["W"], c["H"]
    m2, co, rgb, d, rad = op_inputs(c, grad)
    rs = settings(W, H)
    if batched:
        P = len(c["radii"])
        img, _ = ops.render_gaussians_batched(m2, co, rgb, d, rad, None, [0, P // 3, P], rs, cuda_args)
    else:
        img, *_ = ops.render_gaussians(m2, co, rgb, d, rad, None, rs, cuda_args)
    return img, (m2, co, rgb)


def backward(img, leaves, seed=0):
    g = torch.randn(img.shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    (img * g).sum().backward()
    return [t.grad.clone() for t in leaves]


@pytest.mark.parametrize("batched", [False, True], ids=["single", "batched"])
@pytest.mark.parametrize("grad", [False, True], ids=["forward", "grad"])
def test_instance_hints_and_counts_across_jumping_R(batched, grad):
    from gs_b200 import ops
    scenes = sequence_scenes()
    alone = []
    for c in scenes:
        ops._R_HINT.clear()                              # a fresh state: no hint, buffers sized after the count
        img, leaves = op_render(c, batched, grad)
        alone.append((img.detach().clone(), backward(img, leaves) if grad else None))
    ops._R_HINT.clear()
    Rs = []
    for c, (img0, g0) in zip(scenes, alone):
        collector = {}
        img, leaves = op_render(c, batched, grad, cuda_args={"stats_collector": collector})
        Rs.append(collector["num_rendered"])
        assert torch.equal(img.detach(), img0)
        if grad:
            for a, b, name in zip(backward(img, leaves), g0, ("means2D", "conic_opacity", "rgb")):
                _grad_close(a, b, name)
    assert Rs[2] == 0 and 3e3 < Rs[0] < 3e4 and Rs[1] > 5e5 and 3e4 < Rs[3] < 3e5, Rs


def test_two_forwards_alive_backwards_in_reverse_order():
    from gs_b200 import ops
    a, b = sequence_scenes()[1], sequence_scenes()[3]
    ref = []
    for c in (a, b):
        ops._R_HINT.clear()
        img, leaves = op_render(c, False, True)
        ref.append((img.detach().clone(), backward(img, leaves, seed=7)))
    ops._R_HINT.clear()
    ia, la = op_render(a, False, True)
    ib, lb = op_render(b, False, True)
    gb = backward(ib, lb, seed=7)
    ga = backward(ia, la, seed=7)
    assert torch.equal(ia.detach(), ref[0][0]) and torch.equal(ib.detach(), ref[1][0])
    for got, want in ((ga, ref[0][1]), (gb, ref[1][1])):
        for x, y, name in zip(got, want, ("means2D", "conic_opacity", "rgb")):
            _grad_close(x, y, name)


def test_64_tickets_on_64_streams_read_in_reverse():
    W, H = 640, 480
    lib = _lib.load()
    keep, tickets, refs = [], [], []
    for k in range(64):
        c = bc.size_case(200 + 97 * k, W, H, seed=k, rmax=10 + k)
        refs.append(br.bin_splats(c["means2D"], c["depths"], c["radii"], c["cl"], W, H, with_list=False))
        m2, co, rgb, d, rad = dev_inputs(c)
        cl = gu.to_dev(c["cl"])
        P = len(c["radii"])
        order, offsets = filled(P, SENTINEL), filled(P, SENTINEL)
        rec = torch.empty((P, 12), device=DEV)
        tb = _lib.query("gs_render_count_temp_bytes", P)
        temp = torch.empty((tb,), dtype=torch.uint8, device=DEV)
        keep.append((m2, co, rgb, d, rad, cl, order, offsets, rec, temp, torch.cuda.Stream()))
    torch.cuda.synchronize()
    for k, (m2, co, rgb, d, rad, cl, order, offsets, rec, temp, s) in enumerate(keep):
        t = C.c_void_p()
        _lib.call("gs_render_count_launch", 1, None, m2.shape[0], H, W, m2.data_ptr(), co.data_ptr(), rgb.data_ptr(),
                  d.data_ptr(), rad.data_ptr(), cl.data_ptr(), order.data_ptr(), offsets.data_ptr(), rec.data_ptr(),
                  temp.data_ptr(), temp.numel(), C.byref(t), s.cuda_stream)
        tickets.append(t)
    for k in reversed(range(64)):
        R = C.c_int64(-1)
        assert lib.gs_render_count_read(tickets[k], C.byref(R), keep[k][-1].cuda_stream) == 0
        assert R.value == refs[k]["R"], k
    torch.cuda.synchronize()
    for k in range(64):
        assert np.array_equal(u32(keep[k][7]), refs[k]["offsets"]), k
