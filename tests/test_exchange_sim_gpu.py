"""-m gpu: the splat-exchange and gradient-sync kernels of csrc/distribute.cu with W ranks simulated in one process on one
GPU, against the numpy reference of tests/exchange_ref.py.

No kernel knows whether a destination pointer is a peer's IPC mapping or an ordinary allocation on the same device: all
cross-rank state enters through host tables (strip rows, destination rows, segment tables) or one device array of
all-gathered counts.  So every rank's receive and gradient regions are plain allocations here, and every
collective is a host-side concatenation or split.  Kernel arguments are built with exchange.py's own helpers (_slab_ptrs,
_row_ptrs, _i32, direct_rows, Layout, segments), so the product's glue is under test as well.  What stays with tests/mgpu_parity.py: IPC mapping, NCCL, and the ordering of ranks' streams.

Every output lives in a slab filled with 0xFF bytes, with guard bands around each region: a stray write shows up as a
changed sentinel.  The exchange copies and sums in a fixed order, so all comparisons are bit for bit (int32 views)."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import exchange_ref as xr
import gpu_util as gu
from gs_b200 import _lib, division, exchange, synthetic as syn
from gs_b200.exchange import _i32, _row_ptrs, _slab_ptrs
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

GUARD = 1024       # sentinel bytes on each side of every region
SENTINEL = -1      # int32 view of the 0xFF fill


class Slab:
    """One device allocation filled with 0xFF; region q is nbytes[q] bytes, 256-byte aligned, with at least GUARD
    sentinel bytes before and after it."""

    def __init__(self, nbytes):
        offs, pos = [], GUARD
        for n in nbytes:
            offs.append(pos)
            pos = (pos + int(n) + GUARD + 255) // 256 * 256
        self.buf = torch.full((pos,), 0xFF, dtype=torch.uint8, device=gu.DEV)
        self.guard = torch.ones((pos,), dtype=torch.bool, device=gu.DEV)
        self.regions = []
        for o, n in zip(offs, nbytes):
            self.guard[o:o + int(n)] = False
            self.regions.append(self.buf[o:o + int(n)])

    def f32(self, q, shape):
        return self.regions[q].view(torch.float32).view(shape)

    def i32(self, q, shape):
        return self.regions[q].view(torch.int32).view(shape)

    def words(self, q):
        """Region q as host int32 words."""
        return self.regions[q].cpu().numpy().view(np.int32)

    def guards_intact(self):
        return bool((self.buf[self.guard] == 0xFF).all())


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def region_fields(words, cap):
    """int32 words of a direct-placement receive region (means2D | rgb | conic_opacity | radii | depths, cap rows each)."""
    return dict(means2D=words[:2 * cap].reshape(cap, 2), rgb=words[2 * cap:5 * cap].reshape(cap, 3),
                conic_opacity=words[5 * cap:9 * cap].reshape(cap, 4), radii=words[9 * cap:10 * cap],
                depths=words[10 * cap:11 * cap])


# ---------------------------------------------------------------------------------------------------------------------
# cases: (W, B), uneven P per rank (0, 1, 31, 257, 4099, ~300 k), edge-case splats or real projections, strips from
# division.start_strategy or hand-made ones (empty strips, one-row strips, cameras rendered by some ranks only,
# every rank on every camera), H % 16 != 0
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    "w2b1": dict(W=2, B=1, P=(0, 4099), H=200, Wimg=333, strips="start"),
    "w3b2": dict(W=3, B=2, P=(1, 31, 257), H=200, Wimg=333, strips="start"),
    "w4b4": dict(W=4, B=4, P=(257, 4099, 0, 31), H=200, Wimg=333, strips="hand"),
    "w4b3_projected": dict(W=4, B=3, P=(3000, 2000, 1, 2999), H=136, Wimg=160, strips="start", projected=True),
    "w8b2": dict(W=8, B=2, P=(31, 257, 1, 4099, 0, 300, 1000, 2), H=200, Wimg=333, strips="start"),
    "w16b16": dict(W=16, B=16, P=(300, 0, 1, 31, 257) + (300,) * 11, H=280, Wimg=200, strips="every"),
    "w4b2_300k": dict(W=4, B=2, P=(300_000, 299_999, 300_001, 1), H=200, Wimg=333, strips="hand"),
}


class Case:
    def __init__(self, name):
        c = CASES[name]
        self.W, self.B, self.P, self.H, self.Wimg = c["W"], c["B"], c["P"], c["H"], c["Wimg"]
        W, B, H = self.W, self.B, self.H
        rng = np.random.default_rng(sum(map(ord, name)))
        gy = (H + 15) // 16
        if c["strips"] == "start":
            st, _ = division.start_strategy(list(range(B)), division.StrategyHistory(list(range(B)), gy, W), W, 0)
            self.lo, self.hi = xr.strips_from_strategies(st, W)
        else:
            self.lo, self.hi = xr.hand_strips(rng, W, B, gy, every_rank=c["strips"] == "every")
        self.ids = xr.gpu_ids(self.lo, self.hi)
        self.shards = self._projected(rng) if c.get("projected") else \
            [xr.make_splats(rng, B, p, H, self.Wimg) for p in self.P]
        self.dev = [{f: gu.to_dev(s[f]).contiguous() for f in xr.FIELDS} for s in self.shards]
        o = Oracle(np.float32)
        self.hits = [xr.route(o, H, self.Wimg, s, self.lo, self.hi) for s in self.shards]
        self.cnt = xr.counts(self.hits)
        self.ref = xr.RefLayout(self.cnt)
        self.N = [self.ref.n_recv(j) for j in range(W)]
        self.outputs = [xr.receiver_outputs(self.shards, self.hits, j) for j in range(W)]
        # receiver gradients: normal floats; one camera's pointers are passed as NULL to gs_xchg_pack_grad (its rows
        # must come out as zeros), so the gradients the sources see -- g_eff -- have those rows zeroed
        self.nulls = {(B - 1, f) for f in xr.GRAD_FIELDS} if B > 1 else {(0, "rgb")}
        self.g_full, self.g_eff = [], []
        for j in range(W):
            g = {f: rng.uniform(-1, 1, (self.N[j], xr.WIDTH[f])).astype(np.float32) for f in xr.GRAD_FIELDS}
            e = {f: v.copy() for f, v in g.items()}
            for k, f in self.nulls:
                e[f][self.ref.view[j, k]:self.ref.view[j, k + 1]] = 0.0
            self.g_full.append(g)
            self.g_eff.append(e)
        self.back = xr.backward(self.hits, self.g_eff, self.ref)
        self.lo_c, self.hi_c = _i32(self.lo.reshape(-1)), _i32(self.hi.reshape(-1))
        self.layouts = [exchange.Layout(self.cnt.tolist(), j, self.ids) for j in range(W)]

    def _projected(self, rng):
        """gs_preprocess_forward of a synthetic scene for B cameras, cut into the ranks' shards."""
        n = sum(self.P)
        sc = syn.make_scene(n, self.Wimg, self.H, seed=3, radius_px=10.0)
        per_cam = []
        for cam in syn.make_batch_cameras(self.Wimg, self.H, self.B):
            out, _, _ = gu.preprocess_forward(sc, cam)
            per_cam.append({f: gu.npy(out[f]) for f in xr.FIELDS})
        shards, off = [], 0
        for p in self.P:
            shards.append({f: np.ascontiguousarray(np.stack([pc[f][off:off + p] for pc in per_cam])) for f in xr.FIELDS})
            off += p
        assert sum(int((s["radii"] > 0).sum()) for s in shards) > 0
        return shards

    def ptrs(self, i, f):
        return _slab_ptrs(self.dev[i][f], self.B)


@functools.lru_cache(maxsize=None)   # kept for the module: the row-staged test also compares with the direct pull
def get_case(name):
    return Case(name)


# ---------------------------------------------------------------------------------------------------------------------
# direct placement (the peer-memory path): count -> pack_dev -> pull_grad
# ---------------------------------------------------------------------------------------------------------------------
def xr_count(c, i):
    B, P, W = c.B, c.P[i], c.W
    nblk = max(W * B * ((max(P, 1) + 255) // 256), 1)
    slab = Slab([4 * nblk, 4 * nblk, 4 * W * B])
    blkcnt, blkbase, counts = slab.i32(0, (nblk,)), slab.i32(1, (nblk,)), slab.i32(2, (W, B))
    tb = _lib.query("gs_xr_temp_bytes", B, P, W)
    temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
    _lib.call("gs_xr_count", B, P, W, c.H, c.Wimg, c.ptrs(i, "means2D"), c.ptrs(i, "radii"), c.lo_c, c.hi_c,
              blkcnt.data_ptr(), blkbase.data_ptr(), counts.data_ptr(), temp.data_ptr(), tb, gu.stream())
    return slab, blkcnt, blkbase, counts


def pack_args(c, i, blkbase, bases):
    return (c.B, c.P[i], c.W, c.H, c.Wimg, c.ptrs(i, "means2D"), c.ptrs(i, "rgb"), c.ptrs(i, "conic_opacity"),
            c.ptrs(i, "radii"), c.ptrs(i, "depths"), c.lo_c, c.hi_c, blkbase.data_ptr(), bases)


def run_pack(c, blkbases, cap, allc):
    """Every simulated rank packs into the W receive regions, its destination rows computed on the device from the
    all-gathered counts `allc`.  -> (region slab, row0_dev slab)."""
    W, B = c.W, c.B
    slab = Slab([4 * 11 * cap] * W)
    bases = (C.c_void_p * W)(*[slab.regions[j].data_ptr() for j in range(W)])
    rows = Slab([4 * (W * B + 1)] * W)
    for i in range(W):
        _lib.call("gs_xr_pack_dev", *pack_args(c, i, blkbases[i], bases), allc.data_ptr(), i, rows.regions[i].data_ptr(),
                  C.c_longlong(cap), gu.stream())
    return slab, rows


def check_regions(c, slab, cap):
    assert slab.guards_intact(), "write outside the receive regions"
    for j in range(c.W):
        got = region_fields(slab.words(j), cap)
        n = c.N[j]
        for f in xr.FIELDS:
            assert same(got[f][:n], c.outputs[j][f]), f"receiver {j}: {f}"
            assert (got[f][n:] == SENTINEL).all(), f"receiver {j}: {f} written beyond its {n} rows"


@pytest.mark.parametrize("name", list(CASES))
def test_exchange_sim_direct_placement(name):
    c = get_case(name)
    W, B = c.W, c.B
    # 1. counts per rank, per-block counts add up to them
    blk = []
    for i in range(W):
        slab, blkcnt, blkbase, counts = xr_count(c, i)
        assert np.array_equal(gu.npy(counts), c.cnt[i].T), f"rank {i}: counts"
        if c.P[i]:
            bc = gu.npy(blkcnt).reshape(W, B, -1).astype(np.int64)
            assert np.array_equal(bc.sum(axis=2), c.cnt[i].T), f"rank {i}: per-block counts"
            assert np.array_equal(gu.npy(blkbase).astype(np.int64), np.cumsum(bc.reshape(-1)) - bc.reshape(-1))
        assert slab.guards_intact()
        blk.append((counts, blkbase))
    blkbases = [b for _, b in blk]
    # 2. pack with device rows from the all-gathered counts, laid out as exchange_cat's all_gather leaves them
    cap = (max(c.N) // 4 + 2) * 4
    allc = torch.cat([counts.t().contiguous().reshape(-1) for counts, _ in blk])
    devp, rows = run_pack(c, blkbases, cap, allc)
    for me in range(W):
        r = rows.words(me)
        assert r[:W * B].tolist() == exchange.direct_rows(c.cnt, me)[0] and r[W * B] == 0, f"rank {me}: device rows"
    assert rows.guards_intact()
    check_regions(c, devp, cap)
    small = (max(c.N) - 1) // 4 * 4           # a positive multiple of 4 below the largest receiver total
    if small > 0:
        over, rows = run_pack(c, blkbases, small, allc)
        assert all(rows.words(me)[W * B] == 1 for me in range(W)), "over-capacity flag"
        assert bool((over.buf == 0xFF).all()), "an over-capacity pack wrote rows"
    # 3. pull the gradients back: sum over the destinations in ascending rank order.  The padding float of the 16-byte
    #    d rgb rows is NaN and rows beyond N_j keep the NaN fill: neither may reach a source's gradient.
    grad = Slab([4 * 10 * cap] * W)
    for j in range(W):
        n = c.N[j]
        g = grad.regions[j].view(torch.float32)
        g[:2 * cap].view(cap, 2)[:n] = gu.to_dev(c.g_eff[j]["means2D"])
        drgb = g[2 * cap:6 * cap].view(cap, 4)
        drgb[:n, :3] = gu.to_dev(c.g_eff[j]["rgb"])
        drgb[:n, 3] = float("nan")
        g[6 * cap:10 * cap].view(cap, 4)[:n] = gu.to_dev(c.g_eff[j]["conic_opacity"])
    gbases = (C.c_void_p * W)(*[grad.regions[j].data_ptr() for j in range(W)])
    c.pulled = []
    for i in range(W):
        P = c.P[i]
        out = Slab([4 * B * P * xr.WIDTH[f] for f in xr.GRAD_FIELDS])
        d = [out.f32(q, (B, P, xr.WIDTH[f])) for q, f in enumerate(xr.GRAD_FIELDS)]
        row0, _ = exchange.direct_rows(c.cnt, i)
        _lib.call("gs_xr_pull_grad", B, P, W, c.H, c.Wimg, c.ptrs(i, "means2D"), c.ptrs(i, "radii"), c.lo_c, c.hi_c,
                  blkbases[i].data_ptr(), gbases, _i32(row0), C.c_longlong(cap), _slab_ptrs(d[0], B),
                  _slab_ptrs(d[1], B), _slab_ptrs(d[2], B), gu.stream())
        assert out.guards_intact()
        for q, f in enumerate(xr.GRAD_FIELDS):
            got = gu.npy(d[q])
            assert not np.isnan(got).any(), f"rank {i}: NaN padding or unwritten rows reached d {f}"
            assert same(got, c.back[i][f]), f"rank {i}: d {f}"
        c.pulled.append([gu.npy(t) for t in d])


# ---------------------------------------------------------------------------------------------------------------------
# row staging over NCCL (the fallback): route -> pack -> all-to-all -> unpack; pack_grad -> reverse all-to-all ->
# scatter_grad
# ---------------------------------------------------------------------------------------------------------------------
def staged_grad_rows(c, j):
    """Receiver j's expected 9-float gradient rows in its row-staged receive order (g_eff)."""
    out = np.zeros((c.N[j], exchange.GROW), np.float32)
    for i in range(c.W):
        for k in range(c.B):
            a, b, n = c.ref.recv[j, k, i], c.ref.staged[j, i, k], c.cnt[i, k, j]
            out[b:b + n, 0:2] = c.g_eff[j]["means2D"][a:a + n]
            out[b:b + n, 2:5] = c.g_eff[j]["rgb"][a:a + n]
            out[b:b + n, 5:9] = c.g_eff[j]["conic_opacity"][a:a + n]
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_exchange_sim_row_staged(name):
    c = get_case(name)
    W, B, s = c.W, c.B, gu.stream()
    # the segment table of gs_xchg_unpack / pack_grad holds MAX_SEGMENTS non-empty (source, camera) blocks
    nseg = [int((c.cnt[:, :, j] > 0).sum()) for j in range(W)]
    # 4. route: flags [j][k][i], their exclusive scan, counts [j][k]
    routed, sends = [], []
    for i in range(W):
        P = c.P[i]
        n = max(W * B * P, 1)
        slab = Slab([n, 4 * n, 4 * W * B, 4 * max(c.layouts[i].total_send, 1) * exchange.ROW])
        flags, gpos, counts = slab.regions[0], slab.i32(1, (n,)), slab.i32(2, (W, B))
        tb = _lib.query("gs_xchg_temp_bytes", B, P, W)
        temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
        _lib.call("gs_xchg_route", B, P, W, c.H, c.Wimg, c.ptrs(i, "means2D"), c.ptrs(i, "radii"), c.lo_c, c.hi_c,
                  flags.data_ptr(), gpos.data_ptr(), counts.data_ptr(), temp.data_ptr(), tb, s)
        assert np.array_equal(gu.npy(counts), c.cnt[i].T), f"rank {i}: counts"
        if P:
            f = gu.npy(flags).reshape(W, B, P)
            assert np.array_equal(f, c.hits[i].transpose(2, 0, 1).astype(np.uint8)), f"rank {i}: flags"
            e = f.reshape(-1).astype(np.int64)
            assert np.array_equal(gu.npy(gpos).astype(np.int64), np.cumsum(e) - e), f"rank {i}: gpos"
        # 5. pack: the 11-float send rows in all_to_all_single order
        T = c.layouts[i].total_send
        send = slab.f32(3, (-1, exchange.ROW))
        _lib.call("gs_xchg_pack", B, P, W, flags.data_ptr(), gpos.data_ptr(), c.ptrs(i, "means2D"), c.ptrs(i, "rgb"),
                  c.ptrs(i, "conic_opacity"), c.ptrs(i, "radii"), c.ptrs(i, "depths"), send.data_ptr(), s)
        words = bits(gu.npy(send))
        assert same(gu.npy(send)[:T], xr.send_rows(c.shards[i], c.hits[i])), f"rank {i}: send rows"
        assert (words[T:] == SENTINEL).all() and slab.guards_intact()
        routed.append((flags, gpos, slab))
        sends.append(send[:T])
    # the all-to-all, simulated
    recv = []
    for j in range(W):
        parts = [sends[i].split(c.layouts[i].send_splits)[j] for i in range(W)]
        assert [p.shape[0] for p in parts] == c.layouts[j].recv_splits
        recv.append(torch.cat(parts).contiguous())
    # 6. unpack on every receiver: the reference outputs (== the direct placement's regions)
    for j in range(W):
        lay, n = c.layouts[j], c.N[j]
        vs = [int(v) for v in c.ref.view[j]]
        out = Slab([4 * n * 2, 4 * n * 3, 4 * n * 4, 4 * n, 4 * n])
        o = [out.regions[q] for q in range(5)]
        rs, ln, cam, ds = exchange.segments(lay)
        args = (len(rs), _i32(rs), _i32(ln), _i32(cam), _i32(ds), lay.total_recv, recv[j].data_ptr(), B,
                _row_ptrs(out.f32(0, (n, 2)), vs, B), _row_ptrs(out.f32(1, (n, 3)), vs, B),
                _row_ptrs(out.f32(2, (n, 4)), vs, B), _row_ptrs(out.i32(3, (n,)), vs, B), _row_ptrs(out.f32(4, (n,)), vs, B),
                s)
        if nseg[j] > exchange.MAX_SEGMENTS:
            # 8. more (source, camera) blocks than the segment table holds: a clean error, nothing launched
            with pytest.raises(_lib.GsError, match="segments"):
                _lib.call("gs_xchg_unpack", *args)
            torch.cuda.synchronize()
            assert bool((out.buf == 0xFF).all())
            continue
        _lib.call("gs_xchg_unpack", *args)
        assert out.guards_intact()
        for q, f in enumerate(xr.FIELDS):
            assert same(bits(gu.npy(o[q])), bits(c.outputs[j][f]).reshape(-1)), f"receiver {j}: {f}"
    # 7. backward: pack_grad (one camera NULL -> zeros), the reverse all-to-all, scatter_grad
    grecv = []
    for j in range(W):
        lay, n = c.layouts[j], c.N[j]
        vs = [int(v) for v in c.ref.view[j]]
        g = {f: gu.to_dev(c.g_full[j][f]) for f in xr.GRAD_FIELDS}
        gp = []
        for f in xr.GRAD_FIELDS:
            p = _row_ptrs(g[f], vs, B)
            for k, nf in c.nulls:
                if nf == f:
                    p[k] = None
            gp.append(p)
        rs, ln, cam, ds = exchange.segments(lay)
        rows_out = Slab([4 * n * exchange.GROW])
        args = (len(rs), _i32(rs), _i32(ln), _i32(cam), _i32(ds), lay.total_recv, B, *gp)
        if nseg[j] > exchange.MAX_SEGMENTS:
            with pytest.raises(_lib.GsError, match="segments"):
                _lib.call("gs_xchg_pack_grad", *args, rows_out.regions[0].data_ptr(), s)
            torch.cuda.synchronize()
            assert bool((rows_out.buf == 0xFF).all())
            continue
        _lib.call("gs_xchg_pack_grad", *args, rows_out.regions[0].data_ptr(), s)
        got = gu.npy(rows_out.f32(0, (n, exchange.GROW)))
        assert rows_out.guards_intact() and same(got, staged_grad_rows(c, j)), f"receiver {j}: gradient rows"
        grecv.append(rows_out.f32(0, (n, exchange.GROW)))
    if max(nseg) > exchange.MAX_SEGMENTS:
        return      # the row-staged path cannot serve this step; the direct placement test covers its backward
    for i in range(W):
        # the reverse all-to-all, simulated: rank i receives its block of every receiver's gradient rows, in rank order
        # (at least one row, as _ExchangeSplats allocates it: a zero-size buffer has no address)
        T = c.layouts[i].total_send
        gsend = Slab([4 * max(T, 1) * exchange.GROW])
        gsend.f32(0, (-1, exchange.GROW))[:T] = torch.cat([grecv[j].split(c.layouts[j].recv_splits)[i]
                                                           for j in range(W)])
        P = c.P[i]
        flags, gpos, _ = routed[i]
        out = Slab([4 * B * P * xr.WIDTH[f] for f in xr.GRAD_FIELDS])
        d = [out.f32(q, (B, P, xr.WIDTH[f])) for q, f in enumerate(xr.GRAD_FIELDS)]
        _lib.call("gs_xchg_scatter_grad", B, P, W, flags.data_ptr(), gpos.data_ptr(), gsend.regions[0].data_ptr(),
                  _slab_ptrs(d[0], B), _slab_ptrs(d[1], B), _slab_ptrs(d[2], B), s)
        assert out.guards_intact() and gsend.guards_intact()
        for q, f in enumerate(xr.GRAD_FIELDS):
            got = gu.npy(d[q])
            assert same(got, c.back[i][f]), f"rank {i}: d {f}"
            if getattr(c, "pulled", None) is not None:
                assert same(got, c.pulled[i][q]), f"rank {i}: d {f} differs from gs_xr_pull_grad"


def test_exchange_sim_limits_reached():
    """The (16, 16) case reaches the kernels' 16-rank and 16-camera limits and W*B = 256 threads of k_xr_rows, and a
    receiver there has more (source, camera) blocks than gs_xchg_unpack's segment table holds."""
    c = get_case("w16b16")
    assert (c.W, c.B) == (exchange.MAX_RANKS, exchange.MAX_CAMERAS)
    assert max(int((c.cnt[:, :, j] > 0).sum()) for j in range(c.W)) > exchange.MAX_SEGMENTS


# ---------------------------------------------------------------------------------------------------------------------
# sparse gradient all-reduce (grad_sync, row L2): mask -> OR over ranks -> scan -> pack -> sum -> unpack
# ---------------------------------------------------------------------------------------------------------------------
WIDTHS = (3, 3, 45, 3, 4, 1)


def test_sparse_grad_mask_follows_nonzero():
    """A Gaussian is touched when torch.nonzero would list its _xyz.grad row: NaN counts, -0.0 does not."""
    P = 1000
    rng = np.random.default_rng(5)
    g = rng.normal(size=(P, 3)).astype(np.float32)
    g[rng.random((P, 3)) < 0.5] = 0.0
    g[100:110] = 0.0
    g[110:120] = -0.0
    g[120:130] = [[-0.0, 0.0, -0.0]] * 10
    g[130, 1], g[131, 2], g[132, 0] = np.nan, -np.nan, np.inf
    g[133] = [0.0, -0.0, 1e-45]                                   # the smallest subnormal is non-zero
    slab = Slab([P])
    _lib.call("gs_sparse_grad_mask", P, gu.to_dev(g).data_ptr(), slab.regions[0].data_ptr(), gu.stream())
    xyz = torch.from_numpy(g)
    touched = torch.zeros((P,), dtype=torch.uint8)
    touched[torch.nonzero(xyz)[:, 0].unique()] = 1
    assert np.array_equal(gu.npy(slab.regions[0]), touched.numpy()) and slab.guards_intact()
    assert touched[130:134].tolist() == [1, 1, 1, 1] and not touched[100:130].any()
    _lib.call("gs_sparse_grad_mask", 0, None, None, gu.stream())


@pytest.mark.parametrize("P", [1, 31, 255, 256, 257, 4099, 70001])
def test_sparse_route_scan_column_major(P):
    """gs_route_scan (also the row-staged exchange's and the sparse all-reduce's scan): exclusive ranks of the non-zero
    bytes of a (P, ncols) mask in column-major order, and every column's first rank, for ncols 1 ... 16."""
    rng = np.random.default_rng(P)
    for ncols in range(1, 17):
        mask = np.where(rng.random((P, ncols)) < 0.3, rng.choice([1, 7, 255], (P, ncols)), 0).astype(np.uint8)
        slab = Slab([4 * ncols * P, 4 * (ncols + 1)])
        gpos, colstart = slab.i32(0, (ncols * P,)), slab.i32(1, (ncols + 1,))
        tb = _lib.query("gs_route_scan_temp_bytes", P, ncols)
        temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
        _lib.call("gs_route_scan", P, ncols, gu.to_dev(mask).data_ptr(), gpos.data_ptr(), colstart.data_ptr(),
                  temp.data_ptr(), tb, gu.stream())
        flat = (mask != 0).T.reshape(-1).astype(np.int64)
        exp = np.cumsum(flat) - flat
        assert np.array_equal(gu.npy(gpos).astype(np.int64), exp), ncols
        assert gu.npy(colstart).tolist() == [int(exp[q * P]) for q in range(ncols)] + [int(flat.sum())], ncols
        assert slab.guards_intact()
    slab = Slab([4 * 4])
    _lib.call("gs_route_scan", 0, 3, None, None, slab.regions[0].data_ptr(), None, 0, gu.stream())
    assert gu.npy(slab.i32(0, (4,))).tolist() == [0, 0, 0, 0] and slab.guards_intact()


@pytest.mark.parametrize("R,P", [(2, 0), (2, 1), (3, 4099), (4, 20011)])
def test_sparse_grad_allreduce_simulated(R, P):
    """R replicas of one model: every rank masks, the masks are OR-ed (the all-reduce MAX), one scan, every rank packs
    its touched rows, the rows are summed in rank order (the all-reduce SUM), every rank unpacks.  Touched rows hold the
    fp32 sum bit for bit; untouched rows keep the rank's own gradient, as sync_gradients_sparsely leaves them."""
    rng = np.random.default_rng(R * 100 + P)
    s = gu.stream()
    grads, masks, slabs = [], [], []
    for r in range(R):
        touched = rng.random(P) < 0.1
        g = [rng.normal(size=(P, w)).astype(np.float32) for w in WIDTHS]
        g[0][~touched] = 0.0
        for t in g[1:]:
            t[~touched & (rng.random(P) < 0.5)] = 0.0       # untouched rows may carry other gradients
        grads.append(g)
        slab = Slab([4 * P * w for w in WIDTHS] + [max(P, 1)])
        for q, w in enumerate(WIDTHS):
            slab.f32(q, (P, w)).copy_(gu.to_dev(g[q]))
        _lib.call("gs_sparse_grad_mask", P, slab.regions[0].data_ptr(), slab.regions[6].data_ptr(), s)
        masks.append(gu.npy(slab.regions[6])[:P])
        slabs.append(slab)
    any_mask = np.zeros(P, np.uint8)
    for r in range(R):
        assert np.array_equal(masks[r], (grads[r][0] != 0).any(axis=1).astype(np.uint8))
        any_mask |= masks[r]
    mask_d = gu.to_dev(any_mask if P else np.zeros(1, np.uint8))
    aux = Slab([4 * max(P, 1), 8])
    pos, colstart = aux.i32(0, (max(P, 1),)), aux.i32(1, (2,))
    tb = _lib.query("gs_route_scan_temp_bytes", P, 1)
    temp = torch.empty((tb,), dtype=torch.uint8, device=gu.DEV)
    _lib.call("gs_route_scan", P, 1, mask_d.data_ptr(), pos.data_ptr(), colstart.data_ptr(), temp.data_ptr(), tb, s)
    n = int(gu.npy(colstart)[1])
    assert n == int(any_mask.sum())
    touched_idx = np.nonzero(any_mask)[0]
    rows = []
    for r in range(R):
        out = Slab([4 * max(n, 1) * 59])
        ptrs = (C.c_void_p * 6)(*[slabs[r].regions[q].data_ptr() for q in range(6)])
        _lib.call("gs_sparse_grad_pack", P, mask_d.data_ptr(), pos.data_ptr(), ptrs, out.regions[0].data_ptr(), s)
        got = gu.npy(out.f32(0, (-1, 59)))[:n]
        exp = np.concatenate([g[touched_idx] for g in grads[r]], axis=1)
        assert same(got, exp) and out.guards_intact(), f"rank {r}: packed rows"
        rows.append(got)
    total = rows[0].copy()
    for r in range(1, R):
        total = total + rows[r]
    total_d = gu.to_dev(total if n else np.zeros((1, 59), np.float32))
    for r in range(R):
        ptrs = (C.c_void_p * 6)(*[slabs[r].regions[q].data_ptr() for q in range(6)])
        _lib.call("gs_sparse_grad_unpack", P, mask_d.data_ptr(), pos.data_ptr(), total_d.data_ptr(), ptrs, s)
        assert slabs[r].guards_intact()
        off = 0
        for q, w in enumerate(WIDTHS):
            got = gu.npy(slabs[r].f32(q, (P, w)))
            exp = grads[r][q].copy()
            s_ = grads[0][q][touched_idx].copy()
            for rr in range(1, R):
                s_ = s_ + grads[rr][q][touched_idx]
            exp[touched_idx] = s_
            assert same(got, exp), f"rank {r}: gradient {q}"
            assert same(total[:, off:off + w], s_)
            off += w
