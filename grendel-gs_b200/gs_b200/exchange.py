"""Sparse Gaussian -> pixel-owner all-to-all (and its mirrored backward).

Restates /root/reference/gaussian_renderer/__init__.py:542-698 (all_to_all_communication_final):
every rank projects its own Gaussian shard for all B cameras, then sends each projected splat to the
ranks whose tile-row strip its rectangle touches.  Two paths, chosen per step from values every rank shares:
  * direct placement over NVLink peer memory (PeerBuffers, default when every rank could map them): the pack kernel
    stores every splat into its final row of the destination's receive region, which IS the render's input, and the
    backward pulls the gradient rows from the destinations' gradient regions;
  * row staging over NCCL (no peer buffers, or a step whose rows exceed them): ONE launch per stage for all B cameras
    -- routing flags are laid out [destination][camera][splat], so a single exclusive scan yields every row of the
    send buffer (no W x B nonzero()/index_select/cat, workload_division.py:741-742, __init__.py:590-607) -- ONE
    all_to_all_single of 11-float rows forward (means2D, rgb, conic_opacity, radius, depth) instead of two
    collectives, ONE of 9-float rows backward, and a backward scatter of one thread per local splat (no atomics).
Both need one host sync (the counts) instead of W+2.  Row order is the reference's: per destination, cameras in batch
order, splats in index order; per receiver, sources in rank order.
"""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, ops

ROW, GROW = 11, 9
MAX_CAMERAS, MAX_RANKS, MAX_SEGMENTS = 16, 16, 128   # XB, XW, XSEG of csrc/distribute.cu
MODE = "direct"   # the exchange over peer memory: direct placement (bench.py reports it)


def _t(mark, name):
    """Diagnostics: mark(name) synchronises and charges the time since the last mark (pipeline.Trainer._mark)."""
    if mark is not None:
        mark(name)


# ---------------------------------------------------------------------------------------------------
# pure-Python layout (tested on CPU with gloo)
# ---------------------------------------------------------------------------------------------------
class Layout:
    """Row offsets of one step's exchange, from the all-gathered counts.

    cnt[i][k][j] = number of splats rank i sends to rank j for camera k (zeros where j does not render k).
    """

    def __init__(self, cnt, me, gpu_ids_per_cam):
        # runs on the critical path right after the step's host sync (the GPU is idle until the pack kernel is
        # launched): numpy prefix sums instead of O(W B^2) Python loops
        c = np.asarray(cnt, dtype=np.int64).reshape(len(cnt), len(cnt[0]), len(cnt))     # (W, B, W)
        W, B = c.shape[0], c.shape[1]
        self.W, self.B, self.me = W, B, me
        S = c.sum(axis=1)                                    # S[i][j]: rows rank i sends to rank j
        send_base, recv_base = _excl(S[me]), _excl(S[:, me])
        self.send_splits, self.recv_splits = S[me].tolist(), S[:, me].tolist()
        # camera k, local column c (destination gpu_ids[k][c]) -> first row in the send buffer
        before_send = _excl(c[me], axis=0)                   # [k][j]: rows of cameras < k that go to j
        off = (send_base[None, :] + before_send).tolist()
        self.dst_off = [[off[k][j] for j in gpu_ids_per_cam[k]] for k in range(B)]
        # camera k -> (segment offsets, segment lengths) in the recv buffer, one segment per source rank
        mine = c[:, :, me]                                   # [i][k]: rows rank i sends me for camera k
        self.seg_off = (recv_base[:, None] + _excl(mine, axis=1)).T.tolist()
        self.seg_len = mine.T.tolist()
        self.n_recv = mine.sum(axis=0).tolist()
        self.seg_dst = _excl(mine, axis=0).T.tolist()        # [k][i]: first row of the segment inside camera k's output
        self.total_send, self.total_recv = int(S[me].sum()), int(S[:, me].sum())


def _excl(a, axis=0):
    """Exclusive prefix sum along `axis`."""
    out = np.cumsum(a, axis=axis)
    return out - a


def all_to_all_single(out, inp, out_splits, in_splits, group=None):
    """dist.all_to_all_single on NCCL; isend/irecv emulation elsewhere (gloo has no all_to_all)."""
    if dist.get_backend(group) == "nccl":
        dist.all_to_all_single(out, inp, out_splits, in_splits, group=group)
        return
    W, me = dist.get_world_size(group), dist.get_rank(group)
    outs = list(out.split(out_splits, dim=0))
    ins = list(inp.split(in_splits, dim=0))
    outs[me].copy_(ins[me])
    reqs = []
    for p in range(W):
        if p == me:
            continue
        if in_splits[p]:
            reqs.append(dist.isend(ins[p].contiguous(), p, group=group))
    bufs = {}
    for p in range(W):
        if p == me or not out_splits[p]:
            continue
        bufs[p] = torch.empty_like(outs[p])
        reqs.append(dist.irecv(bufs[p], p, group=group))
    for r in reqs:
        r.wait()
    for p, b in bufs.items():
        outs[p].copy_(b)


# Timing feedback rides on the exchange: the render times a rank wants to share (a few floats, finish_strategy_final's
# all-gather of utils/general_utils.py:249-269) are all-gathered right behind the sizes and read back with them -- no
# collective of their own on the critical path, no extra host sync.  The caller (pipeline.Trainer) passes them as `times`,
# a list of floats (None on steps without feedback, on every rank alike: then no all-gather is issued), and gets every
# rank's list back as a (W, len) float32 array.
_WARNED_OVER_CAPACITY = False


def _gather_times(times, dev, world, group):
    """Enqueue the all-gather of `times` (if any) on the current stream -> device tensor (W * E) or None."""
    if times is None:
        return None
    mine = torch.tensor([float(v) for v in times], dtype=torch.float32, device=dev)
    allp = torch.empty((world * mine.numel(),), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(allp, mine, group=group)
    return allp


def gather_counts(local_counts, group=None, times=None):
    """(B, W) int32 device tensor -> ((W, B, W) integer array cnt[i][k][j], every rank's `times` as a (W, len) float32
    array or None without times); the step's one host sync."""
    W = dist.get_world_size(group)
    flat = local_counts.contiguous().reshape(-1)
    allc = torch.empty((W * flat.numel(),), dtype=flat.dtype, device=flat.device)
    dist.all_gather_into_tensor(allc, flat, group=group)
    allp = _gather_times(times, flat.device, W, group)
    out = allc.reshape((W,) + tuple(local_counts.shape)).cpu().numpy()
    return out, None if allp is None else allp.reshape(W, -1).cpu().numpy()


# ---------------------------------------------------------------------------------------------------
# device side (batched: one launch per stage for all B cameras of the step)
# ---------------------------------------------------------------------------------------------------
def _i32(vals):
    return (C.c_int32 * len(vals))(*[int(v) for v in vals])


def _ptrs(tensors):
    return (C.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])


def segments(layout):
    """(recv_start, length, camera, dst_start) of every (source rank, camera) block of the recv buffer, in recv
    order; dst_start is the block's first row inside that camera's concatenated output."""
    rs, ln, cam, ds = [], [], [], []
    for i in range(layout.W):
        for k in range(layout.B):
            rs.append(layout.seg_off[k][i])
            ln.append(layout.seg_len[k][i])
            cam.append(k)
            ds.append(layout.seg_dst[k][i])
    return rs, ln, cam, ds


def _slab_ptrs(t, B):
    """Device pointers of the B camera slices of a contiguous (B, P, ...) tensor."""
    step = t.stride(0) * t.element_size() if B > 0 and t.dim() > 0 else 0
    base = t.data_ptr()
    return (C.c_void_p * B)(*[base + k * step for k in range(B)])


class PeerBuffers:
    """NVLink peer-memory regions of the direct-placement exchange (include/grendel_gs_b200.h, gs_peer_* / gs_xr_*):
    every rank owns one receive region of `cap_rows` rows (means2D | rgb | conic_opacity | radii | depths, 11 floats per
    row) and one gradient region of `cap_rows` rows (d means2D | d rgb | d conic_opacity, 10 floats per row), exported
    over CUDA IPC and mapped by all peers of the node.  recv[j] / grad[j] are rank j's regions as addresses valid in THIS
    process.  Collective: every rank of `group` must construct it at the same point (handles travel by all_gather)."""

    def __init__(self, world, me, cap_rows, device, group=None):
        self.world, self.me, self.cap_rows, self.group = world, me, (int(cap_rows) + 3) // 4 * 4, group
        self.device = device
        self._owned, self._opened = [], []
        self._views = None
        self.token = torch.zeros((1,), dtype=torch.float32, device=device)
        # every local step that can fail is followed by an agreement (all-reduce MIN), so that either all ranks go on
        # or all ranks raise -- never a rank stuck alone in a collective
        handles, err = [0] * 128, None
        try:
            # gradient region: 10 floats per row (d rgb is padded to 16 bytes)
            for q, nbytes in enumerate((self.cap_rows * ROW * 4, self.cap_rows * (GROW + 1) * 4)):
                ptr, handle = C.c_void_p(), (C.c_ubyte * 64)()
                _lib.call("gs_peer_alloc", nbytes, C.byref(ptr), handle)
                self._owned.append(ptr.value)
                handles[64 * q:64 * q + 64] = list(handle)
        except Exception as e:   # noqa: BLE001
            err = e
        self._agree(err, device, "allocate / export")
        mine = torch.tensor(handles, dtype=torch.uint8, device=device)
        allh = torch.empty((world * 128,), dtype=torch.uint8, device=device)
        dist.all_gather_into_tensor(allh, mine, group=group)
        allh = allh.cpu().reshape(world, 128).tolist()
        self.recv, self.grad = [0] * world, [0] * world
        try:
            for j in range(world):
                for q, table in enumerate((self.recv, self.grad)):
                    if j == me:
                        table[j] = self._owned[q]
                        continue
                    h, p = (C.c_ubyte * 64)(*allh[j][64 * q:64 * q + 64]), C.c_void_p()
                    _lib.call("gs_peer_open", h, C.byref(p))
                    self._opened.append(p.value)
                    table[j] = p.value
        except Exception as e:   # noqa: BLE001
            err = e
        self._agree(err, device, "map the peers' buffers")

    def _agree(self, err, device, what):
        ok = torch.tensor([0.0 if err is not None else 1.0], device=device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
        if float(ok.item()) < 1.0:
            self.close()
            raise RuntimeError(f"peer-memory exchange: could not {what} on every rank (this rank: {err!r})")

    def barrier(self):
        """Stream-ordered: completes on this rank once every rank's stream reached the same call (a 4-byte all-reduce;
        the host does not block).

        Buffer-reuse invariant: a peer writes into this rank's receive region only from its pack kernel, and it launches
        that only after the all-gather of the SAME exchange's counts; it reads this rank's gradient region only in its
        pull kernel, which it enqueues before it joins the next exchange's all-gather.  Those all-gathers run on the
        stream that this rank joins after its consumers of the previous exchange (the render reading the receive region,
        the backward writing the gradient region) were enqueued.  So every remote access is ordered against this rank's
        own accesses as long as (a) every exchange starts with the all-gather of the counts and (b) exchange, consumers
        and collectives share one stream.  A caller that caches counts or moves the consumers to another stream must call
        barrier() after its consumers instead."""
        dist.all_reduce(self.token, op=dist.ReduceOp.MAX, group=self.group)   # MAX of zeros: the value never grows

    def views(self):
        """This rank's own buffers as torch tensors in the structure-of-arrays layout of the direct-placement exchange
        (csrc/distribute.cu "xr"): ((means2D (cap,2), rgb (cap,3), conic_opacity (cap,4), radii (cap) int32, depths (cap)),
        (d means2D, d rgb [a (cap,3) view of 16-byte rows], d conic_opacity)) -- zero-copy views of the peer-visible memory."""
        if self._views is None:
            cap, dev = self.cap_rows, self.device
            r, g = self.recv[self.me], self.grad[self.me]
            f = lambda base, off, shape: _wrap(base + 4 * off * cap, shape, "<f4", dev)
            self._views = ((f(r, 0, (cap, 2)), f(r, 2, (cap, 3)), f(r, 5, (cap, 4)),
                            _wrap(r + 4 * 9 * cap, (cap,), "<i4", dev), f(r, 10, (cap,))),
                           (f(g, 0, (cap, 2)), f(g, 2, (cap, 4))[:, :3], f(g, 6, (cap, 4))))
        return self._views

    def fits_direct(self, cnt):
        """Do every rank's received rows (all cameras) fit the structure-of-arrays regions?  Same answer on every rank."""
        return int(np.asarray(cnt, dtype=np.int64).sum(axis=(0, 1)).max()) <= self.cap_rows

    def close(self):
        for name, ptrs in (("gs_peer_close", self._opened), ("gs_peer_free", self._owned)):
            for p in ptrs:
                try:
                    _lib.call(name, p)
                except _lib.GsError:
                    pass
        self._opened, self._owned = [], []


class _DevMem:
    """__cuda_array_interface__ holder: lets torch view device memory it did not allocate (the IPC-exported buffers)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 3, "strides": None}


def _wrap(ptr, shape, typestr, device):
    return torch.as_tensor(_DevMem(ptr, shape, typestr), device=device)


def direct_rows(cnt, me):
    """Direct-placement layout from the all-gathered counts cnt[i][k][j]:
    -> (dst_row0[j][k] = first row of MY block inside camera k of rank j's arrays, my view_start (B+1))."""
    c = np.asarray(cnt, dtype=np.int64)                        # (W, B, W)
    per_cam = c.sum(axis=0)                                    # [k][j]: rows of camera k on rank j
    view_start = _excl(per_cam, axis=0)                        # [k][j]
    before_me = c[:me].sum(axis=0)                             # [k][j]: rows of ranks < me
    row0 = (view_start + before_me).T                          # [j][k]
    mine = np.concatenate([view_start[:, me], [per_cam[:, me].sum()]])
    return row0.reshape(-1).tolist(), [int(v) for v in mine]


def _row_ptrs(t, starts, B):
    """Device pointers of rows starts[k] (k < B) of a contiguous (N, ...) tensor; NULLs if t is None."""
    if t is None:
        return (C.c_void_p * B)(*[None] * B)
    step = t.stride(0) * t.element_size() if t.shape[0] > 0 else 0
    base = t.data_ptr()
    return (C.c_void_p * B)(*[base + starts[k] * step for k in range(B)])


class _ExchangeSplats(torch.autograd.Function):
    """inputs: means2D (B,P,2), rgb (B,P,3), conic_opacity (B,P,4) of the local shard for the B cameras.
    outputs: the received splats of all B cameras CONCATENATED in camera order -- means2D (N,2), rgb (N,3),
    conic_opacity (N,4) (differentiable), radii (N) int32, depths (N); camera k owns rows
    [view_start[k], view_start[k+1]).  That is the layout the batched render consumes, and it makes both directions
    whole-tensor operations: nothing is sliced, concatenated or re-accumulated per camera."""

    @staticmethod
    def forward(ctx, state, m2, rgb, co):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        layout, group = state["layout"], state["group"]
        B, P, W = state["B"], state["P"], state["W"]
        m2, rgb, co = m2.contiguous(), rgb.contiguous(), co.contiguous()
        radii, depths = state["radii"], state["depths"]
        dev = m2.device
        s = ops._stream()
        send = torch.empty((max(layout.total_send, 1), ROW), dtype=torch.float32, device=dev)
        _lib.call("gs_xchg_pack", B, P, W, state["flags"].data_ptr(), state["gpos"].data_ptr(), _slab_ptrs(m2, B),
                  _slab_ptrs(rgb, B), _slab_ptrs(co, B), _slab_ptrs(radii, B), _slab_ptrs(depths, B), send.data_ptr(), s)
        _t(state["mark"], "x3 pack")
        recv = torch.empty((max(layout.total_recv, 1), ROW), dtype=torch.float32, device=dev)
        all_to_all_single(recv[:layout.total_recv], send[:layout.total_send], layout.recv_splits, layout.send_splits,
                          group)
        _t(state["mark"], "x4 all_to_all")
        vs = state["view_start"]
        N = vs[B]
        om2 = torch.empty((N, 2), dtype=torch.float32, device=dev)
        orgb = torch.empty((N, 3), dtype=torch.float32, device=dev)
        oco = torch.empty((N, 4), dtype=torch.float32, device=dev)
        orad = torch.empty((N,), dtype=torch.int32, device=dev)
        odep = torch.empty((N,), dtype=torch.float32, device=dev)
        rs, ln, cam, ds = state["segs"]
        _lib.call("gs_xchg_unpack", len(rs), _i32(rs), _i32(ln), _i32(cam), _i32(ds), layout.total_recv, recv.data_ptr(),
                  B, _row_ptrs(om2, vs, B), _row_ptrs(orgb, vs, B), _row_ptrs(oco, vs, B), _row_ptrs(orad, vs, B),
                  _row_ptrs(odep, vs, B), s)
        ctx.state = state
        ctx.mark_non_differentiable(orad, odep)
        return om2, orgb, oco, orad, odep

    @staticmethod
    def backward(ctx, g_m2, g_rgb, g_co, *_unused):
        state = ctx.state
        layout, group = state["layout"], state["group"]
        B, P, W = state["B"], state["P"], state["W"]
        dev = state["flags"].device
        s = ops._stream()
        vs = state["view_start"]
        _t(state["mark"], "b1 loss+render backward")
        g_m2, g_rgb, g_co = (None if t is None else t.contiguous() for t in (g_m2, g_rgb, g_co))
        rs, ln, cam, ds = state["segs"]
        grecv = torch.empty((max(layout.total_recv, 1), GROW), dtype=torch.float32, device=dev)
        _lib.call("gs_xchg_pack_grad", len(rs), _i32(rs), _i32(ln), _i32(cam), _i32(ds), layout.total_recv, B,
                  _row_ptrs(g_m2, vs, B), _row_ptrs(g_rgb, vs, B), _row_ptrs(g_co, vs, B), grecv.data_ptr(), s)
        _t(state["mark"], "b2 pack_grad")
        gsend = torch.empty((max(layout.total_send, 1), GROW), dtype=torch.float32, device=dev)
        all_to_all_single(gsend[:layout.total_send], grecv[:layout.total_recv], layout.send_splits, layout.recv_splits,
                          group)
        _t(state["mark"], "b3 all_to_all")
        d_m2 = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
        d_rgb = torch.empty((B, P, 3), dtype=torch.float32, device=dev)
        d_co = torch.empty((B, P, 4), dtype=torch.float32, device=dev)
        _lib.call("gs_xchg_scatter_grad", B, P, W, state["flags"].data_ptr(), state["gpos"].data_ptr(), gsend.data_ptr(),
                  _slab_ptrs(d_m2, B), _slab_ptrs(d_rgb, B), _slab_ptrs(d_co, B), s)
        return None, d_m2, d_rgb, d_co


class _ExchangeSplatsDirect(torch.autograd.Function):
    """Same contract as _ExchangeSplats over the direct-placement kernels: the pack kernel has stored every field into its
    final row of the destination's arrays (launched by exchange_cat right after the counts arrived, so that the GPU idles as
    briefly as possible behind the step's host sync); the outputs ARE views of this rank's peer-visible receive region (no
    unpack), and the backward pulls the gradient rows from the destinations' gradient regions."""

    @staticmethod
    def forward(ctx, state, m2, rgb, co):
        ctx.set_materialize_grads(False)   # undefined output gradients arrive as None, not as zero-filled tensors
        B, peer = state["B"], state["peer"]
        N = state["view_start"][B]
        (v_m2, v_rgb, v_co, v_rad, v_dep), _ = peer.views()
        om2, orgb, oco, orad, odep = v_m2[:N], v_rgb[:N], v_co[:N], v_rad[:N], v_dep[:N]
        ctx.state = state
        ctx.mark_non_differentiable(orad, odep)
        return om2, orgb, oco, orad, odep

    @staticmethod
    def backward(ctx, g_m2, g_rgb, g_co, *_unused):
        state = ctx.state
        B, P, W, peer = state["B"], state["P"], state["W"], state["peer"]
        dev = state["radii"].device
        s = ops._stream()
        N = state["view_start"][B]
        _t(state["mark"], "b1 loss+render backward")
        _, (v_dm2, v_drgb, v_dco) = peer.views()
        for view, g in ((v_dm2, g_m2), (v_drgb, g_rgb), (v_dco, g_co)):   # into the peer-visible gradient region
            if g is None:
                view[:N].zero_()
            else:
                view[:N].copy_(g)
        _t(state["mark"], "b2 pack_grad")
        peer.barrier()
        _t(state["mark"], "b3 all_to_all")
        d_m2 = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
        d_rgb = torch.empty((B, P, 3), dtype=torch.float32, device=dev)
        d_co = torch.empty((B, P, 4), dtype=torch.float32, device=dev)
        _lib.call("gs_xr_pull_grad", B, P, W, state["H"], state["Wimg"], _slab_ptrs(state["m2d"], B),
                  _slab_ptrs(state["radii"], B), state["lo"], state["hi"], state["blkbase"].data_ptr(),
                  (C.c_void_p * W)(*peer.grad), state["row0"], C.c_longlong(peer.cap_rows), _slab_ptrs(d_m2, B),
                  _slab_ptrs(d_rgb, B), _slab_ptrs(d_co, B), s)
        return None, d_m2, d_rgb, d_co


_SIDE = {}


def _read_counts_on_side_stream(dev_tensor, ready_event, shape):
    """Host copy of a small device tensor WITHOUT synchronising the current stream: a side stream waits for `ready_event`
    (recorded right behind the producer), copies into pinned memory and only that copy is waited for."""
    dev = dev_tensor.device
    key = (dev, dev_tensor.numel(), dev_tensor.dtype)
    if key not in _SIDE:
        _SIDE[key] = (torch.cuda.Stream(device=dev), torch.empty((dev_tensor.numel(),), dtype=dev_tensor.dtype).pin_memory())
    side, pinned = _SIDE[key]
    side.wait_event(ready_event)
    with torch.cuda.stream(side):
        pinned.copy_(dev_tensor, non_blocking=True)
        done = torch.cuda.Event()
        done.record(side)
    dev_tensor.record_stream(side)
    done.synchronize()
    return pinned.numpy().reshape(shape).copy()


def open_peer_buffers(world, me, cap_rows, device, group=None):
    """PeerBuffers if every rank of the group could allocate, export and map them, else None on ALL ranks (the
    exchange then uses all_to_all_single).  Collective."""
    if world <= 1 or dist.get_backend(group) != "nccl":
        return None
    try:
        return PeerBuffers(world, me, cap_rows, device, group)   # raises on every rank or on none
    except RuntimeError as e:   # IPC not permitted in this container, out of memory, no peer access ...
        import warnings
        warnings.warn(f"rank {me}: NVLink peer-memory exchange unavailable ({e}); using all_to_all_single")
        return None


def exchange(means2D, rgb, conic_opacity, radii, depths, strategies, settings, world, me, group=None, peer=None):
    """Per-camera view of exchange_cat (the reference's return shape, gaussian_renderer/__init__.py:1010-1023):
    a list of B tuples (means2D, rgb, conic_opacity, radii, depths) -- row slices of the concatenated tensors, empty
    where this rank renders no strip of the camera -- and the all-gathered counts."""
    (m2, c3, co, rad, dep), view_start, cnt, _ = exchange_cat(means2D, rgb, conic_opacity, radii, depths, strategies,
                                                              settings, world, me, group, peer)
    out = []
    for k in range(len(view_start) - 1):
        a, b = view_start[k], view_start[k + 1]
        out.append((m2[a:b], c3[a:b], co[a:b], rad[a:b], dep[a:b]))
    return out, cnt


def exchange_cat(means2D, rgb, conic_opacity, radii, depths, strategies, settings, world, me, group=None, peer=None,
                 times=None, mark=None):
    """means2D (B,P,2), rgb (B,P,3), conic_opacity (B,P,4), radii (B,P) int32, depths (B,P): the local shard projected
    into the B cameras of the step (ops.preprocess_gaussians_batched, or torch.stack of per-camera results).
    peer: PeerBuffers -> splats travel by direct NVLink stores from the pack kernel into their final rows (steps where
    some rank would receive more than the regions hold, and peer=None, go through all_to_all_single).
    times: this rank's render times for the load balancer, all-gathered behind the counts (None: no all-gather; every
    rank must pass None alike).  mark: the diagnostics hook, called with each phase's name, in the backward too.
    Returns ((means2D (N,2), rgb (N,3), conic_opacity (N,4), radii (N), depths (N)), view_start, cnt, gathered times): the
    splats this rank has to render, all cameras concatenated in camera order (camera k = rows [view_start[k],
    view_start[k+1]), none if the rank renders no strip of it), the all-gathered counts cnt[i][k][j] (the reference's
    gpui_to_gpuj_imgk_size), and every rank's `times` as a (W, len) float32 array (None without times)."""
    B, P = means2D.shape[0], means2D.shape[1]
    # the kernels' static limits, checked HERE from values every rank shares (world, bsz, and below the all-gathered
    # counts): a rank-local failure inside a C call between two collectives would leave the other ranks hanging
    if world > MAX_RANKS or B > MAX_CAMERAS:
        raise ValueError(f"exchange supports <= {MAX_RANKS} ranks and <= {MAX_CAMERAS} cameras per step "
                         f"(got {world} ranks, {B} cameras): split the batch")
    dev = means2D.device
    H, Wimg = int(settings[0].image_height), int(settings[0].image_width)
    lo, hi = [0] * (B * world), [0] * (B * world)
    for k, st in enumerate(strategies):
        for c, j in enumerate(st.gpu_ids):
            lo[k * world + j], hi[k * world + j] = st.division_pos[c], st.division_pos[c + 1]
    radii = radii.to(torch.int32).contiguous()
    depths = depths.contiguous()
    m2d = means2D.detach().contiguous()
    if peer is not None:
        # direct placement: per-block hit counts instead of a dense flag array + W*B*P-element scan
        nblk = max(world * B * ((max(P, 1) + 255) // 256), 1)
        blkcnt = torch.empty((nblk,), dtype=torch.int32, device=dev)
        blkbase = torch.empty((nblk,), dtype=torch.int32, device=dev)
        counts = torch.empty((world, B), dtype=torch.int32, device=dev)   # [dest j][camera k]
        tb = _lib.query("gs_xr_temp_bytes", B, P, world)
        temp = torch.empty((tb,), dtype=torch.uint8, device=dev)
        lo_c, hi_c = _i32(lo), _i32(hi)
        _lib.call("gs_xr_count", B, P, world, H, Wimg, _slab_ptrs(m2d, B), _slab_ptrs(radii, B), lo_c, hi_c,
                  blkcnt.data_ptr(), blkbase.data_ptr(), counts.data_ptr(), temp.data_ptr(), tb, ops._stream())
        _t(mark, "x1 route")
        # everything the pack launch needs is prepared BEFORE the all-gather is enqueued: the launch follows it closely
        rgb_c, co_c = rgb.detach().contiguous(), conic_opacity.detach().contiguous()
        pack_args = (B, P, world, H, Wimg, _slab_ptrs(m2d, B), _slab_ptrs(rgb_c, B), _slab_ptrs(co_c, B),
                     _slab_ptrs(radii, B), _slab_ptrs(depths, B), lo_c, hi_c, blkbase.data_ptr(),
                     (C.c_void_p * world)(*peer.recv))
        cap, stream = C.c_longlong(peer.cap_rows), ops._stream()
        # The sizes are all-gathered ON THE DEVICE and the pack kernel derives its destination rows from them there
        # (k_xr_rows), so pack + barrier are enqueued before the host knows the counts; the host copy of the counts -- needed
        # for the tensor shapes of the render -- is read on a side stream meanwhile.  The main stream does not run dry at the
        # exchange's host sync (the reference blocks on the sizes before its all-to-all, gaussian_renderer/__init__.py:609-628).
        flat =counts.t().contiguous().reshape(-1)                    # [camera k][destination j]
        allc = torch.empty((world * flat.numel(),), dtype=torch.int32, device=dev)
        dist.all_gather_into_tensor(allc, flat, group=group)          # cnt[i][k][j]
        allp = _gather_times(times, dev, world, group)
        ev_counts = torch.cuda.Event()
        ev_counts.record()
        row0_dev = torch.empty((world * B + 1,), dtype=torch.int32, device=dev)
        _lib.call("gs_xr_pack_dev", *pack_args, allc.data_ptr(), me, row0_dev.data_ptr(), cap, stream)
        _t(mark, "x3 pack")
        peer.barrier()
        _t(mark, "x4 all_to_all")
        cnt = _read_counts_on_side_stream(allc, ev_counts, (world, B, world))
        gathered = None if allp is None else _read_counts_on_side_stream(allp, ev_counts, (world, -1))
        _t(mark, "x2 gather counts")
        c64 = np.asarray(cnt, dtype=np.int64)
        if peer.fits_direct(c64):   # decided from the all-gathered counts: identical on all ranks (k_xr_rows agrees)
            row0, view_start = direct_rows(c64, me)
            state = dict(group=group, radii=radii, depths=depths, m2d=m2d, blkbase=blkbase, B=B, P=P, W=world, H=H,
                         Wimg=Wimg, lo=lo_c, hi=hi_c, row0=_i32(row0), view_start=view_start, peer=peer, cnt=cnt, me=me,
                         keep=(rgb_c, co_c), mark=mark)
            res = _ExchangeSplatsDirect.apply(state, means2D, rgb, conic_opacity)
            return res, view_start, cnt, gathered
        # does not fit the buffers this step: the row-staged path below (all_to_all_single) handles any size
        global _WARNED_OVER_CAPACITY
        if not _WARNED_OVER_CAPACITY and me == 0:
            import warnings
            warnings.warn(f"exchange: {int(c64.sum(axis=(0, 1)).max())} rows for one rank exceed the peer buffers "
                          f"({peer.cap_rows} rows): this step goes through all_to_all_single (raise peer_cap_rows)")
            _WARNED_OVER_CAPACITY = True
    n = max(B * P * world, 1)
    flags = torch.empty((n,), dtype=torch.uint8, device=dev)
    gpos = torch.empty((n,), dtype=torch.int32, device=dev)
    counts = torch.empty((world, B), dtype=torch.int32, device=dev)   # [dest j][camera k]
    tb = _lib.query("gs_xchg_temp_bytes", B, P, world)
    temp = torch.empty((tb,), dtype=torch.uint8, device=dev)
    _lib.call("gs_xchg_route", B, P, world, H, Wimg, _slab_ptrs(m2d, B), _slab_ptrs(radii, B), _i32(lo), _i32(hi),
              flags.data_ptr(), gpos.data_ptr(), counts.data_ptr(), temp.data_ptr(), tb, ops._stream())
    _t(mark, "x1 route")
    cnt, gathered = gather_counts(counts.t().contiguous(), group, times)   # cnt[i][k][j]
    _t(mark, "x2 gather counts")
    nseg = int((np.asarray(cnt) > 0).sum(axis=(0, 1)).max())   # non-empty (source, camera) blocks of the busiest receiver
    if nseg >= MAX_SEGMENTS:    # identical on every rank: all raise together
        raise ValueError(f"exchange: a rank would receive {nseg} (source, camera) blocks, limit {MAX_SEGMENTS - 1}: "
                         f"use fewer cameras per step")
    layout = Layout(cnt, me, [st.gpu_ids for st in strategies])
    view_start = [0]
    for n in layout.n_recv:
        view_start.append(view_start[-1] + n)
    state = dict(layout=layout, group=group, radii=radii, depths=depths, flags=flags, gpos=gpos, B=B, P=P, W=world,
                 segs=segments(layout), view_start=view_start, mark=mark)
    res = _ExchangeSplats.apply(state, means2D, rgb, conic_opacity)
    return res, view_start, cnt, gathered
