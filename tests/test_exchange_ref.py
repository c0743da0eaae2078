"""CPU: the independent exchange reference (tests/exchange_ref.py) and the product's host-side layout helpers
(gs_b200/exchange.py: Layout, segments, direct_rows, PeerBuffers.fits_direct) agree on random counts and strategies.
The simulated-rank GPU tests build kernel arguments with those helpers and compare the kernels with the reference, so
the two pin each other."""
import numpy as np
import pytest

import exchange_ref as xr
from gs_b200 import division, exchange
from oracle.oracle import Oracle


def _random_counts(rng, W, B, ids):
    cnt = np.zeros((W, B, W), np.int64)
    for i in range(W):
        for k in range(B):
            for j in ids[k]:
                cnt[i, k, j] = rng.integers(0, 40) if rng.random() < 0.8 else 0
    return cnt


def _check_helpers(cnt, ids):
    W, B = cnt.shape[0], cnt.shape[1]
    ref = xr.RefLayout(cnt)
    for me in range(W):
        lay = exchange.Layout(cnt.tolist(), me, ids)
        assert lay.send_splits == [int(ref.send_total[me, j]) for j in range(W)]
        assert lay.recv_splits == [int(ref.send_total[i, me]) for i in range(W)]
        assert lay.total_send == int(ref.send_total[me].sum()) and lay.total_recv == ref.n_recv(me)
        for k in range(B):
            assert lay.dst_off[k] == [int(ref.send[me, j, k]) for j in ids[k]]
            assert lay.seg_off[k] == [int(ref.staged[me, i, k]) for i in range(W)]
            assert lay.seg_len[k] == [int(cnt[i, k, me]) for i in range(W)]
            assert lay.seg_dst[k] == [int(ref.recv[me, k, i] - ref.view[me, k]) for i in range(W)]
            assert lay.n_recv[k] == int(ref.view[me, k + 1] - ref.view[me, k])
        rs, ln, cam, ds = exchange.segments(lay)
        q = [(i, k) for i in range(W) for k in range(B)]
        assert rs == [int(ref.staged[me, i, k]) for i, k in q]
        assert ln == [int(cnt[i, k, me]) for i, k in q]
        assert cam == [k for _, k in q]
        assert ds == [int(ref.recv[me, k, i] - ref.view[me, k]) for i, k in q]
        row0, view_start = exchange.direct_rows(cnt, me)
        assert row0 == [int(ref.recv[j, k, me]) for j in range(W) for k in range(B)]
        assert view_start == [int(v) for v in ref.view[me]]
    # over capacity: some receiver gets more than `cap` rows (k_xr_rows: total > cap; the host: fits_direct)
    most = max(ref.n_recv(j) for j in range(W))
    holder = type("Holder", (), {})()
    for cap in (most - 1, most, most + 1):
        holder.cap_rows = cap
        assert ref.over_capacity(cap) == (cap < most) == (not exchange.PeerBuffers.fits_direct(holder, cnt))


@pytest.mark.parametrize("W,B", [(1, 1), (2, 1), (3, 2), (4, 4), (8, 2), (16, 16), (5, 7)])
def test_reference_layout_equals_host_helpers_on_random_counts(W, B):
    rng = np.random.default_rng(100 * W + B)
    for trial in range(6):
        gy = int(rng.integers(W + 1, 3 * W + 8))
        if trial % 2:
            lo, hi = xr.hand_strips(rng, W, B, gy, every_rank=trial == 3)
        else:
            st, _ = division.start_strategy(list(range(B)), division.StrategyHistory(list(range(B)), gy, W), W, 0)
            lo, hi = xr.strips_from_strategies(st, W)
        ids = xr.gpu_ids(lo, hi)
        _check_helpers(_random_counts(rng, W, B, ids), ids)
    zero = np.zeros((W, B, W), np.int64)
    _check_helpers(zero, [list(range(W))] * B)


@pytest.mark.parametrize("W,B,P", [(2, 1, (0, 257)), (3, 2, (1, 31, 257)), (4, 3, (300, 0, 31, 999))])
def test_reference_payload_round_trip(W, B, P):
    """The reference's own pieces agree with each other on routed splats: its send rows, cut by destination and
    concatenated in source order, are every receiver's arrays; the gradient of a splat is the sum over the ranks
    that received it."""
    rng = np.random.default_rng(W + 10 * B)
    H, Wimg = 200, 333
    o = Oracle(np.float32)
    lo, hi = xr.hand_strips(rng, W, B, (H + 15) // 16)
    shards = [xr.make_splats(rng, B, p, H, Wimg) for p in P]
    hits = [xr.route(o, H, Wimg, s, lo, hi) for s in shards]
    cnt = xr.counts(hits)
    ref = xr.RefLayout(cnt)
    sends = [xr.send_rows(s, h) for s, h in zip(shards, hits)]
    for j in range(W):
        got = xr.receiver_outputs(shards, hits, j)
        staged = np.concatenate([sends[i][ref.send[i, j, 0]:ref.send[i, j, 0] + ref.send_total[i, j]] for i in range(W)])
        assert staged.shape[0] == ref.n_recv(j)
        for k in range(B):
            for i in range(W):
                a, b, n = ref.recv[j, k, i], ref.staged[j, i, k], cnt[i, k, j]
                rows = staged[b:b + n]
                assert np.array_equal(rows[:, 0:2].view(np.uint32), got["means2D"][a:a + n].view(np.uint32))
                assert np.array_equal(rows[:, 2:5].view(np.uint32), got["rgb"][a:a + n].view(np.uint32))
                assert np.array_equal(rows[:, 5:9].view(np.uint32), got["conic_opacity"][a:a + n].view(np.uint32))
                assert np.array_equal(rows[:, 9].astype(np.int32), got["radii"][a:a + n])
                assert np.array_equal(rows[:, 10].view(np.uint32), got["depths"][a:a + n].view(np.uint32))
    grads = [{f: np.full((ref.n_recv(j), xr.WIDTH[f]), 1.0 + j, np.float32) for f in xr.GRAD_FIELDS} for j in range(W)]
    back = xr.backward(hits, grads, ref)
    for i, h in enumerate(hits):
        reached = (h * (1.0 + np.arange(W))).sum(axis=2)          # sum of (1 + j) over the destinations j
        for f in xr.GRAD_FIELDS:
            assert np.array_equal(back[i][f], np.repeat(reached[:, :, None], xr.WIDTH[f], axis=2).astype(np.float32))
    assert sum(int(h.sum()) for h in hits) > 0
