"""CPU tests of the host-side logic: workload division (single process) and the all-to-all layout
over a real 2-rank gloo group (the N>1 path of bench.py / pipeline.Trainer, minus the CUDA kernels)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gs_b200 import division, exchange


# ---------------------------------------------------------------------------------------------------
# division (restates /root/reference/gaussian_renderer/workload_division.py:75-94,852-941)
# ---------------------------------------------------------------------------------------------------
def test_division_pos_uniform_matches_reference_example():
    # SURVEY.md 8a/A8: TILE_Y=68 over 4 ranks -> [0,17,34,51,68]; 67 rows -> [0,16,33,50,67]
    assert division.division_pos_heuristic(torch.ones(68), 4) == [0, 17, 34, 51, 68]
    assert division.division_pos_heuristic(torch.ones(67), 4) == [0, 16, 33, 50, 67]


def test_division_weighted_costs_shift_boundaries():
    h = torch.ones(40)
    h[:10] = 5.0  # top rows are expensive
    pos = division.division_pos_heuristic(h, 2)
    assert pos[0] == 0 and pos[-1] == 40 and pos[1] < 20


@pytest.mark.parametrize("world,bsz,tile_y", [(1, 1, 68), (2, 1, 68), (4, 4, 68), (8, 8, 135), (4, 1, 67), (8, 2, 135), (2, 4, 25)])
def test_start_strategy_partitions_every_row_exactly_once(world, bsz, tile_y):
    uids = list(range(bsz))
    hist = division.StrategyHistory(uids, tile_y, world)
    per_rank = []
    for rank in range(world):
        strategies, tasks = division.start_strategy(uids, hist, world, rank)
        per_rank.append((strategies, tasks))
    s0, t0 = per_rank[0]
    for strategies, tasks in per_rank:  # every rank derives the same plan
        assert [s.division_pos for s in strategies] == [s.division_pos for s in s0]
        assert tasks == t0
    for k, s in enumerate(s0):
        assert s.division_pos[0] == 0 and s.division_pos[-1] == tile_y
        assert len(s.gpu_ids) == len(s.division_pos) - 1
    covered = np.zeros((bsz, tile_y), int)
    for gpu, tl in enumerate(t0):
        assert tl, f"rank {gpu} got no work"
        for (k, lo, hi) in tl:
            covered[k, lo:hi] += 1
    assert (covered == 1).all()
    # ranks own contiguous runs of the concatenated rows, in rank order
    flat = [(k * tile_y + lo, k * tile_y + hi) for tl in t0 for (k, lo, hi) in tl]
    assert all(a[1] == b[0] for a, b in zip(flat, flat[1:]))


def test_strategy_masks_and_pixel_rows():
    hist = division.StrategyHistory([0], 68, 4)
    strategies, _ = division.start_strategy([0], hist, 4, 2)
    s = strategies[0]
    assert s.rank == 2 and s.local_rows() == (34, 51)
    m = s.get_compute_locally(120, "cpu")
    assert m.shape == (68, 120) and m[34:51].all() and not m[:34].any() and not m[51:].any()
    assert s.local_pixel_rows(1080) == (34 * 16, 51 * 16)
    assert strategies[0].strategy_tensor(120, "cpu").tolist() == [0, 17 * 120, 34 * 120, 51 * 120, 68 * 120]
    last = division.start_strategy([0], hist, 4, 3)[0][0]
    assert last.local_pixel_rows(1080) == (51 * 16, 1080)  # last strip is clipped to the image


def test_history_update_rebalances():
    hist = division.StrategyHistory([7], 64, 2)
    strategies, _ = division.start_strategy([7], hist, 2, 0)
    assert strategies[0].division_pos == [0, 32, 64]
    hist.update(strategies, [[30.0], [10.0]])  # rank 0 took 3x longer
    s2, _ = division.start_strategy([7], hist, 2, 0)
    assert s2[0].division_pos[1] < 32


def test_finish_strategy_gate_follows_the_reference():
    """workload_division.py:967-978: no re-estimation during warm-up, on one rank, when every rank can take whole images
    of at most 1080p, or for small images; otherwise the measured times move the boundaries."""
    en = division.heuristics_update_enabled
    assert not en(iteration=5, world_size=4, bsz=1, image_height=2160, image_width=3840, adjust_strategy_warmup_iterations=10)
    assert not en(iteration=50, world_size=1, bsz=1, image_height=2160, image_width=3840)
    assert not en(iteration=50, world_size=4, bsz=1, image_height=2160, image_width=3840, no_heuristics_update=True)
    assert not en(iteration=50, world_size=4, bsz=4, image_height=1080, image_width=1920)      # the bench configuration
    assert not en(iteration=50, world_size=4, bsz=1, image_height=600, image_width=800)
    assert en(iteration=50, world_size=4, bsz=1, image_height=1080, image_width=1920)          # one image over 4 ranks
    assert en(iteration=50, world_size=8, bsz=8, image_height=2160, image_width=3840)          # config c4
    assert division.running_time_of({"forward_render_time": 1.0, "backward_render_time": 2.0, "forward_loss_time": 0.5}) == 4.0
    hist = division.StrategyHistory([3], 135, 2)
    st, _ = division.start_strategy([3], hist, 2, 0)
    assert not division.finish_strategy(hist, st, [[9.0], [3.0]], iteration=1, world_size=2, image_height=1080,
                                        image_width=1920, adjust_strategy_warmup_iterations=5)
    assert division.start_strategy([3], hist, 2, 0)[0][0].division_pos == st[0].division_pos
    assert division.finish_strategy(hist, st, [[9.0], [3.0]], iteration=9, world_size=2, image_height=2160, image_width=3840)
    assert division.start_strategy([3], hist, 2, 0)[0][0].division_pos[1] < st[0].division_pos[1]


def test_feedback_loop_balances_an_uneven_scene():
    """The loop Trainer.step closes (start_strategy -> measured times -> finish_strategy): with a fixed, uneven true
    cost per tile row (the lower third of the image 5x as expensive), the strips move until every rank's time is
    within ~one row of the mean, and stay there."""
    world, tile_y = 4, 135
    true = np.ones(tile_y); true[90:] = 5.0
    hist = division.StrategyHistory([0], tile_y, world)
    spread = []
    for it in range(1, 12):
        st, _ = division.start_strategy([0], hist, world, 0)
        pos = st[0].division_pos
        t = [[float(true[pos[g]:pos[g + 1]].sum())] for g in range(world)]
        spread.append(max(x[0] for x in t) / (sum(x[0] for x in t) / world))
        assert division.finish_strategy(hist, st, t, iteration=it, world_size=world, image_height=2160, image_width=3840)
    assert spread[0] > 2.0                      # uniform strips: the rank with the expensive rows takes > 2x the mean
    assert max(spread[3:]) < 1.1, spread        # balanced after a few iterations (one 5x row = 0.06 of a rank's share)


def test_local_sampling_gives_whole_images():
    hist = division.StrategyHistory([0, 1, 2, 3], 30, 2)
    strategies, tasks = division.start_strategy([0, 1, 2, 3], hist, 2, 1, local_sampling=True)
    assert [s.gpu_ids for s in strategies] == [[0], [0], [1], [1]]
    assert tasks[1] == [(2, 0, 30), (3, 0, 30)]


def test_invalid_division_is_rejected():
    with pytest.raises(ValueError):
        division.DivisionStrategy(0, [0, 1], [0, 10], 20, 0)
    with pytest.raises(ValueError):
        division.DivisionStrategy(0, [0, 1], [0, 12, 12], 12, 0)


# ---------------------------------------------------------------------------------------------------
# exchange layout over gloo, world_size = 2 and 3
# ---------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_data(rank, B, P, world, gpu_ids):
    g = torch.Generator().manual_seed(1000 + rank)
    rows = [torch.rand((P, exchange.ROW), generator=g) + 10 * rank + 100 * k for k in range(B)]
    masks = [torch.rand((P, len(gpu_ids[k])), generator=g) < 0.3 for k in range(B)]
    return rows, masks


def _worker(rank, world, port, B, P, tile_y, q):
    try:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        uids = list(range(B))
        hist = division.StrategyHistory(uids, tile_y, world)
        strategies, _ = division.start_strategy(uids, hist, world, rank)
        gpu_ids = [s.gpu_ids for s in strategies]
        rows, masks = _rank_data(rank, B, P, world, gpu_ids)
        local_counts = torch.zeros((B, world), dtype=torch.int32)
        for k in range(B):
            local_counts[k, torch.tensor(gpu_ids[k])] = masks[k].sum(0).to(torch.int32)
        # the timing feedback rides on the size all-gather (gather_counts(times=...)): every rank gets every rank's row
        cnt, fb = exchange.gather_counts(local_counts, times=[rank + 0.5] + [-1.0] * (B - 1))
        assert fb is not None and fb.shape == (world, B)
        assert fb[:, 0].tolist() == [r + 0.5 for r in range(world)] and (fb[:, 1:] == -1.0).all()
        cnt_again, fb = exchange.gather_counts(local_counts)
        assert cnt_again.tolist() == cnt.tolist() and fb is None
        lay = exchange.Layout(cnt, rank, gpu_ids)
        # torch emulation of gs_pack_rows
        send = torch.full((lay.total_send, exchange.ROW), -1.0)
        for k in range(B):
            for c in range(len(gpu_ids[k])):
                sel = rows[k][masks[k][:, c]]
                send[lay.dst_off[k][c]:lay.dst_off[k][c] + sel.shape[0]] = sel
        assert (send >= 0).all()
        recv = torch.empty((lay.total_recv, exchange.ROW))
        exchange.all_to_all_single(recv, send, lay.recv_splits, lay.send_splits)
        # torch emulation of gs_unpack_rows + the expected answer recomputed from every source's seed
        for k in range(B):
            got = torch.cat([recv[o:o + l] for o, l in zip(lay.seg_off[k], lay.seg_len[k])]) if lay.n_recv[k] else recv[:0]
            exp = []
            for src in range(world):
                r_src, m_src = _rank_data(src, B, P, world, gpu_ids)
                if rank in gpu_ids[k]:
                    exp.append(r_src[k][m_src[k][:, gpu_ids[k].index(rank)]])
            exp = torch.cat(exp) if exp else recv[:0]
            assert torch.equal(got, exp), f"camera {k}"
        # backward: gradient rows travel the reverse route and are summed per local splat
        grecv = torch.zeros((lay.total_recv, exchange.GROW))
        for k in range(B):
            n = lay.n_recv[k]
            g = torch.arange(n, dtype=torch.float32)[:, None] + torch.arange(exchange.GROW)[None] * 0.001 + 1000 * rank + 10000 * k
            o2 = 0
            for o, l in zip(lay.seg_off[k], lay.seg_len[k]):
                grecv[o:o + l] = g[o2:o2 + l]
                o2 += l
        gsend = torch.empty((lay.total_send, exchange.GROW))
        exchange.all_to_all_single(gsend, grecv, lay.send_splits, lay.recv_splits)
        for k in range(B):
            acc = torch.zeros((P, exchange.GROW))
            for c, dest in enumerate(gpu_ids[k]):
                idx = masks[k][:, c].nonzero().squeeze(1)
                acc[idx] += gsend[lay.dst_off[k][c]:lay.dst_off[k][c] + idx.numel()]
                # what `dest` must have assigned to these rows: its camera-k rows from source `rank` start after
                # the rows it received from lower ranks
                before = sum(cnt[i][k][dest] for i in range(rank))
                exp = (before + torch.arange(idx.numel(), dtype=torch.float32))[:, None] + torch.arange(exchange.GROW)[None] * 0.001 + 1000 * dest + 10000 * k
                assert torch.allclose(gsend[lay.dst_off[k][c]:lay.dst_off[k][c] + idx.numel()], exp)
            assert (acc[~masks[k].any(1)] == 0).all()
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
        raise


@pytest.mark.parametrize("world,B,tile_y", [(2, 1, 68), (2, 2, 25), (3, 4, 40)])
def test_exchange_layout_and_gathered_times_over_gloo(world, B, tile_y):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, B, 257, tile_y, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] == "ok" for r in res), res


def test_layout_is_consistent_without_a_group():
    rng = np.random.default_rng(0)
    W, B = 4, 3
    gpu_ids = [[0, 1], [1, 2, 3], [3]]
    cnt = np.zeros((W, B, W), int)
    for i in range(W):
        for k in range(B):
            for j in gpu_ids[k]:
                cnt[i, k, j] = rng.integers(0, 50)
    cnt = cnt.tolist()
    lays = [exchange.Layout(cnt, me, gpu_ids) for me in range(W)]
    for a in range(W):
        for b in range(W):
            assert lays[a].send_splits[b] == lays[b].recv_splits[a]
        assert lays[a].total_recv == sum(lays[a].n_recv)
        # send offsets tile the send buffer without gaps
        spans = sorted((lays[a].dst_off[k][c], cnt[a][k][j]) for k in range(B) for c, j in enumerate(gpu_ids[k]))
        pos = 0
        for off, n in spans:
            assert off == pos or n == 0
            pos = max(pos, off + n)
        assert pos == lays[a].total_send


class _Pinned(torch.Tensor):
    """A pinned host image, without a driver to pin it."""
    def is_pinned(self, *args, **kwargs):
        return True


class _Pageable(torch.Tensor):
    """A pageable host image; pin_memory() needs a driver, so the strip cache's pinned copy is a plain copy here."""
    def pin_memory(self, *args, **kwargs):
        return self.clone()


class _OnDevice(torch.Tensor):
    """An image already on the step's device."""
    is_cuda = property(lambda self: True)


def _gt_scatter_worker(rank, world, port, q):
    import torch.distributed as dist
    from gs_b200 import gt_scatter
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    H, W, B, tile_y = 100, 40, 3, 7
    gts = [torch.from_numpy(np.random.default_rng(k).integers(0, 256, (3, H, W), dtype=np.uint8)) for k in range(B)]
    hist = division.StrategyHistory(list(range(B)), tile_y, world)
    strategies, tasks = division.start_strategy(list(range(B)), hist, world, rank)
    got, h2d = gt_scatter.scatter_gt_strips(gts if rank == 0 else W, tasks, H, "cpu", rank, world)
    ok = set(got) == {t[0] for t in tasks[rank]} and gt_scatter.strip_tasks(strategies, world) == tasks
    for cam, l, r in tasks[rank]:
        y0, y1 = l * 16, min(r * 16, H)
        ok = ok and torch.equal(got[cam], gts[cam][:, y0:y1, :])

    # local_gt: batch position k is camera views[k]; every source gives its local rows [y0, y1) at the expected row0
    views = [2, 0, 1]
    local = {k: st.local_pixel_rows(H) for k, st in enumerate(strategies) if st.local_rows() is not None}
    strip_bytes = sum(3 * (y1 - y0) * W for y0, y1 in local.values())

    def same(pairs, in_place):
        good = len(pairs) == B and all(pairs[k] is None for k in range(B) if k not in local)
        for k, (y0, y1) in local.items():
            t, row0 = pairs[k]
            want = gts[views[k]][:, y0:y1, :]
            good = good and row0 == (0 if in_place else y0) and torch.equal(t[:, y0 - row0:y1 - row0, :], want)
            good = good and (t is images[views[k]] if in_place else tuple(t.shape) == tuple(want.shape))
        return good

    for source in ("scatter", "pinned", "pageable", "held-out", "in place"):
        cache = None if source == "held-out" else {}
        cls = {"pinned": _Pinned, "pageable": _Pageable, "in place": _OnDevice}.get(source)
        images = [g if cls is None else g.as_subclass(cls) for g in gts]
        if source == "scatter" and rank != 0:
            images = None
        pairs, n, ready = gt_scatter.local_gt(images, views, strategies, H, W, "cpu", rank, world,
                                              scatter=source == "scatter", cache=cache)
        ok = ok and ready is None and same(pairs, source == "in place")
        if source == "scatter":
            ok = ok and n == (h2d if rank == 0 else 0)
        else:
            ok = ok and n == (0 if source == "in place" else strip_bytes)
        if source == "pageable":   # the own set's pageable strips stay cached, keyed by camera and rows
            ok = ok and set(cache) == {(views[k], y0, y1) for k, (y0, y1) in local.items()}
        elif cache is not None:
            ok = ok and cache == {}
    q.put((rank, bool(ok), h2d))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gt_strips_scattered_from_rank0_match_the_local_slices(world):
    """loss_distribution.py:2395-2533 with --distributed_dataset_storage: only rank 0 holds pixels; every rank ends up
    with exactly the uint8 rows of its strips (3 cameras over 2 / 3 ranks: strips that start and end mid-image).
    gt_scatter.local_gt, which every training step and evaluation reads its ground truth through, gives each batch
    position's strip rows from each source -- the scatter, pinned and pageable host images (the latter through the
    strip cache, held-out ones without it) and images on the device read in place -- with the expected first row."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29650 + world
    procs = [ctx.Process(target=_gt_scatter_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res), res
    assert res[0][2] > 0 and all(h == 0 for _, _, h in res[1:])      # only rank 0 copied from the host


def _redistribute_worker(rank, world, port, q):
    import torch.distributed as dist
    from gs_b200 import redistribute as rd
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    P = 50 + 37 * rank                                   # uneven shards
    g = torch.Generator().manual_seed(100 + rank)
    shapes = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
    params = {k: torch.nn.Parameter(torch.randn((P,) + s, generator=g)) for k, s in shapes.items()}
    opt = torch.optim.Adam([{"params": [params[k]], "lr": 1e-3, "name": k} for k in rd.NAMES], lr=0.0, eps=1e-15)
    for k in rd.NAMES:
        params[k].grad = torch.randn(params[k].shape, generator=g)
    opt.step()
    before = {k: (params[k].detach().clone(), opt.state[params[k]]["exp_avg"].clone(), opt.state[params[k]]["exp_avg_sq"].clone())
              for k in rd.NAMES}
    dest = torch.randint(0, world, (P,), generator=g)
    need, counts = rd.need_redistribute(P, threshold=1.2)
    res = rd.redistribute(opt, dest)
    # what the reference builds, tensor by tensor: cat over sources i of state_i[destination_i == me]  (:1073-1098)
    gathered = {}
    for k in rd.NAMES:
        for q_, t in enumerate(before[k]):
            mine = [t[dest == j].contiguous() for j in range(world)]
            outs = [None] * world
            dist.all_gather_object(outs, mine)
            gathered[(k, q_)] = torch.cat([outs[i][rank] for i in range(world)], dim=0)
    ok = True
    for k in rd.NAMES:
        p_new = opt.param_groups[rd.NAMES.index(k)]["params"][0]
        st = opt.state[p_new]
        ok = ok and p_new is res[k] and p_new.requires_grad and torch.equal(p_new.detach(), gathered[(k, 0)])
        ok = ok and torch.equal(st["exp_avg"], gathered[(k, 1)]) and torch.equal(st["exp_avg_sq"], gathered[(k, 2)])
        ok = ok and float(st["step"]) == 1.0
    n_new = res["xyz"].shape[0]
    ok = ok and n_new == sum(row[rank] for row in res["counts"]) and res["send_to_gpui_cnt"].shape == (n_new, world)
    for k in rd.NAMES:                                   # the optimizer keeps working on the moved tensors
        res[k].grad = torch.ones_like(res[k])
    opt.step()
    q.put((rank, bool(ok), bool(need), counts, n_new))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_redistribution_in_one_collective_matches_the_reference_tensor_by_tensor(world):
    """scene/gaussian_model.py:1073-1098 + :1262-1329: the fused-row all-to-all reproduces, row for row, the eighteen
    per-tensor exchanges (parameters and Adam moments stay attached to their Gaussian; counts add up)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + world
    procs = [ctx.Process(target=_redistribute_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _, _, _ in res), res
    assert all(need for _, _, need, _, _ in res)                       # 50 * 1.2 < 87: uneven enough
    assert sum(n for *_, n in res) == sum(50 + 37 * r for r in range(world))


def test_device_row_formula_equals_direct_rows():
    """k_xr_rows (csrc/distribute.cu) computes the destination rows of the direct pack ON THE DEVICE from the all-gathered
    counts cnt[i][k][j]; its formula, restated here in plain Python, must equal exchange.direct_rows (the host layout the
    gradient pull and the tensor shapes use) for every rank, and its over-capacity flag the host's decision."""
    import numpy as np
    from gs_b200 import exchange
    rng = np.random.default_rng(3)
    for W, B in ((2, 1), (2, 2), (4, 3), (8, 8), (16, 5)):
        cnt = rng.integers(0, 1000, size=(W, B, W)).astype(np.int64)
        cnt[rng.random(cnt.shape) < 0.2] = 0
        flat = cnt.reshape(-1)
        for me in range(W):
            dev = []
            for j in range(W):
                for k in range(B):
                    r = sum(int(flat[(i * B + kk) * W + j]) for kk in range(k) for i in range(W))
                    r += sum(int(flat[(i * B + k) * W + j]) for i in range(me))
                    dev.append(r)
            row0, view_start = exchange.direct_rows(cnt, me)
            assert dev == row0
            assert view_start[-1] == int(cnt[:, :, me].sum())
        totals = cnt.sum(axis=(0, 1))
        cap = int(totals.max())
        assert not any(int(t) > cap for t in totals) and any(int(t) > cap - 1 for t in totals)


def test_quantised_buffer_sizes():
    """ops._q: sizes that follow data-dependent counts are rounded up to at most 1/16 above the count, monotonically, so a
    slowly varying count maps to few distinct allocation sizes."""
    from gs_b200 import ops
    prev = 0
    for n in list(range(0, 5000, 37)) + [10**5, 10**5 + 1, 5_735_587, 84_000_000, 2**31 - 5]:
        q = ops._q(n)
        assert q >= max(n, 1) and q <= max(n, 1) * 1.0626 + 1024
    xs = sorted(set(ops._q(n) for n in range(5_000_000, 6_000_000, 997)))
    assert len(xs) <= 8          # a 20 % range of instance counts -> a handful of sizes
    for a, b in zip(xs, xs[1:]):
        assert b > a


@pytest.mark.parametrize("n", [1, 2, 5])
def test_gaussian_params_sh_blocks_own_aligned_storage(n):
    """The _raw / _batched kernels need 16-byte aligned SH blocks.  With one Gaussian shs[:, 1:, :] is already
    contiguous, so .contiguous() would hand back a view 12 bytes into the SH tensor."""
    from gs_b200 import pipeline, synthetic as syn
    p = pipeline.GaussianParams(syn.make_scene(n, 64, 48, seed=2), "cpu")
    for t in (p._features_dc, p._features_rest):
        assert t.is_contiguous() and t.storage_offset() == 0 and t.data_ptr() % 16 == 0
    assert p._features_dc.untyped_storage().data_ptr() != p._features_rest.untyped_storage().data_ptr()
