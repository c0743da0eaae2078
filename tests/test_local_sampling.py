"""CPU checks of local sampling (the reference's --local_sampling): the whole-view division against a restatement of
workload_division.py:858-877, every refusal of pipeline.Trainer(local_sampling=True) raised before any collective or
launch (and, over a real gloo group, the construction-time agreement on local_bsz raised on every rank), and ranks
simulated in one process stepping their own views: the load balancer's history is never read or touched and no timing
feedback is queued."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gs_b200 import _lib, division, exchange, pipeline
from gs_b200 import synthetic as syn

TW, TH = 96, 72


def reference_division(B, world, bsz, tile_y):
    """workload_division.py:858-877, restated: (gpu_ids, division_pos) per batch position and gpuid2tasks."""
    gpuid2tasks = [[] for _ in range(world)]
    per_cam = []
    bsz_per_gpu = bsz // world
    for idx in range(B):
        gpu_id = idx // bsz_per_gpu
        gpuid2tasks[gpu_id].append((idx, 0, tile_y))
        per_cam.append(([gpu_id], [0, tile_y]))
    return per_cam, gpuid2tasks


class NoHistory:
    """A StrategyHistory stand-in that only knows TILE_Y: reading its heuristics or updating it fails."""

    def __init__(self, tile_y):
        self.tile_y = tile_y

    def __getattr__(self, name):
        raise AssertionError(f"the whole-view division read StrategyHistory.{name}")


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_whole_view_division_matches_the_reference(world, k):
    B, tile_y = world * k, 17
    want, want_tasks = reference_division(B, world, B, tile_y)
    for rank in range(world):
        for uids in (list(range(B)), [None] * B, [7] * B):   # labels only: the split depends on positions
            for sts, tasks in (division.start_strategy_whole_views(uids, tile_y, world, rank),
                               division.start_strategy(uids, NoHistory(tile_y), world, rank, local_sampling=True)):
                assert [(s.gpu_ids, s.division_pos) for s in sts] == want
                assert tasks == want_tasks
                assert [s.camera_uid for s in sts] == uids
                for p, s in enumerate(sts):
                    mine = p // k == rank
                    assert s.local_rows() == ((0, tile_y) if mine else None)
                    assert s.local_pixel_rows(16 * tile_y - 5) == ((0, 16 * tile_y - 5) if mine else None)


@pytest.mark.parametrize("world,B", [(2, 3), (4, 6), (8, 4), (3, 1)])
def test_whole_view_division_refuses_uneven_batches(world, B):
    with pytest.raises(ValueError, match="divisible"):
        division.start_strategy_whole_views(list(range(B)), 10, world, 0)


def cams_of(n):
    return [syn.make_camera(TW, TH, yaw_deg=3.0 * q, uid=q) for q in range(n)]


def images_held(n, world, rank):
    """--distributed_dataset_storage with local sampling (scene/cameras.py:52-59): a rank holds camera uid when
    uid % world == rank."""
    return [torch.from_numpy(syn.make_gt_image(TW, TH, seed=q)) if q % world == rank else None for q in range(n)]


def local_trainer(cams, gts, local_bsz, **kw):
    return pipeline.Trainer(syn.make_scene(8, TW, TH, seed=0), cams, gts, "cpu", local_sampling=True,
                            local_bsz=local_bsz, **kw)


class Forbidden(Exception):
    pass


@pytest.fixture
def no_collective_or_launch(monkeypatch):
    """Any collective, library call or CUDA stream use raises Forbidden: a refusal must come first."""
    def forbid(*_a, **_k):
        raise Forbidden()
    for name in ("all_gather_into_tensor", "all_gather", "all_reduce", "all_to_all_single", "broadcast"):
        monkeypatch.setattr(dist, name, forbid)
    monkeypatch.setattr(_lib, "call", forbid)
    monkeypatch.setattr(torch.cuda, "current_stream", forbid)


def test_refusals_before_any_collective_or_launch(no_collective_or_launch):
    cams = cams_of(6)
    gts = images_held(6, 1, 0)
    bad_args = [dict(local_bsz=None), dict(local_bsz=0), dict(local_bsz=-2), dict(local_bsz=1.5), dict(local_bsz="2"),
                dict(local_bsz=65), dict(local_bsz=2, distributed_dataset_storage=True),
                dict(local_bsz=2, border_exchange=True)]
    for kw in bad_args:
        with pytest.raises(ValueError):
            local_trainer(cams, gts, **kw)
    with pytest.raises(ValueError, match="hold no training image"):
        local_trainer(cams, None, 2)
    with pytest.raises(ValueError, match="hold no training image"):
        local_trainer(cams, [None] * 6, 2)
    tr = local_trainer(cams, gts, 64)   # 64 views: the batched kernels' limit
    assert tr.local_bsz == 64
    # a rank of three: holds cameras 1 and 4
    tr = local_trainer(cams, images_held(6, 3, 1), 2)
    assert tr.gts_dev[1] is not None and tr.gts_dev[4] is not None
    assert [q for q, g in enumerate(tr.gts_dev) if g is None] == [0, 2, 3, 5]
    tr.rank, tr.world = 1, 3
    for views in (None, [1], [1, 4, 4], [1, 0], [3, 4], [6, 1], [-1, 1], []):
        with pytest.raises(ValueError):
            tr.step(views=views)
    for views in ([1.0, 4], ["1", 4]):
        with pytest.raises(TypeError):
            tr.step(views=views)
    with pytest.raises(Forbidden):   # accepted views reach the device
        tr.step(views=[4, 1])
    assert tr._local_views([4, 4]) == (4, 4)
    assert tr.iteration == 0


def test_default_trainer_keeps_its_views():
    """local_sampling=False: views=None is still every camera, and a None image is not accepted as 'not held'."""
    tr = pipeline.Trainer(syn.make_scene(8, TW, TH, seed=0), cams_of(3), None, "cpu")
    assert not tr.local_sampling and tr.local_bsz is None and tr._cam_table_dev is None
    assert tr._batch_views(None) == (0, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# the agreement on local_bsz over a real gloo group
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _agreement_worker(rank, world, port, case, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    calls = []
    real = dist.all_gather_into_tensor

    def counted(*a, **k):
        calls.append(1)
        return real(*a, **k)
    dist.all_gather_into_tensor = counted
    n = 8
    gts = images_held(n, world, rank)
    kw = dict(peer_exchange=False, load_balance=False)
    if case == "mismatch":
        k = 1 + (rank == world - 1)
    elif case == "too_many":
        k = 64 // world + 1
    elif case == "exchange_limit":
        k = exchange.MAX_CAMERAS // world + 1
    elif case == "bad_on_one_rank":
        k = 0 if rank == 1 else 2
    elif case == "no_images":
        k = 1
        gts = [None] * n if rank == 0 else gts
    else:
        k = 2
    try:
        tr = pipeline.Trainer(syn.make_scene(8 * world, TW, TH, seed=0), cams_of(n), gts, "cpu", rank, world,
                              local_sampling=True, local_bsz=k, **kw)
        res = ("ok", tr.local_bsz, tr.rank, tr.world)
    except ValueError as e:
        res = ("refused", str(e))
    q.put((rank, res, len(calls)))
    dist.all_gather_into_tensor = real
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("case", ["agree", "mismatch", "too_many", "exchange_limit", "bad_on_one_rank", "no_images"])
def test_local_bsz_agreement_over_gloo(case):
    world = 2 if case != "mismatch" else 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_agreement_worker, args=(r, world, port, case, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert all(n == 1 for _, _, n in res), res          # one all-gather, then every rank decides the same
    if case == "agree":
        assert [r[1] for r in res] == [("ok", 2, r, world) for r in range(world)]
        return
    assert all(r[1][0] == "refused" for r in res), res
    assert len({r[1][1] for r in res}) == 1, res         # the same message on every rank
    if case == "mismatch":
        assert "[1, 1, 2]" in res[0][1][1]


# ---------------------------------------------------------------------------------------------------------------------
# ranks simulated in one process: the load balancer is out of the loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_load_balancer(monkeypatch):
    def forbid(*_a, **_k):
        raise AssertionError("a local-sampling step reached the load balancer")
    monkeypatch.setattr(division.StrategyHistory, "update", forbid)
    for mod in (division, pipeline):
        monkeypatch.setattr(mod, "finish_strategy", forbid)
        monkeypatch.setattr(mod, "start_strategy", forbid)
    for name in ("_batch_strategies", "_feed_back_times", "_feedback_before_exchange", "_feedback_after_exchange",
                 "_times_of"):
        monkeypatch.setattr(pipeline.Trainer, name, forbid)


@pytest.mark.parametrize("world,k", [(2, 2), (4, 1), (3, 3)])
def test_simulated_ranks_never_touch_the_history_or_send_feedback(no_load_balancer, world, k):
    n = 12
    cams = cams_of(n)
    trs = []
    for r in range(world):
        # load_balance=True, feedback_lag=1: what would queue and apply timing feedback on the default path
        tr = local_trainer(cams, images_held(n, world, r), k, load_balance=True, feedback_lag=1)
        tr.rank, tr.world = r, world
        trs.append(tr)
    start = {uid: h.clone() for uid, h in trs[0].history.accum_heuristic.items()}
    full = pipeline.ops.pack_cameras([c.settings() for c in trs[0].dcams])
    rng = np.random.default_rng(world * 10 + k)
    for it in range(6):
        mine = [tuple(int(v) for v in rng.choice(np.arange(r, n, world), size=k)) for r in range(world)]
        union = torch.tensor([v for m in mine for v in m], dtype=torch.int64)   # the all-gather, in rank order
        for r, tr in enumerate(trs):
            assert tr._local_views(list(mine[r])) == mine[r]
            sts, _cam_table, span, feedback = tr._step_plan(mine[r])
            assert sts is tr._whole_view_division()                      # built once
            assert span == (r * k, (r + 1) * k) and not feedback          # its own positions, no timing feedback
            # each position is rendered whole by the rank that sampled it and holds its image
            for p, st in enumerate(sts):
                owner = p // k
                assert st.gpu_ids == [owner] and st.division_pos == [0, tr.tile_y]
                assert tr.gts_host[int(union[p])] is not None if owner == r else True
            table = torch.index_select(tr._cam_table_dev, 0, union)       # the device-side gather, on the CPU
            assert torch.equal(table, full[union]) and torch.equal(table, tr._cam_rows[union])
            tr._finish_step(sts, [{} for _ in range(k)], dict(Vp=0, P_local=k * TH * TW), feedback)
            assert tr._sent_feedback is None and tr._pending_feedback == []
    for tr in trs:
        assert tr.iteration == 6
        assert tr.history.history == [] and tr.balance_log == [] and tr._pending_feedback == []
        assert all(torch.equal(tr.history.accum_heuristic[uid], h) for uid, h in start.items())
