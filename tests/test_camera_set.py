"""CPU checks of training over a camera set: the Trainer's view validation, its strip-division cache keyed by the batch's
camera uids, the timing feedback landing on the cameras of the step it was measured on (ranks simulated in one process,
tests/camera_set_sim.py), and the C-ABI refusals of the in-place ground-truth loss in a process that sees no device."""
import os
import subprocess
import sys

import pytest
import torch

from camera_set_sim import SimRanks, run_and_check
from gs_b200 import pipeline
from gs_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# 1088 x 1936: above the size where the reference stops re-estimating row costs for batches of >= world-size views
BIG_W, BIG_H = 1936, 1088


def cams_of(n, w=96, h=64):
    return [syn.make_camera(w, h, yaw_deg=3.0 * k, uid=40 + k) for k in range(n)]


def cpu_trainer(cams, **kw):
    return pipeline.Trainer(syn.make_scene(8, cams[0]["image_width"], cams[0]["image_height"], seed=0), cams, None,
                            "cpu", **kw)


def test_view_validation():
    tr = cpu_trainer(cams_of(5))
    assert tr._batch_views(None) == (0, 1, 2, 3, 4)
    assert tr._batch_views([3, 1, 3]) == (3, 1, 3)
    assert tr._batch_views(torch.tensor([4, 0])) == (4, 0)
    for bad in ([5], [-1], [], [0] * 65):
        with pytest.raises(ValueError):
            tr._batch_views(bad)
    for bad in ([1.0], ["1"], [None]):
        with pytest.raises(TypeError):
            tr._batch_views(bad)
    with pytest.raises(ValueError, match="one image size"):
        cpu_trainer([syn.make_camera(96, 64, uid=0), syn.make_camera(96, 80, uid=1)])
    with pytest.raises(ValueError, match="ground-truth images"):
        pipeline.Trainer(syn.make_scene(8, 96, 64), cams_of(2), [torch.zeros((3, 64, 96), dtype=torch.uint8)], "cpu")


def test_camera_table_rows_follow_the_views():
    cams = cams_of(6)
    tr = cpu_trainer(cams)
    full = pipeline.ops.pack_cameras([c.settings() for c in tr.dcams])
    assert torch.equal(tr._cam_rows, full)
    sub = pipeline.ops.pack_cameras([tr.dcams[i].settings() for i in (4, 1)])
    assert torch.equal(tr._cam_rows[[4, 1]], sub)


def test_strategy_cache_is_keyed_by_uids():
    sim = SimRanks(cams_of(6, BIG_W, BIG_H), world=2)
    tr = sim.trs[1]
    a = tr._batch_strategies((40, 41))
    assert [s.camera_uid for s in a] == [40, 41]
    assert tr._batch_strategies((40, 41)) is a              # same batch, same history version: cached
    b = tr._batch_strategies((41, 40))
    assert b is not a and [s.camera_uid for s in b] == [41, 40]
    masks = {("geometry",): 1}
    tr._bmask_cache.update(masks)
    tr._batch_strategies((45,))                               # another batch: the division-keyed caches stay
    assert tr._bmask_cache == masks and len(tr.balance_log) == 1


@pytest.mark.parametrize("lag", [2, 1])
def test_feedback_passed_by_value_updates_the_cameras_it_was_measured_on(lag):
    """Each camera's cost heuristic -- and so its division -- changes only from the times measured on the steps it was
    in, applied `lag` steps later, also when it is absent from the batch the feedback arrives with."""
    cams = cams_of(6, BIG_W, BIG_H)
    sim = SimRanks(cams, world=2, feedback_lag=lag)
    schedule = [[0], [3, 1], [5], [1, 0, 2], [4], [2], [0, 5], [3]]

    def render_times(rank, k, st):   # a cost that differs per camera, rank and strip height
        lo, hi = st.local_rows()
        return 0.25 * (st.camera_uid - 39) * (hi - lo) * (1 + rank) + 0.5

    untouched = run_and_check(sim, cams, schedule, render_times, lag)
    assert untouched == {c["uid"] for c in cams} - {cams[i]["uid"] for v in schedule[:len(schedule) - lag] for i in v}


REFUSALS = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from gs_b200 import _lib
lib = _lib.load()
H, W = 64, 96
fake = 1 << 20                     # never dereferenced: every call below is refused first
def rows(*r):
    return (C.c_int32 * (4 * len(r)))(*[v for q in r for v in q])
def ptrs(*p):
    return (C.c_void_p * len(p))(*p)
good = rows((0, 32, 0, 32), (32, H, 32, H))
cases = [
    ("misaligned", good, ptrs(fake, fake + 1)),
    ("null", good, ptrs(fake, None)),
    ("past H", rows((0, 32, 0, 32), (32, H + 1, 32, H)), ptrs(fake, fake)),
    ("negative", rows((-16, 32, 0, 32), (32, H, 32, H)), ptrs(fake, fake)),
    ("reversed", rows((0, 32, 0, 32), (40, 32, 40, 32)), ptrs(fake, fake)),
    ("counts", rows((0, 32, 0, 33), (32, H, 32, H)), ptrs(fake, fake)),
]
for name, r4, gp in cases:
    for f in ("gs_loss_forward_batched_gt_full", "gs_loss_forward_batched_gt_full_det"):
        rc = getattr(lib, f)(2, H, W, r4, fake, gp, fake, fake, 1 << 30, None)
        assert rc == -1, (f, name, rc)
    rc = lib.gs_loss_backward_batched_gt_full(2, H, W, r4, fake, gp, fake, fake, fake, fake, None)
    assert rc == -1, (name, rc)
    assert lib.gs_last_error(), name
print("refused", len(cases))
"""


def test_cabi_refusals_without_a_device():
    from gs_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", REFUSALS, os.path.join(ROOT, "grendel-gs_b200")], capture_output=True,
                       text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "refused 6" in r.stdout
