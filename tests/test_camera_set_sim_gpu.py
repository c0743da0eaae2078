"""-m gpu: the load balancer over a camera set, two ranks simulated in one process on one GPU (tests/camera_set_sim.py):
every rank renders its strips of each batch with the real render kernels, forward and backward, and the measured render
times drive the Trainers' own feedback bookkeeping.  A camera's division must move only from the times measured on the
steps it was in, applied feedback_lag steps later -- also when it is absent from the batch that feedback arrives with."""
import pytest
import torch

from camera_set_sim import SimRanks, run_and_check
from gs_b200 import division, ops, pipeline
from gs_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BIG_W, BIG_H = 1936, 1088   # large enough that the reference re-estimates row costs for every batch size


def test_each_camera_moves_only_from_its_own_gathered_render_times():
    cams = [syn.make_camera(BIG_W, BIG_H, yaw_deg=12.0 * k - 30.0, uid=7 + k) for k in range(6)]
    uid_to_cam = {c["uid"]: k for k, c in enumerate(cams)}
    params = pipeline.GaussianParams(syn.make_scene(200_000, BIG_W, BIG_H, seed=4), DEV)
    dcams = [pipeline.DeviceCamera(c, DEV) for c in cams]
    with torch.no_grad():
        proj = [ops.preprocess_gaussians_raw(params._xyz, params._features_dc, params._features_rest, params._scaling,
                                             params._rotation, params._opacity, d.settings()) for d in dcams]
    tile_x = (BIG_W + 15) // 16

    def render_times(rank, k, st):
        """Render this rank's strip of the camera, forward and backward; the time the reference charges for it."""
        cam = uid_to_cam[st.camera_uid]
        m2, rgb, co, radii, depths = (t.detach() for t in proj[cam])
        m2, rgb, co = (t.clone().requires_grad_(True) for t in (m2, rgb, co))
        coll = {}
        image, *_ = ops.render_gaussians(m2, co, rgb, depths, radii, st.get_compute_locally(tile_x, DEV),
                                         dcams[cam].settings(), {"stats_collector": coll})
        image.sum().backward()
        return division.running_time_of(coll)

    for _ in range(2):   # warm the render kernels and the allocator
        render_times(0, 0, division.DivisionStrategy(cams[0]["uid"], [0], [0, (BIG_H + 15) // 16], (BIG_H + 15) // 16, 0))
    schedule = [[0], [3, 1], [5], [1, 0, 2], [4], [2], [0, 5], [3], [2, 4]]
    lag = 2
    sim = SimRanks(cams, world=2, feedback_lag=lag)
    untouched = run_and_check(sim, cams, schedule, render_times, lag)
    measured = {cams[i]["uid"] for v in schedule[:len(schedule) - lag] for i in v}
    assert untouched == {c["uid"] for c in cams} - measured
    # real times are never uniform over the rows: every measured camera's heuristic left the uniform start
    ones = torch.ones((BIG_H + 15) // 16)
    for uid in measured:
        assert not torch.equal(sim.trs[0].history.accum_heuristic[uid], ones), uid
