"""W ranks of a training run over a camera set, simulated in one process: one pipeline.Trainer per rank whose host-side
bookkeeping runs for real -- the strip division of each batch (Trainer._batch_strategies), the timing feedback queued
`feedback_lag` steps (Trainer._feed_back_times) and handed over on the exchange's piggybacked all-gather
(Trainer._feedback_before_exchange / _feedback_after_exchange) -- while the all-gather itself is a host concatenation and
the render times come from the caller.  The Trainers are built for one rank on the CPU (a Trainer for W > 1 opens a
process group) and then told their rank and world size."""
import numpy as np
import torch

from gs_b200 import division, pipeline
from gs_b200 import synthetic as syn


class SimRanks:
    def __init__(self, cams, world, feedback_lag=2):
        self.log = []   # per step: (rank 0's strategies, times[rank][batch camera]) -- -1 where a rank has no strip
        scene = syn.make_scene(8, cams[0]["image_width"], cams[0]["image_height"], seed=0)
        self.world = world
        self.trs = []
        for r in range(world):
            tr = pipeline.Trainer(scene, cams, None, "cpu", feedback_lag=feedback_lag, load_balance=True)
            tr.rank, tr.world = r, world
            tr.history = division.StrategyHistory([c.uid for c in tr.dcams], tr.tile_y, world)
            self.trs.append(tr)

    def step(self, views, render_times):
        """One step over `views`.  render_times(rank, k, strategy) -> ms this rank spent on the strip of batch camera k.
        Returns the strategies every rank used."""
        uids = tuple(self.trs[0].dcams[i].uid for i in views)
        strategies = [tr._batch_strategies(uids) for tr in self.trs]
        # the exchange: every rank hands its piggybacked times in, the all-gather hands all of them out
        ins = [tr._feedback_before_exchange() for tr in self.trs]
        assert all((x is None) == (ins[0] is None) for x in ins)
        gathered = None if ins[0] is None else np.asarray(ins, dtype=np.float32)
        for tr in self.trs:
            tr._feedback_after_exchange(gathered)
        times = []
        for r, (tr, sts) in enumerate(zip(self.trs, strategies)):
            # one batched render per rank: its time is the sum over the rank's strips, in collectors[0]
            t = sum(float(render_times(r, k, st)) for k, st in enumerate(sts) if st.local_rows() is not None)
            collectors = [{} for _ in sts]
            collectors[0] = {"forward_render_time": t, "backward_render_time": 0.0}
            # the times the rank feeds back, as the float32 all-gather carries them
            times.append([float(np.float32(x)) for x in tr._times_of(sts, collectors)])
            tr.iteration += 1
            tr._feed_back_times(sts, collectors)
        self.log.append((strategies[0], times))
        return strategies

    def expected_history(self, n_applied):
        """The cost heuristics after the feedback of the first n_applied steps, applied in step order to the cameras of
        the step each was measured on."""
        tr = self.trs[0]
        h = division.StrategyHistory([c.uid for c in tr.dcams], tr.tile_y, self.world)
        for sts, times in self.log[:n_applied]:
            h.update(sts, times)
        return h


def run_and_check(sim, cams, schedule, render_times, lag):
    """Steps `schedule` and checks, after every step and on every rank, that each camera's cost heuristic is the one its
    own measured steps give, applied `lag` steps later in step order, and that each step's division followed the
    heuristics of its own cameras.  Returns the uids whose division was never fed back (still the uniform split)."""
    untouched = {c["uid"] for c in cams}
    for t, views in enumerate(schedule):
        strategies = sim.step(views, render_times)
        applied = max(0, t + 1 - lag)     # steps whose feedback has arrived by the end of step t
        want = sim.expected_history(applied)
        for tr in sim.trs:
            assert len(tr.history.history) == applied, (t, len(tr.history.history))
            for uid, h in want.accum_heuristic.items():
                assert torch.equal(tr.history.accum_heuristic[uid], h), (t, uid)
        before = sim.expected_history(max(0, t - lag))
        for r in range(sim.world):
            ref = division.start_strategy([cams[i]["uid"] for i in views], before, sim.world, r)[0]
            assert [(s.gpu_ids, s.division_pos) for s in strategies[r]] == [(s.gpu_ids, s.division_pos) for s in ref], t
        for sts, _ in sim.log[:applied]:
            untouched -= {s.camera_uid for s in sts}
    tile_y = sim.trs[0].tile_y
    for uid in untouched:
        for tr in sim.trs:
            assert torch.equal(tr.history.accum_heuristic[uid], torch.ones(tile_y))
    return untouched
