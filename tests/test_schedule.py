"""gs_b200.schedule against the reference's own schedule code (tests/golden/schedule.npz, make_schedule_golden.py):

  * check_update_at_this_iter and get_expon_lr_func, value for value;
  * training_setup's groups (lr, eps, betas) and xyz schedule, bit for bit, in every lr_scale_mode;
  * Schedule.begin / end's decisions over whole runs -- statistics, densify and its size threshold, the redistribution
    gate, the memory gate, the opacity reset, the SH step, the optimizer step -- batch for batch, with the device work
    replaced by recorders and the gates' all-gathers answering the golden's recorded per-rank values."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

from gs_b200 import schedule as sc

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "schedule.npz"))
META = json.loads(str(GOLDEN["meta"]))
COLUMNS = [str(c) for c in GOLDEN["columns"]]


def test_check_update_at_this_iter():
    for it, bsz, interval, residual, want in GOLDEN["check_update"].tolist():
        assert sc.check_update_at_this_iter(it, bsz, interval, residual) == bool(want), (it, bsz, interval, residual)


def test_expon_lr():
    steps = GOLDEN["lr_steps"]
    for row in GOLDEN["expon"]:
        a, b, ds, dm, ms = row[:5]
        f = sc.expon_lr(float(a), float(b), lr_delay_steps=int(ds), lr_delay_mult=float(dm), max_steps=int(ms))
        got = np.asarray([float(f(int(s))) for s in steps], dtype=np.float64)
        assert np.array_equal(got.view(np.int64), row[5:].view(np.int64)), (row[:5], got, row[5:])


@pytest.mark.parametrize("q", range(len(META["setups"])))
def test_group_hyperparameters(q):
    s = META["setups"][q]
    opt = sc.OptimizationParams(lr_scale_mode=s["mode"], bsz=s["bsz"], lr_scale_pos_and_scale=s["lr_scale_pos_and_scale"])
    groups, xyz = sc.group_hyperparameters(opt, s["spatial_lr_scale"])
    assert list(groups) == s["names"]
    got = np.asarray([[float(g["lr"]), float(g["eps"]), float(g["betas"][0]), float(g["betas"][1])]
                      for g in groups.values()], dtype=np.float64)
    want = GOLDEN[f"setup{q}_groups"]
    assert np.array_equal(got.view(np.int64), want.view(np.int64)), (s, got, want)
    lrs = np.asarray([float(xyz(int(i))) for i in GOLDEN["lr_steps"]], dtype=np.float64)
    assert np.array_equal(lrs.view(np.int64), GOLDEN[f"setup{q}_xyz_lr"].view(np.int64))


class Recorder(sc.Schedule):
    """The schedule's decisions with every device operation recorded instead of run."""

    def __init__(self, opt, world, counts, peaks, total_gb):
        self._start(opt, world)
        self.trainer = SimpleNamespace(params=SimpleNamespace(active_sh_degree=0, max_sh_degree=10 ** 9), n_local=1)
        self.optimizer = SimpleNamespace(param_groups=[{"name": "xyz", "lr": 0.0}])
        self.xyz_lr = lambda it: 0.0
        self.counts, self.peaks, self.total_gb = counts, peaks, total_gb
        self.used = {"counts": 0, "peaks": 0}
        self.row = {}

    def _add_stats(self):
        self.row["stats"] = 1

    def _densify(self, size_threshold, noise):
        self.row["densify"] = 1
        self.row["size_threshold"] = 0 if size_threshold is None else size_threshold
        return (0, 0, 0, 0, 1)

    def _redistribute(self):
        self.row["redistribute_call"] = 1
        return super()._redistribute()

    def _move(self):
        self.row["redistributed"] = 1
        return (1, 1)

    def _gather_counts(self):
        c = self.counts[self.used["counts"]]
        self.used["counts"] += 1
        return [int(v) for v in c]

    def _gather_max_reserved_gb(self):
        v = self.peaks[self.used["peaks"]]
        self.used["peaks"] += 1
        return [float(x) for x in v]

    def _total_memory_gb(self):
        return self.total_gb

    def _reset_opacity(self):
        self.row["opacity_reset"] = 1

    def _optimizer_step(self):
        self.row["adam"] = 1


@pytest.mark.parametrize("q", range(len(META["cases"])), ids=[c["name"] for c in META["cases"]])
def test_decision_table(q):
    case = META["cases"][q]
    opt = sc.OptimizationParams(**case["overrides"])
    table = GOLDEN[f"case{q}_table"]
    rec = Recorder(opt, case["world"], GOLDEN[f"case{q}_counts"], GOLDEN[f"case{q}_peaks"], META["total_gb"])
    iterations = list(range(1, opt.iterations + 1, opt.bsz))
    assert [int(r[0]) for r in table] == iterations
    for want in table:
        it = int(want[0])
        rec.row = {}
        deg = rec.trainer.params.active_sh_degree
        rec.begin(it)
        rec.row["sh_up"] = rec.trainer.params.active_sh_degree - deg
        ev = rec.end(it)
        rec.row["disabled"] = int(ev.densification_disabled)
        got = [it] + [int(rec.row.get(c, 0)) for c in COLUMNS[1:]]
        assert got == want.tolist(), (case["name"], dict(zip(COLUMNS, got)), dict(zip(COLUMNS, want.tolist())))
        assert rec.row.get("adam", 0) == int(it < opt.iterations)
        assert (ev.densify is not None) == bool(want[COLUMNS.index("densify")])
        assert (ev.redistribution is not None) == bool(want[COLUMNS.index("redistributed")])
        assert ev.opacity_reset == bool(want[COLUMNS.index("opacity_reset")])
    # every recorded input of the gates was consumed in the reference's order and number
    assert rec.used["counts"] <= len(rec.counts) and rec.used["peaks"] == int(table[:, COLUMNS.index("densify")].sum())


def test_reset_until():
    assert sc.OptimizationParams(bsz=4).reset_until() == 15_004
    assert sc.OptimizationParams(bsz=4, opacity_reset_until_iter=300).reset_until() == 300


@pytest.mark.parametrize("bad", [dict(lr_scale_mode="cubic"), dict(redistribute_gaussians_mode="x"), dict(bsz=0),
                                 dict(densification_interval=0)])
def test_options_refused(bad):
    with pytest.raises(ValueError):
        sc.OptimizationParams(**bad)
