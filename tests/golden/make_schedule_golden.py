"""Generates tests/golden/schedule.npz by CALLING the reference's own schedule code (Grendel-GS):
utils.check_update_at_this_iter, utils.get_expon_lr_func, GaussianModel.training_setup (the optimizer's groups and the
xyz schedule) and densification.densification() (densification.py:5-85) driven over whole runs with a recording stub
model.  Only inputs and outputs are stored; nothing of the reference is copied.

    python tests/golden/make_schedule_golden.py <Grendel-GS checkout>

densification() runs on the CPU: the stub records each call the reference makes on the model (statistics,
densify_and_prune and its size threshold, redistribute_gaussians, reset_opacity); the redistribution gate is the
reference's GaussianModel.need_redistribute_gaussians called on the stub with all_gather_object answering recorded
per-rank Gaussian counts, and the memory gate is the reference's check_memory_usage with the CUDA memory queries and its
float all-gather answering recorded per-rank peaks of reserved memory (80 GiB device).
"""
import io
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else "."
sys.path[:0] = [os.path.join(ROOT, "grendel-gs_b200"), os.path.join(ROOT, "grendel-gs_b200", "shims"), REF]

_zeros = torch.zeros


def zeros_cpu(*a, **k):
    k.pop("device", None)
    return _zeros(*a, **k)


torch.zeros = zeros_cpu
torch.cuda.empty_cache = lambda: None

import utils.general_utils as utils  # noqa: E402  (the reference's)
import scene.gaussian_model as gm    # noqa: E402
import densification as dn           # noqa: E402
from arguments import OptimizationParams  # noqa: E402
from argparse import ArgumentParser  # noqa: E402

TOTAL_GB = 80.0
MAX_CALLS = 320
COLUMNS = ("iteration", "sh_up", "stats", "densify", "size_threshold", "redistribute_call", "redistributed",
           "opacity_reset", "disabled")


class Timers:
    def start(self, _):
        pass

    def stop(self, _):
        pass


class Group:
    def __init__(self, n):
        self.n = n

    def size(self):
        return self.n


def default_opt():
    opt = OptimizationParams(ArgumentParser())
    return {k: v for k, v in vars(opt).items() if not k.startswith("_")}


# (name, overrides of the reference's defaults, world size, memory trip at densify call k or -1)
CASES = [
    ("bsz1", dict(bsz=1, iterations=16000), 4, -1),
    ("bsz3", dict(bsz=3, iterations=16000), 2, -1),
    ("bsz4", dict(bsz=4, iterations=16000), 4, -1),
    ("bsz16", dict(bsz=16, iterations=16000), 2, -1),
    ("bsz32", dict(bsz=32, iterations=16000), 4, -1),
    ("w1", dict(bsz=4, iterations=16000), 1, -1),
    ("odd3", dict(bsz=3, iterations=700, densification_interval=7, opacity_reset_interval=53, densify_from_iter=13,
                  densify_until_iter=500, redistribute_gaussians_frequency=3), 4, -1),
    ("odd5_until", dict(bsz=5, iterations=700, densification_interval=11, opacity_reset_interval=37,
                        densify_from_iter=20, densify_until_iter=600, opacity_reset_until_iter=300,
                        redistribute_gaussians_frequency=4, redistribute_gaussians_threshold=1.3), 2, -1),
    ("odd16", dict(bsz=16, iterations=2000, densification_interval=9, opacity_reset_interval=100,
                   densify_from_iter=30, densify_until_iter=1500, redistribute_gaussians_frequency=5), 4, -1),
    ("trip4", dict(bsz=4, iterations=16000), 2, 40),
    ("trip1_odd", dict(bsz=1, iterations=700, densification_interval=7, opacity_reset_interval=53, densify_from_iter=13,
                       densify_until_iter=500, redistribute_gaussians_frequency=3), 4, 25),
    ("no_redistribute", dict(bsz=3, iterations=3000, densification_interval=7, opacity_reset_interval=200,
                             densify_from_iter=13, densify_until_iter=2000, redistribute_gaussians_frequency=2,
                             redistribute_gaussians_mode="no_redistribute"), 4, -1),
    ("disabled", dict(bsz=4, iterations=3000, disable_auto_densification=True), 2, -1),
]


def case_inputs(seed, world, trip):
    """Per-rank Gaussian counts of each gate all-gather and peak reserved GiB of each memory check."""
    rng = np.random.default_rng(seed)
    base = rng.integers(50_000, 200_000, size=(MAX_CALLS, 1))
    counts = base + (base * rng.uniform(0.0, 0.25, size=(MAX_CALLS, world))).astype(np.int64)
    peaks = np.round(rng.uniform(1.0, 60.0, size=(MAX_CALLS, world)), 3).astype(np.float32).astype(np.float64)
    if trip >= 0:
        peaks[trip:, world - 1] = 75.0
    return counts.astype(np.int64), peaks


def drive(overrides, world, trip, seed):
    args = SimpleNamespace(**default_opt())
    args.redistribute_gaussians_mode = "random_redistribute"
    args.redistribute_gaussians_frequency = 10
    args.redistribute_gaussians_threshold = 1.1
    args.check_gpu_memory = False
    args.log_memory_summary = False
    args.stop_update_param = False
    for k, v in overrides.items():
        setattr(args, k, v)
    if args.opacity_reset_until_iter == -1:            # init_args, arguments/__init__.py:277-278
        args.opacity_reset_until_iter = args.densify_until_iter + args.bsz
    utils.set_args(args)
    utils.TIMERS = Timers()
    utils.LOG_FILE = io.StringIO()
    utils.DENSIFY_ITER = 0
    counts, peaks = case_inputs(seed, world, trip)
    used = {"counts": 0, "peaks": 0}
    row = {}

    def all_gather_object(out, _obj, group=None):
        out[:] = [int(c) for c in counts[used["counts"]]]
        used["counts"] += 1

    def gather_floats(data, group):
        v = peaks[used["peaks"]]
        used["peaks"] += 1
        return [[float(x)] for x in v]

    torch.distributed.all_gather_object = all_gather_object
    utils.our_allgather_among_cpu_processes_float_list = gather_floats
    torch.cuda.memory_allocated = lambda *a: 0
    torch.cuda.max_memory_allocated = lambda *a: 0
    torch.cuda.memory_reserved = lambda *a: 0
    torch.cuda.max_memory_reserved = lambda *a: 0
    torch.cuda.get_device_properties = lambda *a: SimpleNamespace(total_memory=int(TOTAL_GB * 1024 ** 3))

    class Stub:
        max_radii2D = torch.zeros((1,))

        @property
        def get_xyz(self):
            return torch.zeros((1, 3))

        def add_densification_stats(self, *_):
            row["stats"] = 1

        def densify_and_prune(self, max_grad, min_opacity, extent, size_threshold):
            row["densify"] = 1
            row["size_threshold"] = 0 if size_threshold is None else int(size_threshold)

        def redistribute_gaussians(self):
            row["redistribute_call"] = 1
            if args.redistribute_gaussians_mode == "no_redistribute":
                return
            row["redistributed"] = int(gm.GaussianModel.need_redistribute_gaussians(self, Group(world)))

        def reset_opacity(self):
            row["opacity_reset"] = 1

    stub = Stub()
    pkg = {"batched_locally_preprocessed_radii": [torch.ones((1,))],
           "batched_locally_preprocessed_visibility_filter": [torch.ones((1,), dtype=torch.bool)],
           "batched_locally_preprocessed_mean2D": [None]}
    table = []
    for it in range(1, args.iterations + 1, args.bsz):     # train_internal.py:95-97
        row.clear()
        row["sh_up"] = int(utils.check_update_at_this_iter(it, args.bsz, 1000, 0))
        dn.densification(it, SimpleNamespace(cameras_extent=1.0), stub, pkg)
        row["disabled"] = int(args.disable_auto_densification)
        table.append([it] + [row.get(c, 0) for c in COLUMNS[1:]])
    return np.asarray(table, dtype=np.int32), counts, peaks


def check_update_grid():
    rows = []
    for bsz in (1, 2, 3, 4, 7, 16, 32):
        for interval in (1, 2, 3, 5, 7, 10, 100, 1000):
            for residual in (0, 1, 3):
                for it in range(0, 2 * interval + 2 * bsz + 3):
                    rows.append([it, bsz, interval, residual, int(utils.check_update_at_this_iter(it, bsz, interval,
                                                                                                  residual))])
    return np.asarray(rows, dtype=np.int32)


LR_STEPS = np.asarray([-1, 0, 1, 2, 3, 7, 100, 999, 1000, 1001, 7777, 15000, 29999, 30000, 30001, 45000], dtype=np.int64)


def expon_cases():
    out = []
    for (a, b, ds, dm, ms) in ((1.6e-4, 1.6e-6, 0, 1.0, 30000), (1.6e-4 * 3.7, 1.6e-6 * 3.7, 100, 0.01, 1000),
                               (0.0, 0.0, 0, 1.0, 1000), (5e-3, 5e-3, 10, 0.5, 7)):
        f = utils.get_expon_lr_func(a, b, lr_delay_steps=ds, lr_delay_mult=dm, max_steps=ms)
        out.append([a, b, ds, dm, ms] + [float(f(int(s))) for s in LR_STEPS])
    return np.asarray(out, dtype=np.float64)


def setup_case(mode, bsz, pos_scale, spatial):
    args = SimpleNamespace(bsz=bsz, lr_scale_pos_and_scale=pos_scale)
    utils.set_args(args)
    utils.LOG_FILE = io.StringIO()
    targs = SimpleNamespace(**default_opt())
    targs.lr_scale_mode = mode
    targs.lr_scale_pos_and_scale = pos_scale
    m = gm.GaussianModel(3)
    P = 4
    m._xyz = torch.nn.Parameter(torch.zeros((P, 3)))
    m._features_dc = torch.nn.Parameter(torch.zeros((P, 1, 3)))
    m._features_rest = torch.nn.Parameter(torch.zeros((P, 15, 3)))
    m._opacity = torch.nn.Parameter(torch.zeros((P, 1)))
    m._scaling = torch.nn.Parameter(torch.zeros((P, 3)))
    m._rotation = torch.nn.Parameter(torch.zeros((P, 4)))
    m.spatial_lr_scale = spatial
    m.group_for_redistribution = lambda: Group(1)
    m.training_setup(targs)
    groups = [[float(g["lr"]), float(g["eps"]), float(g["betas"][0]), float(g["betas"][1])]
              for g in m.optimizer.param_groups]
    names = [g["name"] for g in m.optimizer.param_groups]
    lrs = [float(m.xyz_scheduler_args(int(s))) for s in LR_STEPS]
    return names, np.asarray(groups, dtype=np.float64), np.asarray(lrs, dtype=np.float64)


def main():
    out = {"columns": np.asarray(COLUMNS), "check_update": check_update_grid(), "lr_steps": LR_STEPS,
           "expon": expon_cases()}
    meta = []
    for q, (name, ov, world, trip) in enumerate(CASES):
        table, counts, peaks = drive(ov, world, trip, seed=100 + q)
        out[f"case{q}_table"], out[f"case{q}_counts"], out[f"case{q}_peaks"] = table, counts, peaks
        meta.append(dict(name=name, overrides=ov, world=world, trip=trip))
        print(f"{name}: {len(table)} batches, densify {table[:, 3].sum()}, redistributed {table[:, 6].sum()}, "
              f"resets {table[:, 7].sum()}, disabled {table[-1, 8]}")
    setups = []
    for mode in ("linear", "sqrt", "accumu"):
        for bsz in (1, 3, 4, 16, 32):
            for pos_scale, spatial in ((1.0, 4.123456789), (0.7, 1.0)):
                names, groups, lrs = setup_case(mode, bsz, pos_scale, spatial)
                q = len(setups)
                out[f"setup{q}_groups"], out[f"setup{q}_xyz_lr"] = groups, lrs
                setups.append(dict(mode=mode, bsz=bsz, lr_scale_pos_and_scale=pos_scale, spatial_lr_scale=spatial,
                                   names=names))
    out["meta"] = np.asarray(json.dumps(dict(cases=meta, setups=setups, total_gb=TOTAL_GB)))
    np.savez_compressed(os.path.join(HERE, "schedule.npz"), **out)


if __name__ == "__main__":
    main()
