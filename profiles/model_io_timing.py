#!/usr/bin/env python
"""What saving and loading a model costs on one GPU (world size 1).

  python profiles/model_io_timing.py [--sizes 2000000 10000000] [--rounds 3] [--dir DIR] [--ref-max 2000000]

For each size, a model of that many Gaussians at SH degree 3 (random raw parameters on the device) is saved and loaded
with gs_b200.model_io: save_ply per rank (point_cloud_rk0_ws1.ply), save_ply gathered (point_cloud.ply), load_ply of
each, save_checkpoint and load_checkpoint (a FusedAdam with moments over the six groups, and the three statistics).
Each time is the host wall clock from the call to its return (every call ends with its data in the file or on the device:
load_* synchronise), median of --rounds rounds.  Files go to --dir (default: a temporary directory), removed afterwards;
a 10 M-Gaussian PLY is 2.5 GB, a checkpoint 7.4 GB.

For the sizes up to --ref-max, the reference's packing step of save_ply (scene/gaussian_model.py:547,
`elements[:] = list(map(tuple, attributes))`, plain numpy) is timed on the same (n, 62) host array, once: it builds one
Python tuple of 62 floats per Gaussian, so its memory grows by about 2.5 kB per Gaussian.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement.  Needs a GPU.
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.join(ROOT, "profiles")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from camera_set_timing import card  # noqa: E402


def model(n, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    shapes = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
    return {k: torch.randn((n,) + s, device=dev, generator=g) for k, s in shapes.items()}


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2_000_000, 10_000_000])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--ref-max", type=int, default=2_000_000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gs_b200 import model_io, pipeline
    from gs_b200 import synthetic as syn
    from gs_b200.optim import FusedAdam
    name, q = card()
    dev = "cuda:0"
    cams = [syn.make_camera(64, 64)]   # the Trainer only holds the model here; nothing is rendered
    for n in a.sizes:
        base = tempfile.mkdtemp(prefix="model_io_timing_", dir=a.dir)
        try:
            tr = pipeline.Trainer(None, cams, None, dev, model=model(n, dev))
            opt = FusedAdam(tr.optimizer_groups(), lr=1e-3, eps=1e-15)
            for p in tr.params.raw_parameters():
                p.grad = torch.ones_like(p)
            opt.step()
            stats = {"max_radii2D": torch.zeros((n,), device=dev), "xyz_gradient_accum": torch.zeros((n, 1), device=dev),
                     "denom": torch.zeros((n, 1), device=dev)}
            legs = {
                "save_ply per-rank": lambda: model_io.save_ply(os.path.join(base, "per_rank"), tr),
                "save_ply gathered": lambda: model_io.save_ply(os.path.join(base, "gathered"), tr, gather=True),
                "load_ply per-rank": lambda: model_io.load_ply(os.path.join(base, "per_rank"), device=dev),
                "load_ply gathered": lambda: model_io.load_ply(os.path.join(base, "gathered"), device=dev),
                "save_checkpoint": lambda: model_io.save_checkpoint(os.path.join(base, "ckpt"), tr, opt, stats, 1),
                "load_checkpoint": lambda: model_io.load_checkpoint(os.path.join(base, "ckpt"), 0, 1, dev),
            }
            times = {k: [] for k in legs}
            for _ in range(a.rounds):
                for k, fn in legs.items():
                    ms, out = wall(fn)
                    times[k].append(ms)
                    del out
            size = os.path.getsize(os.path.join(base, "gathered", "point_cloud.ply"))
            for k, ts in times.items():
                print(json.dumps({"gaussians": n, "leg": k, "median_ms": round(statistics.median(ts), 1),
                                  "rounds_ms": [round(t, 1) for t in ts], "ply_bytes": size, "gpu": name,
                                  "power_limit_max_sm_clock": q}), flush=True)
            if n <= a.ref_max:
                rows = model_io._to_host(model_io.ply_rows(model_io._raw_of(tr)))
                elements = np.empty(n, dtype=[(x, "f4") for x in model_io.attribute_names(3)])
                t = time.perf_counter()
                elements[:] = list(map(tuple, rows))
                ms = (time.perf_counter() - t) * 1e3
                assert np.array_equal(elements.view("<f4").reshape(n, -1).view(np.int32), rows.view(np.int32))
                print(json.dumps({"gaussians": n, "leg": "reference elements[:] = list(map(tuple, attributes))",
                                  "ms": round(ms, 1), "gpu": name, "power_limit_max_sm_clock": q}), flush=True)
                del elements, rows
            del tr, opt, stats
            torch.cuda.empty_cache()
        finally:
            shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
