#!/usr/bin/env python
"""What starting a model from a point cloud costs on one GPU.

  python profiles/point_cloud_timing.py [--sizes 1000000 4000000 16000000 40000000] [--brute 1000000 2000000]
                                        [--init 16000000] [--rounds 3]

Seeded SfM-like clouds (sfm_cloud): dense clusters, a uniform background and far outliers.  For each size in --sizes,
the Morton-tree 3-NN search (simple_knn._C.distCUDA2 on a CUDA tensor, gs_knn3_mean_dist2_range over every point:
bounding box, keys, sort, tree and search, the bounding box read-back included) is timed with CUDA events after one
warm-up call, median of --rounds; for each size in --brute, the exhaustive kernel gs_knn3_mean_dist2 on the same cloud,
once after a warm-up at a small size (one call takes seconds at 2 M points and grows as N^2), and the two answers are
compared bit for bit.  At --init, point_cloud.init_model end to end at world size 1 (host arrays in, the six parameters
on the device out), and the device memory the search's workspace takes.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.join(ROOT, "profiles")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from camera_set_timing import card  # noqa: E402


def sfm_cloud(n, seed=0):
    """(n, 3) float32 and (n, 3) uint8: 85 % in clusters of ~20 k points (sd 0.05 in a 20-unit scene), 14.5 % uniform
    background, 0.5 % outliers a hundred scene sizes out."""
    rng = np.random.default_rng([seed, n])
    kind = rng.random(n)
    centers = rng.uniform(-10.0, 10.0, (max(1, n // 20_000), 3)).astype(np.float32)
    xyz = centers[rng.integers(0, len(centers), n)] + rng.normal(0.0, 0.05, (n, 3)).astype(np.float32)
    bg = (kind >= 0.85) & (kind < 0.995)
    xyz[bg] = rng.uniform(-10.0, 10.0, (int(bg.sum()), 3))
    out = kind >= 0.995
    xyz[out] = rng.normal(0.0, 2000.0, (int(out.sum()), 3))
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    return np.ascontiguousarray(xyz, dtype=np.float32), rgb


def event_ms(fn, rounds):
    times, out = [], None
    for _ in range(rounds):
        out = None   # the previous round's result is freed first: the peak memory is one call's
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), times, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 4_000_000, 16_000_000, 40_000_000])
    ap.add_argument("--brute", type=int, nargs="*", default=[1_000_000, 2_000_000])
    ap.add_argument("--init", type=int, nargs="*", default=[16_000_000])
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gs_b200 import _lib, point_cloud
    from simple_knn import _C as knn
    dev = "cuda:0"
    print(json.dumps({"card": card()}), flush=True)
    knn._dist2_kernel(torch.from_numpy(sfm_cloud(100_000)[0]).to(dev))
    knn._dist2_brute(torch.from_numpy(sfm_cloud(100_000)[0]).to(dev))
    torch.cuda.synchronize()
    for n in sorted(set(a.sizes) | set(a.brute)):
        pts = torch.from_numpy(sfm_cloud(n)[0]).to(dev)
        knn._dist2_kernel(pts)   # warm-up at this size
        ms, times, got = event_ms(lambda: knn._dist2_kernel(pts), a.rounds)
        print(json.dumps({"what": "search", "n": n, "ms": round(ms, 3), "ns_per_point": round(ms * 1e6 / n, 2),
                          "rounds_ms": [round(t, 3) for t in times],
                          "temp_bytes_per_point": round(_lib.query("gs_knn3_temp_bytes", n) / n, 2)}), flush=True)
        if n in a.brute:
            bms, _, ref = event_ms(lambda: knn._dist2_brute(pts), 1)
            same = bool(torch.equal(ref.view(torch.int32), got.view(torch.int32)))
            print(json.dumps({"what": "brute_force", "n": n, "ms": round(bms, 3), "search_ms": round(ms, 3),
                              "speedup": round(bms / ms, 1), "same_bits": same}), flush=True)
        del pts, got
        torch.cuda.empty_cache()
    for n in a.init:
        xyz, rgb = sfm_cloud(n)
        point_cloud.init_model(xyz[:100_000], rgb[:100_000], device=dev)   # warm-up of the elementwise kernels
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        ms, times, (params, _) = event_ms(lambda: point_cloud.init_model(xyz, rgb, 0, 1, 3, dev), a.rounds)
        print(json.dumps({"what": "init_model", "n": n, "ms": round(ms, 1), "rounds_ms": [round(t, 1) for t in times],
                          "peak_device_bytes_per_point": round((torch.cuda.max_memory_allocated() - base) / n, 1)}),
              flush=True)
        del params


if __name__ == "__main__":
    main()
