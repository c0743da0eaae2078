#!/usr/bin/env python
"""What training over a camera set costs: a changing batch of views per step against a fixed batch, on the c2 workload,
and the device memory of the resident ground truth.

  python profiles/camera_set_timing.py [--steps 40] [--warmup 5] [--rounds 3] [--bs 1 4] [--cams 16] [--resident 200]

Step time: for B = 1 and B = 4, one pipeline.Trainer over --cams cameras of the c2 scene (2 M Gaussians, 1920x1080,
synthetic.make_scene seed 0), inputs resident.  Both legs step the same --steps batches of B views, windows that cycle
through the cameras: the "changing" leg takes a new window every step (a new camera table copied from pinned host
memory, a new division lookup), the "fixed" leg holds each window for a block of consecutive steps, so the two differ
only in how often the batch changes, not in which views they render.  CUDA events around --steps steps, the two legs
alternated over --rounds rounds; the median per round and the median of rounds are printed.

Memory: a Trainer holding --resident 1080p images on the device (the reference's --preload_dataset_to_gpu) steps every one
of them once in batches of 4.  Printed: the bytes the images take, the growth of allocated device memory over those steps
with the loss reading the images in place, and the bytes a strip cache keyed by (camera, rows) holds for the same views
when each holds a quarter-height strip (one rank of four), materialised and measured the same way.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return name, q


def step_ms(tr, batches):
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(batches) + 1)]
    torch.cuda.synchronize()
    evs[0].record()
    for i, views in enumerate(batches):
        tr.step(views=views, resident=True)
        evs[i + 1].record()
    torch.cuda.synchronize()
    return statistics.median(evs[i].elapsed_time(evs[i + 1]) for i in range(len(batches)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--resident", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gs_b200 import pipeline, synthetic as syn
    name, q = card()
    print(f"[card] {name}; power.limit, clocks.max.sm = {q}", flush=True)
    cfg = syn.CONFIGS["c2"]
    W, H, N = cfg["width"], cfg["height"], cfg["n"]
    dev = torch.device("cuda", 0)
    scene = syn.make_scene(N, W, H, seed=0)
    cams = [syn.make_camera(W, H, yaw_deg=2.0 * k - a.cams, uid=k) for k in range(a.cams)]
    gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=1 + k)).pin_memory() for k in range(a.cams)]
    tr = pipeline.Trainer(scene, cams, gts, dev)
    for B in a.bs:
        # the same batches in both legs: cycled step by step, or each held for a block of steps
        changing = [[(i * B + j) % a.cams for j in range(B)] for i in range(a.steps)]
        legs = {"fixed": sorted(changing), "changing": changing}
        for batches in legs.values():
            step_ms(tr, batches[:a.warmup])
        per = {k: [] for k in legs}
        for _ in range(a.rounds):
            for k, batches in legs.items():
                per[k].append(step_ms(tr, batches))
        print(json.dumps({"workload": "c2", "B": B, "cameras": a.cams, "gpu": name, "power_limit_max_sm_clock": q,
                          "step_ms": {k: round(statistics.median(v), 4) for k, v in per.items()},
                          "rounds": {k: [round(x, 4) for x in v] for k, v in per.items()}}), flush=True)
    del tr
    torch.cuda.empty_cache()

    # memory of the resident leg: --resident images, every one stepped once
    R = a.resident
    rcams = [syn.make_camera(W, H, yaw_deg=(k % 40) - 20.0, uid=k) for k in range(R)]
    gt0 = torch.from_numpy(syn.make_gt_image(W, H, seed=1)).pin_memory()
    small = syn.make_scene(200_000, W, H, seed=0)
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    tr = pipeline.Trainer(small, rcams, [gt0] * R, dev)
    torch.cuda.synchronize()
    m1 = torch.cuda.memory_allocated()
    tr.step(views=[0, 1, 2, 3], resident=True)   # workspaces of a B = 4 step
    torch.cuda.synchronize()
    m2 = torch.cuda.memory_allocated()
    for i in range(0, R, 4):
        tr.step(views=[(i + j) % R for j in range(4)], resident=True)
    torch.cuda.synchronize()
    m3 = torch.cuda.memory_allocated()
    y0, y1 = H // 4, H // 2   # rank 1 of 4
    cache = {(k, y0, y1): tr.gts_dev[k][:, y0:y1, :].contiguous() for k in range(R)}
    torch.cuda.synchronize()
    m4 = torch.cuda.memory_allocated()
    print(json.dumps({"workload": "c2 images", "resident_images": R, "gpu": name, "power_limit_max_sm_clock": q,
                      "image_bytes": 3 * H * W, "trainer_bytes": m1 - m0,
                      "growth_over_all_views_in_place_bytes": m3 - m2,
                      "strip_cache_quarter_strips_bytes": m4 - m3, "strip_cache_entries": len(cache)}), flush=True)


if __name__ == "__main__":
    main()
