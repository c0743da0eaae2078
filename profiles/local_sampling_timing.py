#!/usr/bin/env python
"""What local sampling costs on one GPU, and the device memory a rank's own images take.

  python profiles/local_sampling_timing.py [--steps 40] [--warmup 5] [--rounds 5] [--bs 1 4] [--cams 16]
                                           [--resident 200] [--worlds 1 2 4 8]

Step time: on the c2 workload (2 M Gaussians, 1920x1080, synthetic.make_scene seed 0), a default pipeline.Trainer and a
pipeline.Trainer(local_sampling=True, local_bsz=B) over --cams cameras step the same --steps batches of B views, a new
batch every step, inputs resident.  At one rank the local-sampling step differs from the default one only in how the
batch's camera table reaches the device (gathered there from a resident (N, 40) table instead of copied from pinned host
memory) and in skipping the strip-division lookup.  CUDA events around --steps steps, the two legs alternated over --rounds
rounds; the median per round and the median of rounds are printed.

Memory: with --resident 1080p training images and W ranks, a rank holds the images of the cameras with uid % W == rank
(scene/cameras.py:52-59).  For each W of --worlds, rank 0's Trainer is built on one GPU with only its own images; printed
are the images it holds, their bytes, and the growth of allocated device memory over the construction.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement.  Multi-GPU step
times are not measured here.  Needs a GPU.
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

import torch  # noqa: E402

from camera_set_timing import card, step_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--resident", type=int, default=200)
    ap.add_argument("--worlds", type=int, nargs="+", default=[1, 2, 4, 8])
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
    default = pipeline.Trainer(scene, cams, gts, dev)
    for B in a.bs:
        local = pipeline.Trainer(scene, cams, gts, dev, local_sampling=True, local_bsz=B)
        batches = [[(i * B + j) % a.cams for j in range(B)] for i in range(a.steps)]
        legs = {"default": default, "local_sampling": local}
        for tr in legs.values():
            step_ms(tr, batches[:a.warmup])
        per = {k: [] for k in legs}
        for _ in range(a.rounds):
            for k, tr in legs.items():
                per[k].append(step_ms(tr, batches))
        print(json.dumps({"workload": "c2", "world": 1, "B": B, "cameras": a.cams, "gpu": name,
                          "power_limit_max_sm_clock": q,
                          "step_ms": {k: round(statistics.median(v), 4) for k, v in per.items()},
                          "rounds": {k: [round(x, 4) for x in v] for k, v in per.items()}}), flush=True)
        del local
    del default
    torch.cuda.empty_cache()

    # memory: rank 0's own images out of --resident, for each world size
    R = a.resident
    rcams = [syn.make_camera(W, H, yaw_deg=(k % 40) - 20.0, uid=k) for k in range(R)]
    gt0 = torch.from_numpy(syn.make_gt_image(W, H, seed=1)).pin_memory()
    small = syn.make_scene(200_000, W, H, seed=0)
    for world in a.worlds:
        held = [gt0 if c["uid"] % world == 0 else None for c in rcams]
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated()
        tr = pipeline.Trainer(small, rcams, held, dev, local_sampling=True, local_bsz=1)
        torch.cuda.synchronize()
        m1 = torch.cuda.memory_allocated()
        n_held = sum(g is not None for g in tr.gts_dev)
        params = sum(t.numel() * t.element_size() for t in tr.params.raw_parameters())
        print(json.dumps({"workload": "c2 images", "resident_images": R, "world": world, "rank": 0, "gpu": name,
                          "power_limit_max_sm_clock": q, "images_held": n_held, "image_bytes": 3 * H * W,
                          "held_image_bytes": n_held * 3 * H * W, "trainer_bytes": m1 - m0,
                          "trainer_bytes_without_parameters": m1 - m0 - params}), flush=True)
        del tr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
