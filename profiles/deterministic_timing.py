#!/usr/bin/env python
"""What the deterministic render and loss cost: default vs deterministic on the c2 workload.

  python profiles/deterministic_timing.py [--steps 40] [--warmup 5] [--rounds 3] [--bs 1 4]

For B = 1 and B = 4 cameras of the c2 scene (2 M Gaussians, 1920x1080, synthetic.make_scene seed 0; B > 1 renders all
cameras in one batched pass), two pipeline.Trainer's over the same scene, deterministic=False and True, inputs resident:
  * Trainer.step: CUDA events around --steps steps, the two trainers alternated over --rounds rounds (median per round);
  * the blend backward ("b10 render": for the deterministic form the memset of the instance rows, the storing
    segment-parallel kernel and the per-splat reduce) and the loss forward ("loss forward": the fused L1 + SSIM kernel
    and its finalize), each from the library's stage timer (gs_profile_read, CUDA events around the launches of the
    stage) over one further window of --steps steps per trainer.
Both trainers also report their instance count R, and the losses of their first step (equal: the forward is unchanged).
Prints the card's name, power limit and maximum SM clock first, then one JSON line per B.  Needs a GPU.
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


def step_ms(tr, steps):
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    torch.cuda.synchronize()
    evs[0].record()
    for i in range(steps):
        tr.step(resident=True)
        evs[i + 1].record()
    torch.cuda.synchronize()
    return statistics.median(evs[i].elapsed_time(evs[i + 1]) for i in range(steps))


def stage_ms(tr, steps):
    from gs_b200 import _lib
    _lib.profile_read()
    _lib.profile_enable(True)
    for _ in range(steps):
        tr.step(resident=True)
    torch.cuda.synchronize()
    st = _lib.profile_read()
    _lib.profile_enable(False)
    return {k: st.get(k, (0.0, 0))[0] / steps for k in ("b10 render", "loss forward")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4])
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gs_b200 import pipeline, synthetic as syn
    name, q = card()
    print(f"[card] {name}; power.limit, clocks.max.sm = {q}", flush=True)
    cfg = syn.CONFIGS["c2"]
    W, H, N = cfg["width"], cfg["height"], cfg["n"]
    dev = torch.device("cuda", 0)
    scene = syn.make_scene(N, W, H, seed=0)
    for B in a.bs:
        cams = syn.make_batch_cameras(W, H, B)
        gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=1 + k)).pin_memory() for k in range(B)]
        trs = {d: pipeline.Trainer(scene, cams, gts, dev, deterministic=d) for d in (False, True)}
        first = {}
        for d, tr in trs.items():
            first[d] = tr.step(resident=False)
            for _ in range(a.warmup):
                tr.step(resident=True)
        R = trs[False].last_info()["R"]
        per = {False: [], True: []}
        for _ in range(a.rounds):
            for d, tr in trs.items():
                per[d].append(step_ms(tr, a.steps))
        stages = {d: stage_ms(tr, a.steps) for d, tr in trs.items()}
        print(json.dumps({
            "workload": "c2", "B": B, "R": R, "gpu": name, "power_limit_max_sm_clock": q,
            "first_loss": {"default": first[False], "deterministic": first[True]},
            "step_ms": {"default": round(statistics.median(per[False]), 4),
                        "deterministic": round(statistics.median(per[True]), 4),
                        "rounds_default": [round(x, 4) for x in per[False]],
                        "rounds_deterministic": [round(x, 4) for x in per[True]]},
            "blend_backward_ms": {"default": round(stages[False]["b10 render"], 4),
                                  "deterministic": round(stages[True]["b10 render"], 4)},
            "loss_forward_ms": {"default": round(stages[False]["loss forward"], 4),
                                "deterministic": round(stages[True]["loss forward"], 4)},
        }), flush=True)
        del trs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
