#!/usr/bin/env python
"""What the schedule's device work costs: the opacity reset and the overhead of Schedule.end.

  python profiles/schedule_timing.py [--iters 200] [--out runs/schedule_timing.json]

  * opacity reset at 1 M and 10 M Gaussians: gs_reset_opacity (densify.reset_opacity: logits rewritten, both moments
    zeroed, in place) against the reference's torch (gaussian_model.py:555-561 with replace_tensor_to_optimizer: the
    expression plus two zeros_like), CUDA events around --iters calls each, mean per call; both are checked to give the
    same bits first.  The kernel's achieved bytes/s from its algorithmic bytes (4 B read + 12 B written per Gaussian)
    against the H100 SXM data sheet's 3.35 TB/s;
  * Schedule.end on an iteration that does not densify (statistics + Adam step) against the same two library calls
    made by hand, host wall time per call behind a synchronise, on a 200 k-Gaussian synthetic scene at 640x480, bsz 4.
Prints the card's name, power limit and maximum SM clock with the JSON result.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return name, q


def events_ms(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def reset_timing(P, iters):
    from gs_b200 import densify
    from gs_b200.optim import FusedAdam
    dev = "cuda:0"
    x = torch.randn((P, 1), device=dev) * 4.0
    p = nn.Parameter(x.clone())
    opt = FusedAdam([{"params": [p], "lr": 0.05, "name": "opacity"}], lr=0.0, eps=1e-15)
    opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.randn_like(x), "exp_avg_sq": torch.rand_like(x)}

    def torch_form(o):
        s = torch.sigmoid(o)
        m = torch.min(s, torch.ones_like(s) * 0.01)
        return torch.log(m / (1 - m)), torch.zeros_like(o), torch.zeros_like(o)

    densify.reset_opacity(opt)
    want = torch_form(x)[0]
    assert torch.equal(p.detach().view(torch.int32), want.view(torch.int32)), "reset bits differ"
    k_ms = events_ms(lambda: densify.reset_opacity(opt), iters)
    t_ms = events_ms(lambda: torch_form(x), iters)
    return dict(P=P, kernel_ms=k_ms, torch_ms=t_ms, speedup=t_ms / k_ms,
                kernel_bytes_per_s=16.0 * P / (k_ms * 1e-3), hbm_share=16.0 * P / (k_ms * 1e-3) / HBM_BYTES_PER_S)


def end_timing(iters):
    from gs_b200 import pipeline, schedule as sc, synthetic as syn
    dev, W, H, N, bsz = "cuda:0", 640, 480, 200_000, 4
    cams = [syn.make_camera(W, H, yaw_deg=2.0 * q - 4.0, uid=q) for q in range(bsz)]
    gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=q)).pin_memory() for q in range(bsz)]
    tr = pipeline.Trainer(syn.make_scene(N, W, H, seed=1), cams, gts, dev)
    # densify_from_iter beyond the run: end() adds the statistics and steps, and never densifies
    sched = sc.Schedule(tr, sc.OptimizationParams(bsz=bsz, iterations=10 ** 9, densify_from_iter=10 ** 9), extent=5.0)
    walls_sched, walls_hand = [], []
    for q in range(iters + 5):
        it = 1 + bsz * q
        sched.begin(it)
        tr.step(views=list(range(bsz)))
        grads = {prm: prm.grad.clone() for prm in tr.params.raw_parameters()}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sched.end(it)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        for prm, g in grads.items():   # the same work again, by hand
            prm.grad = g
        s = sched.stats
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        tr.add_densification_stats(s["xyz_gradient_accum"], s["denom"], s["max_radii2D"])
        sched.optimizer.step()
        sched.optimizer.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        if q >= 5:
            walls_sched.append((t1 - t0) * 1e3)
            walls_hand.append((t3 - t2) * 1e3)
    walls_sched.sort()
    walls_hand.sort()
    return dict(P=N, bsz=bsz, end_ms_median=walls_sched[len(walls_sched) // 2],
                by_hand_ms_median=walls_hand[len(walls_hand) // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("schedule_timing.py needs a GPU")
    name, limits = card()
    res = dict(card=name, power_limit_and_max_sm_clock=limits,
               reset=[reset_timing(P, a.iters) for P in (1_000_000, 10_000_000)], end=end_timing(min(a.iters, 50)))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
