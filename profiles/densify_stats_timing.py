#!/usr/bin/env python
"""What the densification statistics cost: the reference's per-camera torch chain against gs_densify_stats on c2.

  python profiles/densify_stats_timing.py [--iters 50] [--bs 1 4]

For B = 1 and B = 4 cameras of the c2 scene (2 M Gaussians, 1920x1080, synthetic.make_scene seed 0), after real
pipeline.Trainer steps (the statistics read that step's screen-space gradients and radii):
  * device time: CUDA events around --iters calls of each form, on an otherwise idle stream (mean per call);
  * host wall time per call on an idle device, including the host synchronisations the call makes (for the kernel,
    the enqueue only: it makes none);
  * host wall time per call issued right behind a queued Trainer.step: the chain's synchronisations wait for that step;
  * the number of synchronising calls (torch.cuda.set_sync_debug_mode("warn")) per call;
  * the kernel's achieved bytes/s from its algorithmic bytes, 12 B P read (radii + gradients of every view) + 24 P'
    read and written (the three statistics of the P' Gaussians visible in some view), against 3.35 TB/s.
Both forms are checked to give identical bits first.  Prints the card's name, power limit and maximum SM clock, then one
JSON line per B.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return name, q


def reference_chain(accum, denom, max_radii2D, grads, radii):
    """densification.py:15-24 + scene/gaussian_model.py:1046-1052."""
    for g, r in zip(grads, radii):
        visibility_filter = r > 0
        max_radii2D[visibility_filter] = torch.max(max_radii2D[visibility_filter], r[visibility_filter])
        accum[visibility_filter] += torch.norm(g[visibility_filter, :2], dim=-1, keepdim=True)
        denom[visibility_filter] += 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4])
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gs_b200 import densify, pipeline, synthetic as syn
    name, q = card()
    print(f"[card] {name}; power.limit, clocks.max.sm = {q}", flush=True)
    cfg = syn.CONFIGS["c2"]
    W, H, N = cfg["width"], cfg["height"], cfg["n"]
    dev = torch.device("cuda", 0)
    scene = syn.make_scene(N, W, H, seed=0)
    for B in a.bs:
        cams = syn.make_batch_cameras(W, H, B)
        gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=1 + k)).pin_memory() for k in range(B)]
        tr = pipeline.Trainer(scene, cams, gts, dev)
        tr.step(resident=False)
        for _ in range(3):
            tr.step(resident=True)
        torch.cuda.synchronize()
        P = tr.n_local
        grads = tr.means2D.grad if isinstance(tr.means2D, torch.Tensor) else torch.stack([m.grad for m in tr.means2D])
        radii = tr._radii_local
        visible_any = int((radii > 0).any(dim=0).sum())
        fresh = lambda: (torch.zeros((P, 1), device=dev), torch.zeros((P, 1), device=dev), torch.zeros((P,), device=dev))
        forms = {"reference": lambda st: reference_chain(*st, grads.unbind(0), radii.unbind(0)),
                 "kernel": lambda st: tr.add_densification_stats(*st)}
        outs = {}
        for f, fn in forms.items():
            outs[f] = fresh()
            fn(outs[f])
        torch.cuda.synchronize()
        same = all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(outs["kernel"], outs["reference"]))
        res = {"workload": "c2", "B": B, "P": P, "visible_in_some_view": visible_any, "gpu": name,
               "power_limit_max_sm_clock": q, "bit_identical": same}
        for f, fn in forms.items():
            st = fresh()
            for _ in range(3):
                fn(st)
            # device time, idle stream
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                fn(st)
            e1.record()
            torch.cuda.synchronize()
            dev_ms = e0.elapsed_time(e1) / a.iters
            # host wall time per call, idle device
            host = []
            for _ in range(a.iters):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(st)
                host.append((time.perf_counter() - t0) * 1e3)
            # host wall time per call right behind a queued training step
            behind = []
            for _ in range(5):
                torch.cuda.synchronize()
                tr.step(resident=True)
                t0 = time.perf_counter()
                fn(st)
                behind.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("warn")
            try:
                with warnings.catch_warnings(record=True) as w:
                    warnings.simplefilter("always")
                    fn(st)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            syncs = sum("synchroniz" in str(x.message) for x in w)
            res[f] = {"device_ms": round(dev_ms, 5), "host_ms_idle": round(statistics.median(host), 5),
                      "host_ms_behind_step": round(statistics.median(behind), 5), "sync_calls": syncs}
        alg = 12 * B * P + 24 * visible_any
        res["kernel"]["alg_bytes"] = alg
        res["kernel"]["achieved_TBps"] = round(alg / (res["kernel"]["device_ms"] * 1e-3) / 1e12, 4)
        res["kernel"]["share_of_3.35TBps"] = round(alg / (res["kernel"]["device_ms"] * 1e-3) / HBM_BYTES_PER_S, 4)
        print(json.dumps(res), flush=True)
        del tr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
