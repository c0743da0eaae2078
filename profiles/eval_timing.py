#!/usr/bin/env python
"""What held-out view evaluation costs on one GPU.

  python profiles/eval_timing.py [--iters 200] [--rounds 5] [--views 16] [--kernels]

Kernels: on 1920x1080 (c2) images, k_eval_sums (ops.eval_sums_batched) over 1 and 16 views and k_eval_finalize
(ops.eval_finalize), CUDA events around --iters calls, median of --rounds rounds.  A call this short can be bound by the
host's Python, so --kernels (a run of its own) reads the kernels' device times from torch.profiler instead, and sets
k_eval_sums against its memory floor of 15 B per pixel (12 B of fp32 image + 3 B of uint8 ground truth) at 3.35 TB/s.

Evaluation: on the c2 workload (2 M Gaussians, synthetic.make_scene seed 0) a pipeline.Trainer over --views cameras runs
Trainer.evaluate() (every view, one batch; the time per view includes the forward renders and the one host read).  On the
same rendered images, the reference's scoring sequence in torch (train_internal.py:471-478: torch.clamp, l1_loss,
psnr(...).mean().double(), accumulated on the device) is timed per view against ops.eval_sums_batched + eval_finalize over
the same views.  The legs alternate over --rounds rounds; the median per round and the median of rounds are printed.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement.  Multi-GPU times are
not measured here.  Needs a GPU.
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

from camera_set_timing import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def timed_ms(fn, iters):
    """Mean device time of one call over `iters` calls between two events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_us(fn, iters):
    """{kernel name: mean device time in us} of the k_eval_* kernels over `iters` calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("k_eval_sums", "k_eval_finalize"):
            if name in e.key:
                total = getattr(e, "device_time_total", None)
                out[name] = (total if total is not None else e.cuda_time_total) / e.count
    return out


def reference_scoring(images, gts):
    """train_internal.py:471-478 over the views: clamp, l1_loss(...).mean().double(), psnr(...).mean().double()."""
    l1_test = torch.scalar_tensor(0.0, device=images.device, dtype=torch.float64)
    psnr_test = torch.scalar_tensor(0.0, device=images.device, dtype=torch.float64)
    for image, gt in zip(images, gts):
        image = torch.clamp(image, 0.0, 1.0)
        gt_image = torch.clamp(gt / 255.0, 0.0, 1.0)
        l1_test += torch.abs(image - gt_image).mean().mean().double()
        mse = ((image - gt_image) ** 2).view(image.shape[0], -1).mean(1, keepdim=True)
        psnr_test += (20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double()
    return l1_test, psnr_test


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--kernels", action="store_true", help="kernel device times from torch.profiler only")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from gs_b200 import ops, pipeline, synthetic as syn
    name, q = card()
    print(f"[card] {name}; power.limit, clocks.max.sm = {q}", flush=True)
    cfg = syn.CONFIGS["c2"]
    W, H, N = cfg["width"], cfg["height"], cfg["n"]
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)

    # kernels on random images
    for B in (1, a.views):
        img = torch.rand((B, 3, H, W), device=dev, generator=g) * 1.2 - 0.1
        gts = [torch.randint(0, 256, (3, H, W), device=dev, dtype=torch.uint8, generator=g) for _ in range(B)]
        rows, g0 = [(0, H)] * B, [0] * B
        slots = ops.eval_sums_batched(img, gts, rows, g0)
        legs = {"k_eval_sums": lambda: ops.eval_sums_batched(img, gts, rows, g0),
                "k_eval_finalize": lambda: ops.eval_finalize(slots, H, W)}
        for fn in legs.values():
            timed_ms(fn, 10)
        floor_us = 15.0 * B * H * W / HBM_BYTES_PER_S * 1e6
        if a.kernels:
            us = kernel_us(lambda: ops.eval_finalize(ops.eval_sums_batched(img, gts, rows, g0), H, W), a.iters)
            print(json.dumps({"workload": "c2 images", "views": B, "gpu": name, "power_limit_max_sm_clock": q,
                              "kernel_us": {k: round(v, 2) for k, v in us.items()}, "k_eval_sums_bytes": 15 * B * H * W,
                              "k_eval_sums_floor_us": round(floor_us, 2),
                              "k_eval_sums_TB_per_s": round(15.0 * B * H * W / (us["k_eval_sums"] * 1e-6) / 1e12, 3)}),
                  flush=True)
            continue
        per = {k: [] for k in legs}
        for _ in range(a.rounds):
            for k, fn in legs.items():
                per[k].append(timed_ms(fn, a.iters) * 1e3)
        us = {k: statistics.median(v) for k, v in per.items()}
        print(json.dumps({"workload": "c2 images", "views": B, "gpu": name, "power_limit_max_sm_clock": q,
                          "us_per_call": {k: round(v, 2) for k, v in us.items()},
                          "rounds_us": {k: [round(x, 2) for x in v] for k, v in per.items()}}), flush=True)
        del img, gts, slots
    if a.kernels:
        return

    # Trainer.evaluate on c2, and the scoring alone on its rendered images
    scene = syn.make_scene(N, W, H, seed=0)
    cams = [syn.make_camera(W, H, yaw_deg=2.0 * k - a.views, uid=k) for k in range(a.views)]
    gts_host = [torch.from_numpy(syn.make_gt_image(W, H, seed=1 + k)).pin_memory() for k in range(a.views)]
    tr = pipeline.Trainer(scene, cams, gts_host, dev)
    p = tr.params
    with torch.no_grad():
        out = ops.preprocess_gaussians_batched(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                               p._opacity, ops.pack_cameras([c.settings() for c in tr.dcams]), W, H,
                                               p.active_sh_degree)
        Pn = out[0].shape[1]
        images, _ = ops.render_gaussians_batched(out[0].reshape(-1, 2), out[2].reshape(-1, 4), out[1].reshape(-1, 3),
                                                 out[4].reshape(-1), out[3].reshape(-1), None,
                                                 [k * Pn for k in range(a.views + 1)], tr.dcams[0].settings())
        del out
    gts = tr.gts_dev
    rows, g0 = [(0, H)] * a.views, [0] * a.views
    legs = {"evaluate": lambda: tr.evaluate(),
            "reference_scoring": lambda: reference_scoring(images, gts),
            "eval_kernels": lambda: ops.eval_finalize(ops.eval_sums_batched(images, gts, rows, g0), H, W)}
    iters = {"evaluate": 5, "reference_scoring": 20, "eval_kernels": 20}
    for k, fn in legs.items():
        timed_ms(fn, 3)
    per = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, fn in legs.items():
            per[k].append(timed_ms(fn, iters[k]) / a.views)
    print(json.dumps({"workload": "c2", "world": 1, "views": a.views, "bsz": a.views, "gpu": name,
                      "power_limit_max_sm_clock": q,
                      "ms_per_view": {k: round(statistics.median(v), 4) for k, v in per.items()},
                      "rounds_ms_per_view": {k: [round(x, 4) for x in v] for k, v in per.items()}}), flush=True)


if __name__ == "__main__":
    main()
