#!/usr/bin/env python
"""Preprocess and training-step time as a function of the SH degree a model stores (max_sh_degree D = 0..3, K = (D+1)^2
coefficients per Gaussian).

  python profiles/sh_degree_timing.py [--n 2000000] [--width 1920] [--height 1080] [--iters 300] [--steps 50]

On the c2 scene (2 M Gaussians, 1920x1080, synthetic.make_scene seed 0) and for each D:
  * gs_preprocess_{forward,backward}_batched_sh at B = 1 and 4 cameras, CUDA events around --iters launches after
    warm-up (the C ABI called directly: no autograd, no Python between launches);
  * one pipeline.Trainer.step (fused activations, one camera, inputs resident), CUDA events around --steps steps.
The preprocess's algorithmic bytes come from the shapes: per Gaussian the forward reads 44 + 12 K bytes of parameters and
writes 45 B per camera; the backward reads the parameters and 41 B per camera and writes 44 + 12 K bytes of gradients.
Prints the card's name and power limit first, then one JSON line per D.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
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


def timed(fn, iters, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def preprocess_times(params, cams_all, W, H, D, iters):
    from gs_b200 import _lib, ops
    raw = [t.detach() for t in params.raw_parameters()]
    P, K = raw[0].shape[0], (D + 1) ** 2
    dev = raw[0].device
    s = torch.cuda.current_stream().cuda_stream
    out = {}
    for B in (1, 4):
        cams = ops.pack_cameras(cams_all[:B])
        m2, dep, rad, co, rgb, clm = ops._screen_outputs((B, P), dev)
        scr = [t.data_ptr() for t in (m2, dep, rad, co, rgb, clm)]
        g = torch.Generator(device=dev).manual_seed(B)
        gm, gc, gr = (torch.randn((B, P, k), device=dev, generator=g) for k in (2, 4, 3))
        grads = [torch.empty_like(t) for t in raw]

        def fwd():
            _lib.call("gs_preprocess_forward_batched_sh", B, P, D, D, *(t.data_ptr() for t in raw[:4]), 1.0,
                      raw[4].data_ptr(), raw[5].data_ptr(), cams.data_ptr(), W, H, *scr, s)

        def bwd():
            _lib.call("gs_preprocess_backward_batched_sh", B, P, D, D, *(t.data_ptr() for t in raw[:4]), 1.0,
                      raw[4].data_ptr(), raw[5].data_ptr(), cams.data_ptr(), W, H, rad.data_ptr(), clm.data_ptr(),
                      gm.data_ptr(), gc.data_ptr(), gr.data_ptr(), *(t.data_ptr() for t in grads), s)

        tf = timed(fwd, iters)
        tb = timed(bwd, iters)
        fwd_bytes = P * (44 + 12 * K + 45 * B)
        bwd_bytes = P * (44 + 12 * K + 41 * B + 44 + 12 * K)
        out[f"B{B}"] = dict(fwd_ms=round(tf, 4), bwd_ms=round(tb, 4), fwd_bytes=fwd_bytes, bwd_bytes=bwd_bytes,
                            fwd_GBps=round(fwd_bytes / tf / 1e6, 1), bwd_GBps=round(bwd_bytes / tb / 1e6, 1),
                            visible_cam0=int((rad[0] > 0).sum()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--degrees", default="0,1,2,3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sh_degree_timing.py needs a GPU")
    from gs_b200 import build, pipeline, synthetic as syn
    build.build()
    dev = torch.device("cuda", 0)
    name, limit = card()
    print(json.dumps(dict(gpu=name, power_limit_and_max_sm_clock=limit)), flush=True)
    W, H = args.width, args.height
    cams = syn.make_batch_cameras(W, H, 4)
    gt = torch.from_numpy(syn.make_gt_image(W, H)).pin_memory()
    for D in (int(d) for d in args.degrees.split(",")):
        sc = syn.make_scene(args.n, W, H, seed=0, max_sh_degree=D)
        tr = pipeline.Trainer(sc, cams[:1], [gt], dev, max_sh_degree=D)
        settings = [pipeline.DeviceCamera(c, dev).settings(D) for c in cams]
        pre = preprocess_times(tr.params, settings, W, H, D, args.iters)
        step_ms = timed(lambda: tr.step(resident=True), args.steps, warmup=5)
        print(json.dumps(dict(max_sh_degree=D, K=(D + 1) ** 2, n=args.n, width=W, height=H,
                              preprocess_batched=pre, train_step_ms=round(step_ms, 4))), flush=True)
        del tr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
