#!/usr/bin/env python
"""What the image metrics (SSIM / PSNR of the 8-bit renders) cost on one GPU.

  python profiles/image_metrics_timing.py [--rounds 5] [--views 16]

Kernels: on 1920x1080 (c2) images over --views views, the device times of k_quantize_u8 (ops.quantize_u8_batched),
k_image_metric_sums (ops.image_metric_sums_batched) and k_image_metric_finalize from torch.profiler, each set against its
floor: HBM bytes at the data sheet's 3.35 TB/s, and for k_image_metric_sums also its fp64 FMA count at the data sheet's
34 TFLOP/s of fp64 (17 T FMA/s).  k_quantize_u8 moves 12 B of fp32 render in and 3 B out per pixel;
k_image_metric_sums reads 6 B per pixel of window (its halo and column re-reads come from L2) and does, per pixel and
channel, 11 taps x 5 moments in the row pass for 26 / 16 rows per output row and 11 x 5 in the column pass: 144 FMA.

Scoring: on the same c2 renders, per view, the reference's sequence on the device (render.py's clamp and save_image's
quantization, tf.to_tensor's / 255, utils/loss_utils.py ssim with its window built per call, utils/image_utils.py psnr;
without the PNG files) against ours (window assembly, quantize, sums, finalize), alternated over --rounds rounds.
Trainer.image_metrics(): a pipeline.Trainer over --views cameras of the c2 workload (2 M Gaussians), every view in one
batch; the time per view includes the forward renders and the one host read.  Medians of the rounds are printed.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement.  Multi-GPU times are
not measured here.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.join(ROOT, "profiles"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from camera_set_timing import card  # noqa: E402
from eval_timing import timed_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
FP64_FMA_PER_S = 34e12 / 2  # H100 SXM data sheet, fp64 (not the tensor cores)
FMA_PER_PX_CH = 11 * 5 * 26 / 16 + 11 * 5
KERNELS = ("k_quantize_u8", "k_image_metric_sums", "k_image_metric_finalize")


def kernel_us(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in KERNELS:
            if name in e.key:
                total = getattr(e, "device_time_total", None)
                out[name] = (total if total is not None else e.cuda_time_total) / e.count
    return out


def ours(ops, images, gts, H, W):
    B = images.shape[0]
    wins = [torch.empty((6, H, W), dtype=torch.uint8, device=images.device) for _ in range(B)]
    for w, g in zip(wins, gts):
        w[3:].copy_(g)
    ops.quantize_u8_batched(images, [(0, H)] * B, [w[:3] for w in wins], [0] * B)
    return ops.image_metric_finalize(ops.image_metric_sums_batched(wins, [0] * B, [(0, H)] * B, H), H, W)


def reference(metrics_ref, images, gts):
    ssims, psnrs = [], []
    for image, gt in zip(images, gts):
        q = metrics_ref.save_image_quantize(image)
        gq = metrics_ref.save_image_quantize(gt / 255.0)
        a, b = (q.float() / 255).unsqueeze(0), (gq.float() / 255).unsqueeze(0)
        window = metrics_ref.reference_window()[1].expand(3, 1, 11, 11).contiguous().cuda(a.get_device()).type_as(a)
        conv = lambda z: torch.nn.functional.conv2d(z, window, padding=5, groups=3)  # noqa: E731
        mu1, mu2 = conv(a), conv(b)
        mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
        s11, s22, s12 = conv(a * a) - mu1_sq, conv(b * b) - mu2_sq, conv(a * b) - mu1_mu2
        m = ((2 * mu1_mu2 + 0.01 ** 2) * (2 * s12 + 0.03 ** 2)) / ((mu1_sq + mu2_sq + 0.01 ** 2) * (s11 + s22 + 0.03 ** 2))
        ssims.append(m.mean())
        psnrs.append(20 * torch.log10(1.0 / torch.sqrt(((a - b) ** 2).view(1, -1).mean(1, keepdim=True))))
    return ssims, psnrs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--views", type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import metrics_ref
    from gs_b200 import ops, pipeline, synthetic as syn
    name, q = card()
    print(f"[card] {name}; power.limit, clocks.max.sm = {q}", flush=True)
    cfg = syn.CONFIGS["c2"]
    W, H, N, B = cfg["width"], cfg["height"], cfg["n"], a.views
    dev = torch.device("cuda", 0)

    scene = syn.make_scene(N, W, H, seed=0)
    cams = [syn.make_camera(W, H, yaw_deg=2.0 * k - B, uid=k) for k in range(B)]
    gts_host = [torch.from_numpy(syn.make_gt_image(W, H, seed=1 + k)).pin_memory() for k in range(B)]
    tr = pipeline.Trainer(scene, cams, gts_host, dev)
    p = tr.params
    with torch.no_grad():
        out = ops.preprocess_gaussians_batched(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                               p._opacity, ops.pack_cameras([c.settings() for c in tr.dcams]), W, H,
                                               p.active_sh_degree)
        Pn = out[0].shape[1]
        images, _ = ops.render_gaussians_batched(out[0].reshape(-1, 2), out[2].reshape(-1, 4), out[1].reshape(-1, 3),
                                                 out[4].reshape(-1), out[3].reshape(-1), None,
                                                 [k * Pn for k in range(B + 1)], tr.dcams[0].settings())
        del out
    gts = tr.gts_dev

    # kernels, from torch.profiler in a run of their own
    ours(ops, images, gts, H, W)
    us = kernel_us(lambda: ours(ops, images, gts, H, W), 20)
    px = B * H * W
    floors = {"k_quantize_u8": {"hbm_bytes": 15 * px, "hbm_floor_us": 15 * px / HBM_BYTES_PER_S * 1e6},
              "k_image_metric_sums": {"hbm_bytes": 6 * px, "hbm_floor_us": 6 * px / HBM_BYTES_PER_S * 1e6,
                                      "fp64_fma": FMA_PER_PX_CH * 3 * px,
                                      "fp64_floor_us": FMA_PER_PX_CH * 3 * px / FP64_FMA_PER_S * 1e6}}
    print(json.dumps({"workload": "c2 renders", "views": B, "gpu": name, "power_limit_max_sm_clock": q,
                      "kernel_us": {k: round(v, 2) for k, v in us.items()},
                      "floors": {k: {f: round(x, 2) for f, x in v.items()} for k, v in floors.items()},
                      "share_of_binding_floor": {
                          "k_quantize_u8": round(floors["k_quantize_u8"]["hbm_floor_us"] / us["k_quantize_u8"], 3),
                          "k_image_metric_sums": round(max(floors["k_image_metric_sums"]["hbm_floor_us"],
                                                           floors["k_image_metric_sums"]["fp64_floor_us"])
                                                       / us["k_image_metric_sums"], 3)}}), flush=True)

    # per-view scoring, ours against the reference's sequence, and image_metrics with its renders
    got = ours(ops, images, gts, H, W).cpu()
    ref_s, ref_p = reference(metrics_ref, images, gts)
    agree = max(max(abs(got[v, 0].item() - ref_s[v].item()) / abs(ref_s[v].item()),
                    abs(got[v, 1].item() - ref_p[v].item()) / abs(ref_p[v].item())) for v in range(B))
    legs = {"ours": lambda: ours(ops, images, gts, H, W), "reference": lambda: reference(metrics_ref, images, gts),
            "image_metrics": lambda: tr.image_metrics()}
    iters = {"ours": 10, "reference": 3, "image_metrics": 3}
    for k, fn in legs.items():
        timed_ms(fn, 2)
    per = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, fn in legs.items():
            per[k].append(timed_ms(fn, iters[k]) / B)
    print(json.dumps({"workload": "c2", "world": 1, "views": B, "bsz": B, "gpu": name, "power_limit_max_sm_clock": q,
                      "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
                      "max_rel_diff_vs_reference": agree,
                      "ms_per_view": {k: round(statistics.median(v), 4) for k, v in per.items()},
                      "rounds_ms_per_view": {k: [round(x, 4) for x in v] for k, v in per.items()}}), flush=True)


if __name__ == "__main__":
    main()
