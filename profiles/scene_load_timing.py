#!/usr/bin/env python
"""What loading a COLMAP scene with gs_b200.scene costs on the host.

  python profiles/scene_load_timing.py [--views 200] [--obs 50000] [--points 200000] [--rounds 3] [--dir DIR]

Writes a seeded COLMAP dataset of --views views at 1920 x 1080 into --dir (default: a temporary directory, removed
afterwards): sparse/0/{cameras,images,points3D}.bin with --obs 2D observations per image (10 M in images.bin at the
defaults) and --points points with 8-observation tracks, and each view's image twice, as JPEG (quality 95) in images/
and as PNG (PIL's compress_level 1) under the same file names in images_png/.  The images are one smooth seeded texture
with noise, rolled per view.

Times, as host wall clock, median of --rounds rounds:
  * images.bin alone (scene._read_images_bin: the observations are skipped by their count) and points3D.bin alone;
  * read_colmap_scene end to end (the three model files, every image's header, the split, the extent);
  * load_images of every view, JPEG and PNG, on one thread and on the default pool, into pinned memory when a GPU is
    present (pageable otherwise; the JSON says which).
Prints the host's CPU count and model first, then one JSON line per measurement.  Needs no GPU.
"""
import argparse
import json
import os
import shutil
import statistics
import struct
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "grendel-gs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gs_b200 import scene  # noqa: E402

W, H = 1920, 1080


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return "unknown"


def write_dataset(root, views, obs, points):
    from PIL import Image
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse)
    rng = np.random.default_rng(0)
    fx = W / (2 * np.tan(np.radians(60.0) / 2))
    with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<QiiQQ4d", 1, 1, 1, W, H, fx, fx, W / 2, H / 2))
    o = np.zeros(obs, dtype=[("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
    o["x"], o["y"], o["id"] = rng.uniform(0, W, obs), rng.uniform(0, H, obs), rng.integers(-1, points, obs)
    with open(os.path.join(sparse, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", views))
        for k in range(views):
            q = rng.normal(size=4)
            q /= np.linalg.norm(q)
            f.write(struct.pack("<idddddddi", k + 1, *q, *rng.normal(size=3), 1) + b"view_%04d.jpg\x00" % k)
            f.write(struct.pack("<Q", obs) + o.tobytes())
    rec = np.zeros(points, dtype=[("id", "<u8"), ("xyz", "<f8", 3), ("rgb", "u1", 3), ("err", "<f8"), ("n", "<u8"),
                                  ("track", "<i4", 16)])
    rec["id"] = np.arange(1, points + 1)
    rec["xyz"], rec["rgb"] = rng.normal(size=(points, 3)), rng.integers(0, 256, (points, 3))
    rec["err"], rec["n"] = rng.uniform(0, 2, points), 8
    with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", points) + rec.tobytes())
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([128 + 100 * np.sin(xx / 97.0 + c) * np.cos(yy / 61.0 - c) for c in range(3)], axis=-1)
    base = np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)
    for d in ("images", "images_png"):
        os.makedirs(os.path.join(root, d))
    for k in range(views):
        im = Image.fromarray(np.roll(base, 37 * k, axis=1))
        im.save(os.path.join(root, "images", "view_%04d.jpg" % k), quality=95)
        im.save(os.path.join(root, "images_png", "view_%04d.jpg" % k), format="PNG", compress_level=1)


def median_time(fn, rounds):
    ts = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--obs", type=int, default=50_000)
    ap.add_argument("--points", type=int, default=200_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    pin = torch.cuda.is_available()
    pool = min(32, os.cpu_count() or 1)
    print(f"[host] {os.cpu_count()} CPUs, {cpu_model()}; default pool {pool} threads; pinned={pin}", flush=True)
    root = tempfile.mkdtemp(prefix="scene_load_", dir=a.dir)
    try:
        t0 = time.perf_counter()
        write_dataset(root, a.views, a.obs, a.points)
        print(f"[setup] dataset written in {time.perf_counter() - t0:.1f} s", flush=True)
        sparse = os.path.join(root, "sparse", "0")

        def line(what, t, ts, **kw):
            print(json.dumps(dict(what=what, seconds=round(t, 4), rounds=[round(x, 4) for x in ts], views=a.views,
                                  **kw)), flush=True)

        t, ts = median_time(lambda: scene._read_images_bin(os.path.join(sparse, "images.bin")), a.rounds)
        line("images.bin", t, ts, observations=a.views * a.obs,
             mbytes=round(os.path.getsize(os.path.join(sparse, "images.bin")) / 1e6, 1))
        t, ts = median_time(lambda: scene._read_points_bin(os.path.join(sparse, "points3D.bin")), a.rounds)
        line("points3D.bin", t, ts, points=a.points)
        for folder, fmt in (("images", "jpeg"), ("images_png", "png")):
            t, ts = median_time(lambda: scene.read_colmap_scene(root, images=folder), a.rounds)
            line("read_colmap_scene", t, ts, format=fmt, observations=a.views * a.obs, points=a.points)
            views = scene.read_colmap_scene(root, images=folder).train
            for threads in (1, pool):
                t, ts = median_time(lambda: scene.load_images(views, threads=threads, pin=pin), a.rounds)
                line("load_images", t, ts, format=fmt, threads=threads, pinned=pin, width=W, height=H,
                     ms_per_view=round(1e3 * t / a.views, 2))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
