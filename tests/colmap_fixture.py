"""COLMAP models written from scratch for the scene tests: the binary and text forms of cameras, images and points3D
(COLMAP's read_write_model layout), and a small seeded scene that exercises the reader's rules.

The fixture scene has 13 views with non-contiguous ids in unsorted file order, all three accepted camera models with
several intrinsics (and an unused SIMPLE_RADIAL camera the binary reader must walk past), a name with a subdirectory and
one with two dots, RGB and RGBA PNGs and a JPEG at 40 x 30 in images/ and 20 x 15 in images_2/, and a point cloud of
a few hundred points with tracks of 0 to 9 observations.  Every number comes from a seeded generator, so the golden
expectations (tests/golden/make_colmap_golden.py) hold for every checkout."""
import os
import struct

import numpy as np

MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4}
IMAGE_SIZE = (40, 30)       # (W, H) of images/
HALF_SIZE = (20, 15)        # (W, H) of images_2/


def fixture_model(seed=7):
    """-> (cams [(id, model, W, H, params)], images [(id, qvec, tvec, camera id, stored name, number of 2D points)],
    points (xyz (N, 3) float64, rgb (N, 3) int, error (N,), track lengths (N,)))."""
    rng = np.random.default_rng(seed)
    cams = [(11, "PINHOLE", 80, 60, [70.5, 66.25, 40.0, 30.0]),
            (2, "SIMPLE_PINHOLE", 80, 60, [61.3, 40.0, 30.0]),
            (7, "SIMPLE_RADIAL", 80, 60, [60.0, 40.0, 30.0, 0.01]),
            (5, "OPENCV", 96, 72, [80.1, 79.7, 48.0, 36.0, 0.02, -0.01, 0.001, 0.002]),
            (9, "PINHOLE", 80, 60, [55.0, 58.5, 40.5, 29.5])]
    names = ["frame_0009.png", "frame_0002.png", "sub/dir/frame_0011.png", "frame_0001.png", "frame.v2.final.png",
             "frame_0005.jpg", "frame_0013.png", "frame_0004.png", "frame_0010.png", "frame_0003.png",
             "frame_0007.png", "frame_0012.png", "frame_0006.png"]
    ids = [40, 3, 17, 8, 101, 6, 55, 21, 9, 12, 77, 2, 64]
    used = [11, 2, 5, 9]
    images = []
    for k, (iid, name) in enumerate(zip(ids, names)):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        t = rng.normal(size=3) * 2.0
        images.append((iid, q, t, used[k % len(used)], name, int(rng.integers(0, 50))))
    n = 317
    xyz = rng.normal(size=(n, 3)) * 3.0
    rgb = rng.integers(0, 256, (n, 3))
    rgb[:3] = [[0, 0, 0], [255, 255, 255], [1, 128, 254]]
    err = rng.uniform(0.0, 2.0, n)
    tracks = rng.integers(0, 10, n)
    return cams, images, (xyz, rgb, err, tracks)


def write_model(sparse, cams, images, points, fmt="bin", seed=0):
    """The model as COLMAP writes it, in `fmt` ("bin" or "txt"); the 2D observations and tracks are seeded filler."""
    os.makedirs(sparse, exist_ok=True)
    rng = np.random.default_rng(seed)
    xyz, rgb, err, tracks = points
    if fmt == "bin":
        with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(cams)))
            for cid, model, w, h, params in cams:
                f.write(struct.pack("<iiQQ", cid, MODEL_IDS[model], w, h) + struct.pack("<%dd" % len(params), *params))
        with open(os.path.join(sparse, "images.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(images)))
            for iid, q, t, cid, name, m in images:
                f.write(struct.pack("<idddddddi", iid, *q, *t, cid) + name.encode() + b"\x00" + struct.pack("<Q", m))
                for _ in range(m):
                    f.write(struct.pack("<ddq", *rng.uniform(0, 40, 2), int(rng.integers(-1, len(xyz)))))
        with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(xyz)))
            for i in range(len(xyz)):
                f.write(struct.pack("<QdddBBBd", i + 1, *xyz[i], *(int(c) for c in rgb[i]), err[i]))
                f.write(struct.pack("<Q", int(tracks[i])))
                for _ in range(int(tracks[i])):
                    f.write(struct.pack("<ii", int(rng.integers(1, 200)), int(rng.integers(0, 50))))
    else:
        with open(os.path.join(sparse, "cameras.txt"), "w") as f:
            f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
            for cid, model, w, h, params in cams:
                f.write(" ".join([str(cid), model, str(w), str(h)] + [repr(float(p)) for p in params]) + "\n")
        with open(os.path.join(sparse, "images.txt"), "w") as f:
            f.write("# Image list with two lines of data per image:\n")
            for iid, q, t, cid, name, m in images:
                f.write(" ".join([str(iid)] + [repr(float(v)) for v in (*q, *t)] + [str(cid), name]) + "\n")
                obs = [(float(rng.uniform(0, 40)), float(rng.uniform(0, 40)), int(rng.integers(-1, len(xyz))))
                       for _ in range(m)]
                f.write(" ".join("%r %r %d" % o for o in obs) + "\n")
        with open(os.path.join(sparse, "points3D.txt"), "w") as f:
            f.write("# 3D point list with one line of data per point:\n")
            for i in range(len(xyz)):
                track = " ".join("%d %d" % (rng.integers(1, 200), rng.integers(0, 50)) for _ in range(int(tracks[i])))
                f.write(" ".join([str(i + 1)] + [repr(float(v)) for v in xyz[i]] + [str(int(c)) for c in rgb[i]] +
                                 [repr(float(err[i]))]) + (" " + track if track else "") + "\n")


def write_images(folder, names, size, seed=0):
    """Small seeded images under their basenames: RGBA for every third PNG, RGB otherwise, and JPEG for .jpg names."""
    from PIL import Image
    os.makedirs(folder, exist_ok=True)
    rng = np.random.default_rng(seed)
    W, H = size
    for k, name in enumerate(names):
        base = os.path.basename(name)
        if base.endswith(".jpg"):
            Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(folder, base), quality=90)
        elif k % 3 == 0:
            Image.fromarray(rng.integers(0, 256, (H, W, 4), dtype=np.uint8), "RGBA").save(os.path.join(folder, base))
        else:
            Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(folder, base))


def write_fixture(root, fmt="bin", seed=7):
    """The fixture scene under `root` (sparse/0 in `fmt`, images/ and images_2/) -> fixture_model(seed)."""
    cams, images, points = fixture_model(seed)
    write_model(os.path.join(root, "sparse", "0"), cams, images, points, fmt)
    names = [im[4] for im in images]
    write_images(os.path.join(root, "images"), names, IMAGE_SIZE)
    write_images(os.path.join(root, "images_2"), names, HALF_SIZE, seed=1)
    return cams, images, points
