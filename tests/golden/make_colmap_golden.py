"""Regenerate tests/golden/colmap_scene.npz: what the REFERENCE's own readColmapSceneInfo, getWorld2View2,
getProjectionMatrix and storePly -> fetchPly make of the fixture scene of tests/colmap_fixture.py (binary model).

    python tests/golden/make_colmap_golden.py [--reference DIR] [--out FILE]

Needs the reference checkout.  plyfile is replaced by an in-memory stand-in that keeps the structured array storePly
builds and hands it back to fetchPly, so the round trip's numbers are the reference's own casts; nothing is written
into the fixture's dataset directory.  The reference's .txt reader accepts PINHOLE cameras only, so its text path is
not exercised here (tests/test_scene_io.py checks that the .txt model reads as the .bin one does)."""
import argparse
import math
import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(ROOT, "grendel-gs_b200")


def reference_expectations(reference):
    sys.path[:0] = [reference, PKG, os.path.join(PKG, "shims"), os.path.dirname(HERE)]
    import colmap_fixture
    import utils.general_utils as utils
    import scene.dataset_readers as dr
    from utils.graphics_utils import getWorld2View2, getProjectionMatrix

    store = {}

    class PlyElement:
        @staticmethod
        def describe(elements, name):
            return elements

    class PlyData:
        def __init__(self, elements):
            self.vertex = elements[0]

        def write(self, path):
            store[path] = self.vertex

        @staticmethod
        def read(path):
            return {"vertex": store[path]}

    dr.PlyElement, dr.PlyData = PlyElement, PlyData
    utils.GLOBAL_RANK, utils.LOCAL_RANK = 0, 0
    utils.DEFAULT_GROUP = SimpleNamespace(size=lambda: 1)
    out = {}
    with tempfile.TemporaryDirectory() as root:
        colmap_fixture.write_fixture(root, "bin")
        full = dr.readColmapSceneInfo(root, "images", False, 8)
        held = dr.readColmapSceneInfo(root, "images", True, 8)
        half = dr.readColmapSceneInfo(root, "images_2", False, 8)
        assert not os.path.exists(os.path.join(root, "sparse", "0", "points3D.ply"))
    views = full.train_cameras
    out["names"] = np.array([c.image_name for c in views])
    out["names_train_eval"] = np.array([c.image_name for c in held.train_cameras])
    out["names_test_eval"] = np.array([c.image_name for c in held.test_cameras])
    out["R"] = np.stack([c.R for c in views])
    out["T"] = np.stack([c.T for c in views])
    out["FoVx"] = np.array([c.FovX for c in views])
    out["FoVy"] = np.array([c.FovY for c in views])
    out["width"] = np.array([c.width for c in views])
    out["height"] = np.array([c.height for c in views])
    out["FoVx_2"] = np.array([c.FovX for c in half.train_cameras])
    out["FoVy_2"] = np.array([c.FovY for c in half.train_cameras])
    out["width_2"] = np.array([c.width for c in half.train_cameras])
    out["height_2"] = np.array([c.height for c in half.train_cameras])
    out["extent"] = np.float64(full.nerf_normalization["radius"])
    out["extent_eval"] = np.float64(held.nerf_normalization["radius"])
    out["xyz"] = np.asarray(full.point_cloud.points)
    v = store[os.path.join(root, "sparse/0/points3D.ply")]
    out["rgb"] = np.stack([v["red"], v["green"], v["blue"]], axis=1)
    assert np.array_equal(full.point_cloud.colors, out["rgb"] / 255.0)
    # scene/cameras.py:84-94: the host matrices before their transpose and copy to the device
    out["world_view"] = np.stack([getWorld2View2(c.R, c.T, np.array([0.0, 0.0, 0.0]), 1.0) for c in views])
    out["proj"] = np.stack([getProjectionMatrix(znear=0.01, zfar=100.0, fovX=c.FovX, fovY=c.FovY).numpy()
                            for c in views])
    # gaussian_renderer: tanfovx = math.tan(viewpoint_camera.FoVx * 0.5)
    out["tanfovx"] = np.array([math.tan(c.FovX * 0.5) for c in views])
    out["tanfovy"] = np.array([math.tan(c.FovY * 0.5) for c in views])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    ap.add_argument("--out", default=os.path.join(HERE, "colmap_scene.npz"))
    a = ap.parse_args()
    np.savez(a.out, **reference_expectations(a.reference))
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
