"""gs_b200.scene on the CPU: a COLMAP scene read as the reference's readColmapSceneInfo reads it.

  * the fixture scene (tests/colmap_fixture.py) gives the reference's names, order, R, T, FoV, sizes, split, extent,
    point cloud, world-view and projection matrices bit for bit: against tests/golden/colmap_scene.npz, and against the
    reference's own code (tests/golden/make_colmap_golden.py, in a subprocess) when its checkout is present;
  * the .txt model reads as the .bin one does, and sparse/0/points3D.ply takes precedence when present;
  * images decode as PILtoTorch decodes them, for RGB and RGBA PNGs and a JPEG;
  * held_images gives the reference's three holding rules at world sizes 1, 2 and 3;
  * every refusal is raised."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import colmap_fixture as fx
from gs_b200 import point_cloud, scene
from gs_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = "/root/reference"
GOLDEN = os.path.join(ROOT, "tests", "golden", "colmap_scene.npz")


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("colmap"))
    fx.write_fixture(root, "bin")
    return root


def golden_of_reference(tmp_path):
    if not os.path.exists(os.path.join(REFERENCE, "scene", "dataset_readers.py")):
        pytest.skip("the reference checkout is not present")
    out = str(tmp_path / "colmap_scene.npz")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "golden", "make_colmap_golden.py"),
                        "--reference", REFERENCE, "--out", out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(np.load(out))


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def check_against(g, root):
    full = scene.read_colmap_scene(root)
    held = scene.read_colmap_scene(root, eval=True)
    half = scene.read_colmap_scene(root, images="images_2")
    v = full.train
    assert full.test == [] and [x.name for x in v] == list(g["names"])
    assert [x.name for x in held.train] == list(g["names_train_eval"])
    assert [x.name for x in held.test] == list(g["names_test_eval"])
    assert same(np.stack([x.R for x in v]), g["R"]) and same(np.stack([x.T for x in v]), g["T"])
    assert same(np.array([x.FoVx for x in v]), g["FoVx"]) and same(np.array([x.FoVy for x in v]), g["FoVy"])
    assert [x.width for x in v] == list(g["width"]) and [x.height for x in v] == list(g["height"])
    assert [x.width for x in half.train] == list(g["width_2"]) and [x.height for x in half.train] == list(g["height_2"])
    # with -i images_2 the size is the file's and the field of view the full-resolution intrinsics'
    assert same(np.array([x.FoVx for x in half.train]), g["FoVx_2"]) and same(g["FoVx_2"], g["FoVx"])
    assert same(np.array([x.FoVy for x in half.train]), g["FoVy_2"])
    assert np.float64(full.extent) == g["extent"] and np.float64(held.extent) == g["extent_eval"]
    assert same(full.xyz, g["xyz"]) and same(full.rgb, g["rgb"])
    cams = scene.cameras(v, device="cpu")
    for k, c in enumerate(cams):
        assert c["uid"] == k and (c["image_width"], c["image_height"]) == (v[k].width, v[k].height)
        assert same(c["viewmatrix"], np.ascontiguousarray(g["world_view"][k].T))
        assert c["tanfovx"] == g["tanfovx"][k] and c["tanfovy"] == g["tanfovy"][k]
        assert same(syn.projection_matrix(syn.ZNEAR, syn.ZFAR, c["FoVx"], c["FoVy"]), g["proj"][k])
    return full


def test_fixture_matches_golden(dataset):
    check_against(dict(np.load(GOLDEN)), dataset)


def test_fixture_matches_reference_code(dataset, tmp_path):
    g = golden_of_reference(tmp_path)
    check_against(g, dataset)
    committed = dict(np.load(GOLDEN))
    assert set(committed) == set(g) and all(same(committed[k], g[k]) for k in g), "the committed golden is stale"


def test_text_model_reads_as_binary(dataset, tmp_path):
    txt = str(tmp_path / "txt")
    fx.write_fixture(txt, "txt")
    a = scene.read_colmap_scene(dataset, eval=True)
    b = scene.read_colmap_scene(txt, eval=True)
    for x, y in zip(a.train + a.test, b.train + b.test):
        assert x.name == y.name and x.colmap_id == y.colmap_id and (x.width, x.height) == (y.width, y.height)
        assert same(x.R, y.R) and same(x.T, y.T) and x.FoVx == y.FoVx and x.FoVy == y.FoVy
    assert len(a.train) == len(b.train) and len(a.test) == len(b.test) and a.extent == b.extent
    assert same(a.xyz, b.xyz) and same(a.rgb, b.rgb)


def test_points3D_ply_takes_precedence(dataset, tmp_path):
    root = str(tmp_path / "ply")
    shutil.copytree(dataset, root)
    xyz = np.arange(12, dtype=np.float32).reshape(4, 3) * 0.25
    rgb = np.array([[1, 2, 3], [4, 5, 6], [7, 8, 9], [250, 251, 252]], np.uint8)
    rows = np.zeros(4, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                              ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    for k, a in enumerate("xyz"):
        rows[a] = xyz[:, k]
    for k, a in enumerate(("red", "green", "blue")):
        rows[a] = rgb[:, k]
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 4\n" +
              "".join(f"property float {a}\n" for a in ("x", "y", "z", "nx", "ny", "nz")) +
              "".join(f"property uchar {a}\n" for a in ("red", "green", "blue")) + "end_header\n")
    with open(os.path.join(root, "sparse", "0", "points3D.ply"), "wb") as f:
        f.write(header.encode() + rows.tobytes())
    s = scene.read_colmap_scene(root)
    assert same(s.xyz, xyz) and same(s.rgb, rgb)


def test_nothing_is_written_into_the_dataset(dataset):
    before = sorted(os.walk(dataset))
    scene.read_colmap_scene(dataset, eval=True)
    assert sorted(os.walk(dataset)) == before


def test_images_decode_as_piltotorch(dataset):
    from PIL import Image
    s = scene.read_colmap_scene(dataset)
    imgs = scene.load_images(s.train, pin=False)
    modes = set()
    for v, img in zip(s.train, imgs):
        with Image.open(v.image_path) as im:
            modes.add((im.format, im.mode))
            want = np.array(im)[..., :3].transpose(2, 0, 1)
        assert img.dtype == torch.uint8 and img.is_contiguous() and np.array_equal(img.numpy(), want), v.name
    assert {("PNG", "RGB"), ("PNG", "RGBA"), ("JPEG", "RGB")} <= modes
    one = scene.load_images(s.train, threads=1, pin=False)
    assert all(torch.equal(a, b) for a, b in zip(imgs, one))


def test_held_images_rules():
    for world in (1, 2, 3):
        for rank in range(world):
            assert scene.held_images(7, rank, world) == [True] * 7
            assert scene.held_images(7, rank, world, distributed_dataset_storage=True) == [rank == 0] * 7
            assert scene.held_images(7, rank, world, local_sampling=True) == [p % world == rank for p in range(7)]
    with pytest.raises(ValueError, match="distributed_dataset_storage"):
        scene.held_images(7, 0, 2, distributed_dataset_storage=True, local_sampling=True)
    with pytest.raises(ValueError, match="rank"):
        scene.held_images(7, 2, 2)


def test_load_images_holds_only_listed(dataset):
    s = scene.read_colmap_scene(dataset)
    held = scene.held_images(len(s.train), 1, 3, local_sampling=True)
    imgs = scene.load_images(s.train, held, pin=False)
    assert [i is not None for i in imgs] == held


def test_cameras_extent_keeps_its_bits():
    """The shared getNerfppNorm tail gives cameras_extent the bits of its former (N, 3) float64 formula."""
    rng = np.random.default_rng(5)
    for n in (1, 2, 7, 8, 9, 13, 100, 129, 1000):
        c = rng.normal(size=(n, 3)) * rng.uniform(0.1, 50.0)
        cams = [dict(campos=c[i].astype(np.float32)) for i in range(n)]
        centers = np.stack([np.asarray(d["campos"], dtype=np.float64) for d in cams])
        old = float(np.linalg.norm(centers - centers.mean(axis=0, keepdims=True), axis=1).max() * 1.1)
        assert point_cloud.cameras_extent(cams) == old


# -- refusals ----------------------------------------------------------------------------------------------------------
def copy_of(dataset, tmp_path, name="bad"):
    root = str(tmp_path / name)
    shutil.copytree(dataset, root)
    return root


def test_refuses_missing_sparse(tmp_path):
    with pytest.raises(ValueError, match="sparse"):
        scene.read_colmap_scene(str(tmp_path))


@pytest.mark.parametrize("stem", ["cameras", "images", "points3D"])
def test_refuses_truncated_binary(dataset, tmp_path, stem):
    root = copy_of(dataset, tmp_path)
    p = os.path.join(root, "sparse", "0", stem + ".bin")
    data = open(p, "rb").read()
    with open(p, "wb") as f:
        f.write(data[:-5])
    with open(os.path.join(root, "sparse", "0", stem + ".txt"), "w") as f:   # no fallback to text
        f.write("")
    with pytest.raises(ValueError, match=stem + r"\.bin.*truncated"):
        scene.read_colmap_scene(root)


def test_refuses_unknown_camera_id(dataset, tmp_path):
    root = copy_of(dataset, tmp_path)
    cams, images, points = fx.fixture_model()
    images[3] = images[3][:3] + (99,) + images[3][4:]
    fx.write_model(os.path.join(root, "sparse", "0"), cams, images, points)
    with pytest.raises(ValueError, match=r"images\.bin.*camera id 99"):
        scene.read_colmap_scene(root)


def test_refuses_distorted_model(dataset, tmp_path):
    root = copy_of(dataset, tmp_path)
    cams, images, points = fx.fixture_model()
    images[0] = images[0][:3] + (7,) + images[0][4:]   # the SIMPLE_RADIAL camera
    fx.write_model(os.path.join(root, "sparse", "0"), cams, images, points)
    with pytest.raises(ValueError, match="camera 7 is SIMPLE_RADIAL"):
        scene.read_colmap_scene(root)


def test_refuses_missing_image(dataset, tmp_path):
    root = copy_of(dataset, tmp_path)
    os.remove(os.path.join(root, "images", "frame_0004.png"))
    with pytest.raises(ValueError, match="frame_0004.png.*missing"):
        scene.read_colmap_scene(root)


def test_refuses_mixed_sizes(dataset, tmp_path):
    from PIL import Image
    root = copy_of(dataset, tmp_path)
    Image.new("RGB", (41, 30)).save(os.path.join(root, "images", "frame_0004.png"))
    with pytest.raises(ValueError, match="different sizes"):
        scene.read_colmap_scene(root)


def test_refuses_empty_training_set(dataset, tmp_path):
    root = copy_of(dataset, tmp_path)
    cams, images, points = fx.fixture_model()
    fx.write_model(os.path.join(root, "sparse", "0"), cams, images[:1], points)
    assert len(scene.read_colmap_scene(root).train) == 1
    with pytest.raises(ValueError, match="no training view"):
        scene.read_colmap_scene(root, eval=True)


@pytest.mark.parametrize("mode", ["L", "LA", "P", "I;16", "CMYK"])
def test_refuses_image_modes(tmp_path, mode):
    from PIL import Image
    p = str(tmp_path / ("x.jpg" if mode == "CMYK" else "x.png"))
    Image.new(mode, (8, 6)).save(p)
    with pytest.raises(ValueError, match="image mode"):
        scene.decode_image(p)
