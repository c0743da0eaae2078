"""-m gpu: a COLMAP scene loaded by gs_b200.scene drives the renderer and the Trainer on one H100.

  * device matrices: the loader's projmatrix and campos are the bmm and inverse of the golden world-view and projection
    matrices (tests/golden/colmap_scene.npz, the reference's own host matrices) on the device, bit for bit;
  * cameras and images pair up: a scene written in COLMAP form around a known synthetic model is loaded, the model is
    rendered at its held-out cameras (image_metrics(images=True)), the renders become the scene's images, and the
    reloaded images equal the 8-bit renders byte for byte and score PSNR = inf -- a camera / image mismatch, a flipped
    axis or a swapped channel fails here;
  * a model started from the scene's point cloud (init_model) trains over the loaded views with FusedAdam and one
    densify_and_prune at the scene's extent: the loss falls, and evaluate on the held-out views returns finite numbers."""
import math
import os

import numpy as np
import pytest
import torch

import colmap_fixture as fx
import gpu_util as gu
from gs_b200 import densify, pipeline, point_cloud, scene
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "colmap_scene.npz")
W, H, N_VIEWS, N_GAUSS = 160, 112, 12, 30_000


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def test_device_matrices_are_the_references():
    g = np.load(GOLDEN)
    views = [scene.View(str(g["names"][k]), "", k, g["R"][k], g["T"][k], float(g["FoVx"][k]), float(g["FoVy"][k]),
                        int(g["width"][k]), int(g["height"][k])) for k in range(len(g["names"]))]
    cams = scene.cameras(views, gu.DEV)
    for k, c in enumerate(cams):
        # scene/cameras.py:84-100 on the golden host matrices
        vm = torch.tensor(g["world_view"][k]).transpose(0, 1).to(gu.DEV)
        proj = torch.tensor(g["proj"][k]).transpose(0, 1).to(gu.DEV)
        full = vm.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
        campos = vm.inverse()[3, :3]
        assert same_bits(c["viewmatrix"], vm.cpu().numpy()), k
        assert same_bits(c["projmatrix"], full.cpu().numpy()), k
        assert same_bits(c["campos"], campos.cpu().numpy()), k
        assert c["tanfovx"] == g["tanfovx"][k] and c["tanfovy"] == g["tanfovy"][k], k


def rotmat2qvec(M):
    """A unit (w, x, y, z) quaternion of a rotation matrix (COLMAP's convention, the inverse of scene.qvec2rotmat)."""
    w = math.sqrt(max(0.0, 1.0 + M[0, 0] + M[1, 1] + M[2, 2])) / 2
    x = math.copysign(math.sqrt(max(0.0, 1.0 + M[0, 0] - M[1, 1] - M[2, 2])) / 2, M[2, 1] - M[1, 2])
    y = math.copysign(math.sqrt(max(0.0, 1.0 - M[0, 0] + M[1, 1] - M[2, 2])) / 2, M[0, 2] - M[2, 0])
    z = math.copysign(math.sqrt(max(0.0, 1.0 - M[0, 0] - M[1, 1] + M[2, 2])) / 2, M[1, 0] - M[0, 1])
    q = np.array([w, x, y, z])
    return q / np.linalg.norm(q)


def write_scene(root, model):
    """A COLMAP dataset of N_VIEWS cameras around the synthetic model's frustum (PINHOLE, 60 degrees across), with
    black placeholder images of the right size and a point cloud of every third Gaussian with its DC colour."""
    from PIL import Image
    fx_ = W / (2 * math.tan(math.radians(60.0) / 2))
    cams = [(3, "PINHOLE", W, H, [fx_, fx_, W / 2, H / 2])]
    rng = np.random.default_rng(11)
    images = []
    for k in range(N_VIEWS):
        a = math.radians(-8.0 + 16.0 * k / (N_VIEWS - 1))
        R = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
        t = np.array([0.3 * math.sin(3 * a), 0.1 * math.cos(5 * a), 0.2 * a])
        # world_to_view puts R.T top-left: COLMAP's world-to-camera rotation is R.T
        images.append((int(1000 - 7 * k), rotmat2qvec(R.T), t, 3, "view_%02d.png" % ((5 * k) % N_VIEWS), 0))
    rng.shuffle(images)
    pts = model["means3D"][::3].astype(np.float64)
    rgb = np.clip(model["shs"][::3, 0] * point_cloud.C0 + 0.5, 0.0, 1.0) * 255.0
    fx.write_model(os.path.join(root, "sparse", "0"), cams, images,
                   (pts, rgb.astype(np.int64), np.zeros(len(pts)), np.zeros(len(pts), np.int64)))
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    for im in images:
        Image.new("RGB", (W, H)).save(os.path.join(root, "images", im[4]))


def save_png(path, img):
    from PIL import Image
    Image.fromarray(img.permute(1, 2, 0).contiguous().numpy()).save(path)


@pytest.fixture(scope="module")
def rendered_scene(tmp_path_factory):
    """The dataset with every view's image replaced by the model's 8-bit render at the loaded camera."""
    root = str(tmp_path_factory.mktemp("colmap_gpu"))
    model = syn.make_scene(N_GAUSS, W, H, seed=21, radius_px=5.0)
    write_scene(root, model)
    first = scene.read_colmap_scene(root, eval=True, llffhold=4)
    tr = pipeline.Trainer(model, scene.cameras(first.train, gu.DEV), scene.load_images(first.train), gu.DEV,
                          deterministic=True)
    renders = {}
    for views in (first.train, first.test):
        m = tr.image_metrics(cams=scene.cameras(views, gu.DEV), gts=scene.load_images(views), images=True)
        for v, img in zip(views, m["images"]):
            renders[v.name] = img
    for v in first.train + first.test:
        save_png(v.image_path, renders[v.name])
    return root, model, renders


def test_loaded_images_pair_with_loaded_cameras(rendered_scene):
    root, model, renders = rendered_scene
    sc = scene.read_colmap_scene(root, eval=True, llffhold=4)
    assert len(sc.test) == 3 and len(sc.train) == N_VIEWS - 3
    test_imgs = scene.load_images(sc.test)
    assert all(g.is_pinned() for g in test_imgs)
    for v, g in zip(sc.test, test_imgs):
        assert torch.equal(g, renders[v.name]), v.name
    # the views differ from each other, so a pairing mistake cannot pass by accident
    assert not torch.equal(test_imgs[0], test_imgs[1]) and int(test_imgs[0].max()) > 100
    train_imgs = scene.load_images(sc.train)
    tr = pipeline.Trainer(model, scene.cameras(sc.train, gu.DEV), train_imgs, gu.DEV, deterministic=True)
    m = tr.image_metrics(cams=scene.cameras(sc.test, gu.DEV), gts=test_imgs)
    assert torch.isinf(m["psnr_per_view"]).all() and (m["ssim_per_view"] == 1.0).all(), m
    # the same images one view off score finite: the check can tell the pairs apart
    shifted = test_imgs[1:] + test_imgs[:1]
    m = tr.image_metrics(cams=scene.cameras(sc.test, gu.DEV), gts=shifted)
    assert torch.isfinite(m["psnr_per_view"]).all(), m


def test_train_from_the_scene(rendered_scene):
    root, _, _ = rendered_scene
    sc = scene.read_colmap_scene(root, eval=True, llffhold=4)
    cams = scene.cameras(sc.train, gu.DEV)
    gts = scene.load_images(sc.train, scene.held_images(len(sc.train)))
    params, shard = point_cloud.init_model(sc.xyz, sc.rgb, 0, 1, 3, gu.DEV)
    tr = pipeline.Trainer(None, cams, gts, gu.DEV, model=params, shard=shard, deterministic=True)
    lr = {"xyz": 0.00016 * sc.extent, "f_dc": 0.0025, "f_rest": 0.0025 / 20, "opacity": 0.05, "scaling": 0.005,
          "rotation": 0.001}
    opt = FusedAdam(tr.optimizer_groups(lr), lr=0.0, eps=1e-15)
    P0 = tr.n_local

    def fresh_stats():
        P = tr.n_local
        return torch.zeros((P, 1), device=gu.DEV), torch.zeros((P, 1), device=gu.DEV), torch.zeros((P,), device=gu.DEV)

    stats = fresh_stats()
    order = np.random.default_rng(2).permutation(np.tile(np.arange(len(cams)), 600 // len(cams) + 1))
    losses = []
    for it in range(300):
        views = [int(order[2 * it]), int(order[2 * it + 1])]
        losses.append(tr.step(views=views, resident=False))
        tr.add_densification_stats(*stats)
        opt.step(grad_scale=1.0 / len(views))
        if it == 150:
            res = densify.densify_and_prune(opt, stats[0], stats[1], 0.0002, 0.005, sc.extent, 0.01, None)
            tr.adopt_parameters(res)
            stats = fresh_stats()
    assert all(math.isfinite(x) for x in losses)
    first, last = float(np.mean(losses[:20])), float(np.mean(losses[-20:]))
    assert last < 0.7 * first, (first, last)
    assert tr.n_local != P0, "densify_and_prune changed nothing"
    e = tr.evaluate(cams=scene.cameras(sc.test, gu.DEV), gts=scene.load_images(sc.test))
    assert math.isfinite(e["l1"]) and math.isfinite(e["psnr"]), e
    assert torch.isfinite(e["l1_per_view"]).all() and torch.isfinite(e["psnr_per_view"]).all(), e
