"""Loading a COLMAP scene as the reference's Scene does (scene/__init__.py:50-55): its cameras, the held-out split, the
images and the SfM point cloud.  Host-side I/O, like model_io.

* read_colmap_scene: readColmapSceneInfo (scene/dataset_readers.py:83-148, 193-252) with the reference's bits: the
  views in name order, the llffhold split, getNerfppNorm's extent over the training views and the point cloud.
* cameras: the views as camera dicts (synthetic.make_camera's layout) whose matrices are formed as scene/cameras.py:84-100
  forms them, for Trainer(cams=...) and evaluate / image_metrics(cams=...).
* held_images / load_images: which images a rank holds (scene/cameras.py:52-63, utils/camera_utils.py:37-48) and their
  uint8 (3, H, W) host tensors, decoded as PILtoTorch does (utils/general_utils.py:348-361), for
  Trainer(gts_pinned=...) and evaluate / image_metrics(gts=...).

Three deliberate differences from the reference: a corrupt or truncated .bin raises instead of falling back to the .txt
files; the point cloud is converted in memory and nothing is written into the dataset directory (the reference writes
sparse/0/points3D.ply there on rank 0); and the views come in name order, not shuffled -- shuffling is the caller's.
Every rank reads the metadata itself: there is no collective.
"""
import math
import os
import struct
from concurrent.futures import ThreadPoolExecutor
from typing import NamedTuple

import numpy as np
import torch

from . import point_cloud
from . import synthetic

# COLMAP's camera models (src/colmap/sensor/models.h): id -> (name, number of parameters).  The binary reader needs every
# model's parameter count to walk cameras.bin; only the first three are accepted as views' cameras.
CAMERA_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5),
                 4: ("OPENCV", 8), 5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5),
                 8: ("SIMPLE_RADIAL_FISHEYE", 4), 9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}
ACCEPTED_MODELS = ("SIMPLE_PINHOLE", "PINHOLE", "OPENCV")   # OPENCV's distortion is ignored, as the reference does
IMAGE_MODES = ("RGB", "RGBA")   # PILtoTorch's [:3] of any other mode is not the image's RGB


class View(NamedTuple):
    """One registered image: R (the transposed world-to-camera rotation) and T as the reference's CameraInfo holds them,
    FoVx / FoVy from the intrinsics, width / height from the image file."""
    name: str          # the file's basename up to its first dot
    image_path: str
    colmap_id: int     # the image's id in images.bin
    R: np.ndarray      # (3, 3) float64
    T: np.ndarray      # (3,) float64
    FoVx: float
    FoVy: float
    width: int
    height: int


class ColmapScene(NamedTuple):
    train: list        # [View] in name order
    test: list         # [View] in name order; empty without eval
    extent: float      # getNerfppNorm's radius over the training views
    xyz: np.ndarray    # (N, 3) float32
    rgb: np.ndarray    # (N, 3) uint8


def qvec2rotmat(q):
    """COLMAP's world-to-camera rotation of a (w, x, y, z) quaternion (scene/colmap_loader.py:47-66)."""
    w, x, y, z = q
    return np.array([[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def focal2fov(focal, pixels):
    return 2 * math.atan(pixels / (2 * focal))


# -- the COLMAP model files --------------------------------------------------------------------------------------------
class _Bytes:
    """A binary model file read whole, unpacked at a cursor that refuses to run past its end."""

    def __init__(self, path):
        self.path = path
        with open(path, "rb") as f:
            self.data = f.read()
        self.pos = 0

    def take(self, fmt):
        n = struct.calcsize("<" + fmt)
        if self.pos + n > len(self.data):
            raise ValueError(f"{self.path}: truncated at byte {self.pos} ({len(self.data)} bytes)")
        out = struct.unpack_from("<" + fmt, self.data, self.pos)
        self.pos += n
        return out

    def skip(self, n):
        if self.pos + n > len(self.data):
            raise ValueError(f"{self.path}: truncated at byte {self.pos} ({len(self.data)} bytes)")
        self.pos += n

    def name(self):
        end = self.data.find(b"\x00", self.pos)
        if end < 0:
            raise ValueError(f"{self.path}: truncated in an image name at byte {self.pos}")
        s = self.data[self.pos:end].decode("utf-8")
        self.pos = end + 1
        return s

    def done(self):
        if self.pos != len(self.data):
            raise ValueError(f"{self.path}: {len(self.data) - self.pos} bytes after the last entry")


def _read_cameras_bin(path):
    """cameras.bin -> {camera id: (model name, width, height, params)}."""
    f, cams = _Bytes(path), {}
    for _ in range(f.take("Q")[0]):
        cid, model, w, h = f.take("iiQQ")
        if model not in CAMERA_MODELS:
            raise ValueError(f"{path}: camera {cid} has unknown model id {model}")
        name, k = CAMERA_MODELS[model]
        cams[cid] = (name, w, h, np.array(f.take("d" * k)))
    f.done()
    return cams


def _read_images_bin(path):
    """images.bin -> [(image id, qvec, tvec, camera id, name)] in file order.  The 2D observations are skipped by their
    count, not unpacked: a large model holds millions of them."""
    f, out = _Bytes(path), []
    for _ in range(f.take("Q")[0]):
        p = f.take("idddddddi")
        name = f.name()
        f.skip(24 * f.take("Q")[0])   # (x, y, point3D id) as double, double, int64
        out.append((p[0], np.array(p[1:5]), np.array(p[5:8]), p[8], name))
    f.done()
    return out


def _read_points_bin(path):
    """points3D.bin -> (xyz (N, 3) float64, rgb (N, 3) int); the tracks are skipped by their length."""
    f = _Bytes(path)
    n = f.take("Q")[0]
    xyz, rgb = np.empty((n, 3)), np.empty((n, 3), np.int64)
    for i in range(n):
        p = f.take("QdddBBBd")
        xyz[i], rgb[i] = p[1:4], p[4:7]
        f.skip(8 * f.take("Q")[0])    # (image id, point2D index) as int32, int32
    f.done()
    return xyz, rgb


def _text_lines(path):
    with open(path, "r") as f:
        return f.read().splitlines()


def _records(lines):
    """The non-comment, non-empty lines' indices."""
    return [i for i, s in enumerate(lines) if s.strip() and s.strip()[0] != "#"]


def _read_cameras_txt(path):
    lines, cams = _text_lines(path), {}
    names = {v[0] for v in CAMERA_MODELS.values()}
    for i in _records(lines):
        e = lines[i].split()
        if e[1] not in names:
            raise ValueError(f"{path}: camera {e[0]} has unknown model {e[1]}")
        cams[int(e[0])] = (e[1], int(e[2]), int(e[3]), np.array(tuple(map(float, e[4:]))))
    return cams


def _read_images_txt(path):
    """Two lines per image, as the reference reads them: the pose line, then the observations line, taken whatever it
    holds (it is empty for an image without observations)."""
    lines, out, i = _text_lines(path), [], 0
    while i < len(lines):
        s = lines[i].strip()
        i += 1
        if not s or s[0] == "#":
            continue
        e = s.split()
        out.append((int(e[0]), np.array(tuple(map(float, e[1:5]))), np.array(tuple(map(float, e[5:8]))), int(e[8]),
                    e[9]))
        i += 1
    return out


def _read_points_txt(path):
    lines = _text_lines(path)
    rows = [lines[i].split() for i in _records(lines)]
    xyz = np.array([tuple(map(float, e[1:4])) for e in rows]).reshape(-1, 3)
    rgb = np.array([tuple(map(int, e[4:7])) for e in rows], np.int64).reshape(-1, 3)
    return xyz, rgb


def _model_file(sparse, stem):
    """sparse/0/<stem>.bin, or <stem>.txt when the .bin is absent."""
    for ext in (".bin", ".txt"):
        p = os.path.join(sparse, stem + ext)
        if os.path.exists(p):
            return p, ext
    raise ValueError(f"{os.path.join(sparse, stem)}: neither .bin nor .txt exists")


# -- the scene ---------------------------------------------------------------------------------------------------------
def read_colmap_scene(path, images="images", eval=False, llffhold=8):
    """readColmapSceneInfo (scene/dataset_readers.py:193-252) of the COLMAP dataset at `path`, as Scene calls it
    (images: the reference's -i, e.g. "images_4"; llffhold: Scene's default of 8).  -> ColmapScene.

    Per view: R = qvec2rotmat(qvec).T and T = tvec in float64; FoVx / FoVy by focal2fov from the intrinsics' focal
    lengths, width and height; the size from the file images/<basename(name)> (with -i images_4 the field of view stays
    that of the full-resolution intrinsics); the name is that basename up to its first dot.  The views are stable-sorted
    by name; with eval, positions idx % llffhold == 0 are held out.  The extent is getNerfppNorm's radius over the
    training views, from np.linalg.inv of getWorld2View2's float32 matrices.  The point cloud is sparse/0/points3D.ply
    (point_cloud.read_point_cloud) if it exists, else points3D.bin or points3D.txt with the bits of the reference's
    storePly -> fetchPly round trip: xyz rounded to float32, colours as uint8.

    Refused with a ValueError naming the file or view: no sparse/0, a corrupt or truncated .bin, an image whose camera id
    is unknown or whose camera model is not SIMPLE_PINHOLE / PINHOLE / OPENCV, a missing image file, images of different
    sizes, an empty training set, and a point cloud that is missing, has colours outside 0..255 or has no points."""
    from PIL import Image
    sparse = os.path.join(path, "sparse", "0")
    if not os.path.isdir(sparse):
        raise ValueError(f"{sparse}: not a directory (no COLMAP model)")
    cam_path, ext = _model_file(sparse, "cameras")
    img_path, img_ext = _model_file(sparse, "images")
    intr = _read_cameras_bin(cam_path) if ext == ".bin" else _read_cameras_txt(cam_path)
    extr = _read_images_bin(img_path) if img_ext == ".bin" else _read_images_txt(img_path)
    folder = os.path.join(path, images)
    views = []
    for image_id, qvec, tvec, cid, stored in extr:
        if cid not in intr:
            raise ValueError(f"{img_path}: image {image_id} ({stored}) has camera id {cid}, which {cam_path} lacks")
        model, w, h, params = intr[cid]
        if model not in ACCEPTED_MODELS:
            raise ValueError(f"{cam_path}: camera {cid} is {model}; only undistorted models {ACCEPTED_MODELS} are "
                             f"supported (OPENCV's distortion is ignored)")
        fx = params[0]
        fy = params[0] if model == "SIMPLE_PINHOLE" else params[1]
        file = os.path.join(folder, os.path.basename(stored))
        if not os.path.isfile(file):
            raise ValueError(f"{file}: the image of view {stored} is missing")
        with Image.open(file) as im:   # the header only
            width, height = im.size
        views.append(View(os.path.basename(file).split(".")[0], file, int(image_id), np.transpose(qvec2rotmat(qvec)),
                          np.array(tvec), focal2fov(fx, w), focal2fov(fy, h), int(width), int(height)))
    views = sorted(views, key=lambda v: v.name)
    sizes = sorted({(v.width, v.height) for v in views})
    if len(sizes) > 1:
        odd = [v.image_path for v in views if (v.width, v.height) != (views[0].width, views[0].height)]
        raise ValueError(f"{folder}: the images have different sizes (W, H) {sizes}, e.g. {odd[0]}")
    if eval:
        train = [v for i, v in enumerate(views) if i % llffhold != 0]
        test = [v for i, v in enumerate(views) if i % llffhold == 0]
    else:
        train, test = views, []
    if not train:
        raise ValueError(f"{img_path}: no training view ({len(views)} views, eval={eval}, llffhold={llffhold})")
    centers = [np.linalg.inv(synthetic.world_to_view(v.R, v.T))[:3, 3:4] for v in train]
    extent = float(point_cloud.nerfpp_radius(np.hstack(centers)))
    xyz, rgb = _read_points(sparse)
    return ColmapScene(train, test, extent, xyz, rgb)


def _read_points(sparse):
    ply = os.path.join(sparse, "points3D.ply")
    if os.path.exists(ply):
        return point_cloud.read_point_cloud(ply)
    p = os.path.join(sparse, "points3D.bin")
    if os.path.exists(p):
        xyz, rgb = _read_points_bin(p)
    else:
        p = os.path.join(sparse, "points3D.txt")
        if not os.path.exists(p):
            raise ValueError(f"{sparse}: no points3D.ply, points3D.bin or points3D.txt")
        xyz, rgb = _read_points_txt(p)
    if len(xyz) == 0:
        raise ValueError(f"{p}: the point cloud has no points")
    if rgb.min() < 0 or rgb.max() > 255:
        raise ValueError(f"{p}: a colour is outside 0..255")
    return xyz.astype(np.float32), rgb.astype(np.uint8)


def cameras(views, device="cuda", sh_degree=3):
    """Camera dicts in synthetic.make_camera's layout, formed as the reference's Camera forms its matrices
    (scene/cameras.py:84-100): the float32 world-view matrix getWorld2View2(R, T) and the float32 projection
    getProjectionMatrix(0.01, 100, FoVx, FoVy) are built on the host and copied, transposed, to `device`; there
    projmatrix = viewmatrix.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0) and campos = viewmatrix.inverse()[3, :3] are
    computed by the same torch operations, so the bits that decide a render's tiles are the reference's on a CUDA device.
    The matrices come back as host float32 arrays.  uid is the view's position in `views`: pass the list in the order
    the Trainer is to hold it (the reference shuffles its training list with Python's random; this module does not)."""
    out = []
    for uid, v in enumerate(views):
        vm = torch.tensor(synthetic.world_to_view(v.R, v.T)).transpose(0, 1).to(device)
        proj = torch.from_numpy(synthetic.projection_matrix(synthetic.ZNEAR, synthetic.ZFAR, v.FoVx, v.FoVy))
        proj = proj.transpose(0, 1).to(device)
        full = vm.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
        campos = vm.inverse()[3, :3]
        out.append(dict(uid=uid, image_width=v.width, image_height=v.height, FoVx=v.FoVx, FoVy=v.FoVy,
                        tanfovx=math.tan(v.FoVx * 0.5), tanfovy=math.tan(v.FoVy * 0.5),
                        viewmatrix=vm.cpu().contiguous().numpy(), projmatrix=full.cpu().contiguous().numpy(),
                        campos=campos.cpu().contiguous().numpy(), sh_degree=int(sh_degree)))
    return out


# -- the images --------------------------------------------------------------------------------------------------------
def held_images(n, rank=0, world=1, distributed_dataset_storage=False, local_sampling=False):
    """Which of n views' images rank `rank` of `world` holds, as [bool] (scene/cameras.py:52-63,
    utils/camera_utils.py:37-48): every image by default; only rank 0's with distributed_dataset_storage; the views at
    positions p with p % world == rank with local_sampling.  The Trainer refuses the two options together, and so does
    this."""
    if not 0 <= rank < world:
        raise ValueError(f"rank {rank} is not in [0, {world})")
    if distributed_dataset_storage and local_sampling:
        raise ValueError("local_sampling: every rank holds the images of the views it samples; "
                         "distributed_dataset_storage has no meaning with it")
    if local_sampling:
        return [p % world == rank for p in range(n)]
    if distributed_dataset_storage:
        return [rank == 0] * n
    return [True] * n


def decode_image(path, pin=False):
    """PILtoTorch's image (utils/general_utils.py:348-361, camera_utils.py:60): Image.open, np.array, channels first,
    [:3] -> uint8 (3, H, W).  An RGBA image loses its alpha without compositing; no EXIF rotation is applied.  Modes
    other than RGB and RGBA are refused: PILtoTorch would turn them into the wrong channels."""
    from PIL import Image
    with Image.open(path) as im:
        if im.mode not in IMAGE_MODES:
            raise ValueError(f"{path}: image mode {im.mode!r}; only {IMAGE_MODES} decode to the image's RGB")
        a = np.array(im)
    if a.dtype != np.uint8 or a.ndim != 3:
        raise ValueError(f"{path}: decoded to {a.dtype} {a.shape}, not 8-bit channels")
    out = torch.empty((3, a.shape[0], a.shape[1]), dtype=torch.uint8, pin_memory=pin)
    out.copy_(torch.from_numpy(a).permute(2, 0, 1)[:3])
    return out


def load_images(views, held=None, threads=None, pin=True):
    """The images of `views` as uint8 (3, H, W) host tensors (decode_image), pinned by default, and None where
    held[i] is False (held_images): the list Trainer(gts_pinned=...) and evaluate / image_metrics(gts=...) take.
    Decoded on a pool of `threads` threads (default: one per CPU, up to 32); PIL releases the GIL while it decodes."""
    held = [True] * len(views) if held is None else list(held)
    if len(held) != len(views):
        raise ValueError(f"{len(views)} views but {len(held)} holding flags")
    todo = [i for i, h in enumerate(held) if h]
    out = [None] * len(views)
    if not todo:
        return out
    threads = min(32, os.cpu_count() or 1) if threads is None else int(threads)
    with ThreadPoolExecutor(max_workers=max(1, min(threads, len(todo)))) as pool:
        for i, img in zip(todo, pool.map(lambda i: decode_image(views[i].image_path, pin), todo)):
            out[i] = img
    for i in todo:
        if (out[i].shape[2], out[i].shape[1]) != (views[i].width, views[i].height):
            raise ValueError(f"{views[i].image_path}: decoded {tuple(out[i].shape)}, the view is "
                             f"{views[i].width} x {views[i].height}")
    return out
