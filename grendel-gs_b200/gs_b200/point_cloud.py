"""Starting a model from the scene's point cloud: the reference's create_from_pcd, one rank's shard at a time.

* read_point_cloud: fetchPly (scene/dataset_readers.py:150-165) of the SfM cloud `sparse/0/points3D.ply`, the file
  storePly (:167-190) writes: x y z nx ny nz as float, red green blue as uchar.
* init_model: GaussianModel.create_from_pcd (scene/gaussian_model.py:140-232) for one rank: this rank's six raw
  parameters, ready for Trainer(model=..., shard=...).  The 3-NN scale initialisation (distCUDA2) runs for the shard's
  points only, against the whole cloud, by the exact Morton-tree search (simple_knn._C, DESIGN.md 5i).
* cameras_extent: getNerfppNorm's radius (scene/dataset_readers.py:59-80), the spatial_lr_scale of
  model_io.save_checkpoint and the extent of densify.densify_and_prune.

No collective: every rank reads the file and builds its own shard.
"""
import numpy as np
import torch

from . import model_io

C0 = 0.28209479177387814   # utils/sh_utils.py: the degree-0 SH basis constant
COLOURS = ("red", "green", "blue")


def read_point_cloud(path):
    """A points3D.ply -> (xyz float32 (N, 3), rgb uint8 (N, 3)).  Takes any property order, extra properties, comments,
    and x / y / z stored as double (rounded to float32 as torch's .float() does).  Refuses, with a ValueError naming the
    file: what model_io.parse_ply_vertices refuses (ascii or big-endian data, a list property in the vertex element),
    x / y / z missing or not float / double, a colour missing or not uchar, a truncated body and zero points.  The
    reference's fallback to random colours for a file without them is not reproduced."""
    vertices = model_io.parse_ply_vertices(path)
    n, types, dtype, body = vertices
    for a in ("x", "y", "z"):
        if a not in types:
            raise ValueError(f"{path}: attribute {a!r} is missing")
        if model_io._PLY_TYPES[types[a]] not in ("<f4", "<f8"):
            raise ValueError(f"{path}: attribute {a!r} is {types[a]}, not float or double")
    for a in COLOURS:
        if a not in types:
            raise ValueError(f"{path}: colour {a!r} is missing")
        if model_io._PLY_TYPES[types[a]] != "u1":
            raise ValueError(f"{path}: colour {a!r} is {types[a]}, not uchar")
    model_io.check_ply_body(path, vertices)
    if n == 0:
        raise ValueError(f"{path}: the point cloud has no points")
    rec = model_io.read_ply_vertices(path, dtype, body, 0, n)
    xyz = np.stack([rec[a].astype(np.float32) for a in ("x", "y", "z")], axis=1)
    rgb = np.stack([rec[a] for a in COLOURS], axis=1)
    return xyz, rgb


def shard_range(n, rank, world):
    """The Trainer's contiguous shard [n rank // W, n (rank + 1) // W), as model_io.load_ply cuts a model."""
    return n * rank // world, n * (rank + 1) // world


def init_model(xyz, rgb, rank=0, world=1, max_sh_degree=3, device="cuda"):
    """create_from_pcd (scene/gaussian_model.py:140-232) for rank `rank` of `world`.
    xyz (N, 3) float, rgb (N, 3) uint8: the whole cloud (read_point_cloud).  -> (raw params {group name: tensor on
    device}, (lo, hi, N)): Gaussians [lo, hi) of shard_range, for Trainer(None, ..., model=params, shard=(lo, hi, N)).

    Every elementwise step is the reference's own torch sequence on the device (colours / 255.0 in float64, then
    .float(); RGB2SH; features[:, :3, 0]; clamp_min(dist2, 1e-7); log(sqrt(.)).repeat(1, 3); identity quaternions;
    inverse_sigmoid(0.1); the transpose(1, 2).contiguous() layouts), so the shard has the bits of the reference's rows
    [lo, hi).  The reference cuts ceil-sized chunks instead (utils/general_utils.py:272-276); the union over the ranks
    is the same model.

    A fresh reference model starts at active_sh_degree = 0 (GaussianModel.__init__), while GaussianParams.from_raw
    starts at the stored degree: a caller that follows the reference's schedule sets trainer.params.active_sh_degree = 0.
    """
    xyz = np.asarray(xyz)
    rgb = np.asarray(rgb)
    if xyz.ndim != 2 or xyz.shape[1] != 3 or rgb.shape != xyz.shape or rgb.dtype != np.uint8:
        raise ValueError(f"xyz must be (N, 3) and rgb (N, 3) uint8, got {xyz.shape} and {rgb.shape} {rgb.dtype}")
    if not 0 <= rank < world:
        raise ValueError(f"rank {rank} is not in [0, {world})")
    if int(max_sh_degree) not in (0, 1, 2, 3):
        raise ValueError(f"max_sh_degree must be 0..3, got {max_sh_degree}")
    from simple_knn._C import _dist2_range
    n = xyz.shape[0]
    lo, hi = shard_range(n, rank, world)
    K = (int(max_sh_degree) + 1) ** 2
    points = torch.tensor(xyz).float().to(device).contiguous()   # the whole cloud: every shard's neighbours
    with torch.no_grad():
        fused_point_cloud = points[lo:hi].clone()
        fused_color = (torch.tensor(rgb[lo:hi] / 255.0).float().to(device) - 0.5) / C0   # RGB2SH
        m = hi - lo
        features = torch.zeros((m, 3, K)).float().to(device)
        features[:, :3, 0] = fused_color
        features[:, 3:, 1:] = 0.0
        dist2 = torch.clamp_min(_dist2_range(points, lo, hi), 0.0000001)
        scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
        rots = torch.zeros((m, 4), device=device)
        rots[:, 0] = 1
        x = 0.1 * torch.ones((m, 1), dtype=torch.float, device=device)
        opacities = torch.log(x / (1 - x))   # inverse_sigmoid, utils/general_utils.py:279-280
        params = {"xyz": fused_point_cloud, "f_dc": features[:, :, 0:1].transpose(1, 2).contiguous(),
                  "f_rest": features[:, :, 1:].transpose(1, 2).contiguous(), "opacity": opacities,
                  "scaling": scales, "rotation": rots}
    return params, (lo, hi, n)


def cameras_extent(cams):
    """getNerfppNorm's radius (scene/dataset_readers.py:59-80): 1.1 x the largest distance of a camera centre from their
    mean, in float64, from the camera dicts' `campos` (synthetic.make_camera's layout)."""
    if not len(cams):
        raise ValueError("cameras_extent needs at least one camera")
    centers = np.stack([np.asarray(c["campos"], dtype=np.float64).reshape(3) for c in cams])
    return float(nerfpp_radius(centers.T))


def nerfpp_radius(cam_centers):
    """The tail of getNerfppNorm (scene/dataset_readers.py:60-76) over (3, N) camera centres, in their dtype: the largest
    distance from their mean, x 1.1.  numpy's reductions sum in an order set by the memory layout, so the bits depend
    on it: the reference's np.hstack of (3, 1) columns is C-contiguous (scene.read_colmap_scene passes that), while
    cameras_extent passes the transposed view of its (N, 3) rows."""
    center = np.mean(cam_centers, axis=1, keepdims=True)
    dist = np.linalg.norm(cam_centers - center, axis=0, keepdims=True)
    return np.max(dist) * 1.1
