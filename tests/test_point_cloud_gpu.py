"""-m gpu: starting a model from a point cloud on one H100.

  * the Morton-tree 3-NN search (gs_knn3_mean_dist2_range, the CUDA path of distCUDA2) against the exhaustive kernel
    gs_knn3_mean_dist2, bit for bit, over sizes at the leaf and tree-level boundaries and clouds that stress the
    pruning: clusters with far outliers, one repeated point, many duplicates, zero-extent axes, an integer lattice
    (exactly tied distances), an off-origin dense cloud and coordinates near +-1e38 (distances that overflow to inf);
  * query ranges: every rank's range of W = 1..4 is the slice of the whole answer; non-finite input is refused;
  * point_cloud.init_model against create_from_pcd written out in torch with the exhaustive kernel, bit for bit, at SH
    degrees 0..3, its W = 1..4 shards concatenating to the W = 1 model; a Trainer built from it trains, and its PLY
    reads back with the same bits."""
import math

import numpy as np
import pytest
import torch

import gpu_util as gu
import knn_ref
from gs_b200 import model_io, pipeline, point_cloud
from gs_b200 import synthetic as syn
from simple_knn import _C as knn

pytestmark = pytest.mark.gpu

KINDS = ("uniform", "clustered", "identical", "duplicates", "collinear", "coplanar", "lattice", "offset", "huge")
SIZES = (1, 2, 3, 4, 31, 32, 33, 257, 1023, 1024, 1025, 2049, 100_000)


def cloud(kind, n, seed=0):
    """(n, 3) float32 test clouds."""
    rng = np.random.default_rng([seed, n, KINDS.index(kind)])
    if kind == "uniform":
        p = rng.uniform(-1.0, 1.0, (n, 3))
    elif kind == "clustered":   # SfM-like: dense clusters, a sparse background, outliers 1e4 x further out
        centers = rng.uniform(-5.0, 5.0, (max(1, n // 2000), 3))
        p = centers[rng.integers(0, len(centers), n)] + rng.normal(0.0, 0.02, (n, 3))
        bg = rng.random(n) < 0.1
        p[bg] = rng.uniform(-5.0, 5.0, (int(bg.sum()), 3))
        out = rng.random(n) < 0.005
        p[out] = rng.normal(0.0, 5e4, (int(out.sum()), 3))
    elif kind == "identical":
        p = np.tile([[0.3, -0.2, 0.7]], (n, 1))
    elif kind == "duplicates":
        base = rng.uniform(-1.0, 1.0, (max(1, n // 4), 3))
        p = base[rng.integers(0, len(base), n)]
    elif kind == "collinear":   # two zero-extent axes
        p = np.stack([rng.uniform(-2.0, 2.0, n), np.full(n, 1.5), np.full(n, -2.0)], 1)
    elif kind == "coplanar":    # one zero-extent axis
        p = np.stack([rng.uniform(-2.0, 2.0, n), rng.uniform(-1.0, 1.0, n), np.full(n, 3.0)], 1)
    elif kind == "lattice":     # integer grid: many exactly tied distances
        a = max(1, math.ceil(n ** (1 / 3)))
        i = rng.permutation(n)
        p = np.stack([i % a, (i // a) % a, i // (a * a)], 1).astype(np.float64)
    elif kind == "offset":
        p = np.array([30.0, -20.0, 15.0]) + rng.uniform(-0.02, 0.02, (n, 3))
    elif kind == "huge":        # near +-1e38: every distinct pair's distance overflows to inf
        p = rng.choice([-1.0, 1.0], (n, 3)) * rng.uniform(0.5, 1.0, (n, 3)) * 1e38
        if n > 4:
            p[1::3] = p[0]
    return np.ascontiguousarray(p, dtype=np.float32)


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", SIZES)
def test_search_is_the_brute_force(kind, n):
    t = torch.from_numpy(cloud(kind, n)).to(gu.DEV)
    ref = knn._dist2_brute(t).cpu().numpy()
    got = knn._dist2_kernel(t).cpu().numpy()
    assert same_bits(got, ref), (kind, n, int((got.view(np.uint32) != ref.view(np.uint32)).sum()))


@pytest.mark.parametrize("kind,n", [("uniform", 3000), ("offset", 3000), ("clustered", 2049), ("lattice", 1000),
                                    ("huge", 257), ("duplicates", 300), ("uniform", 2), ("uniform", 3), ("uniform", 4)])
def test_both_kernels_are_the_pinned_arithmetic(kind, n):
    """The exhaustive kernel and the search against knn_ref, the numpy restatement of the fp32 arithmetic the exhaustive
    kernel has always compiled to (fma(dz, dz, fma(dx, dx, dy * dy))), bit for bit: pinning the distance in source kept
    distCUDA2's bits."""
    p = cloud(kind, n, seed=7)
    want = knn_ref.mean_dist2(p)
    t = torch.from_numpy(p).to(gu.DEV)
    assert same_bits(knn._dist2_brute(t).cpu().numpy(), want)
    assert same_bits(knn.distCUDA2(t).cpu().numpy(), want)


@pytest.mark.parametrize("kind", ("uniform", "clustered", "duplicates", "lattice"))
def test_search_is_the_brute_force_at_1m(kind):
    t = torch.from_numpy(cloud(kind, 1 << 20)).to(gu.DEV)
    ref = knn._dist2_brute(t).cpu().numpy()
    assert same_bits(knn.distCUDA2(t).cpu().numpy(), ref)


def test_distcuda2_is_the_brute_force():
    """The drop-in distCUDA2 of a CUDA tensor (any float dtype, non-contiguous) gives the exhaustive kernel's bits."""
    p = cloud("clustered", 30_001, seed=3)
    ref = knn._dist2_brute(torch.from_numpy(p).to(gu.DEV)).cpu().numpy()
    t = torch.from_numpy(p.astype(np.float64).T.copy()).to(gu.DEV).T
    assert not t.is_contiguous()
    assert same_bits(knn.distCUDA2(t).cpu().numpy(), ref)


@pytest.mark.parametrize("kind,n", [("clustered", 10_007), ("lattice", 4096), ("uniform", 5), ("uniform", 3),
                                    ("identical", 67)])
def test_rank_ranges_are_slices_of_the_whole(kind, n):
    t = torch.from_numpy(cloud(kind, n, seed=1)).to(gu.DEV)
    whole = knn._dist2_brute(t).cpu().numpy()
    for world in (1, 2, 3, 4):
        parts = []
        for rank in range(world):
            lo, hi = point_cloud.shard_range(n, rank, world)
            part = knn._dist2_range(t, lo, hi).cpu().numpy()
            assert same_bits(part, whole[lo:hi]), (world, rank)
            parts.append(part)
        assert same_bits(np.concatenate(parts), whole)
    assert same_bits(knn._dist2_range(t, n // 3, n // 3 + 1).cpu().numpy(), whole[n // 3:n // 3 + 1])


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_points_are_refused(bad):
    p = cloud("uniform", 1000)
    p[777, 1] = bad
    t = torch.from_numpy(p).to(gu.DEV)
    with pytest.raises(ValueError, match="not finite"):
        knn.distCUDA2(t)
    with pytest.raises(ValueError, match="not finite"):
        knn._dist2_range(t, 0, 10)      # a range without the bad point: the whole cloud is the search space
    with pytest.raises(ValueError, match="not finite"):
        point_cloud.init_model(p, np.zeros_like(p, dtype=np.uint8), 0, 2, 0, gu.DEV)


def test_workspace_size_and_refusal():
    """gs_knn3_temp_bytes grows with N (the sorted points, keys and order alone are 40 bytes per point), and a workspace
    one byte short is refused with GS_ENOMEM before any launch, leaving the output untouched."""
    from gs_b200 import _lib
    need = [_lib.query("gs_knn3_temp_bytes", n) for n in (0, 1, 1000, 1 << 20)]
    assert need == sorted(need) and need[0] > 0 and need[3] >= 40 * (1 << 20)
    n = 1000
    t = torch.from_numpy(cloud("uniform", n)).to(gu.DEV)
    out = torch.full((n,), 5.0, device=gu.DEV)
    temp = torch.empty((need[2],), dtype=torch.uint8, device=gu.DEV)
    stream = torch.cuda.current_stream().cuda_stream
    rc = _lib.query("gs_knn3_mean_dist2_range", n, t.data_ptr(), 0, n, out.data_ptr(), temp.data_ptr(), need[2] - 1,
                    stream)
    assert rc == -3 and b"too small" in _lib.load().gs_last_error()
    assert out.eq(5.0).all()
    _lib.call("gs_knn3_mean_dist2_range", n, t.data_ptr(), 0, n, out.data_ptr(), temp.data_ptr(), need[2], stream)
    assert same_bits(out.cpu().numpy(), knn._dist2_brute(t).cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------
# create_from_pcd
# ---------------------------------------------------------------------------------------------------------------------
def reference_create_from_pcd(xyz, rgb, max_sh_degree):
    """scene/dataset_readers.py:150-165 fetchPly's arrays and scene/gaussian_model.py:140-232 create_from_pcd at world
    size 1, written out in torch, with the exhaustive kernel as distCUDA2."""
    C0 = 0.28209479177387814
    points = np.vstack([xyz[:, 0], xyz[:, 1], xyz[:, 2]]).T
    colors = np.vstack([rgb[:, 0], rgb[:, 1], rgb[:, 2]]).T / 255.0
    fused_point_cloud = torch.tensor(np.asarray(points)).float().cuda().contiguous()
    fused_color = (torch.tensor(np.asarray(colors)).float().cuda() - 0.5) / C0
    features = torch.zeros((fused_color.shape[0], 3, (max_sh_degree + 1) ** 2)).float().cuda()
    features[:, :3, 0] = fused_color
    features[:, 3:, 1:] = 0.0
    dist2 = torch.clamp_min(knn._dist2_brute(torch.from_numpy(np.asarray(points)).float().cuda()), 0.0000001)
    scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
    rots = torch.zeros((fused_point_cloud.shape[0], 4), device="cuda")
    rots[:, 0] = 1
    x = 0.1 * torch.ones((fused_point_cloud.shape[0], 1), dtype=torch.float, device="cuda")
    opacities = torch.log(x / (1 - x))
    return {"xyz": fused_point_cloud, "f_dc": features[:, :, 0:1].transpose(1, 2).contiguous(),
            "f_rest": features[:, :, 1:].transpose(1, 2).contiguous(), "scaling": scales, "rotation": rots,
            "opacity": opacities}


def sfm_cloud(n, seed):
    rng = np.random.default_rng(seed)
    xyz = cloud("clustered", n, seed=seed)
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    rgb[:256, 0] = np.arange(256)   # every byte value
    return xyz, rgb


@pytest.mark.parametrize("D", [0, 1, 2, 3])
def test_init_model_is_create_from_pcd(D):
    xyz, rgb = sfm_cloud(20_011, seed=D)
    ref = reference_create_from_pcd(xyz, rgb, D)
    whole, shard = point_cloud.init_model(xyz, rgb, 0, 1, D, gu.DEV)
    assert shard == (0, len(xyz), len(xyz))
    for k, v in ref.items():
        assert whole[k].shape == v.shape and whole[k].is_contiguous(), k
        assert same_bits(whole[k].cpu().numpy(), v.cpu().numpy()), k
    for world in (2, 3, 4):
        parts = [point_cloud.init_model(xyz, rgb, r, world, D, gu.DEV) for r in range(world)]
        assert [s for _, s in parts] == [(*point_cloud.shard_range(len(xyz), r, world), len(xyz)) for r in range(world)]
        for k in ref:
            cat = torch.cat([p[k] for p, _ in parts]).cpu().numpy()
            assert same_bits(cat, whole[k].cpu().numpy()), (world, k)


def test_trainer_from_the_point_cloud_trains_and_saves(tmp_path):
    W, H, n = 256, 192, 30_000
    cams = [syn.make_camera(W, H, yaw_deg=2.0 * q - 3.0, uid=q) for q in range(4)]
    gts = [torch.from_numpy(syn.make_gt_image(W, H, seed=40 + q)).pin_memory() for q in range(4)]
    xyz = syn.make_scene(n, W, H, seed=5)["means3D"]
    rgb = np.random.default_rng(5).integers(0, 256, (n, 3), dtype=np.uint8)
    path = str(tmp_path / "points3D.ply")
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n + b"".join(
        b"property float %s\n" % a for a in (b"x", b"y", b"z", b"nx", b"ny", b"nz")) +
        b"property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    rec = np.zeros(n, dtype=[(a, "<f4") for a in ("x", "y", "z", "nx", "ny", "nz")] +
                   [(a, "u1") for a in ("red", "green", "blue")])
    for j, a in enumerate("xyz"):
        rec[a] = xyz[:, j]
    for j, a in enumerate(("red", "green", "blue")):
        rec[a] = rgb[:, j]
    with open(path, "wb") as f:
        f.write(header + rec.tobytes())
    xyz2, rgb2 = point_cloud.read_point_cloud(path)
    assert same_bits(xyz2, xyz) and np.array_equal(rgb2, rgb)
    params, shard = point_cloud.init_model(xyz2, rgb2, 0, 1, 3, gu.DEV)
    tr = pipeline.Trainer(None, cams, gts, gu.DEV, model=params, shard=shard)
    tr.params.active_sh_degree = 0
    losses = [tr.step(views=[q % 4, (q + 1) % 4], resident=False) for q in range(4)]
    assert all(math.isfinite(v) for v in losses), losses
    assert tr.params._xyz.grad is not None and torch.isfinite(tr.params._xyz.grad).all()
    folder = str(tmp_path / "point_cloud" / "iteration_0")
    model_io.save_ply(folder, tr)
    back, back_shard, D = model_io.load_ply(folder, device=gu.DEV)
    assert D == 3 and back_shard == shard
    for k, v in params.items():
        assert same_bits(back[k].cpu().numpy(), v.detach().cpu().numpy()), k
