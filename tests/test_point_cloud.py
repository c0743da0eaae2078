"""gs_b200.point_cloud on the CPU: reading the scene's points3D.ply, the shard rule, the cameras' extent, and the argument
checks of the 3-NN search's C ABI.

  * read_point_cloud takes storePly's layout (scene/dataset_readers.py:167-190), other property orders, extra
    properties, comments and double coordinates, and refuses what it cannot read with a ValueError naming the file;
  * shard_range is the Trainer's and model_io.load_ply's contiguous rule, covering every point once;
  * cameras_extent is getNerfppNorm's radius (scene/dataset_readers.py:59-80), restated in numpy from R and T;
  * gs_knn3_mean_dist2_range refuses bad sizes, ranges, pointers and a short workspace before any launch."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from gs_b200 import point_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORE_PLY = [("x", "float", "<f4"), ("y", "float", "<f4"), ("z", "float", "<f4"), ("nx", "float", "<f4"),
             ("ny", "float", "<f4"), ("nz", "float", "<f4"), ("red", "uchar", "u1"), ("green", "uchar", "u1"),
             ("blue", "uchar", "u1")]


def write_ply(path, props, n, values, fmt="binary_little_endian", pre=b"", post=b"", truncate=0):
    """props: [(name, PLY type, numpy type)]; values: {name: array of n}."""
    head = b"ply\nformat %s 1.0\n" % fmt.encode() + pre + b"element vertex %d\n" % n
    head += b"".join(b"property %s %s\n" % (t.encode(), a.encode()) for a, t, _ in props) + post + b"end_header\n"
    rec = np.zeros(n, dtype=[(a, nt) for a, _, nt in props])
    for a, _, _ in props:
        rec[a] = values.get(a, 0)[:n] if a in values else 0
    body = rec.tobytes()
    with open(path, "wb") as f:
        f.write(head + (body[:len(body) - truncate] if truncate else body))


def sample(n, seed=0):
    rng = np.random.default_rng(seed)
    xyz = rng.normal(0.0, 3.0, (n, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    vals = {"x": xyz[:, 0], "y": xyz[:, 1], "z": xyz[:, 2], "red": rgb[:, 0], "green": rgb[:, 1], "blue": rgb[:, 2]}
    return xyz, rgb, vals


def test_reads_storeply_layout(tmp_path):
    xyz, rgb, vals = sample(257)
    path = str(tmp_path / "points3D.ply")
    write_ply(path, STORE_PLY, 257, vals)
    got_xyz, got_rgb = point_cloud.read_point_cloud(path)
    assert got_xyz.dtype == np.float32 and got_xyz.shape == (257, 3)
    assert got_rgb.dtype == np.uint8 and got_rgb.shape == (257, 3)
    assert np.array_equal(got_xyz.view(np.uint32), xyz.view(np.uint32)) and np.array_equal(got_rgb, rgb)


def test_reads_other_orders_extra_properties_comments_and_doubles(tmp_path):
    import torch
    n = 100
    _, rgb, vals = sample(n, seed=1)
    xyz64 = np.random.default_rng(2).normal(0.0, 1e3, (n, 3)) * (1 + 1e-12)
    vals.update(x=xyz64[:, 0], y=xyz64[:, 1], z=xyz64[:, 2], error=np.linspace(0, 1, n), track=np.arange(n))
    props = [("blue", "uchar", "u1"), ("error", "double", "<f8"), ("z", "double", "<f8"), ("red", "uchar", "u1"),
             ("x", "double", "<f8"), ("track", "int", "<i4"), ("green", "uchar", "u1"), ("y", "double", "<f8")]
    path = str(tmp_path / "other.ply")
    write_ply(path, props, n, vals, pre=b"comment written by another tool\nobj_info x\n",
              post=b"element face 0\nproperty list uchar int vertex_indices\n")
    got_xyz, got_rgb = point_cloud.read_point_cloud(path)
    want = torch.tensor(xyz64).float().numpy()   # the reference's torch.tensor(points).float()
    assert np.array_equal(got_xyz.view(np.uint32), want.view(np.uint32))
    assert not np.array_equal(got_xyz.astype(np.float64), xyz64)   # rounding happened
    assert np.array_equal(got_rgb, rgb)


def test_refusals(tmp_path):
    n = 9
    _, _, vals = sample(n)
    no = lambda name: [p for p in STORE_PLY if p[0] != name]
    retype = lambda name, t, nt: [(a, t, nt) if a == name else (a, pt, pnt) for a, pt, pnt in STORE_PLY]
    cases = {
        "ascii": dict(props=STORE_PLY, fmt="ascii"),
        "big-endian": dict(props=STORE_PLY, fmt="binary_big_endian"),
        "list": dict(props=STORE_PLY[:6] + [("vertex_indices", "list uchar int", "<f4")] + STORE_PLY[6:]),
        "no-green": dict(props=no("green")),
        "float-red": dict(props=retype("red", "float", "<f4")),
        "ushort-blue": dict(props=retype("blue", "ushort", "<u2")),
        "no-y": dict(props=no("y")),
        "int-x": dict(props=retype("x", "int", "<i4")),
        "truncated": dict(props=STORE_PLY, truncate=1),
        "empty": dict(props=STORE_PLY, n=0),
    }
    for name, c in cases.items():
        path = str(tmp_path / f"{name}.ply")
        write_ply(path, c["props"], c.get("n", n), vals, fmt=c.get("fmt", "binary_little_endian"),
                  truncate=c.get("truncate", 0))
        with pytest.raises(ValueError, match=f"{name}.ply"):
            point_cloud.read_point_cloud(path)


@pytest.mark.parametrize("n", [0, 1, 3, 7, 1000, 12_345_679])
def test_shard_rule(n):
    for world in (1, 2, 3, 4, 8):
        ranges = [point_cloud.shard_range(n, r, world) for r in range(world)]
        assert ranges[0][0] == 0 and ranges[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        assert all(n // world <= hi - lo <= n // world + 1 for lo, hi in ranges)
        assert ranges == [(n * r // world, n * (r + 1) // world) for r in range(world)]


def test_cameras_extent_is_getnerfppnorm():
    d = np.load(os.path.join(ROOT, "tests", "golden", "cameras.npz"))
    n = len([k for k in d if k.startswith("R_")])
    cams = [dict(campos=d[f"center_{i}"]) for i in range(n)]
    # getNerfppNorm: the centres of inv(getWorld2View2(R, T, translate, scale)) (utils/graphics_utils.py); a dataset's
    # cameras have translate 0 and scale 1, some of these fixtures do not, and the centre is campos either way
    centers = []
    for i in range(n):
        Rt = np.zeros((4, 4))
        Rt[:3, :3] = d[f"R_{i}"].transpose()
        Rt[:3, 3] = d[f"T_{i}"]
        Rt[3, 3] = 1.0
        C2W = np.linalg.inv(Rt)
        C2W[:3, 3] = (C2W[:3, 3] + d[f"trans_{i}"]) * d[f"scale_{i}"]
        centers.append(C2W[:3, 3:4])
    centers = np.hstack(centers)
    center = np.mean(centers, axis=1, keepdims=True)
    radius = np.max(np.linalg.norm(centers - center, axis=0, keepdims=True)) * 1.1
    assert radius > 0
    assert np.allclose(np.stack([d[f"center_{i}"] for i in range(n)], 1), centers, rtol=1e-6, atol=1e-6)
    assert point_cloud.cameras_extent(cams) == pytest.approx(radius, rel=1e-6)
    assert point_cloud.cameras_extent(cams[:1]) == 0.0
    with pytest.raises(ValueError):
        point_cloud.cameras_extent([])


def test_init_model_argument_checks():
    xyz, rgb, _ = sample(10)
    for args in [(xyz[:, :2], rgb), (xyz, rgb.astype(np.int32)), (xyz, rgb[:5])]:
        with pytest.raises(ValueError):
            point_cloud.init_model(*args, device="cpu")
    for rank, world, D in [(2, 2, 3), (-1, 2, 3), (0, 1, 4)]:
        with pytest.raises(ValueError):
            point_cloud.init_model(xyz, rgb, rank, world, D, device="cpu")


KNN_ARGS = r"""
import ctypes, json, sys
sys.path.insert(0, %(pkg)r)
from gs_b200 import _lib
lib = _lib.load()
FAKE = 1 << 20   # a 256-byte aligned address that is never dereferenced: no device is visible to this process
N = 1000
need = 1 << 30   # any size: without a device the workspace cannot be sized, and the check after the arguments fails

def call(N=N, pts=FAKE, q0=0, q1=N, out=FAKE, temp=FAKE, temp_bytes=None):
    return lib.gs_knn3_mean_dist2_range(N, pts, q0, q1, out, temp, need if temp_bytes is None else temp_bytes, None)

print(json.dumps({
    "temp bytes": lib.gs_knn3_temp_bytes(N), "temp bytes error": lib.gs_last_error().decode(),
    "N < 0": call(N=-1, q1=0), "q0 < 0": call(q0=-1), "q1 > N": call(q1=N + 1), "q1 < q0": call(q0=5, q1=4),
    "null points": call(pts=None), "null out": call(out=None), "null temp": call(temp=None),
    "misaligned points": call(pts=FAKE + 2), "misaligned out": call(out=FAKE + 1), "misaligned temp": call(temp=FAKE + 4),
    "empty range, null pointers": call(q0=7, q1=7, pts=None, out=None, temp=None, temp_bytes=0),
    "N 0": call(N=0, q1=0, pts=None, out=None, temp=None, temp_bytes=0),
    "valid": call(), "valid range": call(q0=10, q1=20),
}))
"""


def test_knn_range_argument_checks():
    """gs_knn3_mean_dist2_range refuses bad sizes, ranges and pointers before any launch.  The calls run in a process
    that sees no device, so a check that stops working ends in a CUDA error and never touches one.  There the workspace
    cannot be sized (CUB sizes its scratch for the current device): gs_knn3_temp_bytes says so with 0 and an error
    text, and a call that passes the argument checks fails with GS_ECUDA before anything is launched.  The short
    workspace (GS_ENOMEM) is checked on the device (tests/test_point_cloud_gpu.py)."""
    code = KNN_ARGS % dict(pkg=os.path.join(ROOT, "grendel-gs_b200"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out.pop("temp bytes") == 0 and "device" in out.pop("temp bytes error")
    for case in ("N < 0", "q0 < 0", "q1 > N", "q1 < q0", "null points", "null out", "null temp", "misaligned points",
                 "misaligned out", "misaligned temp"):
        assert out[case] == -1, (case, out[case])                 # GS_EINVAL
    assert out["empty range, null pointers"] == 0 and out["N 0"] == 0
    assert out["valid"] == -2 and out["valid range"] == -2         # GS_ECUDA: passed every check, no device to size for


def _round32(x):
    """The float32 nearest to the Fraction x, ties to even."""
    from fractions import Fraction
    f = np.float32(float(x))
    cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    err = [abs(Fraction(float(c)) - x) for c in cands]
    best = min(err)
    ties = [c for c, e in zip(cands, err) if e == best]
    return min(ties, key=lambda c: int(np.array(c, np.float32).view(np.uint32)) & 1)


def test_fma32_is_correctly_rounded():
    """knn_ref.fma32, the restatement's single-rounding FMA, against exact rational arithmetic, on random operands and
    on sums built to sit on or next to a float32 rounding tie."""
    from fractions import Fraction
    import knn_ref
    rng = np.random.default_rng(11)
    a = rng.normal(0.0, 1.0, 3000).astype(np.float32)
    c = (rng.normal(0.0, 1.0, 3000) * 10.0 ** rng.integers(-6, 6, 3000)).astype(np.float32)
    near = -(a.astype(np.float64) * a).astype(np.float32)          # c ~ -a*a: cancellation
    c[:1000] = near[:1000]
    ulp = np.spacing(np.abs(c[1000:2000])).astype(np.float32)
    c[1000:2000] = (c[1000:2000] + ulp / np.float32(2)).astype(np.float32)
    got = knn_ref.fma32(a, a, c)
    for j in range(len(a)):
        want = _round32(Fraction(float(a[j])) * Fraction(float(a[j])) + Fraction(float(c[j])))
        assert np.float32(got[j]).view(np.uint32) == np.float32(want).view(np.uint32), (a[j], c[j])


def test_operand_order_matters():
    """The kernels' order fma(dz, dz, fma(dx, dx, dy * dy)) and the other natural order fma(dz, dz, fma(dy, dy, dx * dx))
    give different fp32 distances on about 15 % of the pairs of a uniform cloud, so a bit-exact test of the restatement
    tells them apart."""
    import knn_ref
    p = np.random.default_rng(0).uniform(-1.0, 1.0, (400, 3)).astype(np.float32)
    dx, dy, dz = (p[:, None, j] - p[None, :, j] for j in range(3))
    other = knn_ref.fma32(dz, dz, knn_ref.fma32(dy, dy, dx * dx))
    assert (knn_ref.dist2_pairs(p, p).view(np.uint32) != other.view(np.uint32)).mean() > 0.05


def test_model_files_keep_their_first_fault(tmp_path):
    """model_io's reader checks the model's attributes before the body's length, as it always has: a file that is both
    truncated and missing an attribute is refused for the attribute."""
    from gs_b200 import model_io
    props = [(a, "float", "<f4") for a in model_io.attribute_names(0) if a != "rot_3"]
    path = str(tmp_path / "two_faults.ply")
    write_ply(path, props, 5, {}, truncate=3)
    with pytest.raises(ValueError, match="'rot_3' is missing"):
        model_io.read_ply(path, 0)
    write_ply(path, props + [("rot_3", "float", "<f4")], 5, {}, truncate=3)
    with pytest.raises(ValueError, match="truncated"):
        model_io.read_ply(path, 0)
