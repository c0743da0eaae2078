"""gs_b200.model_io on the CPU: the reference's PLY point clouds and per-rank checkpoints, written and read at any world
size.

  * the PLY header is the one plyfile writes, with construct_list_of_attributes' names (scene/gaussian_model.py:404-417);
  * the body is the fp32 little-endian rows, and write -> read gives the same bits, special values included;
  * the reader takes comments, shuffled and extra properties, and refuses what it cannot read with a ValueError;
  * per-rank PLY sets of W0 ranks load at any W as the Trainer's contiguous shards of one model, as a gathered file does;
  * per-rank checkpoints of W0 ranks load at every W the reference's rules allow, optimizer moments and step included;
  * the gathered save over 2 and 3 gloo processes writes the bytes of a one-process save of the whole model."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gs_b200 import model_io, pipeline
from gs_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = "/root/reference"
NAMES = model_io.GROUP_ORDER


def names_of(D):
    K = (D + 1) ** 2
    return (["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + ["f_rest_%d" % i for i in range(3 * K - 3)] +
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"])


def raw_model(n, D, seed, special=True):
    """Random raw parameters; with special, every tensor also carries -0.0, +-inf, NaN payloads and subnormals."""
    g = torch.Generator().manual_seed(seed)
    K = (D + 1) ** 2
    shapes = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (K - 1, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
    out = {}
    for k, s in shapes.items():
        t = torch.randn((n,) + s, generator=g)
        if special and t.numel():
            bits = torch.tensor([0x80000000, 0x7F800000, 0xFF800000, 0x7FC00001, 0xFFA12345, 0x7F812345, 0x00000001,
                                 0x807FFFFF], dtype=torch.int64).to(torch.int32).view(torch.float32)
            flat = t.reshape(-1)
            idx = torch.randperm(flat.numel(), generator=g)[:min(flat.numel(), 64)]
            flat[idx] = bits[torch.arange(idx.numel()) % bits.numel()]
        out[k] = t
    return out


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def fake_rank(params, rank=0, world=1, group=None, active=None):
    """What save_ply / save_checkpoint read of a Trainer: its raw parameters, rank, world size and group."""
    gp = pipeline.GaussianParams.from_raw(params, "cpu")
    if active is not None:
        gp.active_sh_degree = active
    return SimpleNamespace(params=gp, rank=rank, world=world, group=group)


def shard(params, lo, hi):
    return {k: v[lo:hi] for k, v in params.items()}


def cat(parts):
    return {k: torch.cat([p[k] for p in parts]) for k in NAMES}


# ---------------------------------------------------------------------------------------------------------------------
# header and body
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,F", [(0, 17), (1, 26), (2, 41), (3, 62)])
def test_header_is_plyfiles(D, F):
    want = (b"ply\nformat binary_little_endian 1.0\nelement vertex 7\n" +
            b"".join(b"property float " + a.encode() + b"\n" for a in names_of(D)) + b"end_header\n")
    assert len(names_of(D)) == F
    assert model_io.ply_header(7, D) == want
    assert model_io.attribute_names(D) == names_of(D)


REF_NAMES = r"""
import json, sys
sys.path[:0] = [%(ref)r, %(pkg)r, %(shims)r]
import torch
from scene.gaussian_model import GaussianModel
g = GaussianModel.__new__(GaussianModel)
out = {}
for D in range(4):
    K = (D + 1) ** 2
    g._features_dc, g._features_rest = torch.zeros(2, 1, 3), torch.zeros(2, K - 1, 3)
    g._scaling, g._rotation = torch.zeros(2, 3), torch.zeros(2, 4)
    out[D] = g.construct_list_of_attributes()
print(json.dumps(out))
"""


def test_attribute_names_are_the_references():
    if not os.path.exists(os.path.join(REFERENCE, "scene", "gaussian_model.py")):
        pytest.skip("the reference checkout is not present")
    pkg = os.path.join(ROOT, "grendel-gs_b200")
    code = REF_NAMES % dict(ref=REFERENCE, pkg=pkg, shims=os.path.join(pkg, "shims"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    import json
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for D in range(4):
        assert got[str(D)] == model_io.attribute_names(D), D


@pytest.mark.parametrize("D", [0, 1, 2, 3])
def test_round_trip_keeps_every_bit(tmp_path, D):
    n = 53
    p = raw_model(n, D, seed=D)
    path = model_io.save_ply(str(tmp_path), fake_rank(p))
    assert os.path.basename(path) == "point_cloud_rk0_ws1.ply"
    data = open(path, "rb").read()
    header = model_io.ply_header(n, D)
    assert data.startswith(header)
    # the body: fp32 little-endian rows, x y z, zero normals, channel-major SH, opacity, scales, rotation
    rows = np.frombuffer(data[len(header):], dtype="<f4").reshape(n, -1)
    want = torch.cat([p["xyz"], torch.zeros(n, 3), p["f_dc"].transpose(1, 2).flatten(1),
                      p["f_rest"].transpose(1, 2).flatten(1), p["opacity"], p["scaling"], p["rotation"]], dim=1)
    assert same_bits(torch.from_numpy(rows.copy()), want)
    names = names_of(D)
    for j in range(3 * (D + 1) ** 2 - 3):   # f_rest_j is coefficient j % (K-1) + 1 of channel j // (K-1)
        K1 = (D + 1) ** 2 - 1
        col = torch.from_numpy(rows[:, names.index("f_rest_%d" % j)].copy())
        assert same_bits(col, p["f_rest"][:, j % K1, j // K1]), j
    got, (lo, hi, total), deg = model_io.load_ply(str(tmp_path))
    assert (lo, hi, total, deg) == (0, n, n, D)
    for k in NAMES:
        assert same_bits(got[k], p[k]), k
        assert got[k].is_contiguous() and got[k].storage_offset() == 0


# ---------------------------------------------------------------------------------------------------------------------
# the reader: what other tools write, and what it refuses
# ---------------------------------------------------------------------------------------------------------------------
def write_custom(path, fields, n, fmt="binary_little_endian", pre=b"", body=None, extra_lines=b""):
    """A PLY file with a vertex element of the given (name, ply type, numpy type, values) fields, in that order."""
    rec = np.zeros(n, dtype=[(name, nt) for name, _, nt, _ in fields])
    for name, _, _, v in fields:
        rec[name] = v
    head = (b"ply\nformat " + fmt.encode() + b" 1.0\n" + pre + b"element vertex %d\n" % n +
            b"".join(b"property %s %s\n" % (pt.encode(), name.encode()) for name, pt, _, _ in fields) + extra_lines +
            b"end_header\n")
    with open(path, "wb") as f:
        f.write(head + (rec.tobytes() if body is None else body))


def std_fields(rows, D, order=None):
    names = names_of(D)
    order = range(len(names)) if order is None else order
    return [(names[j], "float", "<f4", rows[:, j]) for j in order]


def test_reader_takes_comments_shuffled_and_extra_properties(tmp_path):
    D, n = 2, 31
    p = raw_model(n, D, seed=9)
    rows = model_io.ply_rows(p).numpy()
    order = np.random.default_rng(3).permutation(len(names_of(D)))
    fields = std_fields(rows, D, order)
    fields.insert(5, ("red", "uchar", "u1", np.arange(n) % 256))
    fields.insert(11, ("confidence", "double", "<f8", np.linspace(0, 1, n)))
    fields.append(("id", "int", "<i4", np.arange(n)))
    path = str(tmp_path / "point_cloud.ply")
    write_custom(path, fields, n, pre=b"comment written by another tool\nobj_info some info\n",
                 extra_lines=b"element face 0\nproperty list uchar int vertex_indices\n")
    got, _, deg = model_io.load_ply(str(tmp_path), max_sh_degree=D)
    assert deg == D
    for k in NAMES:
        assert same_bits(got[k], p[k]), k


def test_reader_refusals(tmp_path):
    D, n = 1, 9
    rows = model_io.ply_rows(raw_model(n, D, seed=1, special=False)).numpy()
    cases = {
        "ascii": dict(fields=std_fields(rows, D), fmt="ascii"),
        "big-endian": dict(fields=std_fields(rows, D), fmt="binary_big_endian"),
        "list": dict(fields=std_fields(rows, D)[:9] + [("vertex_indices", "list uchar int", "<f4", 0)] +
                     std_fields(rows, D)[9:]),
        "double": dict(fields=[(a, "double" if a == "opacity" else pt, "<f8" if a == "opacity" else nt, v)
                               for a, pt, nt, v in std_fields(rows, D)]),
        "int": dict(fields=[(a, "int" if a == "x" else pt, "<i4" if a == "x" else nt, v)
                            for a, pt, nt, v in std_fields(rows, D)]),
        "missing": dict(fields=[f for f in std_fields(rows, D) if f[0] != "rot_3"]),
        "truncated": dict(fields=std_fields(rows, D), truncate=5),
    }
    for name, c in cases.items():
        path = str(tmp_path / f"{name}.ply")
        fields = c["fields"]
        body = None
        if "truncate" in c:
            rec = np.zeros(n, dtype=[(a, nt) for a, _, nt, _ in fields])
            body = rec.tobytes()[:-c["truncate"]]
        write_custom(path, fields, n, fmt=c.get("fmt", "binary_little_endian"), body=body)
        with pytest.raises(ValueError, match=f"{name}.ply"):
            model_io.read_ply(path, D)
    # an f_rest count that is not 3K - 3 for the requested degree, or for any degree
    good = str(tmp_path / "good.ply")
    write_custom(good, std_fields(rows, D), n)
    assert model_io.read_ply(good, D)[1] == D
    for D_req in (0, 2, 3):
        with pytest.raises(ValueError, match="good.ply"):
            model_io.read_ply(good, D_req)
    odd = str(tmp_path / "odd.ply")
    write_custom(odd, [f for f in std_fields(rows, D) if f[0] != "f_rest_8"], n)
    with pytest.raises(ValueError, match="odd.ply"):
        model_io.read_ply(odd)


# ---------------------------------------------------------------------------------------------------------------------
# PLY sets at any world size
# ---------------------------------------------------------------------------------------------------------------------
def test_ply_sets_reshard_to_contiguous_shards(tmp_path):
    n, D = 103, 3
    model = raw_model(n, D, seed=4)
    gathered = tmp_path / "gathered"
    model_io.save_ply(str(gathered), fake_rank(model), gather=True)
    assert os.listdir(gathered) == ["point_cloud.ply"]
    for W0 in (1, 2, 3, 4):
        folder = tmp_path / f"ws{W0}"
        for r in range(W0):
            model_io.save_ply(str(folder), fake_rank(shard(model, n * r // W0, n * (r + 1) // W0), r, W0))
        assert sorted(os.listdir(folder)) == [f"point_cloud_rk{r}_ws{W0}.ply" for r in range(W0)]
        for src in (folder, gathered):
            for W in (1, 2, 3, 4):
                parts = []
                for r in range(W):
                    got, (lo, hi, total), deg = model_io.load_ply(str(src), r, W, max_sh_degree=D)
                    assert (lo, hi, total, deg) == (n * r // W, n * (r + 1) // W, n, D)
                    for k in NAMES:
                        assert same_bits(got[k], model[k][lo:hi]), (W0, W, r, k)
                    parts.append(got)
                whole = cat(parts)
                assert all(same_bits(whole[k], model[k]) for k in NAMES)


def test_ply_folder_refusals(tmp_path):
    m = raw_model(10, 0, seed=2, special=False)
    for r in (0, 2):    # rank 1 of 3 missing
        model_io.save_ply(str(tmp_path / "gap"), fake_rank(shard(m, r, r + 1), r, 3))
    with pytest.raises(ValueError, match="missing"):
        model_io.load_ply(str(tmp_path / "gap"))
    model_io.save_ply(str(tmp_path / "mixed"), fake_rank(m, 0, 1))
    model_io.save_ply(str(tmp_path / "mixed"), fake_rank(shard(m, 0, 5), 0, 2))
    model_io.save_ply(str(tmp_path / "mixed"), fake_rank(shard(m, 5, 10), 1, 2))
    with pytest.raises(ValueError, match="several world sizes"):
        model_io.load_ply(str(tmp_path / "mixed"))
    os.makedirs(tmp_path / "empty")
    with pytest.raises(FileNotFoundError):
        model_io.load_ply(str(tmp_path / "empty"))


# ---------------------------------------------------------------------------------------------------------------------
# checkpoints
# ---------------------------------------------------------------------------------------------------------------------
def stepped_adam(gp, seed, steps=2):
    """torch.optim.Adam over the six groups (gaussian_model.py:257-292) of a GaussianParams, after a few steps."""
    g = torch.Generator().manual_seed(seed)
    ps = {k: getattr(gp, attr) for k, attr in model_io.ATTR.items()}
    opt = torch.optim.Adam([{"params": [ps[k]], "lr": 1e-3 * (i + 1), "name": k} for i, k in enumerate(NAMES)],
                           lr=0.0, eps=1e-15)
    for _ in range(steps):
        for k in NAMES:
            ps[k].grad = torch.randn(ps[k].shape, generator=g)
        opt.step()
    return ps, opt


def write_checkpoints(folder, n, W0, D=3, seed=0):
    """W0 ranks, uneven shards, each with a stepped Adam and statistics -> the per-rank sources."""
    model = raw_model(n, D, seed=seed, special=False)
    g = torch.Generator().manual_seed(seed + 1)
    sources = []
    for r in range(W0):
        lo, hi = n * r // W0, n * (r + 1) // W0
        tr = fake_rank(shard(model, lo, hi), r, W0, active=1)
        ps, opt = stepped_adam(tr.params, seed=100 * seed + r)
        P = hi - lo
        stats = {"max_radii2D": torch.rand((P,), generator=g), "xyz_gradient_accum": torch.rand((P, 1), generator=g),
                 "denom": torch.randint(0, 9, (P, 1), generator=g).float()}
        path = model_io.save_checkpoint(str(folder), tr, opt, stats, next_iteration=17, spatial_lr_scale=2.5)
        assert os.path.basename(path) == f"chkpnt_ws={W0}_rk={r}.pth"
        sources.append(dict(params={k: ps[k].detach() for k in NAMES}, stats=stats,
                            state={k: opt.state[ps[k]] for k in NAMES}))
    return sources


def expected_part(sources, rank, world):
    """The reference's rules (general_utils.py:667-709), restated on the sources: -> list of (source, a, b) pieces."""
    F = len(sources)
    if F == world:
        return [(sources[rank], 0, None)]
    if F > world:
        return [(sources[i], 0, None) for i in range(rank, F, world)]
    src = sources[rank % F]
    n = src["params"]["xyz"].shape[0]
    chunk = n // (world // F) + 1
    part = rank // F
    return [(src, min(part * chunk, n), min((part + 1) * chunk, n))]


def pieces(pcs, get):
    return torch.cat([get(s)[a:b] for s, a, b in pcs])


@pytest.mark.parametrize("W0", [1, 2, 4, 8])
def test_checkpoints_reshard_with_optimizer_state(tmp_path, W0):
    n = 203
    sources = write_checkpoints(tmp_path, n, W0, seed=W0)
    ranks_total = 0
    for W in range(1, 9):
        if not (W == W0 or (W < W0 and W0 % W == 0) or (W > W0 and W % W0 == 0)):
            with pytest.raises(ValueError, match="cannot be loaded"):
                model_io.load_checkpoint(str(tmp_path), 0, W)
            continue
        got_total = 0
        for r in range(W):
            ck = model_io.load_checkpoint(str(tmp_path), r, W)
            pcs = expected_part(sources, r, W)
            assert ck.active_sh_degree == 1 and ck.next_iteration == 17 and ck.spatial_lr_scale == 2.5
            for k in NAMES:
                assert same_bits(ck.params[k], pieces(pcs, lambda s: s["params"][k])), (W, r, k)
                st = ck.optimizer_state["state"][NAMES.index(k)]
                for m in ("exp_avg", "exp_avg_sq"):
                    assert same_bits(st[m], pieces(pcs, lambda s: s["state"][k][m])), (W, r, k, m)
                assert float(st["step"]) == 2.0
            for k in model_io.STAT_NAMES:
                assert same_bits(ck.stats[k], pieces(pcs, lambda s: s["stats"][k])), (W, r, k)
            assert [g["name"] for g in ck.optimizer_state["param_groups"]] == list(NAMES)
            got_total += ck.params["xyz"].shape[0]
        assert got_total == n   # every Gaussian on exactly one rank
        ranks_total += 1
    assert ranks_total >= 2


def test_checkpoint_refusals(tmp_path):
    write_checkpoints(tmp_path / "three", 30, 3)
    for W in (2, 4, 5):
        with pytest.raises(ValueError, match="cannot be loaded"):
            model_io.load_checkpoint(str(tmp_path / "three"), 0, W)
    # merged files of different runs: the steps differ
    write_checkpoints(tmp_path / "steps", 40, 2)
    path = os.path.join(tmp_path / "steps", "chkpnt_ws=2_rk=1.pth")
    capture, it = torch.load(path, weights_only=True)
    capture[10]["state"][0]["step"] = torch.tensor(5.0)
    torch.save((capture, it), path)
    with pytest.raises(ValueError, match="step"):
        model_io.load_checkpoint(str(tmp_path / "steps"), 0, 1)
    os.remove(os.path.join(tmp_path / "three", "chkpnt_ws=3_rk=1.pth"))
    with pytest.raises(ValueError, match="ranks"):
        model_io.load_checkpoint(str(tmp_path / "three"), 0, 3)


def test_checkpoint_is_the_references_capture_tuple(tmp_path):
    sources = write_checkpoints(tmp_path, 12, 1)
    capture, it = torch.load(os.path.join(tmp_path, "chkpnt_ws=1_rk=0.pth"), weights_only=True)
    assert it == 17 and len(capture) == 12 and capture[0] == 1 and capture[11] == 2.5
    for q, k in enumerate(model_io.CAPTURE_NAMES):
        assert isinstance(capture[1 + q], torch.nn.Parameter) and same_bits(capture[1 + q], sources[0]["params"][k])
    for q, k in enumerate(model_io.STAT_NAMES):
        assert same_bits(capture[7 + q], sources[0]["stats"][k])
    # restore()'s optimizer takes the state: torch.optim.Adam over the six groups in the reference's order
    ps = {k: torch.nn.Parameter(capture[1 + model_io.CAPTURE_NAMES.index(k)]) for k in NAMES}
    opt = torch.optim.Adam([{"params": [ps[k]], "lr": 0.0, "name": k} for k in NAMES], lr=0.0, eps=1e-15)
    opt.load_state_dict(capture[10])
    assert torch.equal(opt.state[ps["opacity"]]["exp_avg"], sources[0]["state"]["opacity"]["exp_avg"])


def test_torch_adam_state_loads_into_fused_adam_and_back(tmp_path):
    sources = write_checkpoints(tmp_path, 25, 1, D=1)
    ck = model_io.load_checkpoint(str(tmp_path), 0, 1)
    cams = [syn.make_camera(48, 32, uid=0)]
    tr = pipeline.Trainer(None, cams, None, "cpu", model=ck.params)
    assert tr.params.max_sh_degree == 1 and tr.n_total == 25
    for k, attr in model_io.ATTR.items():
        assert same_bits(getattr(tr.params, attr), sources[0]["params"][k])
    fused = model_io.load_fused_adam(tr, ck)
    for g in fused.param_groups:
        st = fused.state[g["params"][0]]
        src = sources[0]["state"][g["name"]]
        assert same_bits(st["exp_avg"], src["exp_avg"]) and same_bits(st["exp_avg_sq"], src["exp_avg_sq"])
        assert st["step"].device.type == "cpu" and float(st["step"]) == 2.0
    back = torch.optim.Adam(tr.optimizer_groups(), lr=0.0, eps=1e-15)
    back.load_state_dict(fused.state_dict())
    for g, g0 in zip(back.param_groups, ck.optimizer_state["param_groups"]):
        assert g["lr"] == g0["lr"] and g["name"] == g0["name"] and g["betas"] == g0["betas"] and g["eps"] == g0["eps"]
        st = back.state[g["params"][0]]
        assert same_bits(st["exp_avg"], sources[0]["state"][g["name"]]["exp_avg"])


# ---------------------------------------------------------------------------------------------------------------------
# the gathered save over gloo
# ---------------------------------------------------------------------------------------------------------------------
def _gather_worker(rank, world, port, folder, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        n = 61 + 7 * world
        model = raw_model(n, 2, seed=world)
        lo, hi = (0, 5) if rank == 0 else (5 + (n - 5) * (rank - 1) // (world - 1), 5 + (n - 5) * rank // (world - 1))
        cams = [syn.make_camera(48, 32, uid=0)]
        tr = pipeline.Trainer(None, cams, None, "cpu", rank, world, model=shard(model, lo, hi), shard=(lo, hi, n),
                              peer_exchange=False, load_balance=False)
        path = model_io.save_ply(folder, tr, gather=True)
    except Exception as e:   # reported to the test, which ends the other workers
        q.put((rank, None, repr(e)))
        raise
    q.put((rank, path, None))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gathered_save_over_gloo_is_the_one_process_file(tmp_path, world):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29760 + world
    folder = str(tmp_path / "gathered")
    procs = [ctx.Process(target=_gather_worker, args=(r, world, port, folder, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = sorted(q.get(timeout=180) for _ in range(world))
    finally:   # no worker outlives the test, whatever happened in it
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(err is None for _, _, err in res), res
    assert res[0][1] == os.path.join(folder, "point_cloud.ply") and all(p is None for _, p, _ in res[1:])
    n = 61 + 7 * world
    one = str(tmp_path / "one")
    model_io.save_ply(one, fake_rank(raw_model(n, 2, seed=world)), gather=True)
    assert os.listdir(folder) == ["point_cloud.ply"]
    assert open(res[0][1], "rb").read() == open(os.path.join(one, "point_cloud.ply"), "rb").read()
