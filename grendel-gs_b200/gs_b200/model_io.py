"""Saving and loading trained models in the reference's formats, at any world size.

* PLY point clouds (scene/gaussian_model.py:404-553 save_ply, :572-769 load_ply): binary little-endian PLY 1.0, one
  `vertex` element of float properties `x y z nx ny nz f_dc_0..2 f_rest_0..(3K-4) opacity scale_0..2 rot_0..3`
  (K = (D+1)^2 for a model stored at SH degree D), normals zero, SH channel-major (`transpose(1, 2).flatten(1)`), the
  raw parameters (log-scales, opacity logits, unnormalised quaternions).  These are the files 3DGS viewers open.
  Per rank (`point_cloud_rk<r>_ws<W>.ply`, every rank its shard) or gathered (`point_cloud.ply`, rank 0, rank order).
* Checkpoints (train_internal.py:288-313, utils/general_utils.py:516-709): `chkpnt_ws=<W>_rk=<r>.pth` holding
  `torch.save((capture(), next_iteration))` with the 12 entries of GaussianModel.capture() (gaussian_model.py:70-84),
  read back at another world size by merging or splitting files.

Host-side I/O beside the training step, like densification and redistribution: a Gaussian's PLY row is packed on the
device by the fused-row packing the redistribution uses (redistribute.fused_rows) and copied to pinned host memory once.
DESIGN.md 5h states the formats, the resharding rules and the two places where this module differs from the reference.
"""
import os
import re
from typing import NamedTuple

import numpy as np
import torch
import torch.distributed as dist

from .exchange import all_to_all_single
from .optim import GROUPS, NAMES, FusedAdam, group_params
from .redistribute import fused_rows

# the capture() order of the six parameters (gaussian_model.py:70-84), the checkpoint tuple's, is not the group order
CAPTURE_NAMES = ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity")
STAT_NAMES = ("max_radii2D", "xyz_gradient_accum", "denom")
ATTR, GROUP_ORDER = GROUPS, NAMES   # group name -> GaussianParams attribute; the optimizer's group order


# ---------------------------------------------------------------------------------------------------------------------
# PLY files
# ---------------------------------------------------------------------------------------------------------------------
def attribute_names(max_sh_degree):
    """construct_list_of_attributes (gaussian_model.py:404-417) for a model stored at SH degree max_sh_degree."""
    K = (int(max_sh_degree) + 1) ** 2
    return (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] +
            [f"f_rest_{i}" for i in range(3 * K - 3)] + ["opacity"] + [f"scale_{i}" for i in range(3)] +
            [f"rot_{i}" for i in range(4)])


def ply_header(n, max_sh_degree):
    """The header plyfile writes for PlyData([PlyElement.describe(elements, "vertex")]) of n float rows."""
    props = "".join(f"property float {a}\n" for a in attribute_names(max_sh_degree))
    return f"ply\nformat binary_little_endian 1.0\nelement vertex {int(n)}\n{props}end_header\n".encode("ascii")


def ply_rows(params):
    """{group name: raw tensor} -> (P, 17 / 26 / 41 / 62) float32 rows in attribute_names order, on the tensors' device:
    normals zero, f_dc / f_rest channel-major as save_ply's transpose(1, 2).flatten(1)."""
    with torch.no_grad():
        xyz = params["xyz"].detach()
        parts = [xyz, torch.zeros_like(xyz), params["f_dc"].detach().transpose(1, 2),
                 params["f_rest"].detach().transpose(1, 2), params["opacity"].detach(), params["scaling"].detach(),
                 params["rotation"].detach()]
        return fused_rows([t.to(torch.float32) for t in parts])[0]


def params_from_ply_rows(rows, max_sh_degree):
    """The inverse of ply_rows: (m, F) rows -> {group name: own dense tensor} on the rows' device."""
    K = (int(max_sh_degree) + 1) ** 2
    m, o = rows.shape[0], 9 + 3 * (K - 1)
    own = lambda t: t.clone(memory_format=torch.contiguous_format)
    return {"xyz": own(rows[:, 0:3]), "f_dc": own(rows[:, 6:9].reshape(m, 3, 1).transpose(1, 2)),
            "f_rest": own(rows[:, 9:o].reshape(m, 3, K - 1).transpose(1, 2)), "opacity": own(rows[:, o:o + 1]),
            "scaling": own(rows[:, o + 1:o + 4]), "rotation": own(rows[:, o + 4:o + 8])}


def _to_host(rows):
    """One device-to-host copy of the rows, into pinned memory when they are on the device."""
    host = torch.empty(rows.shape, dtype=torch.float32, pin_memory=rows.is_cuda)
    host.copy_(rows)
    return host.numpy()


def _replace(path, write):
    """write(file) into path + ".tmp", then rename over path: a reader never sees a partly written file."""
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        write(f)
    os.replace(tmp, path)


def write_ply(path, rows, max_sh_degree):
    """(n, F) float32 rows (host numpy or a tensor) -> one PLY file of the reference's layout."""
    if isinstance(rows, torch.Tensor):
        rows = _to_host(rows)
    rows = np.ascontiguousarray(rows, dtype="<f4")
    F = len(attribute_names(max_sh_degree))
    if rows.ndim != 2 or rows.shape[1] != F:
        raise ValueError(f"{path}: rows must be (n, {F}) at SH degree {max_sh_degree}, got {rows.shape}")
    header = ply_header(rows.shape[0], max_sh_degree)

    def write(f):
        f.write(header)
        f.write(memoryview(rows).cast("B"))
    _replace(path, write)


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2",
              "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4",
              "float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8"}


class PlyLayout(NamedTuple):
    path: str
    n: int                   # vertices
    dtype: np.dtype          # one vertex record
    body: int                # byte offset of the first vertex
    max_sh_degree: int


class PlyVertices(NamedTuple):
    """The vertex element of a checked binary little-endian PLY file."""
    n: int                   # vertices
    types: dict              # property name -> PLY type name
    dtype: np.dtype          # one vertex record
    body: int                # byte offset of the first vertex


def parse_ply_vertices(path):
    """Parse the generic part of a PLY header.  Accepts comment / obj_info lines, any property order and extra scalar
    properties; refuses, with a ValueError naming the file: ascii or big-endian data, a first element other than
    `vertex`, list properties in it and unknown or repeated properties.  A reader checks the properties it needs, then
    the body's length (check_ply_body), so a file with several faults is named for the same one whichever reader."""
    with open(path, "rb") as f:
        head = f.read(1 << 16)
        while b"end_header\n" not in head:
            more = f.read(1 << 16)
            if not more or len(head) > 1 << 20:
                raise ValueError(f"{path}: not a PLY file (no end_header line)")
            head += more
    end = head.index(b"end_header\n") + len(b"end_header\n")
    try:
        lines = head[:end].decode("ascii").split("\n")[:-1]
    except UnicodeDecodeError:
        raise ValueError(f"{path}: the PLY header is not ASCII") from None
    if lines[0] != "ply":
        raise ValueError(f"{path}: not a PLY file")
    fmt, n, props, element = None, None, [], None
    for line in lines[1:-1]:
        w = line.split()
        if not w or w[0] in ("comment", "obj_info"):
            continue
        if w[0] == "format":
            fmt = w[1:]
        elif w[0] == "element":
            if element is None and w[1] != "vertex":
                raise ValueError(f"{path}: the first element is {w[1]!r}, not 'vertex'")
            element = w[1]
            if element == "vertex":
                n = int(w[2])
        elif w[0] == "property":
            if element != "vertex":
                continue   # properties of later elements, which come after the vertices in the body
            if w[1] == "list":
                raise ValueError(f"{path}: list property {w[-1]!r} in the vertex element is not supported")
            if w[1] not in _PLY_TYPES:
                raise ValueError(f"{path}: unknown property type {w[1]!r} of {w[2]!r}")
            props.append((w[2], w[1]))
        else:
            raise ValueError(f"{path}: unexpected header line {line!r}")
    if fmt != ["binary_little_endian", "1.0"]:
        raise ValueError(f"{path}: format {' '.join(fmt or ['missing'])}; only binary_little_endian 1.0 is read")
    if n is None:
        raise ValueError(f"{path}: no vertex element")
    types = dict(props)
    if len(types) != len(props):
        raise ValueError(f"{path}: a vertex property name appears twice")
    return PlyVertices(n, types, np.dtype([(name, _PLY_TYPES[t]) for name, t in props]), end)


def check_ply_body(path, vertices):
    """Refuses, with a ValueError naming the file, a body shorter than the vertex records of parse_ply_vertices."""
    n, _, dtype, end = vertices
    if os.path.getsize(path) < end + n * dtype.itemsize:
        raise ValueError(f"{path}: truncated: {n} vertices of {dtype.itemsize} bytes need "
                         f"{end + n * dtype.itemsize} bytes, the file has {os.path.getsize(path)}")


def read_ply_vertices(path, dtype, body, a, b):
    """Vertex records [a, b) of a checked file (parse_ply_vertices' dtype and body) -> numpy structured array."""
    with open(path, "rb") as f:
        f.seek(body + a * dtype.itemsize)
        buf = bytearray((b - a) * dtype.itemsize)   # writable: torch.from_numpy takes it without a copy
        f.readinto(buf)
    return np.frombuffer(buf, dtype=dtype, count=b - a)


def read_ply_header(path, max_sh_degree=None):
    """Parse and check a PLY header of a model: parse_ply_vertices, then refuses, with a ValueError naming the file, a
    needed attribute that is missing or not float and an f_rest count other than 3K - 3 for the requested degree (any
    degree 0..3 when max_sh_degree is None), then check_ply_body."""
    vertices = parse_ply_vertices(path)
    n, types, dtype, end = vertices
    n_rest = sum(1 for name in types if re.fullmatch(r"f_rest_\d+", name))
    if max_sh_degree is None:
        if n_rest not in (0, 9, 24, 45):
            raise ValueError(f"{path}: {n_rest} f_rest properties is no SH degree 0..3 (0, 9, 24 or 45)")
        max_sh_degree = {0: 0, 9: 1, 24: 2, 45: 3}[n_rest]
    elif n_rest != 3 * (int(max_sh_degree) + 1) ** 2 - 3:
        raise ValueError(f"{path}: {n_rest} f_rest properties, SH degree {max_sh_degree} stores "
                         f"{3 * (int(max_sh_degree) + 1) ** 2 - 3}")
    for a in attribute_names(max_sh_degree):
        if a in ("nx", "ny", "nz"):
            continue   # the normals are written but never read (load_raw_ply does not)
        if a not in types:
            raise ValueError(f"{path}: attribute {a!r} is missing")
        if _PLY_TYPES[types[a]] != "<f4":
            raise ValueError(f"{path}: attribute {a!r} is {types[a]}, not float")
    check_ply_body(path, vertices)
    return PlyLayout(path, n, dtype, end, int(max_sh_degree))


def read_ply_rows(layout, a=0, b=None):
    """Vertices [a, b) of a checked file -> (b - a, F) float32 rows in attribute_names order (normals zero)."""
    b = layout.n if b is None else b
    names = attribute_names(layout.max_sh_degree)
    rec = read_ply_vertices(layout.path, layout.dtype, layout.body, a, b)
    if list(layout.dtype.names) == names:   # the layout this module writes: the records are the rows
        return rec.view("<f4").reshape(b - a, len(names))
    rows = np.zeros((b - a, len(names)), dtype="<f4")
    for j, name in enumerate(names):
        if name not in ("nx", "ny", "nz"):
            rows[:, j] = rec[name]
    return rows


def read_ply(path, max_sh_degree=None):
    """One PLY file -> (rows (n, F) float32 numpy, stored SH degree)."""
    layout = read_ply_header(path, max_sh_degree)
    return read_ply_rows(layout), layout.max_sh_degree


def _raw_of(trainer):
    return {name: getattr(trainer.params, attr) for name, attr in ATTR.items()}


def _counts_over_ranks(n, world, group, device):
    dev = device if dist.get_backend(group) == "nccl" else "cpu"
    allc = torch.empty((world,), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(allc, torch.tensor([int(n)], dtype=torch.int64, device=dev), group=group)
    return [int(v) for v in allc.cpu().tolist()]


def save_ply(folder, trainer, gather=False):
    """Scene.save (scene/__init__.py:180-184) -> save_ply into folder (<model>/point_cloud/iteration_<it>).
    trainer: a Trainer (its params, rank, world and group are read).  gather=False: every rank writes its shard to
    point_cloud_rk<r>_ws<W>.ply, as the reference does at every world size (_rk0_ws1 at W = 1, gaussian_model.py:473-509).
    gather=True: rank 0 writes the whole model, shards in rank order, to point_cloud.ply (:425-471).  The shards travel
    as one PLY row per Gaussian in ONE all_to_all_single in which only rank 0 receives, sized by one all-gather (the
    reference: six tensors, each with W - 1 send / recv pairs).  Returns the path written on this rank, or None."""
    rank, world, group = trainer.rank, trainer.world, trainer.group
    D = trainer.params.max_sh_degree   # write_ply refuses rows of another degree
    rows = ply_rows(_raw_of(trainer))
    if not gather:
        os.makedirs(folder, exist_ok=True)
        path = os.path.join(folder, f"point_cloud_rk{rank}_ws{world}.ply")
        write_ply(path, rows, D)
        return path
    if world > 1:
        counts = _counts_over_ranks(rows.shape[0], world, group, rows.device)
        recv_splits = counts if rank == 0 else [0] * world
        out = torch.empty((sum(recv_splits), rows.shape[1]), dtype=rows.dtype, device=rows.device)
        all_to_all_single(out, rows, recv_splits, [rows.shape[0]] + [0] * (world - 1), group)
        rows = out
    if rank != 0:
        return None
    os.makedirs(folder, exist_ok=True)
    path = os.path.join(folder, "point_cloud.ply")
    write_ply(path, rows, D)
    return path


def ply_files(folder):
    """load_ply's choice of files (gaussian_model.py:765-769): point_cloud.ply if it exists, else every
    point_cloud_rk<r>_ws<W0>.ply, r = 0..W0-1, in rank order.  A folder with a missing rank or several W0 is refused."""
    one = os.path.join(folder, "point_cloud.ply")
    if os.path.exists(one):
        return [one]
    found = {}
    for f in os.listdir(folder):
        m = re.fullmatch(r"point_cloud_rk(\d+)_ws(\d+)\.ply", f)
        if m:
            found[(int(m.group(2)), int(m.group(1)))] = os.path.join(folder, f)
    sizes = sorted({ws for ws, _ in found})
    if not sizes:
        raise FileNotFoundError(f"{folder}: neither point_cloud.ply nor point_cloud_rk<r>_ws<W>.ply files")
    if len(sizes) > 1:
        raise ValueError(f"{folder}: per-rank PLY files of several world sizes {sizes}")
    W0 = sizes[0]
    missing = [r for r in range(W0) if (W0, r) not in found]
    extra = [r for ws, r in found if r >= W0]
    if missing or extra:
        raise ValueError(f"{folder}: per-rank PLY files of world size {W0}: ranks {missing} missing, {extra} out of range")
    return [found[(W0, r)] for r in range(W0)]


def load_ply(folder, rank=0, world=1, max_sh_degree=None, device="cpu"):
    """Scene(load_ply_path) -> load_ply (gaussian_model.py:572-769), this rank's part.  The files of ply_files, read as
    one model in their order; the rank takes Gaussians [n rank // W, n (rank + 1) // W), the Trainer's contiguous shard
    (the reference slices by n // W + 1 instead, :698-716; the union is the same model), reading only those rows.
    max_sh_degree: the degree the files must store (None: whatever they store, the same in every file).
    -> (params {group name: tensor on device}, (lo, hi, n_total), stored SH degree).  As at :640, the model's
    active_sh_degree is the stored degree (GaussianParams.from_raw / Trainer(model=...) start there)."""
    layouts = []
    for path in ply_files(folder):
        layouts.append(read_ply_header(path, max_sh_degree if not layouts else layouts[0].max_sh_degree))
    D = layouts[0].max_sh_degree
    n = sum(lay.n for lay in layouts)
    lo, hi = n * rank // world, n * (rank + 1) // world
    parts, start = [], 0
    for lay in layouts:
        a, b = max(lo, start) - start, min(hi, start + lay.n) - start
        if a < b:
            parts.append(read_ply_rows(lay, a, b))
        start += lay.n
    if not parts:
        parts = [np.zeros((0, len(attribute_names(D))), dtype="<f4")]
    rows = torch.from_numpy(np.concatenate(parts) if len(parts) > 1 else parts[0]).to(device)
    return params_from_ply_rows(rows, D), (lo, hi, n), D


# ---------------------------------------------------------------------------------------------------------------------
# checkpoints
# ---------------------------------------------------------------------------------------------------------------------
class Checkpoint(NamedTuple):
    """A loaded checkpoint, named.  capture() gives the reference's 12-entry tuple back."""
    active_sh_degree: int
    params: dict             # {group name: tensor}
    stats: dict              # {"max_radii2D", "xyz_gradient_accum", "denom"}
    optimizer_state: dict    # torch.optim.Optimizer.state_dict() of the six groups
    spatial_lr_scale: float
    next_iteration: int

    def capture(self):
        return ((self.active_sh_degree,) + tuple(self.params[k] for k in CAPTURE_NAMES) +
                tuple(self.stats[k] for k in STAT_NAMES) + (self.optimizer_state, self.spatial_lr_scale))


def checkpoint_path(folder, rank, world):
    return os.path.join(folder, f"chkpnt_ws={world}_rk={rank}.pth")


def save_checkpoint(folder, trainer, optimizer, stats, next_iteration, spatial_lr_scale=0.0):
    """train_internal.py:288-313: this rank writes torch.save((capture(), next_iteration)) to
    <folder>/chkpnt_ws=<W>_rk=<r>.pth, capture() as gaussian_model.py:70-84 builds it.  trainer: a Trainer (its params,
    rank and world are read); optimizer: the six-group optimizer over the trainer's parameters (FusedAdam or
    torch.optim.Adam); stats: {"max_radii2D", "xyz_gradient_accum", "denom"}, the densification statistics the caller
    keeps.  The file loads into the reference's restore() and torch.optim.Adam.  -> the path written."""
    params = _raw_of(trainer)
    for k, p in group_params(optimizer, ordered=True).items():
        if p is not params[k]:
            raise ValueError(f"optimizer group {k!r} does not hold the trainer's parameter (adopt_parameters "
                             "after densification or redistribution)")
    P = int(params["xyz"].shape[0])
    for k in STAT_NAMES:
        if k not in stats or stats[k].shape[0] != P:
            raise ValueError(f"stats[{k!r}] must have one row per Gaussian ({P})")
    capture = ((int(trainer.params.active_sh_degree),) + tuple(params[k] for k in CAPTURE_NAMES) +
               tuple(stats[k] for k in STAT_NAMES) + (optimizer.state_dict(), spatial_lr_scale))
    os.makedirs(folder, exist_ok=True)
    path = checkpoint_path(folder, trainer.rank, trainer.world)
    _replace(path, lambda f: torch.save((capture, int(next_iteration)), f))
    return path


def checkpoint_files(folder):
    """The chkpnt_ws=<F>_rk=<r>.pth files of a folder in rank order: one F, every rank 0..F-1."""
    found = {}
    for f in os.listdir(folder):
        m = re.fullmatch(r"chkpnt_ws=(\d+)_rk=(\d+)\.pth", f)
        if m:
            found[(int(m.group(1)), int(m.group(2)))] = os.path.join(folder, f)
    sizes = sorted({ws for ws, _ in found})
    if not sizes:
        raise FileNotFoundError(f"{folder}: no chkpnt_ws=<W>_rk=<r>.pth files")
    if len(sizes) > 1:
        raise ValueError(f"{folder}: checkpoint files of several world sizes {sizes}")
    F = sizes[0]
    if sorted(r for _, r in found) != list(range(F)):
        raise ValueError(f"{folder}: checkpoint files of world size {F} need ranks 0..{F - 1}, found "
                         f"{sorted(r for _, r in found)}")
    return [found[(F, r)] for r in range(F)]


def _read_checkpoint(path, device):
    capture, next_iteration = torch.load(path, map_location=device, weights_only=True)
    if len(capture) != 12:
        raise ValueError(f"{path}: capture() has 12 entries, this file {len(capture)}")
    return Checkpoint(int(capture[0]), dict(zip(CAPTURE_NAMES, capture[1:7])), dict(zip(STAT_NAMES, capture[7:10])),
                      capture[10], capture[11], int(next_iteration))


def _rows_of(t, P):
    return isinstance(t, torch.Tensor) and t.dim() >= 1 and t.shape[0] == P


def _merge(cks, paths):
    """merge_multiple_checkpoints (general_utils.py:516-564) with the optimizer state merged too: every per-Gaussian
    tensor -- parameters, statistics, and the Adam moments -- concatenated in file order; per-group scalars (Adam's
    step) must agree across the files."""
    first = cks[0]
    params = {k: torch.cat([c.params[k].detach() for c in cks]) for k in CAPTURE_NAMES}
    stats = {k: torch.cat([c.stats[k] for c in cks]) for k in STAT_NAMES}
    opt = first.optimizer_state
    state = {}
    for idx in opt["state"]:
        if any(idx not in c.optimizer_state["state"] for c in cks):
            raise ValueError(f"{paths}: optimizer state of group {idx} is in some files only")
        entry = {}
        for key, v in opt["state"][idx].items():
            vals = [c.optimizer_state["state"][idx][key] for c in cks]
            if all(_rows_of(x, int(c.params["xyz"].shape[0])) for x, c in zip(vals, cks)):
                entry[key] = torch.cat(vals)
            elif all(torch.equal(torch.as_tensor(x).cpu(), torch.as_tensor(v).cpu()) for x in vals):
                entry[key] = v
            else:
                raise ValueError(f"{paths}: optimizer {key!r} of group {idx} differs between the files "
                                 f"({[float(torch.as_tensor(x)) for x in vals]}): they are not of one run")
        state[idx] = entry
    if any(set(c.optimizer_state["state"]) != set(state) for c in cks):
        raise ValueError(f"{paths}: the files hold optimizer state of different groups")
    return first._replace(params=params, stats=stats, optimizer_state={"state": state, "param_groups": opt["param_groups"]})


def _part(ck, parts, part):
    """get_part_of_checkpoints (general_utils.py:567-606): part `part` of `parts` chunks of n // parts + 1 Gaussians,
    optimizer moments included."""
    n = int(ck.params["xyz"].shape[0])
    chunk = n // parts + 1
    a, b = min(part * chunk, n), min((part + 1) * chunk, n)
    cut = lambda t: t[a:b].clone() if _rows_of(t, n) else t
    state = {idx: {key: cut(v) for key, v in e.items()} for idx, e in ck.optimizer_state["state"].items()}
    return ck._replace(params={k: cut(v.detach()) for k, v in ck.params.items()},
                       stats={k: cut(v) for k, v in ck.stats.items()},
                       optimizer_state={"state": state, "param_groups": ck.optimizer_state["param_groups"]})


def load_checkpoint(folder, rank, world, device="cpu"):
    """utils.load_checkpoint (general_utils.py:667-709) for rank `rank` of `world`, every tensor mapped to device.
    F files of one run (checkpoint_files):
      F == W: the rank's own file;
      F a multiple of W: files rank, rank + W, rank + 2W, ... merged in that order;
      W a multiple of F: part rank // F of file rank % F, in chunks of n // (W / F) + 1 Gaussians;
      otherwise a ValueError, raised on every rank alike, before anything is read.
    Unlike the reference, which drops the optimizer state when F != W (opt_dict = None, :546, :589) so that Adam
    restarts from zero moments and step 0, the moments are per-Gaussian rows and are merged and split with the
    parameters, and merged files must carry the same step: a run resumed at any world size starts from the optimizer
    state it stopped with.  -> Checkpoint."""
    paths = checkpoint_files(folder)
    F = len(paths)
    if F == world:
        return _read_checkpoint(paths[rank], device)
    if F > world and F % world == 0:
        mine = paths[rank::world]
        return _merge([_read_checkpoint(p, device) for p in mine], mine)
    if F < world and world % F == 0:
        return _part(_read_checkpoint(paths[rank % F], device), world // F, rank // F)
    raise ValueError(f"{folder}: {F} checkpoint files cannot be loaded at world size {world}: the file count must be a "
                     "multiple or a divisor of the world size")


def load_fused_adam(trainer, checkpoint, **kw):
    """A FusedAdam over trainer.optimizer_groups() with the checkpoint's optimizer state loaded (learning rates, betas,
    eps, step and moments: the saved groups replace the new ones, as torch.optim's load_state_dict does).  The groups
    must be the reference's six, in its order.  kw: FusedAdam's constructor arguments (grad_scale)."""
    opt = FusedAdam(trainer.optimizer_groups(), lr=0.0, eps=1e-15, **kw)
    opt.load_state_dict(checkpoint.optimizer_state)
    group_params(opt, ordered=True)   # the saved groups, which replaced the new ones
    for st in opt.state.values():   # the step counter lives on the host, as FusedAdam creates it
        if "step" in st:
            st["step"] = torch.as_tensor(st["step"], dtype=torch.float32).cpu()
    return opt
