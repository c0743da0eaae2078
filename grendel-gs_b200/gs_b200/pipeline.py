"""Host-side training-step pipeline around the operators: the call sequence of
Grendel-GS train_internal.py:139-196 (strategy -> GT load -> preprocess (+ all-to-all) -> render ->
loss -> backward) written against our C-ABI operators, for bench.py, smoke() and the tests.

The reference's own Python (gaussian_renderer/*.py) runs unchanged on top of the drop-in
`diff_gaussian_rasterization` package; this module is the equivalent harness for use without a reference checkout,
with the same partitioning rules:
  * Gaussians sharded evenly across ranks (scene/gaussian_model.py:181-194),
  * pixels sharded by contiguous tile rows per camera (workload_division.py:852-941),
  * one sparse all-to-all of projected splats per step and its mirror in backward
    (gaussian_renderer/__init__.py:542-698).
"""

import contextlib
import operator
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import gt_scatter, ops
from .optim import GROUPS
from .division import (DivisionStrategy, StrategyHistory, finish_strategy, heuristics_update_enabled,  # noqa: F401
                       start_strategy, start_strategy_whole_views)


class RasterSettings:
    """Attribute bag with the 12 fields of GaussianRasterizationSettings (gaussian_renderer/__init__.py:930-943)."""
    __slots__ = ("image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
                 "projmatrix", "sh_degree", "campos", "prefiltered", "debug")

    def __init__(self, **kw):
        for k in self.__slots__:
            setattr(self, k, kw[k])


class DeviceCamera:
    """Camera constants resident on the GPU (scene/cameras.py:84-100 keeps them as cuda tensors too)."""

    def __init__(self, cam, device, bg=(0.0, 0.0, 0.0)):
        self.uid = cam.get("uid", 0)
        self.image_height, self.image_width = int(cam["image_height"]), int(cam["image_width"])
        self.tanfovx, self.tanfovy = float(cam["tanfovx"]), float(cam["tanfovy"])
        self.sh_degree = int(cam["sh_degree"])
        self.viewmatrix = torch.as_tensor(cam["viewmatrix"], dtype=torch.float32).to(device)
        self.projmatrix = torch.as_tensor(cam["projmatrix"], dtype=torch.float32).to(device)
        self.campos = torch.as_tensor(cam["campos"], dtype=torch.float32).to(device)
        self.bg = torch.tensor(bg, dtype=torch.float32, device=device)

    def settings(self, sh_degree=None):
        return RasterSettings(image_height=self.image_height, image_width=self.image_width, tanfovx=self.tanfovx,
                              tanfovy=self.tanfovy, bg=self.bg, scale_modifier=1.0, viewmatrix=self.viewmatrix,
                              projmatrix=self.projmatrix, sh_degree=self.sh_degree if sh_degree is None else sh_degree,
                              campos=self.campos, prefiltered=False, debug=False)


class GaussianParams(nn.Module):
    """The six raw nn.Parameter tensors of GaussianModel (scene/gaussian_model.py:219-228) with its
    activations (:109-129).  Built from an ACTIVATED synthetic scene by inverting the activations.
    max_sh_degree: the SH degree the model stores (--sh_degree, gaussian_model.py:51-53): the first (D+1)^2 coefficients
    of scene["shs"] are kept, _features_rest is (P,(D+1)^2-1,3) (:150-156); active_sh_degree starts at it."""

    def __init__(self, scene, device, max_sh_degree=3):
        super().__init__()
        if not 0 <= int(max_sh_degree) <= 3:
            raise ValueError(f"max_sh_degree must be 0..3, got {max_sh_degree}")
        K = (int(max_sh_degree) + 1) ** 2
        if scene["shs"].shape[1] < K:
            raise ValueError(f"the scene stores {scene['shs'].shape[1]} SH coefficients, max_sh_degree "
                             f"{max_sh_degree} needs {K}")
        t = lambda a: torch.as_tensor(a, dtype=torch.float32).to(device)
        shs = t(scene["shs"][:, :K])
        op = t(scene["opacities"]).clamp(1e-6, 1 - 1e-6)
        self._xyz = nn.Parameter(t(scene["means3D"]).contiguous())
        # own storage, not views of shs: with one Gaussian shs[:, 1:, :] is already contiguous, so .contiguous() would
        # return a view 12 bytes into shs, and the kernels need 16-byte aligned SH blocks
        self._features_dc = nn.Parameter(shs[:, :1, :].clone(memory_format=torch.contiguous_format))
        self._features_rest = nn.Parameter(shs[:, 1:, :].clone(memory_format=torch.contiguous_format))
        self._scaling = nn.Parameter(torch.log(t(scene["scales"])).contiguous())
        self._rotation = nn.Parameter(t(scene["rotations"]).contiguous())
        self._opacity = nn.Parameter(torch.log(op / (1 - op)).contiguous())
        self.max_sh_degree = int(max_sh_degree)
        self.active_sh_degree = self.max_sh_degree

    RAW_SHAPES = {"xyz": (3,), "f_dc": (1, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}

    @classmethod
    def from_raw(cls, raw, device):
        """The six raw parameters as they are stored (a PLY shard or a checkpoint, model_io): raw = {group name
        (optim.GROUPS): tensor}, taken bit for bit, with no activation inverted.  max_sh_degree comes from _features_rest's
        (P, (D+1)^2 - 1, 3); active_sh_degree starts at it."""
        if set(raw) != set(GROUPS):
            raise ValueError(f"raw parameters need the groups {sorted(GROUPS)}, got {sorted(raw)}")
        P = int(raw["xyz"].shape[0])
        for name, tail in cls.RAW_SHAPES.items():
            if tuple(raw[name].shape) != (P,) + tail:
                raise ValueError(f"raw parameter {name} must be {(P,) + tail}, got {tuple(raw[name].shape)}")
        rest = tuple(raw["f_rest"].shape)
        if len(rest) != 3 or rest[0] != P or rest[2] != 3:
            raise ValueError(f"raw parameter f_rest must be (P, (D+1)^2 - 1, 3) for D = 0..3, got {rest}")
        max_sh_degree = ops.stored_sh_degree(rest[1] + 1, f"raw parameter f_rest {rest}")
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        for name, attr in GROUPS.items():
            t = raw[name].detach().to(device=device, dtype=torch.float32)
            if not t.is_contiguous() or t.storage_offset() != 0:   # the kernels need 16-byte aligned, dense rows
                t = t.clone(memory_format=torch.contiguous_format)
            setattr(self, attr, nn.Parameter(t))
        self.max_sh_degree = max_sh_degree
        self.active_sh_degree = self.max_sh_degree
        return self

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_scaling(self):
        return torch.exp(self._scaling)

    @property
    def get_rotation(self):
        return torch.nn.functional.normalize(self._rotation)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    @property
    def get_features(self):
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    def raw_parameters(self):
        return [getattr(self, attr) for attr in ops.RAW_ORDER]


def train_step_single(params, dcam, gt_u8_dev, lambda_dssim=0.2, collector=None, compute_locally=None):
    """One camera on one rank: preprocess -> render -> fused L1+SSIM -> backward.  Returns the loss tensor
    (gradients land in params.*.grad) and the projected means2D (its .grad feeds densification)."""
    rs = dcam.settings(params.active_sh_degree)
    cuda_args = {"stats_collector": collector if collector is not None else {}}
    means2D, rgb, conic_opacity, radii, depths = ops.preprocess_gaussians(
        params.get_xyz, params.get_scaling, params.get_rotation, params.get_features, params.get_opacity, rs, cuda_args)
    means2D.retain_grad()
    image, *_ = ops.render_gaussians(means2D, conic_opacity, rgb, depths, radii, compute_locally, rs, cuda_args)
    loss = ops.fused_loss(image, gt_u8_dev, 0, dcam.image_height, lambda_dssim)
    loss.backward()
    return loss, means2D, radii


def sum_over_ranks(gathered):
    """(W, n, 2) per-rank [Ll1, ssim] records -> (n, 2): ((rank 0 + rank 1) + rank 2) + ..., in rank order, so the bits
    depend only on which partial each rank holds, not on a collective's reduction order."""
    total = gathered[0]
    for r in range(1, gathered.shape[0]):
        total = total + gathered[r]
    return total


def loss_table(gathered, index, lambda_dssim):
    """The drained records as one table: (W, n, 2) gathered [Ll1, ssim] and (n,) camera indices -> (n, 4) float64 rows
    (camera index, Ll1, ssim, loss).  loss = (1 - lambda) Ll1 + lambda (1 - ssim) in float32, as train_internal.py:220-222
    forms batched_loss; the float32 values widen exactly."""
    pairs = sum_over_ranks(gathered)
    loss = (1.0 - lambda_dssim) * pairs[:, 0] + lambda_dssim * (1.0 - pairs[:, 1])
    return torch.cat([index.to(torch.float64)[:, None], pairs.to(torch.float64), loss.to(torch.float64)[:, None]], 1)


def loss_entries(rows, steps):
    """loss_table's rows as host lists and the steps' (iteration, B), oldest first -> one entry per step:
    {"iteration", "views", "l1", "ssim", "loss"}, the views' values in batch order."""
    out, off = [], 0
    for iteration, B in steps:
        part = rows[off:off + B]
        off += B
        out.append({"iteration": int(iteration), "views": [int(r[0]) for r in part], "l1": [r[1] for r in part],
                    "ssim": [r[2] for r in part], "loss": [r[3] for r in part]})
    return out


class Trainer:
    """Distributed training-step harness (one process per GPU).

    Gaussians are sharded evenly by contiguous chunks (scene/gaussian_model.py:181-194); the B cameras of a
    step are divided into tile-row strips over the W ranks (division.start_strategy); projected splats reach
    their strip owners through exchange.exchange_cat (skipped when W == 1, like gaussian_renderer/__init__.py:968).
    Every batch renders all its local strips in one batched render (ops.render_gaussians_batched) instead of the
    reference's per-camera loop (render_final, gaussian_renderer/__init__.py:1217-1288), and scores them in one batched
    loss (ops.fused_l1_ssim_batched).
    """

    def __init__(self, scene, cams, gts_pinned, device, rank=0, world=1, lambda_dssim=0.2, group=None,
                 border_exchange=False, peer_exchange=None, peer_cap_rows=None, shard=None, load_balance=True,
                 heuristic_decay=0.0, distributed_dataset_storage=False, feedback_lag=None, max_sh_degree=3,
                 deterministic=False, local_sampling=False, local_bsz=None, model=None):
        """cams, gts_pinned: the camera set -- N cameras and their uint8 (3,H,W) host images, all of one size (the reference
        keeps one global TILE_Y); each step trains on the views it lists (step(views=...)), all N by default.
        scene: the WHOLE scene (sliced here into this rank's contiguous shard), or -- shard=(lo, hi, n_total) -- only
        this rank's Gaussians [lo, hi) of an n_total-Gaussian scene (synthetic.make_scene_shard).
        load_balance: feed the measured render times back into the strip division after every step
        (finish_strategy_final, workload_division.py:944-998; only where the reference's gate enables it).
        distributed_dataset_storage: only rank 0 holds the ground-truth images (gts_pinned may be None elsewhere); the
        strips of a resident=False step are scattered from rank 0's GPU (loss_distribution.py:2395-2533, gt_scatter.py)
        instead of being read from every rank's own host copy.
        feedback_lag: 0 = the reference's sequencing (finish_strategy_final right after the step: the render times are
        read, all-gathered and applied before the next step starts, so the host waits for the device at the end of every
        step and cannot enqueue ahead).  > 0 (default 2, GS_B200_FEEDBACK_LAG) = the times of the step `feedback_lag`
        steps back, whose events have long completed, ride on the NEXT exchange's size all-gather (exchange_cat(times=...)):
        no collective of their own, no host sync; the strips move the same way, `feedback_lag` steps later.
        max_sh_degree: the SH degree the model stores (GaussianParams).
        deterministic: every render and loss of the step runs its atomic-free form (ops.render_gaussians(...,
        deterministic=True)), so two runs of the same steps on the same inputs give the same bits in every loss, gradient
        and, through FusedAdam and densification, parameter.  False leaves the choice to
        torch.use_deterministic_algorithms.  This holds for a FIXED strip division: with more than one rank and
        load_balance=True the strips follow measured render times, which differ from run to run, so that combination is
        refused.  (The exchange sums gradients in a fixed rank order already; the NCCL all-reduce of replicated-Gaussian
        gradient sync is outside this guarantee.)
        local_sampling: the reference's --local_sampling (train_internal.py:113-132, workload_division.py:858-877).  Each
        rank trains on local_bsz views of its own images per step (step(views=...)); the W * local_bsz views of all ranks
        form the batch, and batch position p is rendered whole by rank p // local_bsz.  gts_pinned[i] is None for the
        cameras whose images this rank does not hold; only the held images go to the device.  The ranks' view indices are
        all-gathered on the device and the batch's camera table is gathered there from a resident (N, 40) table, so the
        host never learns the other ranks' views.  The division reads no render times: none are gathered or fed back.
        model: instead of an activated scene (scene=None), this rank's six raw parameters as stored -- {group name
        (optim.GROUPS): tensor}, a shard of a PLY or checkpoint from model_io -- taken bit for bit (GaussianParams.from_raw);
        max_sh_degree then comes from their shape and the argument is not read.  shard=(lo, hi, n_total) gives the whole
        model's size; without it n_total is this rank's count at world size 1, and their sum over the ranks (one small
        all-reduce) otherwise."""
        self.local_sampling, self.local_bsz = bool(local_sampling), None
        if self.local_sampling:
            self._check_local_sampling(gts_pinned, device, world, group, local_bsz, distributed_dataset_storage,
                                       border_exchange)
        if deterministic and world > 1 and load_balance and not self.local_sampling:
            raise ValueError("deterministic=True needs a fixed strip division: pass load_balance=False when world > 1 "
                             "(the load balancer moves the strips by measured times)")
        # None: the operators follow torch.use_deterministic_algorithms
        self.deterministic = True if deterministic else None
        from . import exchange as _ex
        self._ex = _ex
        # splats travel by direct NVLink stores from the pack kernel and their gradients are pulled back over NVLink
        # (exchange.PeerBuffers) instead of all_to_all_single; peer_exchange=None: on unless GS_B200_EXCHANGE=nccl.
        # Buffers hold peer_cap_rows rows (default 1.25 x the scene's Gaussians); a step that needs more falls back to
        # all_to_all_single.
        if peer_exchange is None:
            import os as _os
            peer_exchange = _os.environ.get("GS_B200_EXCHANGE", "p2p") != "nccl"
        self._peer = None
        if model is not None:
            if scene is not None:
                raise ValueError("pass an activated scene or the raw parameters (model=...), not both")
            n = self._model_total(model, shard, device, world, group)
        else:
            n = scene["means3D"].shape[0] if shard is None else int(shard[2])
        if world > 1 and peer_exchange:
            # every splat of every local camera can land on one rank (bsz views of the scene): rows of the largest
            # receive / send total.  1.25 x the scene per view, capped by what a step can produce.
            cap = int(peer_cap_rows) if peer_cap_rows else int(1.25 * n) + 65536
            if self.local_sampling and not peer_cap_rows:   # a rank receives its local_bsz views whole
                cap = int(1.25 * n * self.local_bsz) + 65536
            self._peer = _ex.open_peer_buffers(world, rank, cap, device, group)
        if world > 1:
            # NCCL connects the point-to-point channels of all_to_all_single lazily, on first use: ~7 s on an 8-GPU box.  The
            # exchange needs them only when a step exceeds the peer buffers (and the redistribution after densification
            # always does): pay for the set-up here, not inside whichever training step happens to be the first.
            import torch.distributed as _dist
            if _dist.get_backend(group) == "nccl":
                _w = torch.zeros((world,), dtype=torch.float32, device=device)
                _dist.all_to_all_single(torch.empty_like(_w), _w, group=group)
        self.device, self.rank, self.world, self.group = device, rank, world, group
        self.lambda_dssim = lambda_dssim
        self.border_exchange = border_exchange   # legacy row L1: exchange 5 halo rows so strip losses sum to the full-image loss
        if model is not None:
            self.params = GaussianParams.from_raw(model, device)
            lo, hi = 0, self.params._xyz.shape[0]
        elif shard is None:
            lo, hi = n * rank // world, n * (rank + 1) // world
            self.params = GaussianParams({k: v[lo:hi] for k, v in scene.items()}, device, max_sh_degree)
        else:
            lo, hi = int(shard[0]), int(shard[1])
            if scene["means3D"].shape[0] != hi - lo:
                raise ValueError("shard=(lo, hi, n_total) does not match the scene passed")
            self.params = GaussianParams(scene, device, max_sh_degree)
        self.n_local, self.n_total = hi - lo, n
        self.load_balance, self.heuristic_decay = load_balance, heuristic_decay
        if feedback_lag is None:
            import os as _os
            feedback_lag = int(_os.environ.get("GS_B200_FEEDBACK_LAG", "2"))
        self.feedback_lag = max(0, int(feedback_lag))
        self._pending_feedback = []     # steps whose render times have not been fed back yet, oldest first
        self._sent_feedback = None      # the step whose times ride on the exchange of the current step
        self.iteration = 0
        self.balance_log = []      # (iteration, division rows of camera 0) whenever the division moved
        self.dcams = [DeviceCamera(c, device) for c in cams]
        if not self.dcams:
            raise ValueError("a Trainer needs at least one camera")
        self.H, self.W = self.dcams[0].image_height, self.dcams[0].image_width
        sizes = {(c.image_height, c.image_width) for c in self.dcams}
        if gts_pinned is not None:
            if len(gts_pinned) != len(self.dcams):
                raise ValueError(f"{len(self.dcams)} cameras but {len(gts_pinned)} ground-truth images")
            sizes |= {(int(g.shape[-2]), int(g.shape[-1])) for g in gts_pinned if g is not None}
        if len(sizes) > 1:
            raise ValueError(f"all cameras and images of a Trainer must share one image size (one TILE_Y, as in the "
                             f"reference); got (H, W) = {sorted(sizes)}")
        self.tile_y, self.tile_x = (self.H + 15) // 16, (self.W + 15) // 16
        self.distributed_dataset_storage = bool(distributed_dataset_storage) and world > 1
        self.gts_host = gts_pinned                      # uint8 (3,H,W) pinned host tensors
        # the "inputs resident" leg keeps every image on the device (--preload_dataset_to_gpu, scene/cameras.py:67-68); its
        # loss reads the strip rows in place (ops.fused_l1_ssim_batched(gt_full=True)).  Not needed by ranks without
        # pixels in distributed-storage mode.
        if self.local_sampling:   # only the images this rank holds
            self.gts_dev = [None if g is None else g.to(device) for g in gts_pinned]
        else:
            self.gts_dev = [g.to(device) for g in gts_pinned] if gts_pinned is not None else None
        self.history = StrategyHistory([c.uid for c in self.dcams], self.tile_y, world)
        self._strip_cache = {}     # pinned copies of the strips of non-pinned host images (resident=False)
        # (N,40) host table of the batched preprocess: a step copies the rows of its views to the device
        self._cam_rows = ops.pack_cameras([c.settings() for c in self.dcams]).cpu()
        self._cams_dev = None      # (views, (B,40) device table) of the last step
        # local sampling: the whole (N,40) table stays on the device, and a step gathers its batch's rows there
        self._cam_table_dev = self._cam_rows.to(device) if self.local_sampling else None
        self._whole_views = None   # ((world, rank), the whole-view division of a local-sampling batch)
        self._strategy_cache = None   # ((history version, the batch's camera uids), strategies)
        self._bmask_cache = {}
        self._copy_stream = None
        self._loss_host = None
        self._info = {}
        self._h2d = 0
        # per-view [Ll1, ssim] of every step since the last train_losses(): (slots, 2) fp32 and (slots,) int64 camera
        # indices on the device, grown geometrically; the host keeps (iteration, B) per step.  Only local sampling at
        # world size > 1 has batches whose camera indices the host does not know: the index buffer is filled then, and
        # the host lists them (_rec_host_index) otherwise.
        self._rec_pairs = self._rec_index = None
        self._rec_used, self._rec_steps, self._rec_host_index = 0, [], []
        self._rec_index_on_device = self.local_sampling and world > 1
        # the border path's (1 - lambda, -lambda): a strip's loss is its [Ll1, ssim] dotted with it, plus lambda, the
        # arithmetic of ops.fused_loss
        lam = float(lambda_dssim)
        self._loss_w = (torch.tensor([1.0 - lam, -lam], dtype=torch.float32, device=device)
                        if border_exchange else None)

    @staticmethod
    def _model_total(model, shard, device, world, group):
        """n_total of a Trainer built from raw parameters (the peer buffers are sized from it)."""
        P = int(model["xyz"].shape[0])
        if shard is not None:
            if int(shard[1]) - int(shard[0]) != P:
                raise ValueError(f"shard=(lo, hi, n_total) = {tuple(shard)} does not match the {P} Gaussians passed")
            return int(shard[2])
        if world == 1:
            return P
        import torch.distributed as dist
        dev = device if dist.get_backend(group) == "nccl" else "cpu"
        t = torch.tensor([P], dtype=torch.int64, device=dev)
        dist.all_reduce(t, group=group)
        return int(t.item())

    def _check_local_sampling(self, gts_pinned, device, world, group, local_bsz, distributed_dataset_storage,
                              border_exchange):
        """The construction-time refusals of local sampling, before any other collective.  local_bsz and the number of
        images each rank holds are all-gathered first (one small collective, none at world 1) and every rank decides from
        the gathered values, so a rank whose value differs raises together with the others instead of leaving them
        waiting in a collective."""
        if distributed_dataset_storage:
            raise ValueError("local_sampling: every rank holds the images of the views it samples; "
                             "distributed_dataset_storage has no meaning with it")
        if border_exchange:
            raise ValueError("local_sampling renders and scores whole views: border_exchange=True does not apply")
        try:
            k = operator.index(local_bsz)
        except TypeError:
            k = 0   # refused below, on every rank
        held = 0 if gts_pinned is None else sum(g is not None for g in gts_pinned)
        every = [[k, held]]
        if world > 1:
            import torch.distributed as dist
            allv = torch.empty((world * 2,), dtype=torch.int64, device=device)
            dist.all_gather_into_tensor(allv, torch.tensor([k, held], dtype=torch.int64, device=device), group=group)
            every = allv.reshape(world, 2).tolist()
        ks = [int(e[0]) for e in every]
        if ks[0] < 1 or any(v != ks[0] for v in ks):
            raise ValueError(f"local_sampling needs one positive local_bsz on every rank, got {ks} (in rank order)")
        if world * ks[0] > ops.MAX_VIEWS:
            raise ValueError(f"local_sampling: a batch of world size x local_bsz = {world * ks[0]} views exceeds the "
                             f"{ops.MAX_VIEWS} views of the batched kernels")
        from .exchange import MAX_CAMERAS
        if world > 1 and world * ks[0] > MAX_CAMERAS:
            raise ValueError(f"local_sampling: the exchange carries at most {MAX_CAMERAS} views per step, "
                             f"world size x local_bsz = {world * ks[0]}")
        empty = [r for r, e in enumerate(every) if int(e[1]) == 0]
        if empty:
            raise ValueError(f"local_sampling: rank(s) {empty} hold no training image (gts_pinned[i] is the image of "
                             f"camera i where the rank holds it, None elsewhere)")
        self.local_bsz = ks[0]

    def _mark(self, name):
        """GS_B200_TRACE=1: synchronise and accumulate wall-clock per phase (diagnostics only)."""
        if not self._trace_on:
            return
        import time
        torch.cuda.synchronize()
        now = time.perf_counter()
        self.trace[name] = self.trace.get(name, 0.0) + (now - self._t_last) * 1e3
        self._t_last = now

    def step(self, views=None, resident=True):
        """One forward + loss + backward over a batch of the camera set.  views: indices into the cameras, in batch
        order (a camera may appear more than once); None = all cameras in order.  The caller chooses them (the reference
        draws --bsz per step, train_internal.py:134).  resident=False copies the GT strips from pinned host memory inside
        the step and reads the loss back (the end-to-end leg); returns the loss as a float then.
        With local_sampling, views are this rank's own local_bsz views (required).
        Every step keeps its views' [Ll1, ssim] on the device for train_losses()."""
        views = self._local_views(views) if self.local_sampling else self._batch_views(views)
        ops.STEP_STREAM = torch.cuda.current_stream().cuda_stream   # every kernel of the step goes to this stream
        try:
            return self._step(views, resident)
        finally:
            ops.STEP_STREAM = None

    def evaluate(self, views=None, *, cams=None, gts=None, bsz=None):
        """training_report's L1 / PSNR (train_internal.py:355-490) over a set of views, rendered forward-only.
        cams / gts None: the Trainer's own cameras, scored against its own images (the reference's "train" config).
        cams + gts: a held-out set of camera dicts of the Trainer's image size and their uint8 (3,H,W) images, on the
        device (read in place) or on the host (pinned or not; a rank copies only its own strip rows).  With
        distributed_dataset_storage the images are rank 0's, scattered by strip as the training step scatters them (the
        other ranks' gts entries may be None).  views: indices into the chosen set, in order (None = all); choosing them
        -- the reference's truncation to whole batches and its sample of the training views -- is the caller's.
        bsz: views per batch, default all of them up to 64 on one rank and exchange.MAX_CAMERAS on several.

        Each batch runs the forward of a training step (_forward) over a fresh strip division of the listed views (the
        reference builds a fresh DivisionStrategyHistoryFinal per evaluation, :387) at the active SH degree, and
        ops.eval_sums_batched scores the local strips per tile row.  The slots of all batches are summed over the ranks in
        ONE all-reduce, exact because each tile row is local to one rank, and finalized on the device, so every view's
        numbers are the same bits at any world size, strip division and bsz.  One host read, at the end.  The training
        state -- division history, queued timing feedback, iteration, means2D / radii, gradients -- is left as it was.
        -> {"l1", "psnr": the means over the views (floats), "l1_per_view", "psnr_per_view": (n,) float64 on the device}"""
        args = self._eval_args("evaluate", views, cams, gts, bsz)
        with self._eval_state():
            return self._evaluate(*args)

    def image_metrics(self, views=None, *, cams=None, gts=None, bsz=None, images=False):
        """The SSIM and PSNR that render.py + metrics.py report for a trained scene (render.py:97-138,
        metrics.py:26-80), computed on the device from forward-only strip renders.  views, cams, gts and bsz are those of
        evaluate, and so are the refusals, the Trainer's background and active SH degree, and the untouched training state.

        Each local strip is quantized to 8 bits as render.py's clamp and save_image quantize it (ops.quantize_u8_batched)
        into a window with its ground truth; the 5 rows on each side that the 11 x 11 SSIM window reads come from the
        neighbouring strips' owners (image_halo.exchange_halos, one all_to_all_single per batch).
        ops.image_metric_sums_batched scores the windows per tile row in fp64, the slots of all batches are summed over
        the ranks in ONE all-reduce, exact because each tile row is local to one rank, and finalized on the device: every
        view's numbers are the same bits at any world size, strip division and bsz.  With images=False, one host read, at
        the end.  images=True also gathers the 8-bit renders on rank 0 (image_halo.gather_images, batch by batch, into
        host memory) for the caller to write; LPIPS, which needs downloaded network weights, is not computed.
        -> {"ssim", "psnr": the means over the views (floats), "ssim_per_view", "psnr_per_view": (n,) float64 on the
        device, "images": a list of the n uint8 (3,H,W) CPU renders in view order on rank 0 if images=True, else None}"""
        args = self._eval_args("image_metrics", views, cams, gts, bsz)
        with self._eval_state():
            return self._image_metrics(*args, bool(images))

    def train_losses(self):
        """The training loss of every view of every step since the last call, as the reference reports it each step
        (train_internal.py:211-238): per view [Ll1, ssim], both normalised by the full image's 3 H W, summed over the
        ranks, and (1 - lambda) Ll1 + lambda (1 - ssim).  A collective, like evaluate: every rank calls it after the same
        steps.  The steps' records are all-gathered in one all_gather_into_tensor (none at world size 1) and added in rank
        order on the device (sum_over_ranks), so the bits depend on the strip division only, not on NCCL's reduction
        order; one host read.  The records are then cleared.
        -> one entry per step, oldest first: {"iteration": the step's number (Trainer.iteration after it), "views": its
        camera indices in batch order, "l1", "ssim", "loss": lists of floats, one per view}; [] when no step is pending."""
        n = self._rec_used
        if n == 0:
            return []
        mine = self._rec_pairs[:n]
        if self.world > 1:
            import torch.distributed as dist
            allp = torch.empty((self.world * n, 2), dtype=torch.float32, device=self.device)
            dist.all_gather_into_tensor(allp, mine, group=self.group)
            gathered = allp.reshape(self.world, n, 2)
        else:
            gathered = mine[None]
        steps = self._rec_steps
        if self._rec_index_on_device:
            index = self._rec_index[:n]
        else:
            index = torch.tensor(self._rec_host_index, dtype=torch.int64).to(self.device)
        rows = loss_table(gathered, index, self.lambda_dssim).tolist()   # the call's one host read
        mine.zero_()   # unused slots stay +0.0 for the positions a later step has no strip of
        self._rec_used, self._rec_steps, self._rec_host_index = 0, [], []
        return loss_entries(rows, steps)

    def _record_losses(self, views, B, span=None, l1_ssim=None, strips=()):
        """Keep this step's (B, 2) [Ll1, ssim] in batch-position order: the span (lo, hi) of l1_ssim, or (k, (1,2) pair)
        per local strip; every other position stays +0.0.  Device copies into the record buffer, no host sync.  The
        camera indices stay on the host when it knows the batch; under local sampling at world size > 1 they are copied
        from the device-gathered batch index."""
        off = self._rec_used
        if self._rec_pairs is None or off + B > self._rec_pairs.shape[0]:
            cap = max(256, 2 * (0 if self._rec_pairs is None else self._rec_pairs.shape[0]), off + B)
            pairs = torch.zeros((cap, 2), dtype=torch.float32, device=self.device)
            index = torch.zeros((cap,), dtype=torch.int64, device=self.device)
            if off:
                pairs[:off].copy_(self._rec_pairs[:off]); index[:off].copy_(self._rec_index[:off])
            self._rec_pairs, self._rec_index = pairs, index
        if l1_ssim is not None:
            self._rec_pairs[off + span[0]:off + span[1]].copy_(l1_ssim.detach())
        for k, pair in strips:
            self._rec_pairs[off + k].copy_(pair.detach().reshape(2))
        if self._rec_index_on_device:
            self._rec_index[off:off + B].copy_(self._batch_index)
        else:
            self._rec_host_index.extend(views)
        self._rec_used = off + B
        self._rec_steps.append((self.iteration + 1, B))

    def _eval_args(self, name, views, cams, gts, bsz):
        """The refusals of evaluate / image_metrics, from the arguments alone, before any collective or launch.
        -> (device cameras, their images, views, bsz).  The Trainer's own images are its resident ones, or with
        distributed_dataset_storage rank 0's host images, scattered."""
        from .exchange import MAX_CAMERAS
        if cams is not None or gts is not None:
            if cams is None or gts is None:
                raise ValueError(f"{name}: pass cams and gts together (a held-out set), or neither (the Trainer's own)")
            if len(gts) != len(cams):
                raise ValueError(f"{name}: {len(cams)} cameras but {len(gts)} ground-truth images")
            dcams = [DeviceCamera(c, self.device) for c in cams]
            for dc in dcams:
                dc.bg = self.dcams[0].bg   # the Trainer's background, as training renders it
            sizes = {(c.image_height, c.image_width) for c in dcams}
            sizes |= {(int(g.shape[-2]), int(g.shape[-1])) for g in gts if g is not None}
            if sizes - {(self.H, self.W)}:
                raise ValueError(f"{name}: the held-out images must have the Trainer's size (H, W) = {(self.H, self.W)}, "
                                 f"got {sorted(sizes)}")
            for k, g in enumerate(gts):
                if g is not None and (g.dtype != torch.uint8 or tuple(g.shape) != (3, self.H, self.W)):
                    raise ValueError(f"{name}: gts[{k}] must be uint8 (3, {self.H}, {self.W}), got {g.dtype} "
                                     f"{tuple(g.shape)}")
                if g is not None and g.is_cuda and g.device != torch.device(self.device):
                    raise ValueError(f"{name}: gts[{k}] is on {g.device}, the Trainer on {self.device}")
            if (not self.distributed_dataset_storage or self.rank == 0) and any(g is None for g in gts):
                raise ValueError(f"{name}: a ground-truth image is None (only ranks other than 0 of a "
                                 "distributed_dataset_storage Trainer may leave them out)")
            gts = list(gts)
        else:
            if self.gts_dev is None and not self.distributed_dataset_storage:
                raise ValueError(f"{name}: this Trainer holds no images of its cameras; pass a held-out set")
            if self.local_sampling:
                raise ValueError(f"{name}: a local-sampling Trainer holds only its own rank's images, so it cannot score "
                                 "its camera set; pass a held-out set (cams=..., gts=...) on every rank")
            dcams, gts = self.dcams, self.gts_host if self.distributed_dataset_storage else self.gts_dev
        N = len(dcams)
        views = tuple(range(N)) if views is None else tuple(operator.index(v) for v in views)
        if not views:
            raise ValueError(f"{name}: no views listed")
        bad = [v for v in views if not 0 <= v < N]
        if bad:
            raise ValueError(f"{name}: views {bad} are not in the set (0..{N - 1})")
        cap = ops.MAX_VIEWS if self.world == 1 else MAX_CAMERAS
        if bsz is None:
            bsz = min(len(views), cap)
        bsz = operator.index(bsz)
        if not 1 <= bsz <= cap:
            raise ValueError(f"{name}: bsz must be in 1..{cap} at world size {self.world}, got {bsz}")
        return dcams, gts, views, bsz

    @contextlib.contextmanager
    def _eval_state(self):
        """Forward-only scoring: no gradients, no tracing, every kernel on the current stream; the tracing switch and the
        operators' pinned stream are restored afterwards."""
        saved = (getattr(self, "_trace_on", False), ops.STEP_STREAM)
        self._trace_on = False
        ops.STEP_STREAM = torch.cuda.current_stream().cuda_stream
        try:
            with torch.no_grad():
                yield
        finally:
            self._trace_on, ops.STEP_STREAM = saved

    def _eval_batches(self, dcams, gts, views, bsz):
        """The batches of an evaluation, bsz views each: a fresh strip division of the listed views (one history per
        call), each local strip's ground truth, and the forward.  Yields (strategies, rows, pairs, fw) per batch: rows[k]
        the local pixel rows of view k ((0, 0): none); pairs[k] its ground truth as gt_scatter.local_gt gives it, None or
        (tensor, row0); fw the _forward namespace."""
        p, H = self.params, self.H
        history = StrategyHistory(sorted({dcams[v].uid for v in views}), self.tile_y, self.world)
        for b0 in range(0, len(views), bsz):
            bviews = views[b0:b0 + bsz]
            bcams = [dcams[v] for v in bviews]
            strategies = start_strategy([c.uid for c in bcams], history, self.world, self.rank)[0]
            settings = [c.settings(p.active_sh_degree) for c in bcams]
            pairs = gt_scatter.local_gt(gts, bviews, strategies, H, self.W, self.device, self.rank, self.world,
                                        self.group, scatter=self.distributed_dataset_storage)[0]
            rows = [st.local_pixel_rows(H) or (0, 0) for st in strategies]
            fw = self._forward(settings[0], strategies, {}, lambda: ops.pack_cameras(settings), (0, len(bcams)),
                               training=False)
            yield strategies, rows, pairs, fw

    def _per_view(self, slots, finalize):
        """The slots of every batch summed over the ranks in ONE all-reduce and finalized batch by batch on the device.
        -> ((n, 2) per-view values, their means over the views as floats: the call's one host read)."""
        sizes = [s.shape[0] for s in slots]
        slots = torch.cat(slots) if len(slots) > 1 else slots[0]
        if self.world > 1:   # every tile row is non-zero on one rank only: the sum is exact in any order
            import torch.distributed as dist
            dist.all_reduce(slots, op=dist.ReduceOp.SUM, group=self.group)
        per_view = [finalize(s, self.H, self.W) for s in slots.split(sizes)]
        per_view = torch.cat(per_view) if len(per_view) > 1 else per_view[0]
        return per_view, (per_view.sum(0) / per_view.shape[0]).tolist()

    def _evaluate(self, dcams, gts, views, bsz):
        slots = [ops.eval_sums_batched(fw.images, [None if g is None else g[0] for g in pairs], rows,
                                       [0 if g is None else g[1] for g in pairs])
                 for _, rows, pairs, fw in self._eval_batches(dcams, gts, views, bsz)]
        per_view, means = self._per_view(slots, ops.eval_finalize)
        return {"l1": means[0], "psnr": means[1], "l1_per_view": per_view[:, 0], "psnr_per_view": per_view[:, 1]}

    def _image_metrics(self, dcams, gts, views, bsz, images):
        from . import image_halo
        H, W = self.H, self.W
        slots, pictures = [], []
        for strategies, rows, pairs, fw in self._eval_batches(dcams, gts, views, bsz):
            # per local strip a (6, rows, W) window of the strip and its halo: 8-bit render in channels 0-2, ground truth
            # in 3-5; the strip's own rows filled here, the halo rows by the neighbours' owners
            wins, win_row0 = [], []
            for (y0, y1), g in zip(rows, pairs):
                if g is None:
                    wins.append(None); win_row0.append(0)
                    continue
                (gt, row0), (a, b) = g, image_halo.window_rows((y0, y1), H)
                win = torch.empty((6, b - a, W), dtype=torch.uint8, device=self.device)
                win[3:, y0 - a:y1 - a].copy_(gt[:, y0 - row0:y1 - row0])
                wins.append(win); win_row0.append(a)
            ops.quantize_u8_batched(fw.images, rows, [None if w is None else w[:3] for w in wins], win_row0)
            if self.world > 1:
                image_halo.exchange_halos(wins, win_row0, strategies, H, W, self.rank, self.world, self.group, self.device)
            if any(w is not None for w in wins):
                slots.append(ops.image_metric_sums_batched(wins, win_row0, rows, H))
            else:   # no strip of this batch here: every slot is +0.0
                slots.append(torch.zeros((len(rows), self.tile_y, 2), dtype=torch.float64, device=self.device))
            if images:
                strips = [None if w is None else w[:3, y0 - a:y1 - a]
                          for w, a, (y0, y1) in zip(wins, win_row0, rows)]
                got = image_halo.gather_images(strips, strategies, H, W, self.rank, self.world, self.group, self.device)
                if got is not None:
                    pictures.extend(got)
        per_view, means = self._per_view(slots, ops.image_metric_finalize)   # the image copies are complete too
        return {"ssim": means[0], "psnr": means[1], "ssim_per_view": per_view[:, 0], "psnr_per_view": per_view[:, 1],
                "images": pictures if images and (self.rank == 0 or self.world == 1) else None}

    def _local_views(self, views):
        """This rank's views of a local-sampling step, refused before any collective or launch unless they are exactly
        local_bsz cameras whose images this rank holds."""
        if views is None:
            raise ValueError(f"local_sampling: step(views=...) takes this rank's {self.local_bsz} views")
        views = self._batch_views(views)
        if len(views) != self.local_bsz:
            raise ValueError(f"local_sampling: {len(views)} views passed, local_bsz is {self.local_bsz}")
        missing = [v for v in views if self.gts_host[v] is None]
        if missing:
            raise ValueError(f"local_sampling: this rank does not hold the images of views {missing}")
        return views

    def _whole_view_division(self):
        """The division of every local-sampling batch: position p whole on rank p // local_bsz.  It depends on positions
        only, so it is built once (per rank and world size) and never reads the load balancer's history."""
        key = (self.world, self.rank)
        if self._whole_views is None or self._whole_views[0] != key:
            B = self.world * self.local_bsz
            self._whole_views = (key, start_strategy_whole_views([None] * B, self.tile_y, self.world, self.rank)[0])
        return self._whole_views[1]

    def _gathered_camera_table(self, views):
        """(B,40) camera table of a local-sampling batch, built on the device: this rank's view indices are all-gathered in
        rank order (all_gather_into_tensor, as train_internal.py:119-128, without its read-back to the host) and the rows
        of the resident (N,40) table are picked at them.  The host never learns the other ranks' views."""
        mine = torch.tensor(views, dtype=torch.int64).pin_memory().to(self.device, non_blocking=True)
        if self.world > 1:
            import torch.distributed as dist
            idx = torch.empty((self.world * self.local_bsz,), dtype=torch.int64, device=self.device)
            dist.all_gather_into_tensor(idx, mine, group=self.group)
        else:
            idx = mine
        self._batch_index = idx                    # the batch's camera indices and table, kept until the next step
        self._batch_table = torch.index_select(self._cam_table_dev, 0, idx)
        return self._batch_table

    def _read_loss(self, loss_sum):
        """The step's loss as a float, through a pinned host word (the resident=False leg)."""
        if self._loss_host is None:
            self._loss_host = torch.zeros((1,), dtype=torch.float32).pin_memory()
        self._loss_host.copy_(loss_sum.detach().reshape(1), non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return float(self._loss_host[0])

    def _batch_views(self, views):
        N = len(self.dcams)
        if views is None:
            return tuple(range(N))
        views = tuple(operator.index(v) for v in views)   # TypeError for anything but integers
        if not 1 <= len(views) <= 64:   # GS_MAX_VIEWS of the batched kernels
            raise ValueError(f"a step trains on 1 to 64 views, got {len(views)}")
        for v in views:
            if not 0 <= v < N:
                raise ValueError(f"view {v} is not a camera of this Trainer (0..{N - 1})")
        return views

    def _batch_strategies(self, uids):
        """The strip division of a batch, cached per (history version, the batch's camera uids): it follows the cost
        heuristics of exactly those cameras.  The division-keyed mask / strip caches are only dropped when the load
        balancer moved the strips (a new history version), so batches that come and go keep theirs."""
        ver = len(self.history.history)   # the division only changes when the cost heuristic is updated
        prev = self._strategy_cache
        if prev is not None and prev[0] == (ver, uids):
            return prev[1]
        new = start_strategy(list(uids), self.history, self.world, self.rank)[0]
        moved = prev is None or len(new) != len(prev[1]) or any(
            a.gpu_ids != b.gpu_ids or a.division_pos != b.division_pos for a, b in zip(new, prev[1]))
        self._strategy_cache = ((ver, uids), new)
        if moved and (prev is None or prev[0][0] != ver):   # per-division caches belong to the old boundaries
            self._strip_cache.clear(); self._bmask_cache.clear()
            self.balance_log.append((self.iteration, [list(st.division_pos) for st in new],
                                     [list(st.gpu_ids) for st in new]))
        return new

    def _camera_table(self, views):
        """(B,40) device camera table of the batched preprocess: the views' rows gathered into pinned host memory and
        copied asynchronously (no host sync; the pinned block is not reused before the copy has run).  Kept while the
        views stay the same."""
        if self._cams_dev is None or self._cams_dev[0] != views:
            stage = torch.empty((len(views), self._cam_rows.shape[1]), dtype=torch.float32, pin_memory=True)
            torch.index_select(self._cam_rows, 0, torch.tensor(views, dtype=torch.int64), out=stage)
            self._cams_dev = (views, stage.to(self.device, non_blocking=True))
        return self._cams_dev[1]

    def _step_plan(self, views):
        """What sets a local-sampling step apart from the default one, decided once at the top of the step.
        -> (the batch's division, cam_table() -> its (B,40) device camera table, the span (lo, hi) of the batch positions
        this rank renders -- position p is the view views[p - lo] --, whether the render times are fed back)."""
        if self.local_sampling:   # the B = W x local_bsz views of all ranks, each rendered whole by the rank that drew it
            k = self.local_bsz
            return (self._whole_view_division(), lambda: self._gathered_camera_table(views),
                    (self.rank * k, (self.rank + 1) * k), False)
        strategies = self._batch_strategies(tuple(self.dcams[i].uid for i in views))
        return strategies, lambda: self._camera_table(views), (0, len(views)), True

    def _step(self, views, resident):
        import os as _os, time as _time
        self._trace_on = _os.environ.get("GS_B200_TRACE") == "1"
        if self._trace_on:
            if not hasattr(self, "trace"):
                self.trace = {}
            torch.cuda.synchronize()
            self._t_last = _time.perf_counter()
        p = self.params
        for t in p.raw_parameters():
            t.grad = None
        strategies, cam_table, (lo, hi), feedback = self._step_plan(views)
        rs = self.dcams[views[0]].settings(p.active_sh_degree)   # image size and background, shared by every view
        # "Asynchronously load ground-truth image to GPU" (loss_distribution.py:2399): host strips are copied on a side
        # stream while preprocess / binning / blend run, and the loss waits for them
        if not resident and self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        gt, self._h2d, ready = gt_scatter.local_gt(
            self.gts_dev if resident else self.gts_host, views, strategies[lo:hi], self.H, self.W, self.device,
            self.rank, self.world, self.group, scatter=self.distributed_dataset_storage and not resident,
            cache=self._strip_cache, stream=None if resident else self._copy_stream)
        collectors = [{} for _ in range(hi - lo)]
        fw = self._forward(rs, strategies, collectors[0], cam_table, (lo, hi), training=True, feedback=feedback)
        self.means2D, self._radii_local = fw.means2D, fw.radii
        if ready is not None:
            cur = torch.cuda.current_stream()
            cur.wait_event(ready)
            for g in gt:
                if g is not None:
                    g[0].record_stream(cur)
        if self.border_exchange:
            # the legacy row L1: one loss per local strip, summed in view order; a strip of a view split over several
            # ranks is widened by the 5 halo rows its neighbours render, so the strip losses sum to the full-image loss.
            # Each strip's [Ll1, ssim] is kept for the record; its loss is ops.fused_loss's arithmetic on it (the same
            # launch, dot with (1 - lambda, -lambda), + lambda), so the loss and gradients keep their bits.
            loss_sum, pairs = None, []
            for k, st in enumerate(strategies):
                if gt[k] is None:
                    continue
                rows = st.local_pixel_rows(self.H)
                if len(st.gpu_ids) > 1:
                    from . import border
                    image, (r0, r1), _ = border.add_remote_border_rows(fw.images[k], st, self.H, self.group)
                    g, rows4, gt_full = self.gts_dev[views[k]], (r0, r1, *rows), True
                else:   # the view is this rank's alone, so its strip is every row: the strip form
                    image, rows4, g, gt_full = fw.images[k], (*rows, *rows), gt[k][0], False
                pair = ops.fused_l1_ssim_batched(image[None], [g], [rows4], deterministic=self.deterministic,
                                                 gt_full=gt_full)
                pairs.append((k, pair))
                loss = torch.dot(pair.reshape(-1), self._loss_w) + float(self.lambda_dssim)
                loss_sum = loss if loss_sum is None else loss_sum + loss
            self._record_losses(views, len(strategies), strips=pairs)
        else:
            # the resident image of a one-view batch that is local whole is read as a strip of every row (no host-side
            # row tables); every other resident image is read in place at its strip rows
            gt_full = resident and not (len(views) == 1 and fw.rows4[0] == (0, self.H, 0, self.H))
            l1_ssim = ops.fused_l1_ssim_batched(fw.images, [None if g is None else g[0] for g in gt], fw.rows4,
                                                deterministic=self.deterministic, gt_full=gt_full)
            # sum over the local strips of (1 - lambda) Ll1 + lambda (1 - ssim)
            loss_sum = torch.dot(l1_ssim.reshape(-1), fw.coef) + fw.const
            self._record_losses(views, len(strategies), span=(lo, hi), l1_ssim=l1_ssim)
        self._mark("r render+loss")
        loss_sum.backward()
        self._mark("b4 backward (rest)")
        self._finish_step(strategies, collectors, dict(Vp=int(fw.view_start[-1]) - int(fw.view_start[0]),
                                                       P_local=sum((r[1] - r[0]) * self.W for r in fw.rows4)), feedback)
        self._mark("t time feedback")
        if resident:
            return None
        return self._read_loss(loss_sum)

    def _finish_step(self, strategies, collectors, counts, feedback):
        """The host bookkeeping after a step, and with feedback its render times queued for (or, with feedback_lag=0,
        applied to) the load balancer."""
        self._collectors, self._strategies, self._counts = collectors, strategies, counts
        self.iteration += 1
        if feedback:
            self._feed_back_times(strategies, collectors)

    def _preprocess(self, rs, cam_table, B, training):
        """This rank's Gaussians projected into the B views of a batch -> (means2D (B,P,2), rgb, conic_opacity, radii,
        depths): a one-view batch with its settings rs, more over the (B,40) device camera table cam_table(), built only
        then (ops._PreprocessRaw).  training: means2D keeps its gradient, which densification reads (means2D.grad of
        camera k, densification.py:24)."""
        p = self.params
        out = ops._PreprocessRaw.apply(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation, p._opacity, B,
                                       rs, cam_table, (self.W, self.H, p.active_sh_degree, 1.0))
        if training:
            out[0].retain_grad()
        return out

    @staticmethod
    def _concat(batched):
        """On one rank the (B,P,.) projections ARE the concatenation of the views' splats: camera k = rows [k P, (k+1) P).
        -> (concatenated tensors, view_start)."""
        B, Pn = batched[0].shape[:2]
        return tuple(t.reshape(B * Pn, *t.shape[2:]) for t in batched), [k * Pn for k in range(B + 1)]

    def _forward(self, rs, strategies, collector, cam_table, span, training, feedback=False):
        """The forward of one batch: preprocess (_preprocess) -> exchange of the projected splats (exchange_cat, W > 1) or
        their concatenation (W == 1) -> one batched render of the batch positions span = (lo, hi): every position for the
        strip division, this rank's own views for local sampling.  rs: the raster settings the views share (a one-view
        batch's own).  cam_table(): the (B,40) device camera table of the batched preprocess.  collector: the render's
        stats collector.  training: the screen-space gradient is retained (evaluate: not).  feedback: the load balancer's
        render times ride on the exchange.
        -> namespace of means2D (B,P,2) and radii (B,P) (this rank's pre-exchange values, which densification reads),
        images (hi - lo,3,H,W), the span's rows4 and loss weights coef / const, and its view_start."""
        B, (lo, hi) = len(strategies), span
        batched = self._preprocess(rs, cam_table, B, training)
        self._mark("p preprocess")
        if self.world > 1:
            times = self._feedback_before_exchange() if feedback else None
            cat, view_start, _cnt, gathered = self._ex.exchange_cat(*batched, strategies, [rs], self.world, self.rank,
                                                                    self.group, self._peer, times=times, mark=self._mark)
            if feedback:
                self._feedback_after_exchange(gathered)
        else:
            cat, view_start = self._concat(batched)
        self._mark("x5 unpack")
        view_start = view_start[lo:hi + 1]   # the positions outside the span have no rows here
        mk = (span, tuple((tuple(st.gpu_ids), tuple(st.division_pos), st.rank) for st in strategies))
        if mk not in self._bmask_cache:
            m = torch.zeros((hi - lo, self.tile_y, self.tile_x), dtype=torch.uint8, device=self.device)
            rows4, coef, const = [], [], 0.0
            for k, st in enumerate(strategies[lo:hi]):
                r = st.local_rows()
                if r is None:   # no strip of this camera here: no tiles, no loss term
                    rows4.append((0, 0, 0, 0))
                    coef += [0.0, 0.0]
                    continue
                m[k, r[0]:r[1]] = 1
                y0, y1 = st.local_pixel_rows(self.H)
                rows4.append((y0, y1, y0, y1))
                coef += [1.0 - self.lambda_dssim, -self.lambda_dssim]
                const += self.lambda_dssim
            self._bmask_cache[mk] = (m.reshape(hi - lo, -1), rows4,
                                     torch.tensor(coef, dtype=torch.float32, device=self.device), const)
        cl, rows4, coef, const = self._bmask_cache[mk]
        m2, rgb, co, radii, depths = cat
        images, _stats = ops.render_gaussians_batched(m2, co, rgb, depths, radii, cl, view_start, rs,
                                                      {"stats_collector": collector}, deterministic=self.deterministic)
        return SimpleNamespace(means2D=batched[0], radii=batched[3], images=images, rows4=rows4, coef=coef, const=const,
                               view_start=view_start)

    def _times_of(self, strategies, collectors):
        """This rank's gpu_camera_running_time row for one step: the render time of each camera it rendered a strip of.
        One batched render served all local strips; with several, its time is apportioned by strip height (the
        reference times every camera's render separately, render_final __init__.py:1217-1288)."""
        from .division import running_time_of
        mine = [-1.0] * len(strategies)
        rows = [(st.local_rows()[1] - st.local_rows()[0]) if st.local_rows() is not None else 0 for st in strategies]
        n_local = sum(1 for r in rows if r)
        if n_local:
            t = running_time_of(collectors[0])
            for k, r in enumerate(rows):
                if r:
                    mine[k] = t if n_local == 1 else t * r / sum(rows)
        return mine

    def _feedback_before_exchange(self):
        """feedback_lag > 0: the render times of the step `feedback_lag` steps back (its events have completed: the host is
        never more than one step ahead of the device), for the exchange to all-gather behind the sizes -> this rank's
        times, or None when no step's feedback is due."""
        self._sent_feedback = None
        if self.feedback_lag > 0 and len(self._pending_feedback) >= self.feedback_lag:
            self._sent_feedback = self._pending_feedback.pop(0)
            return self._times_of(self._sent_feedback[0], self._sent_feedback[1])
        return None

    def _feedback_after_exchange(self, times):
        """times: every rank's times as the exchange all-gathered them, (W, B) (None: none were sent)."""
        if self._sent_feedback is None:
            return
        strategies, _collectors, iteration = self._sent_feedback
        self._sent_feedback = None
        if times is not None:
            finish_strategy(self.history, strategies, times.tolist(), iteration, self.world, self.H, self.W,
                            self.heuristic_decay)

    def _feed_back_times(self, strategies, collectors):
        """finish_strategy_final (workload_division.py:944-998) + the time all-gather (utils/general_utils.py:249-269):
        every rank contributes the render time of each camera it rendered a strip of; the per-row cost heuristic is
        rebuilt from them and the strips of a later step move.  Only where the reference's gate enables it (more than
        one rank, and not when whole <= 1080p images can be handed out)."""
        import torch.distributed as dist
        B = len(strategies)
        if not (self.load_balance and self.world > 1 and
                heuristics_update_enabled(self.iteration, self.world, B, self.H, self.W)):
            self._pending_feedback.clear()
            return
        if self.feedback_lag > 0:   # fed back later, on the size all-gather of a coming exchange (_feedback_before_exchange)
            self._pending_feedback.append((strategies, collectors, self.iteration))
            return
        mine = self._times_of(strategies, collectors)
        loc = torch.tensor(mine, dtype=torch.float32, device=self.device)
        allt = torch.empty((self.world * B,), dtype=torch.float32, device=self.device)
        dist.all_gather_into_tensor(allt, loc, group=self.group)
        times = allt.reshape(self.world, B).cpu().tolist()       # gpu_camera_running_time[gpu][camera]
        finish_strategy(self.history, strategies, times, self.iteration, self.world, self.H, self.W, self.heuristic_decay)

    def add_densification_stats(self, xyz_gradient_accum, denom, max_radii2D):
        """The densification statistics of the last step (densification.py:15-24), in place, one launch, no host sync:
        densify.add_densification_stats over this rank's screen-space gradients and pre-exchange radii of every camera of
        the step (the reference's batched_locally_preprocessed_mean2D / _radii).  xyz_gradient_accum, denom: (P, 1),
        max_radii2D: (P,), float32, P = n_local."""
        from . import densify
        densify.add_densification_stats(xyz_gradient_accum, denom, max_radii2D, self.means2D.grad, self._radii_local)

    GROUP_OF = GROUPS

    def optimizer_groups(self, lrs=None):
        """The reference's six single-tensor groups over this trainer's parameters (scene/gaussian_model.py:257-292)."""
        lrs = lrs or {"xyz": 0.00016, "f_dc": 0.0025, "f_rest": 0.0025 / 20, "opacity": 0.05, "scaling": 0.005,
                      "rotation": 0.001}            # arguments/__init__.py:110-119
        return [{"params": [getattr(self.params, attr)], "lr": lrs[name], "name": name} for name, attr in GROUPS.items()]

    def adopt_parameters(self, new):
        """After densification / redistribution replaced the optimizer's tensors: new = {group name: nn.Parameter}."""
        for name, attr in GROUPS.items():
            setattr(self.params, attr, new[name])
        self.n_local = int(new["xyz"].shape[0])

    def last_info(self):
        """Realised sizes of the last step on this rank: V visible, V' splats rendered, R instances."""
        V = int((self._radii_local > 0).sum())
        R = self._collectors[0]["num_rendered"]   # the step's one render
        return dict(V=V, Vp=self._counts["Vp"], P_local=self._counts["P_local"], R=R)

    def io_bytes_per_step(self):
        """(host->device, device->host) bytes of the last resident=False step: GT strips in, loss out
        (+ the 8-byte instance count the step's one render reads back)."""
        return int(self._h2d), 4 + 8
