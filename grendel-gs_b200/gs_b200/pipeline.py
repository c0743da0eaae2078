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

from . import ops
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
        """The six raw parameters as they are stored (a PLY shard or a checkpoint, model_io): raw = {group name (Trainer.
        GROUP_OF): tensor}, taken bit for bit, with no activation inverted.  max_sh_degree comes from _features_rest's
        (P, (D+1)^2 - 1, 3); active_sh_degree starts at it."""
        if set(raw) != set(Trainer.GROUP_OF):
            raise ValueError(f"raw parameters need the groups {sorted(Trainer.GROUP_OF)}, got {sorted(raw)}")
        P = int(raw["xyz"].shape[0])
        for name, tail in cls.RAW_SHAPES.items():
            if tuple(raw[name].shape) != (P,) + tail:
                raise ValueError(f"raw parameter {name} must be {(P,) + tail}, got {tuple(raw[name].shape)}")
        Km1 = raw["f_rest"].shape[1] if raw["f_rest"].dim() == 3 else -1
        if raw["f_rest"].dim() != 3 or tuple(raw["f_rest"].shape) != (P, Km1, 3) or Km1 + 1 not in (1, 4, 9, 16):
            raise ValueError(f"raw parameter f_rest must be (P, (D+1)^2 - 1, 3) for D = 0..3, got "
                             f"{tuple(raw['f_rest'].shape)}")
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        for name, attr in Trainer.GROUP_OF.items():
            t = raw[name].detach().to(device=device, dtype=torch.float32)
            if not t.is_contiguous() or t.storage_offset() != 0:   # the kernels need 16-byte aligned, dense rows
                t = t.clone(memory_format=torch.contiguous_format)
            setattr(self, attr, nn.Parameter(t))
        self.max_sh_degree = int(round((Km1 + 1) ** 0.5)) - 1
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
        return [self._xyz, self._features_dc, self._features_rest, self._scaling, self._rotation, self._opacity]


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


class Trainer:
    """Distributed training-step harness (one process per GPU).

    Gaussians are sharded evenly by contiguous chunks (scene/gaussian_model.py:181-194); the B cameras of a
    step are divided into tile-row strips over the W ranks (division.start_strategy); projected splats reach
    their strip owners through exchange.exchange (skipped when W == 1, like gaussian_renderer/__init__.py:968).
    """

    def __init__(self, scene, cams, gts_pinned, device, rank=0, world=1, lambda_dssim=0.2, group=None,
                 fused_activations=True, border_exchange=False, batched_render=True, peer_exchange=None,
                 peer_cap_rows=None, shard=None, load_balance=True, heuristic_decay=0.0,
                 distributed_dataset_storage=False, feedback_lag=None, max_sh_degree=3, deterministic=False,
                 local_sampling=False, local_bsz=None, model=None):
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
        steps back, whose events have long completed, ride on the NEXT exchange's size all-gather (exchange.PIGGYBACK_IN):
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
        (GROUP_OF): tensor}, a shard of a PLY or checkpoint from model_io -- taken bit for bit (GaussianParams.from_raw);
        max_sh_degree then comes from their shape and the argument is not read.  shard=(lo, hi, n_total) gives the whole
        model's size; without it n_total is this rank's count at world size 1, and their sum over the ranks (one small
        all-reduce) otherwise."""
        self.local_sampling, self.local_bsz = bool(local_sampling), None
        if self.local_sampling:
            self._check_local_sampling(gts_pinned, device, world, group, local_bsz, distributed_dataset_storage,
                                       fused_activations, batched_render, border_exchange)
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
        # bin + blend + loss of all B cameras in one pass (ops.render_gaussians_batched) instead of the reference's
        # per-camera loop (render_final, gaussian_renderer/__init__.py:1217-1288); False keeps the per-camera calls
        self.batched_render = batched_render
        self.device, self.rank, self.world, self.group = device, rank, world, group
        self.lambda_dssim = lambda_dssim
        self.fused_activations = fused_activations
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
        self._mask_cache = {}
        self._bmask_cache = {}
        self._n_renders = 0
        self._copy_stream = None
        self._loss_host = None
        self._local_coef = None    # local sampling: (the loss weights of the local_bsz views, the constant term)
        self._info = {}
        self._h2d = 0

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
                              fused_activations, batched_render, border_exchange):
        """The construction-time refusals of local sampling, before any other collective.  local_bsz and the number of
        images each rank holds are all-gathered first (one small collective, none at world 1) and every rank decides from
        the gathered values, so a rank whose value differs raises together with the others instead of leaving them
        waiting in a collective."""
        if distributed_dataset_storage:
            raise ValueError("local_sampling: every rank holds the images of the views it samples; "
                             "distributed_dataset_storage has no meaning with it")
        if not fused_activations or not batched_render or border_exchange:
            raise ValueError("local_sampling runs the fused-activation batched preprocess and render over whole views: "
                             "fused_activations=False, batched_render=False and border_exchange=True do not apply")
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

    # -- ground truth strips (load_camera_from_cpu_to_all_gpu, loss_distribution.py:2395-2533) ------------
    def _strip_h2d(self, host, y0, y1, cache_key=None):
        """Rows [y0, y1) of a (3,H,W) uint8 host image -> a (3, rows, W) device strip: the rows of one channel are
        contiguous in the image, so the strip is three asynchronous copies straight out of a pinned image -- no staging
        copy, and nothing to re-pin when the load balancer moves the strip boundaries (a pinned staging strip per division
        cost several ms of cudaHostAlloc every time the strips of a 4K view moved).  A pageable image with a cache_key
        goes through a pinned copy of the strip kept in the strip cache; without one, the three copies stage through
        pageable memory."""
        if not host.is_pinned() and cache_key is not None:
            key = (cache_key, y0, y1, False)
            if key not in self._strip_cache:
                self._strip_cache[key] = host[:, y0:y1, :].contiguous().pin_memory()
            return self._strip_cache[key].to(self.device, non_blocking=True)
        d = torch.empty((3, y1 - y0, self.W), dtype=torch.uint8, device=self.device)
        for c in range(3):
            d[c].copy_(host[c, y0:y1, :], non_blocking=True)
        return d

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
        With local_sampling, views are this rank's own local_bsz views (required), and the step is _step_local."""
        views = self._local_views(views) if self.local_sampling else self._batch_views(views)
        ops.STEP_STREAM = torch.cuda.current_stream().cuda_stream   # every kernel of the step goes to this stream
        try:
            return self._step_local(views, resident) if self.local_sampling else self._step(views, resident)
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

    def _eval_args(self, name, views, cams, gts, bsz):
        """The refusals of evaluate / image_metrics, from the arguments alone, before any collective or launch.
        -> (device cameras, their images, views, bsz, held_out)."""
        from .exchange import MAX_CAMERAS
        held_out = cams is not None or gts is not None
        if held_out:
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
            host = list(gts)
        else:
            if self.gts_dev is None and not self.distributed_dataset_storage:
                raise ValueError(f"{name}: this Trainer holds no images of its cameras; pass a held-out set")
            if self.local_sampling:
                raise ValueError(f"{name}: a local-sampling Trainer holds only its own rank's images, so it cannot score "
                                 "its camera set; pass a held-out set (cams=..., gts=...) on every rank")
            dcams, host = self.dcams, self.gts_host
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
        return dcams, host, views, bsz, held_out

    @contextlib.contextmanager
    def _eval_state(self):
        """Forward-only scoring: no gradients, no tracing, every kernel on the current stream; the step's globals are
        restored afterwards."""
        saved = (ops.LAST_R_TOTAL, getattr(self, "_trace_on", False), self._ex.TRACE, ops.STEP_STREAM)
        self._trace_on, self._ex.TRACE = False, None
        ops.STEP_STREAM = torch.cuda.current_stream().cuda_stream
        try:
            with torch.no_grad():
                yield
        finally:
            ops.LAST_R_TOTAL, self._trace_on, self._ex.TRACE, ops.STEP_STREAM = saved

    def _eval_batches(self, dcams, host, views, bsz, held_out):
        """The batches of an evaluation, bsz views each: a fresh strip division of the listed views (one history per
        call), each local strip's ground truth, and the forward.  Yields (strategies, rows, gts, gt_row0, fw) per batch:
        rows[k] the local pixel rows of view k ((0, 0): none); gts[k] a device image holding rows [gt_row0[k], ...) of its
        ground truth -- a resident image in place, or a strip -- or None; fw the _forward namespace."""
        p, H = self.params, self.H
        history = StrategyHistory(sorted({dcams[v].uid for v in views}), self.tile_y, self.world)
        for b0 in range(0, len(views), bsz):
            bviews = views[b0:b0 + bsz]
            bcams = [dcams[v] for v in bviews]
            strategies, tasks = start_strategy([c.uid for c in bcams], history, self.world, self.rank)
            settings = [c.settings(p.active_sh_degree) for c in bcams]
            # each local strip's ground truth and its first row: resident images in place, host images by strip rows
            gts, gt_row0, rows = [], [], []
            if self.distributed_dataset_storage:
                from . import gt_scatter
                strips, _ = gt_scatter.scatter_gt_strips([host[v] for v in bviews] if self.rank == 0 else self.W, tasks,
                                                         H, self.device, self.rank, self.world, self.group)
            for k, st in enumerate(strategies):
                r = st.local_pixel_rows(H)
                if r is None:
                    gts.append(None); gt_row0.append(0); rows.append((0, 0))
                    continue
                rows.append(r)
                if self.distributed_dataset_storage:
                    gts.append(strips[k]); gt_row0.append(r[0])
                elif not held_out:
                    gts.append(self.gts_dev[bviews[k]]); gt_row0.append(0)
                elif host[bviews[k]].is_cuda:
                    gts.append(host[bviews[k]]); gt_row0.append(0)
                else:
                    gts.append(self._strip_h2d(host[bviews[k]], r[0], r[1])); gt_row0.append(r[0])
            collectors = [{} for _ in bcams]
            fw = self._forward(settings, strategies, collectors, lambda: ops.pack_cameras(settings), training=False)
            yield strategies, rows, gts, gt_row0, fw

    def _sum_slots_over_ranks(self, slots):
        if self.world > 1:   # every tile row is non-zero on one rank only: the sum is exact in any order
            import torch.distributed as dist
            dist.all_reduce(slots, op=dist.ReduceOp.SUM, group=self.group)
        return slots

    def _evaluate(self, dcams, host, views, bsz, held_out):
        batches, slots = [], []
        for strategies, rows, gts, gt_row0, fw in self._eval_batches(dcams, host, views, bsz, held_out):
            if fw.images is not None:
                s = ops.eval_sums_batched(fw.images, gts, rows, gt_row0)
            else:   # per-camera renders; the slots of cameras without a strip here stay +0.0
                s = torch.zeros((len(strategies), self.tile_y, 3, 2), dtype=torch.float64, device=self.device)
                for k, image, _n in fw.per_camera:
                    s[k] = ops.eval_sums_batched(image.unsqueeze(0), gts[k:k + 1], rows[k:k + 1], gt_row0[k:k + 1])[0]
            slots.append(s)
            batches.append(len(strategies))
        slots = self._sum_slots_over_ranks(torch.cat(slots) if len(slots) > 1 else slots[0])
        per_view, b0 = [], 0
        for b in batches:
            per_view.append(ops.eval_finalize(slots[b0:b0 + b], self.H, self.W))
            b0 += b
        per_view = torch.cat(per_view) if len(per_view) > 1 else per_view[0]
        means = (per_view.sum(0) / len(views)).tolist()   # the call's one host read
        return {"l1": means[0], "psnr": means[1], "l1_per_view": per_view[:, 0], "psnr_per_view": per_view[:, 1]}

    def _image_metrics(self, dcams, host, views, bsz, held_out, images):
        from . import image_halo
        H, W = self.H, self.W
        batches, slots, pictures = [], [], []
        for strategies, rows, gts, gt_row0, fw in self._eval_batches(dcams, host, views, bsz, held_out):
            # per local strip a (6, rows, W) window of the strip and its halo: 8-bit render in channels 0-2, ground truth
            # in 3-5; the strip's own rows filled here, the halo rows by the neighbours' owners
            wins, win_row0 = [], []
            for k, (y0, y1) in enumerate(rows):
                if y1 == y0:
                    wins.append(None); win_row0.append(0)
                    continue
                a, b = image_halo.window_rows((y0, y1), H)
                win = torch.empty((6, b - a, W), dtype=torch.uint8, device=self.device)
                win[3:, y0 - a:y1 - a].copy_(gts[k][:, y0 - gt_row0[k]:y1 - gt_row0[k]])
                wins.append(win); win_row0.append(a)
            if fw.images is not None:
                ops.quantize_u8_batched(fw.images, rows, [None if w is None else w[:3] for w in wins], win_row0)
            for k, image, _n in fw.per_camera:
                ops.quantize_u8_batched(image.unsqueeze(0), rows[k:k + 1], [wins[k][:3]], win_row0[k:k + 1])
            if self.world > 1:
                image_halo.exchange_halos(wins, win_row0, strategies, H, W, self.rank, self.world, self.group, self.device)
            if any(w is not None for w in wins):
                slots.append(ops.image_metric_sums_batched(wins, win_row0, rows, H))
            else:   # no strip of this batch here: every slot is +0.0
                slots.append(torch.zeros((len(rows), self.tile_y, 2), dtype=torch.float64, device=self.device))
            batches.append(len(strategies))
            if images:
                strips = [None if w is None else w[:3, y0 - a:y1 - a]
                          for w, a, (y0, y1) in zip(wins, win_row0, rows)]
                got = image_halo.gather_images(strips, strategies, H, W, self.rank, self.world, self.group, self.device)
                if got is not None:
                    pictures.extend(got)
        slots = self._sum_slots_over_ranks(torch.cat(slots) if len(slots) > 1 else slots[0])
        per_view, b0 = [], 0
        for b in batches:
            per_view.append(ops.image_metric_finalize(slots[b0:b0 + b], H, W))
            b0 += b
        per_view = torch.cat(per_view) if len(per_view) > 1 else per_view[0]
        means = (per_view.sum(0) / len(views)).tolist()   # the call's one host read; the image copies are complete too
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

    def _step_local(self, views, resident):
        """One local-sampling step.  Every rank projects its Gaussian shard into all B = W x local_bsz views of the batch
        (the camera table gathered on the device), the exchange hands each rank the splats of its own views, and the rank
        renders them whole in one batched render and scores them against its own images.  No timing feedback: the
        division does not read it."""
        self._trace_on = False
        self._ex.TRACE = None
        p = self.params
        for t in p.raw_parameters():
            t.grad = None
        self._h2d = 0
        ops.LAST_R_TOTAL = 0
        k, B, H = self.local_bsz, self.world * self.local_bsz, self.H
        strategies = self._whole_view_division()
        rs = self.dcams[views[0]].settings(p.active_sh_degree)   # image size and background, shared by every view
        gt_ready = []
        if not resident:   # the whole own images from pinned host memory, on the copy stream, while the render runs
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream(device=self.device)
            for v in views:
                with torch.cuda.stream(self._copy_stream):
                    d = self._strip_h2d(self.gts_host[v], 0, H, cache_key=v)
                    self._h2d += d.numel()
                    ev = torch.cuda.Event()
                    ev.record(self._copy_stream)
                gt_ready.append((d, ev))
        if B == 1:   # one view on one rank: the per-camera preprocess, as the default one-view step runs it
            out = ops.preprocess_gaussians_raw(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                               p._opacity, rs)
            out[0].retain_grad()
            self.means2D = [out[0]]
            batched = tuple(t.unsqueeze(0) for t in out)
        else:
            batched = ops.preprocess_gaussians_batched(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                                       p._opacity, self._gathered_camera_table(views), self.W, self.H,
                                                       p.active_sh_degree)
            batched[0].retain_grad()   # (B,P,2): densification reads the screen-space gradients of all B views
            self.means2D = batched[0]
        self._radii_local = batched[3]
        if self.world > 1:
            self._ex.PIGGYBACK_IN = None   # no render times ride on the exchange
            cat, view_start, _cnt = self._ex.exchange_cat(*batched, strategies, [rs], self.world, self.rank, self.group,
                                                          self._peer)
            view_start = view_start[self.rank * k:(self.rank + 1) * k + 1]   # the other views have no rows here
        else:
            Pn = batched[0].shape[1]
            cat = (batched[0].reshape(-1, 2), batched[1].reshape(-1, 3), batched[2].reshape(-1, 4),
                   batched[3].reshape(-1), batched[4].reshape(-1))
            view_start = [q * Pn for q in range(B + 1)]
        collectors = [{} for _ in range(k)]
        m2, rgb, co, radii, depths = cat
        images, _stats = ops.render_gaussians_batched(m2, co, rgb, depths, radii, None, view_start, rs,
                                                      {"stats_collector": collectors[0]}, deterministic=self.deterministic)
        if resident:   # the whole resident images, read in place
            gts = [self.gts_dev[v] for v in views]
        else:
            gts = []
            for gt, ev in gt_ready:
                torch.cuda.current_stream().wait_event(ev)
                gt.record_stream(torch.cuda.current_stream())
                gts.append(gt)
        if self._local_coef is None:   # the weights and constant the default batched step forms for whole strips
            coef, const = [], 0.0
            for _ in range(k):
                coef += [1.0 - self.lambda_dssim, -self.lambda_dssim]
                const += self.lambda_dssim
            self._local_coef = (torch.tensor(coef, dtype=torch.float32, device=self.device), const)
        coef, const = self._local_coef
        l1_ssim = ops.fused_l1_ssim_batched(images, gts, [(0, H, 0, H)] * k, deterministic=self.deterministic,
                                            gt_full=resident)
        loss_sum = torch.dot(l1_ssim.reshape(-1), coef) + const
        loss_sum.backward()
        self._n_renders = 1
        self._finish_local_step(strategies, collectors, int(view_start[-1]) - int(view_start[0]))
        if resident:
            return None
        return self._read_loss(loss_sum)

    def _finish_local_step(self, strategies, collectors, n_splats):
        """The host bookkeeping after a local-sampling step.  Nothing is queued for the load balancer."""
        self._collectors, self._strategies = collectors, strategies
        self._counts = dict(Vp=n_splats, P_local=self.local_bsz * self.H * self.W)
        self.iteration += 1

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
            self._strip_cache.clear(); self._mask_cache.clear(); self._bmask_cache.clear()
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

    def _step(self, views, resident):
        import os as _os, time as _time
        self._trace_on = _os.environ.get("GS_B200_TRACE") == "1"
        self._ex.TRACE = self._mark if self._trace_on else None
        if self._trace_on:
            if not hasattr(self, "trace"):
                self.trace = {}
            torch.cuda.synchronize()
            self._t_last = _time.perf_counter()
        p = self.params
        for t in p.raw_parameters():
            t.grad = None
        self._h2d = 0
        ops.LAST_R_TOTAL = 0
        dcams = [self.dcams[i] for i in views]
        strategies = self._batch_strategies(tuple(c.uid for c in dcams))
        self._tasks = [[(k, st.division_pos[st.gpu_ids.index(g)], st.division_pos[st.gpu_ids.index(g) + 1])
                        for k, st in enumerate(strategies) if g in st.gpu_ids] for g in range(self.world)]
        settings = [c.settings(p.active_sh_degree) for c in dcams]
        # "Asynchronously load ground-truth image to GPU" (loss_distribution.py:2399): the strips this rank needs are
        # copied from pinned host memory on a side stream while preprocess / binning / blend run, and the loss waits
        # on the copy's event.
        gt_ready = {}
        if not resident and self.distributed_dataset_storage:
            from . import gt_scatter
            batch_host = [self.gts_host[i] for i in views] if self.rank == 0 else self.W
            strips, h2d = gt_scatter.scatter_gt_strips(batch_host, self._tasks, self.H,
                                                       self.device, self.rank, self.world, self.group)
            self._h2d += h2d
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            gt_ready = {k: (t, ev) for k, t in strips.items()}
        elif not resident:
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream(device=self.device)
            for k, st in enumerate(strategies):
                rows = st.local_pixel_rows(self.H)
                if rows is None:
                    continue
                with torch.cuda.stream(self._copy_stream):
                    d = self._strip_h2d(self.gts_host[views[k]], rows[0], rows[1], cache_key=views[k])
                    self._h2d += d.numel()
                    ev = torch.cuda.Event()
                    ev.record(self._copy_stream)
                gt_ready[k] = (d, ev)
        collectors = [{} for _ in dcams]
        fw = self._forward(settings, strategies, collectors, lambda: self._camera_table(views), training=True)
        self.means2D, self._radii_local, self._n_renders = fw.means2D, fw.radii, fw.n_renders
        loss_sum = None
        Vp = Pl = 0
        if fw.images is not None:   # one batched render of every local strip
            rows4, coef, const = fw.rows4, fw.coef, fw.const
            gts = []
            for k, (y0, y1, _c0, _c1) in enumerate(rows4):
                if y1 == y0:
                    gts.append(None)
                elif resident:   # the whole resident image, read in place
                    gts.append(self.gts_dev[views[k]])
                else:
                    gt, ev = gt_ready[k]
                    torch.cuda.current_stream().wait_event(ev)
                    gt.record_stream(torch.cuda.current_stream())
                    gts.append(gt)
            l1_ssim = ops.fused_l1_ssim_batched(fw.images, gts, rows4, deterministic=self.deterministic, gt_full=resident)
            # sum over the local strips of (1 - lambda) Ll1 + lambda (1 - ssim)
            loss_sum = torch.dot(l1_ssim.reshape(-1), coef) + const
            Vp = int(fw.view_start[-1])
            Pl = sum((r[1] - r[0]) * self.W for r in rows4)
        for k, image, n_splats in fw.per_camera:
            st = strategies[k]
            y0, y1 = st.local_pixel_rows(self.H)
            if self.border_exchange and self.world > 1 and len(st.gpu_ids) > 1:
                from . import border
                image, (r0, r1), _ = border.add_remote_border_rows(image, st, self.H, self.group)
                loss = ops.fused_loss(image, self.gts_dev[views[k]], r0, r1, self.lambda_dssim, y0, y1,
                                      deterministic=self.deterministic, gt_full=True)
            else:
                if resident:
                    gt = self.gts_dev[views[k]]
                else:
                    gt, ev = gt_ready[k]
                    torch.cuda.current_stream().wait_event(ev)
                    gt.record_stream(torch.cuda.current_stream())
                # a strip of every row is the resident image itself: the strip form reads it with no host-side row
                # tables (the single-rank step); only a part of the image needs the in-place form
                loss = ops.fused_loss(image, gt, y0, y1, self.lambda_dssim, deterministic=self.deterministic,
                                      gt_full=resident and (y0, y1) != (0, self.H))
            loss_sum = loss if loss_sum is None else loss_sum + loss
            Vp += n_splats
            Pl += (y1 - y0) * self.W
        self._mark("r render+loss")
        loss_sum.backward()
        self._mark("b4 backward (rest)")
        self._collectors, self._strategies = collectors, strategies
        self._counts = dict(Vp=Vp, P_local=Pl)
        self.iteration += 1
        self._feed_back_times(strategies, collectors)
        self._mark("t time feedback")
        if resident:
            return None
        return self._read_loss(loss_sum)

    def _forward(self, settings, strategies, collectors, cam_table, training):
        """The forward of one batch, on the path the Trainer's options select: preprocess (all cameras in one batched launch
        with fused activations, else per camera) -> exchange of the projected splats (W > 1) -> render (one batched render
        of every local strip, else one render per camera with a strip here).  cam_table(): the (B,40) device camera table
        of the batched preprocess.  training=False (evaluate): no screen-space gradient is retained and no render times
        ride on the exchange.
        -> namespace of means2D and radii (this rank's pre-exchange values, which densification reads); images (B,3,H,W)
        of the batched render with its rows4 / coef / const / view_start, or None; per_camera [(camera index, image (3,H,W),
        splats rendered)] of the per-camera renders; n_renders."""
        p = self.params
        if not self.fused_activations:  # the reference's five activation kernels + cat (__init__.py:902-906)
            xyz, scaling, rotation, feats, opacity = p.get_xyz, p.get_scaling, p.get_rotation, p.get_features, p.get_opacity
        screen = []
        B = len(settings)
        use_batched = self.batched_render and B > 1 and not self.border_exchange
        if self.fused_activations and B > 1:
            # all B cameras in ONE launch: every Gaussian is read once and projected into each camera
            bm2, brgb, bco, bradii, bdepths = ops.preprocess_gaussians_batched(
                p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation, p._opacity, cam_table(),
                self.W, self.H, p.active_sh_degree)
            if training:
                bm2.retain_grad()   # (B,P,2): densification reads bm2.grad[k] (means2D.grad of camera k, densification.py:24)
            batched = (bm2, brgb, bco, bradii, bdepths)
            if self.world == 1 and not use_batched:
                for k in range(B):
                    screen.append((bm2[k], brgb[k], bco[k], bradii[k], bdepths[k]))
            settings_loop = []
        else:
            batched = None
            settings_loop = settings
        for k, rs in enumerate(settings_loop):
            if self.fused_activations:
                out = ops.preprocess_gaussians_raw(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                                   p._opacity, rs)
            else:
                out = ops.preprocess_gaussians(xyz, scaling, rotation, feats, opacity, rs,
                                               {"stats_collector": collectors[k]})
            if training:
                out[0].retain_grad()
            screen.append(out)
        means2D = batched[0] if batched is not None else [s[0] for s in screen]
        self._mark("p preprocess")
        if batched is None and (self.world > 1 or use_batched):
            # per-camera results (B == 1 or unfused activations): stack into (B,P,.)
            batched = tuple(torch.stack([s[q] for s in screen]) for q in range(5))
        cat = view_start = None
        if self.world > 1:
            if training:
                self._feedback_before_exchange()
            else:
                self._ex.PIGGYBACK_IN = None
            if use_batched:
                cat, view_start, cnt = self._ex.exchange_cat(*batched, strategies, settings, self.world, self.rank,
                                                             self.group, self._peer)
            else:
                redistributed, cnt = self._ex.exchange(*batched, strategies, settings, self.world, self.rank, self.group,
                                                       self._peer)
            if training:
                self._feedback_after_exchange()
        elif use_batched:   # (B,P,.) stacked IS the concatenation: camera k = rows [k P, (k+1) P)
            Pn = batched[0].shape[1]
            cat = (batched[0].reshape(-1, 2), batched[1].reshape(-1, 3), batched[2].reshape(-1, 4),
                   batched[3].reshape(-1), batched[4].reshape(-1))
            view_start = [k * Pn for k in range(B + 1)]
        else:
            redistributed = screen
        radii = (batched[3] if batched is not None else
                 screen[0][3].unsqueeze(0) if len(screen) == 1 else torch.stack([s[3] for s in screen]))
        self._mark("x5 unpack")
        fw = SimpleNamespace(means2D=means2D, radii=radii, images=None, view_start=view_start, per_camera=[],
                             n_renders=0)
        if use_batched:
            mk = tuple((tuple(st.gpu_ids), tuple(st.division_pos), st.rank) for st in strategies)
            if mk not in self._bmask_cache:
                m = torch.zeros((B, self.tile_y, self.tile_x), dtype=torch.uint8, device=self.device)
                rows4, coef, const = [], [], 0.0
                for k, st in enumerate(strategies):
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
                self._bmask_cache[mk] = (m.reshape(B, -1), rows4,
                                         torch.tensor(coef, dtype=torch.float32, device=self.device), const)
            cl, fw.rows4, fw.coef, fw.const = self._bmask_cache[mk]
            m2, rgb, co, radii, depths = cat
            fw.images, _stats = ops.render_gaussians_batched(m2, co, rgb, depths, radii, cl, view_start, settings[0],
                                                             {"stats_collector": collectors[0]},
                                                             deterministic=self.deterministic)
            fw.n_renders = 1
            return fw
        for k, st in enumerate(strategies):
            rows = st.local_rows()
            if rows is None:
                continue
            fw.n_renders += 1
            m2, rgb, co, radii, depths = redistributed[k]
            ck = (tuple(st.gpu_ids), tuple(st.division_pos), st.rank)
            if ck not in self._mask_cache:
                self._mask_cache[ck] = st.get_compute_locally(self.tile_x, self.device)
            cl = self._mask_cache[ck]
            image, *_ = ops.render_gaussians(m2, co, rgb, depths, radii, cl, settings[k],
                                             {"stats_collector": collectors[k]}, deterministic=self.deterministic)
            fw.per_camera.append((k, image, m2.shape[0]))
        return fw

    def _times_of(self, strategies, collectors, n_renders):
        """This rank's gpu_camera_running_time row for one step: the render time of each camera it rendered a strip of."""
        from .division import running_time_of
        B = len(strategies)
        mine = [-1.0] * B
        rows = [(st.local_rows()[1] - st.local_rows()[0]) if st.local_rows() is not None else 0 for st in strategies]
        if n_renders == 1 and sum(1 for r in rows if r) > 1:
            # one batched render served all local strips: its time is apportioned by strip height (the reference times
            # every camera's render separately, render_final __init__.py:1217-1288)
            t = running_time_of(collectors[0])
            for k, r in enumerate(rows):
                if r:
                    mine[k] = t * r / sum(rows)
        else:
            for k, r in enumerate(rows):
                if r:
                    c = collectors[k] if "forward_render_time" in collectors[k] else collectors[0]
                    mine[k] = running_time_of(c)
        return mine

    def _feedback_before_exchange(self):
        """feedback_lag > 0: hand the render times of the step `feedback_lag` steps back (its events have completed: the
        host is never more than one step ahead of the device) to the exchange, which all-gathers them behind the sizes."""
        self._ex.PIGGYBACK_IN, self._sent_feedback = None, None
        if self.feedback_lag > 0 and len(self._pending_feedback) >= self.feedback_lag:
            entry = self._pending_feedback.pop(0)
            self._ex.PIGGYBACK_IN = self._times_of(entry[0], entry[1], entry[3])
            self._sent_feedback = entry

    def _feedback_after_exchange(self):
        if self._sent_feedback is None:
            return
        strategies, _collectors, iteration, _n = self._sent_feedback
        times = self._ex.PIGGYBACK_OUT
        self._ex.PIGGYBACK_IN, self._sent_feedback = None, None
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
            self._pending_feedback.append((strategies, collectors, self.iteration, self._n_renders))
            return
        mine = self._times_of(strategies, collectors, self._n_renders)
        loc = torch.tensor(mine, dtype=torch.float32, device=self.device)
        allt = torch.empty((self.world * B,), dtype=torch.float32, device=self.device)
        dist.all_gather_into_tensor(allt, loc, group=self.group)
        times = allt.reshape(self.world, B).cpu().tolist()       # gpu_camera_running_time[gpu][camera]
        finish_strategy(self.history, strategies, times, self.iteration, self.world, self.H, self.W, self.heuristic_decay)

    def add_densification_stats(self, xyz_gradient_accum, denom, max_radii2D):
        """The densification statistics of the last step (densification.py:15-24), in place, one launch, no host sync:
        densify.add_densification_stats over this rank's screen-space gradients and pre-exchange radii of every camera of
        the step (the reference's batched_locally_preprocessed_mean2D / _radii), whichever of the batched or per-camera
        preprocess the step ran.  xyz_gradient_accum, denom: (P, 1), max_radii2D: (P,), float32, P = n_local."""
        from . import densify
        grads = self.means2D.grad if isinstance(self.means2D, torch.Tensor) else [m.grad for m in self.means2D]
        densify.add_densification_stats(xyz_gradient_accum, denom, max_radii2D, grads, self._radii_local)

    GROUP_OF = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
                "scaling": "_scaling", "rotation": "_rotation"}

    def optimizer_groups(self, lrs=None):
        """The reference's six single-tensor groups over this trainer's parameters (scene/gaussian_model.py:257-292)."""
        lrs = lrs or {"xyz": 0.00016, "f_dc": 0.0025, "f_rest": 0.0025 / 20, "opacity": 0.05, "scaling": 0.005,
                      "rotation": 0.001}            # arguments/__init__.py:110-119
        return [{"params": [getattr(self.params, attr)], "lr": lrs[name], "name": name} for name, attr in self.GROUP_OF.items()]

    def adopt_parameters(self, new):
        """After densification / redistribution replaced the optimizer's tensors: new = {group name: nn.Parameter}."""
        for name, attr in self.GROUP_OF.items():
            setattr(self.params, attr, new[name])
        self.n_local = int(new["xyz"].shape[0])

    def last_info(self):
        """Realised sizes of the last step on this rank: V visible, V' splats rendered, R instances."""
        V = int((self._radii_local > 0).sum())
        R = ops.LAST_R_TOTAL
        return dict(V=V, Vp=self._counts["Vp"], P_local=self._counts["P_local"], R=R)

    def io_bytes_per_step(self):
        """(host->device, device->host) bytes of the last resident=False step: GT strips in, loss out
        (+ the 8-byte instance count each render reads back)."""
        return int(self._h2d), 4 + 8 * self._n_renders
