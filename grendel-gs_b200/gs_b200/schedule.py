"""The reference's training schedule around Trainer.step: the optimizer set-up and what happens between two steps.

Per batch [iteration, iteration + bsz) the caller runs

    schedule.begin(iteration)      # update_learning_rate, oneupSHdegree       (train_internal.py:100-113)
    trainer.step(views)            # forward, loss, backward
    event = schedule.end(iteration)   # densification(), then the Adam step   (train_internal.py:271-329)

and owns everything else (views, saving, evaluation, logging).  end() is densification.py:5-85 with its device work
done by this library -- densify.add_densification_stats, densify.densify_and_prune, redistribute.redistribute,
densify.reset_opacity -- and the optimizer step of train_internal.py:316-329 by FusedAdam.  Every decision is the
reference's: the same intervals (check_update_at_this_iter), thresholds, counters and gates, in the same order.

The densify counter and the "densification disabled" flag are the reference's process globals (utils.DENSIFY_ITER,
args.disable_auto_densification): they are not in a checkpoint, so on resume they restart at 0 and at the configured
value, as they do in the reference.
"""
import operator
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import densify
from . import model_io
from . import redistribute as rd
from .optim import FusedAdam

LR_SCALE_MODES = ("linear", "sqrt", "accumu")
REDISTRIBUTE_MODES = ("random_redistribute", "no_redistribute")


@dataclass
class OptimizationParams:
    """arguments/__init__.py:107-133 (OptimizationParams) with the reference's names and defaults, plus the batch size,
    the redistribution options of DistributionParams (:149-155) and sh_step, the SH-degree interval the reference
    hard-codes (train_internal.py:112).  opacity_reset_until_iter = -1 stands for densify_until_iter + bsz
    (init_args, :277-278)."""
    iterations: int = 30_000
    position_lr_init: float = 0.00016
    position_lr_final: float = 0.0000016
    position_lr_delay_mult: float = 0.01
    position_lr_max_steps: int = 30_000
    feature_lr: float = 0.0025
    opacity_lr: float = 0.05
    scaling_lr: float = 0.005
    lr_scale_loss: float = 1.0
    lr_scale_pos_and_scale: float = 1.0
    rotation_lr: float = 0.001
    percent_dense: float = 0.01
    lambda_dssim: float = 0.2
    densification_interval: int = 100
    opacity_reset_interval: int = 3000
    densify_from_iter: int = 500
    densify_until_iter: int = 15_000
    densify_grad_threshold: float = 0.0002
    densify_memory_limit_percentage: float = 0.9
    disable_auto_densification: bool = False
    opacity_reset_until_iter: int = -1
    random_background: bool = False
    min_opacity: float = 0.005
    lr_scale_mode: str = "sqrt"
    bsz: int = 1
    redistribute_gaussians_mode: str = "random_redistribute"
    redistribute_gaussians_frequency: int = 10
    redistribute_gaussians_threshold: float = 1.1
    sh_step: int = 1000

    def __post_init__(self):
        if self.lr_scale_mode not in LR_SCALE_MODES:
            raise ValueError(f"lr_scale_mode {self.lr_scale_mode!r} not supported ({LR_SCALE_MODES})")
        if self.redistribute_gaussians_mode not in REDISTRIBUTE_MODES:
            raise ValueError(f"redistribute_gaussians_mode {self.redistribute_gaussians_mode!r} not supported "
                             f"({REDISTRIBUTE_MODES})")
        for name in ("bsz", "densification_interval", "opacity_reset_interval", "redistribute_gaussians_frequency",
                     "sh_step"):
            if operator.index(getattr(self, name)) < 1:
                raise ValueError(f"{name} must be a positive integer")

    def reset_until(self):
        """The last batch start + bsz at which the opacity may be reset."""
        u = self.opacity_reset_until_iter
        return self.densify_until_iter + self.bsz if u == -1 else u


def check_update_at_this_iter(iteration, bsz, update_interval, update_residual):
    """utils/general_utils.py:146-160: does the batch [iteration, iteration + bsz) reach an iteration that is
    update_residual modulo update_interval (within the batch's position in the current or the next interval)?"""
    lo = iteration % update_interval
    hi = lo + bsz
    return (lo <= update_residual < hi) or (lo <= update_residual + update_interval < hi)


def expon_lr(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """get_expon_lr_func (utils/general_utils.py:364-396): the log-linear decay from lr_init to lr_final over
    max_steps, in numpy float64 as the reference evaluates it."""
    def helper(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * np.sin(0.5 * np.pi * np.clip(step / lr_delay_steps, 0, 1))
        else:
            delay_rate = 1.0
        t = np.clip(step / max_steps, 0, 1)
        return delay_rate * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)
    return helper


def group_hyperparameters(opt, spatial_lr_scale):
    """training_setup (scene/gaussian_model.py:244-330) without the tensors: -> ({group name: {"lr", "eps", "betas"}}
    in the reference's group order, the xyz learning-rate schedule).  The values are the reference's Python / numpy
    floats, formed in its order: the groups start at torch.optim.Adam(l, lr=0.0, eps=1e-15)'s betas and eps, then
    lr_scale_mode "linear" multiplies the learning rates by bsz, "sqrt" multiplies them by sqrt(bsz), divides eps by it
    and raises the betas to the power bsz, and "accumu" leaves them."""
    pos = opt.lr_scale_pos_and_scale
    lrs = {"xyz": opt.position_lr_init * spatial_lr_scale * pos, "f_dc": opt.feature_lr,
           "f_rest": opt.feature_lr / 20.0, "opacity": opt.opacity_lr, "scaling": opt.scaling_lr * pos,
           "rotation": opt.rotation_lr}
    bsz = opt.bsz
    if opt.lr_scale_mode == "linear":
        lr_scale = bsz
    elif opt.lr_scale_mode == "sqrt":
        lr_scale = np.sqrt(bsz)
    else:
        lr_scale = 1
    groups = {}
    for name, lr in lrs.items():
        g = {"lr": lr, "eps": 1e-15, "betas": (0.9, 0.999)}
        if opt.lr_scale_mode == "linear":
            g["lr"] *= lr_scale
        elif opt.lr_scale_mode == "sqrt":
            g["lr"] *= lr_scale
            g["eps"] /= lr_scale
            g["betas"] = tuple(beta ** bsz for beta in g["betas"])
        groups[name] = g
    xyz = expon_lr(lr_init=opt.position_lr_init * spatial_lr_scale * lr_scale * pos,
                   lr_final=opt.position_lr_final * spatial_lr_scale * lr_scale * pos,
                   lr_delay_mult=opt.position_lr_delay_mult, max_steps=opt.position_lr_max_steps)
    return groups, xyz


@dataclass
class Event:
    """What end(iteration) did.  densify: densify_and_prune's counts (kept, clones, children per copy, split-selected,
    new total) or None; redistribution: this rank's Gaussian count (before, after) when the redistribution ran, else
    None; opacity_reset: the opacity was reset; densification_disabled: the memory gate has stopped densification (now or
    earlier)."""
    iteration: int
    densify: Optional[tuple] = None
    redistribution: Optional[tuple] = None
    opacity_reset: bool = False
    densification_disabled: bool = False


class Schedule:
    """The optimizer and the per-iteration decisions of a run over one Trainer (one rank; every rank builds its own and
    calls it at the same iterations).

    opt: OptimizationParams.  extent: the scene's cameras_extent (densify and prune thresholds).  spatial_lr_scale: the
    model's (create_from_pcd receives cameras_extent, scene/__init__.py), default extent.  checkpoint: a
    model_io.Checkpoint to resume from -- the trainer must hold its parameters (Trainer(model=checkpoint.params)); its
    SH degree, densification statistics and optimizer state are taken; without one the run starts fresh at SH degree 0
    with zero statistics (point_cloud.py asks the caller to set active_sh_degree = 0)."""

    def __init__(self, trainer, opt, extent, spatial_lr_scale=None, checkpoint=None):
        self.trainer, self.extent = trainer, float(extent)
        self.spatial_lr_scale = self.extent if spatial_lr_scale is None else float(spatial_lr_scale)
        self._start(opt, trainer.world)
        hyper, self.xyz_lr = group_hyperparameters(opt, self.spatial_lr_scale)
        grad_scale = 1.0 if opt.lr_scale_mode == "accumu" else 1.0 / opt.bsz
        dev, P = trainer.device, trainer.n_local
        if checkpoint is None:
            groups = trainer.optimizer_groups({k: g["lr"] for k, g in hyper.items()})
            for g in groups:   # Python floats of the reference's values: a checkpoint's groups load with weights_only
                h = hyper[g["name"]]
                g["lr"], g["eps"], g["betas"] = float(h["lr"]), float(h["eps"]), tuple(float(b) for b in h["betas"])
            self.optimizer = FusedAdam(groups, lr=0.0, eps=1e-15, grad_scale=grad_scale)
            trainer.params.active_sh_degree = 0
            fresh = densify.fresh_stats(P, dev)
            self.stats = {k: fresh[k] for k in model_io.STAT_NAMES}
        else:
            self.optimizer = model_io.load_fused_adam(trainer, checkpoint, grad_scale=grad_scale)
            trainer.params.active_sh_degree = int(checkpoint.active_sh_degree)
            self.stats = {k: checkpoint.stats[k].to(dev).contiguous() for k in model_io.STAT_NAMES}
            for k, t in self.stats.items():
                if t.shape[0] != P:
                    raise ValueError(f"checkpoint statistic {k!r} has {t.shape[0]} rows, the trainer {P} Gaussians")

    def _start(self, opt, world):
        """The host state of the decisions: the reference's densify counter and disabled flag."""
        self.opt, self.world = opt, int(world)
        self.densify_iter = 0
        self.densification_disabled = bool(opt.disable_auto_densification)

    def checkpoint_stats(self):
        """The densification statistics as model_io.save_checkpoint takes them."""
        return dict(self.stats)

    def begin(self, iteration):
        """Before the step of [iteration, iteration + bsz): the xyz learning rate of the schedule, then one more SH
        degree at every sh_step.  -> the xyz learning rate."""
        lr = float(self.xyz_lr(iteration))
        for g in self.optimizer.param_groups:
            if g["name"] == "xyz":
                g["lr"] = lr
        if check_update_at_this_iter(iteration, self.opt.bsz, self.opt.sh_step, 0):
            p = self.trainer.params
            if p.active_sh_degree < p.max_sh_degree:
                p.active_sh_degree += 1
        return lr

    def end(self, iteration, noise=None):
        """After the step of [iteration, iteration + bsz): densification.py:5-85, then the optimizer step while
        iteration < iterations.  noise: standard-normal draws for the split (densify.densify_and_prune), default
        drawn on the device.  -> Event."""
        o, bsz = self.opt, self.opt.bsz
        ev = Event(iteration)
        if not self.densification_disabled and iteration <= o.densify_until_iter:
            self._add_stats()
            if iteration > o.densify_from_iter and check_update_at_this_iter(iteration, bsz, o.densification_interval, 0):
                ev.densify = self._densify(20 if iteration > o.opacity_reset_interval else None, noise)
                if self.densify_iter % o.redistribute_gaussians_frequency == 0:
                    ev.redistribution = self._redistribute()
                self._memory_gate()
                self.densify_iter += 1
            if check_update_at_this_iter(iteration, bsz, o.opacity_reset_interval, 0) and iteration + bsz <= o.reset_until():
                self._reset_opacity()
                ev.opacity_reset = True
        if iteration < o.iterations:
            self._optimizer_step()
        ev.densification_disabled = self.densification_disabled
        return ev

    # -- the decisions' inputs and the device work (a test substitutes recorders for these) -------------------------
    def _add_stats(self):
        s = self.stats
        self.trainer.add_densification_stats(s["xyz_gradient_accum"], s["denom"], s["max_radii2D"])

    def _adopt(self, res):
        self.trainer.adopt_parameters(res)
        self.stats = {k: res[k] for k in model_io.STAT_NAMES}

    def _densify(self, size_threshold, noise):
        o, s = self.opt, self.stats
        res = densify.densify_and_prune(self.optimizer, s["xyz_gradient_accum"], s["denom"], o.densify_grad_threshold,
                                        o.min_opacity, self.extent, o.percent_dense, size_threshold, noise=noise)
        self._adopt(res)
        return res["counts"]

    def _redistribute(self):
        """redistribute_gaussians (scene/gaussian_model.py:1261-1329) with its gate: -> (before, after) or None."""
        if self.opt.redistribute_gaussians_mode == "no_redistribute" or not self._redistribution_gate():
            return None
        return self._move()

    def _move(self):
        before = self.trainer.n_local
        self._adopt(rd.redistribute(self.optimizer, group=self.trainer.group))
        return before, self.trainer.n_local

    def _redistribution_gate(self):
        """need_redistribute_gaussians (:1246-1259): never at world size 1; always when the densify counter equals the
        frequency (the first redistribution, no collective); otherwise when min * threshold < max over the ranks'
        counts."""
        if self.world == 1:
            return False
        if self.densify_iter == self.opt.redistribute_gaussians_frequency:
            return True
        counts = self._gather_counts()
        return min(counts) * self.opt.redistribute_gaussians_threshold < max(counts)

    def _gather_counts(self):
        return rd.need_redistribute(self.trainer.n_local, self.trainer.group)[1]

    def _memory_gate(self):
        """check_memory_usage(before_densification_stop=True) (utils/general_utils.py:303-345): the ranks' peak
        reserved memory in GiB, gathered as fp32, against densify_memory_limit_percentage of the device's total; over it,
        densification stops for the rest of the run on every rank."""
        peaks = self._gather_max_reserved_gb()
        if max(peaks) > self.opt.densify_memory_limit_percentage * self._total_memory_gb():
            self.densification_disabled = True

    def _gather_max_reserved_gb(self):
        dev = torch.device(self.trainer.device)
        mine = torch.cuda.max_memory_reserved(dev) / 1024 / 1024 / 1024
        if self.world == 1:
            return [float(np.float32(mine))]
        import torch.distributed as dist
        on = dev if dist.get_backend(self.trainer.group) == "nccl" else "cpu"
        allv = torch.empty((self.world,), dtype=torch.float32, device=on)
        dist.all_gather_into_tensor(allv, torch.tensor([mine], dtype=torch.float32, device=on), group=self.trainer.group)
        return allv.cpu().tolist()

    def _total_memory_gb(self):
        return torch.cuda.get_device_properties(torch.device(self.trainer.device)).total_memory / 1024 / 1024 / 1024

    def _reset_opacity(self):
        densify.reset_opacity(self.optimizer)

    def _optimizer_step(self):
        self.optimizer.step()
        self.optimizer.zero_grad(set_to_none=True)
