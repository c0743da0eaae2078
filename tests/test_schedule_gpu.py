"""-m gpu: the training schedule on one H100 (gs_b200.schedule, densify.reset_opacity / gs_reset_opacity).

  * the opacity reset is the reference's torch expression, bit for bit, at the edges (logits around logit(0.01), the
    logit whose sigmoid is exactly 0.01f, large of either sign, non-finite, P = 0, 1, not a multiple of 4, unaligned,
    ~2^24); both moments are zero afterwards, "step" is kept, and the next optimizer step skips the opacity;
  * the reference's gradient division `param.grad /= bsz` is, on CUDA, FusedAdam's grad_scale = 1 / bsz, bit for bit;
  * Schedule-driven runs at bsz 1 and 4 over a few hundred iterations with shortened intervals (densify with and without
    the size threshold, SH steps, two opacity resets) equal a hand-written restatement of the reference's sequence on
    the library's primitives: every parameter, moment, step, statistic, loss and per-iteration count;
  * a run saved mid-way and resumed through Schedule(checkpoint=...) gives the uninterrupted run's bits;
  * the memory gate, forced by a tiny densify_memory_limit_percentage, stops densification."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import gpu_util as gu
from gs_b200 import densify, model_io, pipeline
from gs_b200 import schedule as sc
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu

TW, TH, N_VIEWS, N_GAUSS = 256, 192, 8, 12000
ITERS = 300


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def torch_reset(o):
    """gaussian_model.py:555-561: inverse_sigmoid(torch.min(get_opacity, torch.ones_like(get_opacity) * 0.01))."""
    s = torch.sigmoid(o)
    m = torch.min(s, torch.ones_like(s) * 0.01)
    return torch.log(m / (1 - m))


def edge_logits(P, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((P,), generator=g) * 6.0
    special = []
    c = np.float32(np.log(0.01 / 0.99))
    for d in range(-40, 41):   # the fp32 neighbours of logit(0.01) on both sides
        special.append(float(np.float32(c) + np.float32(d) * np.spacing(c)))
    special += [0.0, -0.0, 1e-30, -1e-30, 30.0, -30.0, 88.0, -88.0, 104.0, -104.0, 1e30, -1e30, 3.4e38, -3.4e38,
                float("inf"), float("-inf"), float("nan")]
    k = min(P, len(special))
    x[:k] = torch.tensor(special[:k])
    return x.reshape(P, 1)


def exact_one_hundredth():
    """A logit whose fp32 sigmoid on the device is exactly 0.01f (found by walking the neighbours of logit(0.01))."""
    c = np.float32(np.log(0.01 / 0.99))
    cand = torch.tensor([float(c + np.float32(d) * np.spacing(c)) for d in range(-200, 201)], device=gu.DEV)
    hit = cand[torch.sigmoid(cand) == torch.tensor(0.01, dtype=torch.float32, device=gu.DEV)]
    return hit


def opt_with_state(p, step=7.0, seed=0):
    opt = FusedAdam([{"params": [p], "lr": 0.05, "name": "opacity"}], lr=0.0, eps=1e-15)
    g = torch.Generator(device=gu.DEV).manual_seed(seed)
    opt.state[p] = {"step": torch.tensor(step), "exp_avg": torch.randn(p.shape, device=gu.DEV, generator=g),
                    "exp_avg_sq": torch.rand(p.shape, device=gu.DEV, generator=g)}
    return opt


@pytest.mark.parametrize("P,offset", [(0, 0), (1, 0), (5, 0), (1023, 0), (4099, 1), (4096, 3), ((1 << 24) + 3, 0)])
def test_reset_opacity_bits(P, offset):
    x = edge_logits(P, seed=P).to(gu.DEV)
    buf = torch.empty((P + offset,), device=gu.DEV)   # offset > 0: not 16-byte aligned, the scalar path
    buf[offset:] = x.reshape(-1)
    p = nn.Parameter(buf[offset:].view(P, 1))
    p.grad = torch.ones_like(p)
    opt = opt_with_state(p)
    want = torch_reset(x)
    assert densify.reset_opacity(opt) is p
    torch.cuda.synchronize()
    assert same(p, want)
    st = opt.state[p]
    assert float(st["step"]) == 7.0
    assert torch.equal(bits(st["exp_avg"]), torch.zeros_like(bits(st["exp_avg"])))
    assert torch.equal(bits(st["exp_avg_sq"]), torch.zeros_like(bits(st["exp_avg_sq"])))
    assert p.grad is None
    opt.step()                     # no gradient: the opacity and its step stay as the reset left them
    assert same(p, want) and float(st["step"]) == 7.0


def test_reset_opacity_at_exactly_one_hundredth_and_without_state():
    """Logits whose sigmoid is 0.01f (where fp32 has one), their neighbours, and logits whose sigmoid is above 0.01,
    where min() yields 0.01f itself: all take the round trip.  No optimizer state yet: only the opacity changes."""
    hit = exact_one_hundredth()
    c = np.float32(np.log(0.01 / 0.99))
    near = torch.tensor([float(c + np.float32(d) * np.spacing(c)) for d in range(-8, 9)], device=gu.DEV)
    x = torch.cat([hit, near, torch.tensor([-4.0, 0.0, 2.5], device=gu.DEV)]).reshape(-1, 1)
    p = nn.Parameter(x.clone())
    opt = FusedAdam([{"params": [p], "lr": 0.05, "name": "opacity"}], lr=0.0, eps=1e-15)   # no state yet
    densify.reset_opacity(opt)
    want = torch_reset(x)
    print(f"[reset] {hit.numel()} fp32 logit(s) with sigmoid == 0.01f")
    assert same(p, want)
    assert len(opt.state) == 0


@pytest.mark.parametrize("bsz", [1, 2, 3, 5, 6, 7, 9, 12, 17, 31, 32, 48, 64])
def test_grad_division_is_the_reciprocal_product(bsz):
    """torch on CUDA divides a tensor by a Python scalar as a product with the fp32 reciprocal; FusedAdam's
    grad_scale = 1 / bsz reaches the kernel as that same fp32 value."""
    g = torch.Generator(device=gu.DEV).manual_seed(bsz)
    x = torch.randn((1 << 20,), device=gu.DEV, generator=g) * torch.exp(torch.randn((1 << 20,), device=gu.DEV,
                                                                                     generator=g) * 10)
    d = x.clone()
    d /= bsz
    assert same(d, x * np.float32(1.0 / bsz))
    # one Adam step: the reference's `/=` then torch.optim.Adam, against FusedAdam with grad_scale
    p0 = torch.randn((4099, 3), device=gu.DEV, generator=g)
    grad = torch.randn((4099, 3), device=gu.DEV, generator=g)
    a, b = nn.Parameter(p0.clone()), nn.Parameter(p0.clone())
    lr, eps, betas = 0.0025 * np.sqrt(bsz), 1e-15 / np.sqrt(bsz), [0.9 ** bsz, 0.999 ** bsz]
    ref = torch.optim.Adam([{"params": [a], "lr": lr, "eps": eps, "betas": betas}], lr=0.0, eps=1e-15)
    fused = FusedAdam([{"params": [b], "lr": lr, "eps": eps, "betas": betas}], lr=0.0, eps=1e-15, grad_scale=1.0 / bsz)
    for _ in range(3):
        a.grad = grad.clone()
        a.grad /= bsz
        b.grad = grad.clone()
        ref.step()
        fused.step()
    assert same(a, b)
    assert same(ref.state[a]["exp_avg"], fused.state[b]["exp_avg"])
    assert same(ref.state[a]["exp_avg_sq"], fused.state[b]["exp_avg_sq"])


# ---------------------------------------------------------------------------------------------------------------------
# whole runs
# ---------------------------------------------------------------------------------------------------------------------
def camera_set():
    cams = [syn.make_camera(TW, TH, yaw_deg=1.5 * q - 5.0, uid=q) for q in range(N_VIEWS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=30 + q)).pin_memory() for q in range(N_VIEWS)]
    return cams, gts


def views_of(it, bsz):
    return [(it - 1 + b) % N_VIEWS for b in range(bsz)]


def short_schedule(bsz, grad_threshold):
    return sc.OptimizationParams(bsz=bsz, iterations=ITERS, densify_from_iter=20, densification_interval=25,
                                 opacity_reset_interval=100, densify_until_iter=240, sh_step=50,
                                 densify_grad_threshold=grad_threshold)


class Setup:
    def __init__(self, bsz):
        self.cams, self.gts = camera_set()
        self.scene = syn.make_scene(N_GAUSS, TW, TH, seed=12, max_sh_degree=3)
        self.noise = torch.randn((8 * N_GAUSS, 3), generator=torch.Generator().manual_seed(3)).to(gu.DEV)
        tr = self.trainer()
        self.extent = float(torch.exp(tr.params._scaling.detach()).max(dim=1).values.median()) / 0.01
        # a gradient threshold that selects some Gaussians: the 0.85 quantile of a few steps' mean gradients
        a, d, m = (torch.zeros((tr.n_local, 1), device=gu.DEV), torch.zeros((tr.n_local, 1), device=gu.DEV),
                   torch.zeros((tr.n_local,), device=gu.DEV))
        for it in range(1, 9):
            tr.step(views=views_of(it, bsz))
            tr.add_densification_stats(a, d, m)
        self.threshold = float(torch.quantile((a / d).nan_to_num(0.0), 0.85))
        self.opt = short_schedule(bsz, self.threshold)

    def trainer(self, model=None):
        if model is not None:
            return pipeline.Trainer(None, self.cams, self.gts, gu.DEV, model=model, deterministic=True)
        return pipeline.Trainer(self.scene, self.cams, self.gts, gu.DEV, deterministic=True)


def run_schedule(setup, tr, sched, iterations):
    log = []
    for it in iterations:
        sched.begin(it)
        loss = tr.step(views=views_of(it, setup.opt.bsz), resident=False)
        ev = sched.end(it, noise=setup.noise)
        log.append((it, loss, ev.densify, ev.opacity_reset, tr.n_local, tr.params.active_sh_degree))
    return log


def run_by_hand(setup, tr):
    """train_internal.py:95-329 and densification.py:5-85 at world size 1, restated on the library's primitives, with
    the opacity reset and the gradient division in the reference's torch."""
    o, bsz = setup.opt, setup.opt.bsz
    scale = np.sqrt(bsz)                                                            # lr_scale_mode "sqrt"
    lrs = {"xyz": o.position_lr_init * setup.extent * 1.0, "f_dc": o.feature_lr, "f_rest": o.feature_lr / 20.0,
           "opacity": o.opacity_lr, "scaling": o.scaling_lr * 1.0, "rotation": o.rotation_lr}
    groups = tr.optimizer_groups({k: v * scale for k, v in lrs.items()})
    for g in groups:
        g["eps"], g["betas"] = 1e-15 / scale, [0.9 ** bsz, 0.999 ** bsz]
    opt = FusedAdam(groups, lr=0.0, eps=1e-15)
    lr_init, lr_final = o.position_lr_init * setup.extent * scale * 1.0, o.position_lr_final * setup.extent * scale * 1.0
    tr.params.active_sh_degree = 0
    P = tr.n_local
    stats = {"max_radii2D": torch.zeros((P,), device=gu.DEV), "xyz_gradient_accum": torch.zeros((P, 1), device=gu.DEV),
             "denom": torch.zeros((P, 1), device=gu.DEV)}
    log = []

    def hit(it, interval):
        return sc.check_update_at_this_iter(it, bsz, interval, 0)

    for it in range(1, o.iterations + 1, bsz):
        t = np.clip(it / o.position_lr_max_steps, 0, 1)
        opt.param_groups[0]["lr"] = 1.0 * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)
        if hit(it, o.sh_step) and tr.params.active_sh_degree < tr.params.max_sh_degree:
            tr.params.active_sh_degree += 1
        loss = tr.step(views=views_of(it, bsz), resident=False)
        counts, reset = None, False
        if it <= o.densify_until_iter:
            tr.add_densification_stats(stats["xyz_gradient_accum"], stats["denom"], stats["max_radii2D"])
            if it > o.densify_from_iter and hit(it, o.densification_interval):
                res = densify.densify_and_prune(opt, stats["xyz_gradient_accum"], stats["denom"], o.densify_grad_threshold,
                                                o.min_opacity, setup.extent, o.percent_dense,
                                                20 if it > o.opacity_reset_interval else None, noise=setup.noise)
                tr.adopt_parameters(res)
                stats = {k: res[k] for k in model_io.STAT_NAMES}
                counts = res["counts"]
            if hit(it, o.opacity_reset_interval) and it + bsz <= o.densify_until_iter + bsz:
                g = opt.param_groups[3]
                old = g["params"][0]
                with torch.no_grad():
                    new = nn.Parameter(torch_reset(old.detach()).requires_grad_(True))
                st = opt.state.pop(old)
                st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(new), torch.zeros_like(new)
                g["params"][0] = new
                opt.state[new] = st
                tr.adopt_parameters({x["name"]: x["params"][0] for x in opt.param_groups})
                reset = True
        if it < o.iterations:
            for p in tr.params.raw_parameters():
                if p.grad is not None:
                    p.grad /= bsz
            opt.step()
            opt.zero_grad(set_to_none=True)
        log.append((it, loss, counts, reset, tr.n_local, tr.params.active_sh_degree))
    return tr, opt, stats, log


def state_of(tr, opt, stats):
    out = {}
    for g in opt.param_groups:
        p = g["params"][0]
        assert p is getattr(tr.params, pipeline.Trainer.GROUP_OF[g["name"]])
        st = opt.state[p]
        out[g["name"]] = (p.detach(), st["exp_avg"], st["exp_avg_sq"], float(st["step"]), float(g["lr"]))
    out.update(stats)
    return out


def assert_same_state(a, b):
    assert set(a) == set(b)
    for k in a:
        if k in model_io.STAT_NAMES:
            assert same(a[k], b[k]), k
        else:
            for q in range(5):
                if q < 3:
                    assert same(a[k][q], b[k][q]), (k, q)
                else:
                    assert a[k][q] == b[k][q], (k, q, a[k][q], b[k][q])


SETUPS = {}


def setup_for(bsz):
    if bsz not in SETUPS:
        SETUPS[bsz] = Setup(bsz)
    return SETUPS[bsz]


@pytest.mark.parametrize("bsz", [1, 4])
def test_schedule_equals_the_reference_sequence(bsz):
    s = setup_for(bsz)
    tr = s.trainer()
    sched = sc.Schedule(tr, s.opt, s.extent)
    log_a = run_schedule(s, tr, sched, range(1, ITERS + 1, bsz))
    a = state_of(tr, sched.optimizer, sched.checkpoint_stats())
    del tr, sched
    trh, opt_h, stats_h, log_b = run_by_hand(s, s.trainer())
    b = state_of(trh, opt_h, stats_h)
    densified = [e for e in log_a if e[2] is not None]
    print(f"[schedule] bsz {bsz}: threshold {s.threshold:.3e}, Gaussians {N_GAUSS} -> {log_a[-1][4]}, densify counts "
          f"{[e[2] for e in densified]}, resets at {[e[0] for e in log_a if e[3]]}")
    assert log_a == log_b
    # the run reached every decision it is meant to exercise
    assert any(e[2][1] + e[2][3] > 0 for e in densified)
    assert any(e[0] > s.opt.opacity_reset_interval for e in densified)       # the size threshold applies
    assert sum(e[3] for e in log_a) == 2
    assert log_a[-1][5] == 3 and log_a[0][5] == 0
    assert_same_state(a, b)


@pytest.mark.parametrize("bsz", [1, 4])
def test_resume_gives_the_uninterrupted_bits(tmp_path, bsz):
    s = setup_for(bsz)
    iters = list(range(1, ITERS + 1, bsz))
    half = iters[len(iters) // 2]                       # resumes between two densifications, after the first reset
    tr = s.trainer()
    sched = sc.Schedule(tr, s.opt, s.extent)
    log_a = run_schedule(s, tr, sched, iters)
    a = state_of(tr, sched.optimizer, sched.checkpoint_stats())
    del tr, sched

    tr = s.trainer()
    sched = sc.Schedule(tr, s.opt, s.extent)
    log_b = run_schedule(s, tr, sched, [i for i in iters if i < half])
    model_io.save_checkpoint(str(tmp_path), tr, sched.optimizer, sched.checkpoint_stats(), next_iteration=half)
    del tr, sched
    ck = model_io.load_checkpoint(str(tmp_path), 0, 1, gu.DEV)
    tr = s.trainer(model=ck.params)
    sched = sc.Schedule(tr, s.opt, s.extent, checkpoint=ck)
    assert tr.params.active_sh_degree == ck.active_sh_degree > 0
    log_b += run_schedule(s, tr, sched, range(ck.next_iteration, ITERS + 1, bsz))
    b = state_of(tr, sched.optimizer, sched.checkpoint_stats())
    assert log_a == log_b
    assert_same_state(a, b)


def test_memory_gate_stops_densification():
    s = setup_for(4)
    opt = short_schedule(4, s.threshold)
    opt.densify_memory_limit_percentage = 1e-9
    tr = s.trainer()
    sched = sc.Schedule(tr, opt, s.extent)
    events = []
    for it in range(1, 121, 4):
        sched.begin(it)
        tr.step(views=views_of(it, 4))
        stopped = sched.densification_disabled
        before = {k: v.clone() for k, v in sched.stats.items()}
        events.append(sched.end(it, noise=s.noise))
        if stopped:                 # no statistics are gathered once densification has stopped
            for k in before:
                assert same(before[k], sched.stats[k]), k
    first = next(i for i, e in enumerate(events) if e.densify is not None)
    assert events[first].densification_disabled
    assert all(e.densification_disabled for e in events[first:])
    assert not any(e.densify is not None or e.opacity_reset for e in events[first + 1:])
    assert not any(e.densification_disabled for e in events[:first])
