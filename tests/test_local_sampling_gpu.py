"""-m gpu: local sampling (pipeline.Trainer(local_sampling=True)) on one GPU.

At one rank a local-sampling Trainer must be the default Trainer, bit for bit under deterministic=True: loss, the six
parameter gradients, the screen-space gradients, the densification statistics, and a FusedAdam run with a densify/prune
over changing views; its camera table, gathered on the device, must be the host-gathered one.  With W = 2 and 4 ranks
simulated in one process (the direct-placement kernels of tests/test_exchange_sim_gpu.py, every receive region a plain
allocation), each owner's receive region must hold exactly the splats of its own views, sources in rank order, and its
batched render and loss of them must equal a one-rank render of the same views over the whole scene.  Comparisons are
of int32 bit patterns."""
import numpy as np
import pytest
import torch

import exchange_ref as xr
from gs_b200 import densify, division, exchange, ops, pipeline
from gs_b200 import synthetic as syn
from gs_b200.exchange import _i32, _slab_ptrs
from gs_b200.optim import FusedAdam
from oracle.oracle import Oracle
from test_exchange_sim_gpu import region_fields, run_pack, xr_count

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TW, TH, N_CAMS, N_GAUSS = 256, 200, 12, 20_000


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


@pytest.fixture(scope="module")
def camera_set():
    scene = syn.make_scene(N_GAUSS, TW, TH, seed=0)
    cams = [syn.make_camera(TW, TH, yaw_deg=4.0 * q - 20.0, uid=100 + q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=10 + q)).pin_memory() for q in range(N_CAMS)]
    return scene, cams, gts


def pair(scene, cams, gts, k):
    """(default Trainer, local-sampling Trainer) on one rank, deterministic."""
    return (pipeline.Trainer(scene, cams, gts, DEV, deterministic=True),
            pipeline.Trainer(scene, cams, gts, DEV, deterministic=True, local_sampling=True, local_bsz=k))


def grads_of(tr):
    return [t.grad.detach().clone() for t in tr.params.raw_parameters()]


def screen_grads(tr):
    return tr.means2D.grad if isinstance(tr.means2D, torch.Tensor) else torch.stack([m.grad for m in tr.means2D])


def assert_same_step(a, b, what):
    for q, (x, y) in enumerate(zip(grads_of(a), grads_of(b))):
        assert same_bits(x, y), f"{what}: gradient of parameter {q} differs"
    assert same_bits(screen_grads(a), screen_grads(b)), f"{what}: screen-space gradients differ"


def assert_no_load_balancer(tr):
    assert tr.history.history == [] and tr.balance_log == [] and tr._pending_feedback == []
    assert tr._strategy_cache is None and tr._sent_feedback is None
    assert all(torch.equal(h, torch.ones(tr.tile_y)) for h in tr.history.accum_heuristic.values())


# (a) one rank: the local-sampling step is the default step
@pytest.mark.parametrize("views", [[7, 2, 9, 0], [5], [3, 3]])
@pytest.mark.parametrize("resident", [True, False])
def test_one_rank_local_step_is_the_default_step(camera_set, views, resident):
    scene, cams, gts = camera_set
    default, local = pair(scene, cams, gts, len(views))
    la = default.step(views=views, resident=resident)
    lb = local.step(views=views, resident=resident)
    if not resident:
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (la, lb)
    assert_same_step(default, local, f"views {views}, resident={resident}")
    stats = []
    for tr in (default, local):
        s = (torch.zeros((tr.n_local, 1), device=DEV), torch.zeros((tr.n_local, 1), device=DEV),
             torch.zeros((tr.n_local,), device=DEV))
        tr.add_densification_stats(*s)
        stats.append(s)
    assert all(same_bits(x, y) for x, y in zip(*stats)), "densification statistics"
    assert local.last_info() == default.last_info()
    if len(views) > 1:   # (b) the camera table gathered on the device is the host-gathered one
        assert same_bits(local._batch_table, default._cams_dev[1])
        assert same_bits(local._batch_table, local._cam_rows[list(views)].to(DEV))
        assert local._batch_index.tolist() == list(views)
    assert_no_load_balancer(local)


SCHEDULES = {4: ([7, 2, 9, 0], [3, 11, 4, 4], [11, 3, 4, 1], [7, 2, 9, 0], [0, 0, 5, 6], [10, 1, 6, 8]),
             1: ([7], [3], [11], [7], [0], [10])}
DENSIFY_AFTER = 2


def _densify(opt, accum, denom, params, noise):
    extent = float(torch.exp(params._scaling.detach()).max(dim=1).values.median()) / 0.01
    grads = (accum / denom.clamp(min=1))[:, 0]
    return densify.densify_and_prune(opt, accum, denom, float(torch.quantile(grads, 0.8)), 0.005, extent, 0.01, None,
                                     noise=noise)


@pytest.mark.parametrize("k", [4, 1])
def test_one_rank_local_training_run_is_the_default_run(camera_set, k):
    """Six steps over changing views with FusedAdam and a densify/prune after the third: the same losses, gradients,
    statistics, densification counts and parameters, bit for bit."""
    scene, cams, gts = camera_set
    noise = torch.randn((2 * N_GAUSS, 3), generator=torch.Generator().manual_seed(3)).to(DEV)
    lr = dict(xyz=1e-3, f_dc=1e-2, f_rest=1e-3, opacity=5e-2, scaling=5e-3, rotation=1e-3)
    trs = pair(scene, cams, gts, k)
    opts = [FusedAdam(tr.optimizer_groups(lr), lr=0.0, eps=1e-15) for tr in trs]
    stats = [None, None]
    for it, views in enumerate(SCHEDULES[k]):
        la, lb = (tr.step(views=views, resident=False) for tr in trs)
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (it, la, lb)
        assert_same_step(*trs, f"step {it} {views}")
        for w, tr in enumerate(trs):
            if stats[w] is None:
                P = tr.n_local
                stats[w] = (torch.zeros((P, 1), device=DEV), torch.zeros((P, 1), device=DEV), torch.zeros((P,), device=DEV))
            tr.add_densification_stats(*stats[w])
        assert all(same_bits(x, y) for x, y in zip(*stats)), f"step {it}: densification statistics"
        for opt in opts:
            opt.step(grad_scale=1.0 / len(views))
        if it == DENSIFY_AFTER:
            res = [_densify(opt, s[0], s[1], tr.params, noise) for opt, s, tr in zip(opts, stats, trs)]
            assert res[0]["counts"] == res[1]["counts"] and res[0]["counts"][1] + res[0]["counts"][3] > 0, res[0]["counts"]
            for tr, r in zip(trs, res):
                tr.adopt_parameters(r)
            stats = [None, None]
        for name, attr in pipeline.Trainer.GROUP_OF.items():
            assert same_bits(getattr(trs[0].params, attr), getattr(trs[1].params, attr)), f"step {it}: parameter {name}"
    assert_no_load_balancer(trs[1])


def test_one_rank_refusals_leave_the_last_step(camera_set):
    scene, cams, gts = camera_set
    held = [g if q % 2 == 0 else None for q, g in enumerate(gts)]
    tr = pipeline.Trainer(scene, cams, held, DEV, deterministic=True, local_sampling=True, local_bsz=2)
    assert sum(g is not None for g in tr.gts_dev) == N_CAMS // 2      # only the held images are on the device
    tr.step(views=[4, 0])
    before = [bits(t).clone() for t in grads_of(tr)]
    for views in (None, [4], [4, 0, 2], [4, 1], [13, 0]):
        with pytest.raises(ValueError):
            tr.step(views=views)
    assert all(torch.equal(bits(t), b) for t, b in zip(grads_of(tr), before))
    assert tr.iteration == 1


# (c) W ranks simulated on one GPU: direct placement over whole views, then the owner's render and loss
class SimCase:
    """The shape test_exchange_sim_gpu's helpers read: B, P, W, H, Wimg, lo_c, hi_c, ptrs(i, field)."""

    def __init__(self, W, B, P, H, Wimg, strategies, dev):
        self.W, self.B, self.P, self.H, self.Wimg = W, B, P, H, Wimg
        self.lo, self.hi = xr.strips_from_strategies(strategies, W)
        self.lo_c, self.hi_c = _i32(self.lo.reshape(-1)), _i32(self.hi.reshape(-1))
        self.dev = dev

    def ptrs(self, i, f):
        return _slab_ptrs(self.dev[i][f], self.B)


def _render_and_loss(m2, co, rgb, depths, radii, view_start, rs, gts):
    images, _ = ops.render_gaussians_batched(m2, co, rgb, depths, radii, None, view_start, rs, deterministic=True)
    k = len(gts)
    l1_ssim = ops.fused_l1_ssim_batched(images, gts, [(0, TH, 0, TH)] * k, deterministic=True, gt_full=True)
    return images, l1_ssim


@pytest.mark.parametrize("W,k", [(2, 2), (4, 1), (4, 2)])
def test_simulated_ranks_render_their_own_views_whole(camera_set, W, k):
    scene, cams, gts = camera_set
    B, n = W * k, N_GAUSS - N_GAUSS % W
    # every rank samples k views among the cameras it holds (uid % W == rank)
    rng = np.random.default_rng(W * 10 + k)
    mine = [[int(v) for v in rng.choice([q for q in range(N_CAMS) if cams[q]["uid"] % W == r], size=k, replace=False)]
            for r in range(W)]
    union = [v for m in mine for v in m]
    dcams = [pipeline.DeviceCamera(c, DEV) for c in cams]
    rs = dcams[0].settings()
    table = ops.pack_cameras([dcams[v].settings() for v in union])
    shards = [pipeline.GaussianParams({f: a[n * i // W:n * (i + 1) // W] for f, a in scene.items()}, DEV) for i in range(W)]
    whole = pipeline.GaussianParams({f: a[:n] for f, a in scene.items()}, DEV)

    def project(p, cam_table):
        with torch.no_grad():
            out = ops.preprocess_gaussians_batched(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                                   p._opacity, cam_table, TW, TH, 3)
        return dict(zip(xr.FIELDS, (t.contiguous() for t in out)))

    proj = [project(s, table) for s in shards]
    strategies = division.start_strategy_whole_views(union, (TH + 15) // 16, W, 0)[0]
    c = SimCase(W, B, tuple(s._xyz.shape[0] for s in shards), TH, TW, strategies, proj)
    # route: the per-rank counts, all-gathered as exchange_cat lays them out
    blk = [xr_count(c, i) for i in range(W)]
    cnt = np.stack([gu_counts.cpu().numpy().T for _, _, _, gu_counts in blk]).astype(np.int64)   # cnt[i][k][j]
    shards_np = [{f: t.cpu().numpy() for f, t in d.items()} for d in proj]
    hits = [xr.route(Oracle(np.float32), TH, TW, s, c.lo, c.hi) for s in shards_np]
    assert np.array_equal(cnt, xr.counts(hits))
    for i in range(W):   # nothing of another rank's views reaches an owner, and every visible splat reaches its owner
        for p in range(B):
            assert cnt[i, p, :].sum() == cnt[i, p, p // k] == int((shards_np[i]["radii"][p] > 0).sum())
    N = [int(cnt[:, :, j].sum()) for j in range(W)]
    cap = (max(N) // 4 + 2) * 4
    allc = torch.cat([counts.t().contiguous().reshape(-1) for _, _, _, counts in blk])
    regions, _rows = run_pack(c, [b for _, _, b, _ in blk], cap, allc)
    assert regions.guards_intact()
    # the one-rank reference: the whole scene projected into each owner's views
    for j in range(W):
        own = list(range(j * k, (j + 1) * k))
        got = region_fields(regions.words(j), cap)
        ref = project(whole, table[own[0]:own[-1] + 1])
        vis = [ref["radii"][q] > 0 for q in range(k)]
        # (1) the receive region holds the visible splats of the owner's views, view by view, sources in rank order --
        # shards are contiguous, so that is the whole scene's index order
        for f in xr.FIELDS:
            want = torch.cat([ref[f][q][vis[q]] for q in range(k)]).cpu().numpy()
            assert np.array_equal(got[f][:N[j]].reshape(want.shape), np.ascontiguousarray(want).view(np.int32)), \
                f"owner {j}: {f}"
            assert (got[f][N[j]:] == -1).all(), f"owner {j}: {f} written beyond its rows"
        _, view_start = exchange.direct_rows(cnt, j)
        vs = view_start[j * k:(j + 1) * k + 1]
        assert vs[0] == 0 and vs[-1] == N[j] and vs == [0] + list(np.cumsum([int(v.sum()) for v in vis]))
        # (2) the owner's batched render and loss of its region == the one-rank render of the same views
        region = {f: torch.from_numpy(np.ascontiguousarray(got[f][:N[j]])).to(DEV) for f in xr.FIELDS}
        r_m2, r_rgb, r_co = (region[f].view(torch.float32).clone().requires_grad_(True)
                             for f in ("means2D", "rgb", "conic_opacity"))
        r_rad, r_dep = region["radii"], region["depths"].view(torch.float32)
        img_a, loss_a = _render_and_loss(r_m2, r_co, r_rgb, r_dep, r_rad, vs, rs, [gts[union[p]].to(DEV) for p in own])
        P = ref["means2D"].shape[1]
        w_m2, w_rgb, w_co = (ref[f].reshape(k * P, -1).clone().requires_grad_(True)
                             for f in ("means2D", "rgb", "conic_opacity"))
        img_b, loss_b = _render_and_loss(w_m2, w_co, w_rgb, ref["depths"].reshape(-1), ref["radii"].reshape(-1),
                                         [q * P for q in range(k + 1)], rs, [gts[union[p]].to(DEV) for p in own])
        assert same_bits(img_a, img_b), f"owner {j}: images"
        assert same_bits(loss_a, loss_b), f"owner {j}: losses"
        g = torch.randn((k, 2), generator=torch.Generator().manual_seed(j)).to(DEV)
        ga = torch.autograd.grad(loss_a, (r_m2, r_rgb, r_co), g)
        gb = torch.autograd.grad(loss_b, (w_m2, w_rgb, w_co), g)
        sel = torch.cat([vis[q] for q in range(k)])
        for f, a, b in zip(("means2D", "rgb", "conic_opacity"), ga, gb):
            assert same_bits(a, b[sel]), f"owner {j}: d {f}"
