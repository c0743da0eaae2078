"""-m gpu: saving and loading a trained model on one H100 (gs_b200.model_io).

  * exact resume: 2k deterministic training steps (FusedAdam, densification statistics, densify_and_prune on both sides
    of the checkpoint) give the same bits as k steps, a checkpoint, a fresh Trainer and FusedAdam from it, and k more --
    in every parameter, Adam moment and step, statistic and per-step loss; at SH degree 3 and 1, and with the active
    degree below the stored one;
  * PLY round trip: a Trainer loaded from the per-rank or the gathered PLY of a trained one evaluates to the same bits
    (evaluate and image_metrics with the 8-bit renders)."""
import pytest
import torch

import gpu_util as gu
from gs_b200 import densify, model_io, pipeline
from gs_b200 import synthetic as syn
from gs_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu

TW, TH, N_VIEWS, N_GAUSS = 256, 192, 8, 20000
K_STEPS = 4
DENSIFY_AFTER = (1, 5)   # one densification before the checkpoint, one after it from statistics that span it
BSZ = 2


def camera_set():
    cams = [syn.make_camera(TW, TH, yaw_deg=1.5 * q - 5.0, uid=q) for q in range(N_VIEWS)]
    gts = [torch.from_numpy(syn.make_gt_image(TW, TH, seed=30 + q)).pin_memory() for q in range(N_VIEWS)]
    return cams, gts


def zero_stats(P):
    return {"max_radii2D": torch.zeros((P,), device=gu.DEV), "xyz_gradient_accum": torch.zeros((P, 1), device=gu.DEV),
            "denom": torch.zeros((P, 1), device=gu.DEV)}


def advance(tr, opt, stats, iterations, noise):
    """Training iterations: a batch of BSZ views, the statistics, the Adam step, and densify_and_prune where due."""
    losses = []
    for it in iterations:
        views = [(BSZ * it + b) % N_VIEWS for b in range(BSZ)]
        losses.append(tr.step(views=views, resident=False))
        tr.add_densification_stats(stats["xyz_gradient_accum"], stats["denom"], stats["max_radii2D"])
        opt.step(grad_scale=1.0 / BSZ)
        if it in DENSIFY_AFTER:
            p = tr.params
            grads = (stats["xyz_gradient_accum"] / stats["denom"]).nan_to_num(0.0)
            extent = float(torch.exp(p._scaling.detach()).max(dim=1).values.median()) / 0.01
            res = densify.densify_and_prune(opt, stats["xyz_gradient_accum"], stats["denom"],
                                            float(torch.quantile(grads, 0.8)), 0.005, extent, 0.01, 0, noise=noise)
            tr.adopt_parameters(res)
            stats = {k: res[k] for k in model_io.STAT_NAMES}
    return losses, stats


def state_of(tr, opt, stats):
    out = {}
    for g in opt.param_groups:
        prm = g["params"][0]
        assert prm is getattr(tr.params, pipeline.Trainer.GROUP_OF[g["name"]])
        st = opt.state[prm]
        out[g["name"]] = (prm.detach(), st["exp_avg"], st["exp_avg_sq"], float(st["step"]))
    out.update(stats)
    return out


def bits_equal(a, b):
    if isinstance(a, float):
        return a == b
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.int32),
                                                                   b.contiguous().view(torch.int32))


@pytest.mark.parametrize("D_max,active", [(3, 3), (1, 1), (3, 1)])
def test_resume_from_a_checkpoint_is_exact(tmp_path, D_max, active):
    cams, gts = camera_set()
    sc = syn.make_scene(N_GAUSS, TW, TH, seed=12 + D_max, max_sh_degree=D_max)
    noise = torch.randn((8 * N_GAUSS, 3), generator=torch.Generator().manual_seed(3)).to(gu.DEV)

    def fresh():
        tr = pipeline.Trainer(sc, cams, gts, gu.DEV, max_sh_degree=D_max, deterministic=True)
        tr.params.active_sh_degree = active
        return tr, FusedAdam(tr.optimizer_groups(), lr=0.0, eps=1e-15), zero_stats(tr.n_local)

    tr, opt, stats = fresh()                                       # run A: 2k steps
    la, stats = advance(tr, opt, stats, range(2 * K_STEPS), noise)
    a = state_of(tr, opt, stats)
    del tr, opt, stats

    tr, opt, stats = fresh()                                       # run B: k steps, checkpoint, k steps
    lb, stats = advance(tr, opt, stats, range(K_STEPS), noise)
    model_io.save_checkpoint(str(tmp_path), tr, opt, stats, next_iteration=K_STEPS)
    del tr, opt, stats
    ck = model_io.load_checkpoint(str(tmp_path), 0, 1, gu.DEV)
    assert ck.next_iteration == K_STEPS and ck.active_sh_degree == active
    tr = pipeline.Trainer(None, cams, gts, gu.DEV, model=ck.params, deterministic=True)
    tr.params.active_sh_degree = ck.active_sh_degree
    assert tr.params.max_sh_degree == D_max
    opt = model_io.load_fused_adam(tr, ck)
    lb2, stats = advance(tr, opt, ck.stats, range(K_STEPS, 2 * K_STEPS), noise)
    b = state_of(tr, opt, stats)

    print(f"[resume] D {D_max} active {active}: losses {la}; Gaussians {a['xyz'][0].shape[0]}")
    assert la == lb + lb2
    assert a["xyz"][0].shape[0] != N_GAUSS   # the densifications changed the model
    assert set(a) == set(b)
    for k in a:
        if k in model_io.STAT_NAMES:
            assert bits_equal(a[k], b[k]), k
        else:
            for q in range(4):
                assert bits_equal(a[k][q], b[k][q]), (k, q)


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int64), b.view(torch.int64))


@pytest.mark.parametrize("gather", [False, True], ids=["per_rank", "gathered"])
def test_ply_round_trip_evaluates_to_the_same_bits(tmp_path, gather):
    cams, gts = camera_set()
    sc = syn.make_scene(N_GAUSS, TW, TH, seed=5)
    tr = pipeline.Trainer(sc, cams, gts, gu.DEV, deterministic=True)
    opt = FusedAdam(tr.optimizer_groups(), lr=0.0, eps=1e-15)
    for it in range(3):
        tr.step(views=[it, it + 3])
        opt.step(grad_scale=0.5)
    path = model_io.save_ply(str(tmp_path), tr, gather=gather)
    assert path.endswith("point_cloud.ply" if gather else "point_cloud_rk0_ws1.ply")
    params, shard, D = model_io.load_ply(str(tmp_path), 0, 1, max_sh_degree=3, device=gu.DEV)
    assert shard == (0, N_GAUSS, N_GAUSS) and D == 3
    again = pipeline.Trainer(None, cams, gts, gu.DEV, model=params, shard=shard, deterministic=True)
    for name, attr in pipeline.Trainer.GROUP_OF.items():
        a, b = getattr(tr.params, attr).detach(), getattr(again.params, attr).detach()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), name
    views = [0, 5, 2, 7, 7]
    e1, e2 = tr.evaluate(views), again.evaluate(views)
    assert _same(e1["l1_per_view"], e2["l1_per_view"]) and _same(e1["psnr_per_view"], e2["psnr_per_view"])
    m1, m2 = tr.image_metrics(views, images=True), again.image_metrics(views, images=True)
    assert _same(m1["ssim_per_view"], m2["ssim_per_view"]) and _same(m1["psnr_per_view"], m2["psnr_per_view"])
    assert len(m1["images"]) == len(views) and all(torch.equal(x, y) for x, y in zip(m1["images"], m2["images"]))
    print(f"[ply] {'gathered' if gather else 'per-rank'}: L1 {e1['l1']:.9f} PSNR {e1['psnr']:.6f} SSIM {m1['ssim']:.9f}")
