"""Multi-GPU check of the per-view training loss report (run under torch.distributed.run, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 \
        tests/mgpu_train_losses.py

W ranks step the same batches, drain Trainer.train_losses() on every rank, and rank 0 compares each view's [Ll1, ssim,
loss] with a one-rank Trainer over the whole scene stepping the same views:
  * the strip division with border_exchange=True (every strip's SSIM window holds its neighbours' 5 halo rows):
    Ll1 and ssim within W float32 ulps of the one-rank value (tests/test_train_losses_gpu.py states the bound), the loss
    within what those differences and its own rounding allow;
  * the strip division without it: Ll1 within the same bound; the SSIM of a split view sees the strip edges, as the
    reference's strip loss does, so its difference is only reported;
  * local sampling (each rank draws local_bsz views of the images it holds; the batch is the ranks' views in rank order):
    every view is rendered whole by one rank, within the same bound (whether it is bit for bit is reported);
  * distributed_dataset_storage=True (only rank 0 holds the images and scatters each rank's strips), with and without
    border_exchange: every resident=False step's loss and gradients, and the drained entries, are the bits of the default
    Trainer at the same world size.
Every rank's drained entries must be the same (the records are summed over the ranks)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from gs_b200 import pipeline, synthetic as syn  # noqa: E402

W_IMG, H_IMG, N_CAMS, N_GAUSS = 320, 272, 16, 30000
LAM = 0.2


def scene_of(world):
    n = N_GAUSS - N_GAUSS % world
    scene = syn.make_scene(n, W_IMG, H_IMG, seed=21, radius_px=8.0)
    cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=3.0 * q - 20.0, uid=q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=50 + q)).pin_memory() for q in range(N_CAMS)]
    return scene, cams, gts


def same_on_every_rank(entries, dev, world):
    flat = torch.tensor([v for e in entries for k in ("views", "l1", "ssim", "loss") for v in e[k]], dtype=torch.float64,
                        device=dev)
    parts = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(parts, flat)
    return all(torch.equal(p.view(torch.int64), flat.view(torch.int64)) for p in parts)


def compare(got, want, world, check_ssim):
    """-> (within the bound, bit for bit, the largest |ssim| difference in ulps)."""
    ok, exact, worst = True, True, 0.0
    for a, b in zip(got, want):
        ok = ok and a["views"] == b["views"]
        for q in range(len(b["views"])):
            d = {k: abs(np.float64(a[k][q]) - np.float64(b[k][q])) for k in ("l1", "ssim", "loss")}
            ulp = {k: float(np.spacing(np.float32(abs(b[k][q])))) for k in ("l1", "ssim", "loss")}
            bl1, bssim = world * ulp["l1"], world * ulp["ssim"]
            ok = ok and d["l1"] <= bl1
            if check_ssim:
                ok = ok and d["ssim"] <= bssim and d["loss"] <= (1 - LAM) * bl1 + LAM * bssim + 2 * ulp["loss"]
            exact = exact and all(np.float32(a[k][q]) == np.float32(b[k][q]) for k in ("l1", "ssim", "loss"))
            worst = max(worst, d["ssim"] / ulp["ssim"])
    return ok and len(got) == len(want), exact, worst


def check_division(dev, rank, world, border, steps=4, log=print):
    scene, cams, gts = scene_of(world)
    tr = pipeline.Trainer(scene, cams, gts, dev, rank, world, lambda_dssim=LAM, deterministic=True, load_balance=False,
                          border_exchange=border)
    one = pipeline.Trainer(scene, cams, gts, dev, lambda_dssim=LAM, deterministic=True) if rank == 0 else None
    rng = np.random.default_rng(5)
    for it in range(steps):
        views = [int(v) for v in rng.choice(N_CAMS, size=int(rng.integers(1, 9)))]
        tr.step(views=views, resident=it % 2 == 1)
        if one is not None:
            one.step(views=views)
    entries = tr.train_losses()
    same = same_on_every_rank(entries, dev, world)
    ok, exact, worst = True, True, 0.0
    if rank == 0:
        ok, exact, worst = compare(entries, one.train_losses(), world, check_ssim=border)
        log(f"[mgpu-tl] world {world} strip division, border_exchange={border}: "
            f"{'within bound' if ok else 'DIFFERENT'}, bit-exact {exact}, largest ssim difference {worst:.1f} ulp")
    flag = torch.tensor([1.0 if ok and same else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item() > 0)


def check_dataset_storage(dev, rank, world, border, steps=4, log=print):
    scene, cams, gts = scene_of(world)
    kw = dict(lambda_dssim=LAM, deterministic=True, load_balance=False, border_exchange=border)
    # border_exchange reads the strips of views split over several ranks from every rank's resident images
    tr = pipeline.Trainer(scene, cams, gts if rank == 0 or border else None, dev, rank, world,
                          distributed_dataset_storage=True, **kw)
    ref = pipeline.Trainer(scene, cams, gts, dev, rank, world, **kw)
    rng = np.random.default_rng(9)
    same = True
    for _ in range(steps):
        views = [int(v) for v in rng.choice(N_CAMS, size=int(rng.integers(1, 9)))]
        a, b = tr.step(views=views, resident=False), ref.step(views=views, resident=False)
        same = same and np.float32(a).view(np.int32) == np.float32(b).view(np.int32)
        same = same and all(torch.equal(x.grad.view(torch.int32), y.grad.view(torch.int32))
                            for x, y in zip(tr.params.raw_parameters(), ref.params.raw_parameters()))
    same = same and tr.train_losses() == ref.train_losses()
    flag = torch.tensor([1.0 if same else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    ok = bool(flag.item() > 0)
    log(f"[mgpu-tl] world {world} distributed_dataset_storage, border_exchange={border}: "
        f"{'bit-exact' if ok else 'DIFFERENT'} against the default Trainer")
    return ok


def check_local_sampling(dev, rank, world, local_bsz, steps=3, log=print):
    scene, cams, gts = scene_of(world)
    held = [g if q % world == rank else None for q, g in enumerate(gts)]
    tr = pipeline.Trainer(scene, cams, held, dev, rank, world, lambda_dssim=LAM, deterministic=True,
                          local_sampling=True, local_bsz=local_bsz)
    one = pipeline.Trainer(scene, cams, gts, dev, lambda_dssim=LAM, deterministic=True) if rank == 0 else None
    rng = np.random.default_rng(7)
    for it in range(steps):
        mine = [[int(v) for v in rng.choice(np.arange(r, N_CAMS, world), size=local_bsz)] for r in range(world)]
        tr.step(views=mine[rank], resident=it % 2 == 1)
        if one is not None:
            one.step(views=[v for m in mine for v in m])
    entries = tr.train_losses()
    same = same_on_every_rank(entries, dev, world)
    ok = True
    if rank == 0:
        ok, exact, _ = compare(entries, one.train_losses(), world, check_ssim=True)
        log(f"[mgpu-tl] world {world} local sampling, local_bsz {local_bsz}: "
            f"{'within bound' if ok else 'DIFFERENT'}, bit-exact {exact}")
    flag = torch.tensor([1.0 if ok and same else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item() > 0)


def main():
    sys.stdout.reconfigure(line_buffering=True)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    log = (lambda m: print(m, flush=True)) if rank == 0 else (lambda m: None)
    results = [check_division(dev, rank, world, border, log=log) for border in (True, False)]
    results += [check_local_sampling(dev, rank, world, k, log=log) for k in (1, 2)]
    results += [check_dataset_storage(dev, rank, world, border, log=log) for border in (True, False)]
    ok = all(results)
    log(f"[mgpu-tl] {'PASS' if ok else 'FAIL'} world_size {world}")
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
