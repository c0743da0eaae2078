"""Multi-GPU check of saving and loading a model (run under torch.distributed.run, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29516 \
        tests/mgpu_model_io.py

W ranks train a few deterministic steps over their shards, then save per-rank PLY files, a gathered PLY and per-rank
checkpoints into one directory on the node.
  * PLY at W' = W (every rank) and at W' = 1 (rank 0 alone, over the whole model): Trainers loaded from the per-rank and
    from the gathered files evaluate to the bits of the training Trainer -- evaluate is world-size independent (DESIGN.md
    5f), so a reload at any world size scores the same;
  * checkpoints at W' = W and at W' = 1: the loaded state -- parameters, Adam moments and step, statistics -- is the
    training state gathered in rank order, and a Trainer resumed from the W' = 1 load evaluates to the same bits."""
import os
import shutil
import sys
import tempfile

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from gs_b200 import model_io, pipeline, synthetic as syn  # noqa: E402
from gs_b200.optim import FusedAdam  # noqa: E402

W_IMG, H_IMG, N_CAMS, N_GAUSS = 320, 264, 6, 30000


def bits(t):
    return t.detach().contiguous().view(torch.int32 if t.element_size() == 4 else torch.int64)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def gathered(t, world):
    """This rank's rows of every rank, concatenated in rank order, on every rank (CPU)."""
    out = [None] * world
    dist.all_gather_object(out, t.detach().cpu())
    return torch.cat(out)


def check(dev, rank, world, log=print):
    scene = syn.make_scene(N_GAUSS, W_IMG, H_IMG, seed=31, radius_px=8.0)
    cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=3.0 * q - 7.0, uid=q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=60 + q)).pin_memory() for q in range(N_CAMS)]
    tr = pipeline.Trainer(scene, cams, gts, dev, rank, world, load_balance=False, deterministic=True)
    opt = FusedAdam(tr.optimizer_groups(), lr=0.0, eps=1e-15)
    stats = {"max_radii2D": torch.zeros((tr.n_local,), device=dev),
             "xyz_gradient_accum": torch.zeros((tr.n_local, 1), device=dev),
             "denom": torch.zeros((tr.n_local, 1), device=dev)}
    for it in range(3):
        tr.step(views=[it, it + 3])
        tr.add_densification_stats(stats["xyz_gradient_accum"], stats["denom"], stats["max_radii2D"])
        opt.step(grad_scale=0.5)
    box = [tempfile.mkdtemp(prefix="mgpu_model_io_") if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    base = box[0]
    ok = True
    try:
        model_io.save_ply(os.path.join(base, "per_rank"), tr)
        model_io.save_ply(os.path.join(base, "gathered"), tr, gather=True)
        model_io.save_checkpoint(os.path.join(base, "ckpt"), tr, opt, stats, next_iteration=3)
        dist.barrier()
        want = tr.evaluate()
        want = (want["l1_per_view"], want["psnr_per_view"])

        def scores(t):
            e = t.evaluate()
            return e["l1_per_view"], e["psnr_per_view"]

        for kind in ("per_rank", "gathered"):
            params, shard, _ = model_io.load_ply(os.path.join(base, kind), rank, world, device=dev)
            again = pipeline.Trainer(None, cams, gts, dev, rank, world, model=params, shard=shard, load_balance=False)
            got = scores(again)
            good = all(same(x, y) for x, y in zip(got, want))
            log(f"[mgpu-model-io] world {world} PLY {kind} reloaded at W' = {world}: "
                f"{'bit-exact' if good else 'DIFFERENT'}")
            ok = ok and good
            if rank == 0:
                params, shard, _ = model_io.load_ply(os.path.join(base, kind), 0, 1, device=dev)
                one = pipeline.Trainer(None, cams, gts, dev, model=params, shard=shard)
                good = all(same(x, y) for x, y in zip(scores(one), want))
                log(f"[mgpu-model-io] world {world} PLY {kind} reloaded at W' = 1: {'bit-exact' if good else 'DIFFERENT'}")
                ok = ok and good
                del one
            dist.barrier()
        # the training state gathered in rank order: what a W' = 1 load of the checkpoint must hold
        src = {name: gathered(getattr(tr.params, attr), world) for name, attr in pipeline.Trainer.GROUP_OF.items()}
        mom = {g["name"]: (gathered(opt.state[g["params"][0]]["exp_avg"], world),
                           gathered(opt.state[g["params"][0]]["exp_avg_sq"], world),
                           float(opt.state[g["params"][0]]["step"])) for g in opt.param_groups}
        st = {k: gathered(v, world) for k, v in stats.items()}
        ck = model_io.load_checkpoint(os.path.join(base, "ckpt"), rank, world, dev)
        good = all(same(ck.params[k], getattr(tr.params, a)) for k, a in pipeline.Trainer.GROUP_OF.items())
        log(f"[mgpu-model-io] world {world} checkpoint at W' = {world}: {'own state' if good else 'DIFFERENT'}")
        ok = ok and good
        if rank == 0:
            ck = model_io.load_checkpoint(os.path.join(base, "ckpt"), 0, 1, dev)
            one = pipeline.Trainer(None, cams, gts, dev, model=ck.params)
            fused = model_io.load_fused_adam(one, ck)
            good = all(same(ck.params[k].cpu(), src[k]) for k in src)
            good = good and all(same(ck.stats[k].cpu(), st[k]) for k in st)
            for g in fused.param_groups:
                s = fused.state[g["params"][0]]
                m, v, step = mom[g["name"]]
                good = good and same(s["exp_avg"].cpu(), m) and same(s["exp_avg_sq"].cpu(), v) and float(s["step"]) == step
            good = good and all(same(x, y) for x, y in zip(scores(one), want))
            log(f"[mgpu-model-io] world {world} checkpoint resumed at W' = 1: gathered state and evaluation "
                f"{'bit-exact' if good else 'DIFFERENT'}")
            ok = ok and good
    finally:
        dist.barrier()
        if rank == 0:
            shutil.rmtree(base, ignore_errors=True)
    flag = torch.tensor([1.0 if ok else 0.0], device=dev)
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
    ok = check(dev, rank, world, log=log)
    log(f"[mgpu-model-io] {'PASS' if ok else 'FAIL'} world_size {world}")
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
