"""Multi-GPU check of the training schedule (run under torch.distributed.run, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29531 \
        tests/mgpu_schedule.py

W ranks train their shards through gs_b200.schedule.Schedule with short intervals and densify every few iterations.
  * redistribution fires exactly where the reference's gate says (need_redistribute_gaussians: the densify counter is a
    multiple of the frequency, and equal to it or min * threshold < max over the ranks' counts before the move), on
    every rank alike, and the whole model's Gaussian count is the same before and after each move;
  * the memory gate: the limit is set between the ranks' peak reserved memory and that peak plus 1 GiB, and rank 0
    alone then holds a 2 GiB block; at the next densification every rank stops densifying, and none before."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from gs_b200 import pipeline, schedule as sc, synthetic as syn  # noqa: E402

W_IMG, H_IMG, N_CAMS, N_GAUSS = 320, 264, 6, 30000
BSZ, ITERS, BLOCK_AT = 2, 61, 41


def gathered(values, dev):
    t = torch.tensor(values, dtype=torch.float64, device=dev)
    out = torch.empty((dist.get_world_size(), t.numel()), dtype=torch.float64, device=dev)
    dist.all_gather_into_tensor(out, t)
    return out.cpu().tolist()


def check(dev, rank, world, log=print):
    scene = syn.make_scene(N_GAUSS, W_IMG, H_IMG, seed=31, radius_px=8.0)
    cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=3.0 * q - 7.0, uid=q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=60 + q)).pin_memory() for q in range(N_CAMS)]
    tr = pipeline.Trainer(scene, cams, gts, dev, rank, world, load_balance=False, deterministic=True)
    extent = float(torch.exp(tr.params._scaling.detach()).max(dim=1).values.median()) / 0.01
    # a gradient threshold that selects a few percent of the Gaussians, one value on every rank
    a, d, m = (torch.zeros((tr.n_local, 1), device=dev), torch.zeros((tr.n_local, 1), device=dev),
               torch.zeros((tr.n_local,), device=dev))
    for it in range(4):
        tr.step(views=[(it + b) % N_CAMS for b in range(BSZ)])
        tr.add_densification_stats(a, d, m)
    threshold = max(r[0] for r in gathered([float(torch.quantile((a / d).nan_to_num(0.0), 0.95))], dev))
    torch.cuda.synchronize(dev)
    total = torch.cuda.get_device_properties(dev).total_memory / 1024 ** 3
    base = max(r[0] for r in gathered([torch.cuda.max_memory_reserved(dev) / 1024 ** 3], dev))
    # peaks grow a little as the model grows: the limit sits 1 GiB over today's peak, the block adds 2 GiB
    opt = sc.OptimizationParams(bsz=BSZ, iterations=ITERS, densify_from_iter=2, densification_interval=4,
                                opacity_reset_interval=30, densify_until_iter=ITERS, sh_step=10,
                                densify_grad_threshold=threshold, redistribute_gaussians_frequency=2,
                                redistribute_gaussians_threshold=1.01,
                                densify_memory_limit_percentage=(base + 1.0) / total)
    sched = sc.Schedule(tr, opt, extent)
    ok, block, fired, tripped_at = True, None, 0, None
    for it in range(1, ITERS + 1, BSZ):
        if it == BLOCK_AT and rank == 0:
            block = torch.empty((2 << 30,), dtype=torch.uint8, device=dev)
        sched.begin(it)
        tr.step(views=[(it + b) % N_CAMS for b in range(BSZ)])
        counter, disabled = sched.densify_iter, sched.densification_disabled
        ev = sched.end(it)
        if ev.densify is None:
            continue
        # the gate as the reference forms it, from the counts after this densification (one extra all-gather)
        n_after = ev.redistribution[0] if ev.redistribution else tr.n_local
        counts = [int(r[0]) for r in gathered([n_after], dev)]
        want = counter % opt.redistribute_gaussians_frequency == 0 and (
            counter == opt.redistribute_gaussians_frequency or min(counts) * opt.redistribute_gaussians_threshold < max(counts))
        rows = gathered([float(ev.redistribution is not None), float(ev.densification_disabled), float(tr.n_local)], dev)
        if any(bool(r[0]) != want for r in rows):
            log(f"[mgpu-schedule] iteration {it}: redistribution {[r[0] for r in rows]}, gate {want} (counts {counts})")
            ok = False
        if ev.redistribution is not None:
            fired += 1
            if sum(int(r[2]) for r in rows) != sum(counts):
                log(f"[mgpu-schedule] iteration {it}: {sum(counts)} Gaussians before the move, "
                    f"{sum(int(r[2]) for r in rows)} after")
                ok = False
        if len({r[1] for r in rows}) != 1:
            log(f"[mgpu-schedule] iteration {it}: memory-gate decisions differ between ranks: {[r[1] for r in rows]}")
            ok = False
        if ev.densification_disabled and not disabled:
            tripped_at = it
    if tripped_at is None or tripped_at < BLOCK_AT:
        log(f"[mgpu-schedule] the memory gate tripped at {tripped_at}, expected the first densification after {BLOCK_AT}")
        ok = False
    if fired == 0:
        log("[mgpu-schedule] no redistribution fired")
        ok = False
    log(f"[mgpu-schedule] world {world}: {fired} redistributions, memory gate at iteration {tripped_at}, "
        f"{tr.n_local} Gaussians on rank {rank}")
    del block
    return ok


def main():
    sys.stdout.reconfigure(line_buffering=True)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    log = (lambda m: print(m, flush=True)) if rank == 0 else (lambda m: None)
    ok = check(dev, rank, world, log=log)
    flags = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    ok = bool(flags.item())
    log(f"[mgpu-schedule] {'PASS' if ok else 'FAIL'} world_size {world}")
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
