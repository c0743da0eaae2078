"""Multi-GPU check of local sampling (run under torch.distributed.run, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513 \
        tests/mgpu_local_sampling.py

W ranks each hold the images of the cameras with uid % W == rank and step local_bsz views of their own with
pipeline.Trainer(local_sampling=True, deterministic=True).  A one-rank Trainer over the whole scene, stepping the union
batch (the ranks' views in rank order), is the reference: the W ranks' losses must add up to its loss, and their
gathered parameter gradients must equal its gradients.  Whether the gradients agree bit for bit is reported as well
(each view is rendered whole by one rank, as on one rank; the loss adds per-rank partial sums in another order)."""
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

NAMES = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")
W_IMG, H_IMG, N_CAMS, N_GAUSS = 320, 272, 16, 30000
RTOL = 1e-5


def check(dev, rank, world, local_bsz, steps=3, log=print):
    n = N_GAUSS - N_GAUSS % world
    scene = syn.make_scene(n, W_IMG, H_IMG, seed=21, radius_px=8.0)
    cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=3.0 * q - 20.0, uid=q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=50 + q)).pin_memory() for q in range(N_CAMS)]
    held = [g if q % world == rank else None for q, g in enumerate(gts)]
    tr = pipeline.Trainer(scene, cams, held, dev, rank, world, deterministic=True, local_sampling=True,
                          local_bsz=local_bsz)
    one = pipeline.Trainer(scene, cams, gts, dev, deterministic=True) if rank == 0 else None
    rng = np.random.default_rng(7)
    ok, exact = True, True
    for it in range(steps):
        # every rank draws the same schedule, so each knows the union batch only for this check
        mine = [[int(v) for v in rng.choice(np.arange(r, N_CAMS, world), size=local_bsz)] for r in range(world)]
        loss = tr.step(views=mine[rank], resident=False)
        losses = [torch.zeros((), device=dev) for _ in range(world)]
        dist.all_gather(losses, torch.tensor(loss, device=dev))
        grads = {}
        for name in NAMES:
            g = getattr(tr.params, name).grad.contiguous()
            parts = [torch.empty_like(g) for _ in range(world)]
            dist.all_gather(parts, g)
            grads[name] = torch.cat(parts)
        if rank == 0:
            ref_loss = one.step(views=[v for m in mine for v in m], resident=False)
            got = float(sum(float(x) for x in losses))
            step_ok = abs(got - ref_loss) <= RTOL * abs(ref_loss)
            for name in NAMES:
                a, b = grads[name].double(), getattr(one.params, name).grad.double()
                tol = RTOL * b.abs() + RTOL * b.abs().mean()
                step_ok = step_ok and bool(((a - b).abs() <= tol).all())
                exact = exact and torch.equal(grads[name], getattr(one.params, name).grad)
            log(f"[mgpu-ls] world {world} local_bsz {local_bsz} step {it}: views {mine}, loss {got:.7f} vs one rank "
                f"{ref_loss:.7f}, gradients {'bit-exact' if exact else 'within tolerance' if step_ok else 'DIFFERENT'}")
            ok = ok and step_ok
    flag = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    assert tr.history.history == [] and tr._pending_feedback == []
    return bool(flag.item() > 0), exact


def main():
    sys.stdout.reconfigure(line_buffering=True)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    log = (lambda m: print(m, flush=True)) if rank == 0 else (lambda m: None)
    results = [check(dev, rank, world, k, log=log) for k in sorted({1, max(1, 16 // world // 2)})]
    ok = all(r[0] for r in results)
    log(f"[mgpu-ls] {'PASS' if ok else 'FAIL'} world_size {world}; bit-exact gradients: {[r[1] for r in results]}")
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
