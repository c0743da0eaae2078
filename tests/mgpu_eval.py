"""Multi-GPU check of held-out view evaluation (run under torch.distributed.run, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29514 \
        tests/mgpu_eval.py

W ranks, each holding its shard of the scene, evaluate the camera set and a held-out set with pipeline.Trainer.evaluate at
several batch sizes, over the peer-memory exchange and over all_to_all_single (peer_exchange=False), and with
distributed_dataset_storage=True, where only rank 0 holds the images and scatters each rank's strips.  A one-rank Trainer
over the whole scene on rank 0 is the reference: every view's L1 and PSNR must be the same bits.  The slots of a view are
non-zero on the one rank that owns each tile row, so their all-reduce is exact; the renders of the strips are those of
the whole view, so the sums are too."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from gs_b200 import pipeline, synthetic as syn  # noqa: E402

W_IMG, H_IMG, N_CAMS, N_GAUSS = 320, 264, 12, 30000


def check(dev, rank, world, peer, dds=False, log=print):
    n = N_GAUSS - N_GAUSS % world
    scene = syn.make_scene(n, W_IMG, H_IMG, seed=21, radius_px=8.0)
    cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=3.0 * q - 15.0, uid=q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=50 + q)).pin_memory() for q in range(N_CAMS)]
    held_cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=2.0 * q - 9.0, uid=100 + q) for q in range(5)]
    held_gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=80 + q)) for q in range(5)]
    if dds:   # only rank 0 holds the images, its own and the held-out ones
        gts, held_gts = [g if rank == 0 else None for g in gts], [g if rank == 0 else None for g in held_gts]
    tr = pipeline.Trainer(scene, cams, None if dds and rank != 0 else gts, dev, rank, world, load_balance=False,
                          peer_exchange=peer, distributed_dataset_storage=dds)
    one = pipeline.Trainer(scene, cams, gts, dev) if rank == 0 else None
    ok = True
    for what, kw, views in (("own", {}, [4, 0, 11, 7, 7, 2, 9]), ("held-out", dict(cams=held_cams, gts=held_gts),
                                                                    [3, 1, 4, 0])):
        for bsz in (1, 3, None):
            got = tr.evaluate(views, bsz=bsz, **kw)
            if rank == 0:
                want = one.evaluate(views, **kw)
                same = (torch.equal(got["l1_per_view"], want["l1_per_view"]) and
                        torch.equal(got["psnr_per_view"], want["psnr_per_view"]))
                log(f"[mgpu-eval] world {world} {'peer' if peer else 'nccl'}{' dataset on rank 0' if dds else ''} {what} "
                    f"bsz {bsz}: L1 {got['l1']:.9f} "
                    f"PSNR {got['psnr']:.6f} vs one rank {want['l1']:.9f} / {want['psnr']:.6f}: "
                    f"{'bit-exact' if same else 'DIFFERENT'}")
                ok = ok and same
    flag = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    assert tr.history.history == [] and tr.iteration == 0
    return bool(flag.item() > 0)


def main():
    sys.stdout.reconfigure(line_buffering=True)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    log = (lambda m: print(m, flush=True)) if rank == 0 else (lambda m: None)
    ok = all([check(dev, rank, world, peer, dds, log=log) for peer, dds in ((True, False), (False, False), (True, True))])
    log(f"[mgpu-eval] {'PASS' if ok else 'FAIL'} world_size {world}")
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
