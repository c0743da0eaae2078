"""Multi-GPU check of the image metrics (run under torch.distributed.run, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29516 \
        tests/mgpu_image_metrics.py

W ranks, each holding its shard of the scene, score the camera set and a held-out set with pipeline.Trainer.image_metrics
at several batch sizes, over the peer-memory exchange and over all_to_all_single (peer_exchange=False).  A one-rank
Trainer over the whole scene on rank 0 is the reference: every view's SSIM and PSNR must be the same bits, and the 8-bit
renders gathered on rank 0 must be the same bytes.  The halo rows come from the neighbouring strips' owners, whose
renders of those rows are those of the whole view; H = 264 leaves a last tile row of 8 rows."""
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


def check(dev, rank, world, peer, log=print):
    n = N_GAUSS - N_GAUSS % world
    scene = syn.make_scene(n, W_IMG, H_IMG, seed=21, radius_px=8.0)
    cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=3.0 * q - 15.0, uid=q) for q in range(N_CAMS)]
    gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=50 + q)).pin_memory() for q in range(N_CAMS)]
    held_cams = [syn.make_camera(W_IMG, H_IMG, yaw_deg=2.0 * q - 9.0, uid=100 + q) for q in range(5)]
    held_gts = [torch.from_numpy(syn.make_gt_image(W_IMG, H_IMG, seed=80 + q)) for q in range(5)]
    tr = pipeline.Trainer(scene, cams, gts, dev, rank, world, load_balance=False, peer_exchange=peer)
    one = pipeline.Trainer(scene, cams, gts, dev) if rank == 0 else None
    ok = True
    for what, kw, views in (("own", {}, [4, 0, 11, 7, 7, 2, 9]), ("held-out", dict(cams=held_cams, gts=held_gts),
                                                                    [3, 1, 4, 0])):
        for bsz in (1, 3, None):
            got = tr.image_metrics(views, bsz=bsz, images=True, **kw)
            if rank == 0:
                want = one.image_metrics(views, images=True, **kw)
                same = (torch.equal(got["ssim_per_view"], want["ssim_per_view"]) and
                        torch.equal(got["psnr_per_view"], want["psnr_per_view"]))
                same_images = len(got["images"]) == len(views) and all(
                    torch.equal(a, b) for a, b in zip(got["images"], want["images"]))
                log(f"[mgpu-image-metrics] world {world} {'peer' if peer else 'nccl'} {what} bsz {bsz}: "
                    f"SSIM {got['ssim']:.9f} PSNR {got['psnr']:.6f} vs one rank {want['ssim']:.9f} / {want['psnr']:.6f}: "
                    f"{'bit-exact' if same else 'DIFFERENT'}; images {'equal' if same_images else 'DIFFERENT'}")
                ok = ok and same and same_images
            else:
                ok = ok and got["images"] is None
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
    ok = all([check(dev, rank, world, peer, log=log) for peer in (True, False)])
    log(f"[mgpu-image-metrics] {'PASS' if ok else 'FAIL'} world_size {world}")
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
