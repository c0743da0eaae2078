"""Multi-GPU parity (run under torch.distributed.run, one rank per GPU; also called by bench.py at N > 1, outside its
timed regions, so that every SCALE line carries a parity verdict):
pixel-sharded render + sparse all-to-all + mirrored backward must reproduce what a single rank computes.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
        tests/mgpu_parity.py

Checks, for bsz = world size (every rank renders one whole view), bsz = 1 (ONE view cut into `world` tile-row strips) and
bsz = world/2 (two strips per view):
  1. strips rendered by the W ranks, summed with all_reduce (train_internal.py:466-469), equal the oracle's full
     render; tile lists are partition independent so pixels agree to fp32 rounding, non-local tiles are exactly 0;
  2. the per-shard parameter gradients, gathered, match the oracle evaluated with the SAME strip-wise loss
     (zero-padded SSIM at strip edges, loss_distribution.py:2553-2576) within 1e-4;
  1b. the NVLink peer-memory exchange equals all_to_all_single bit for bit, forward rows and backward gradients;
  3. the fused sparse gradient all-reduce (replicated Gaussians, row L2) equals the dense all-reduce;
  4. border-pixel exchange (row L1): strip losses add up to the full-image loss, gradients equal the single-GPU ones;
  5. the timing feedback moves the strips of an uneven 4K-class division and the step stays correct afterwards.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "grendel-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from gs_b200 import division, ops, pipeline, synthetic as syn  # noqa: E402

NAMES = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")
RTOL = 1e-4          # |err| <= RTOL |ref| + RTOL rms(ref)   (tests/gpu_util.py: the bar of the single-GPU tests)
MAX_OUTSIDE = 1e-3
VIEW_W, VIEW_H = 320, 272   # 17 tile rows: can be cut into 8 strips of >= 2 rows


def _gather_grads(tr, world):
    grads = {}
    for n in NAMES:
        g = getattr(tr.params, n).grad.contiguous()
        parts = [torch.empty_like(g) for _ in range(world)]  # equal shards: N divisible by world in these tests
        dist.all_gather(parts, g)
        grads[n] = torch.cat(parts).cpu().numpy()
    return grads


def _raw_param_grads(scene, e):
    """Oracle gradients w.r.t. the activated inputs -> gradients of the raw GaussianModel parameters."""
    op, q, gq = scene["opacities"], scene["rotations"], e["rotations"]
    return {"_xyz": e["means3D"], "_features_dc": e["shs"][:, :1], "_features_rest": e["shs"][:, 1:],
            "_scaling": e["scales"] * scene["scales"], "_opacity": e["opacities"] * op * (1 - op),
            "_rotation": gq - q * (q * gq).sum(1, keepdims=True)}


def _compare(grads, ref, log, tag):
    worst, out = 0.0, 0.0
    for n in NAMES:
        a, b = grads[n].astype(np.float64), ref[n].astype(np.float64)
        rms = np.sqrt((b ** 2).mean())
        err = np.abs(a - b)
        badf = float((err > RTOL * np.abs(b) + RTOL * rms).mean())
        w = float((err / (np.abs(b) + rms + 1e-30)).max())
        log(f"[mgpu] {tag} grad {n}: rms {rms:.3e} max_abs_err {err.max():.3e} worst_rel {w:.2e} outside tol {badf:.1e}")
        worst, out = max(worst, w), max(out, badf)
    return worst, out


def views_check(dev, rank, world, B, scene, log, oracle):
    """Checks 1 + 2 for B views per step.  Returns a dict (rank 0: verdict; other ranks: {})."""
    W, H = VIEW_W, VIEW_H
    cams = syn.make_batch_cameras(W, H, B)
    gts = [syn.make_gt_image(W, H, seed=50 + k) for k in range(B)]
    tr = pipeline.Trainer(scene, cams, [torch.from_numpy(g).pin_memory() for g in gts], dev, rank, world)
    loss = tr.step(resident=False)
    strategies, _ = division.start_strategy([c.uid for c in tr.dcams], tr.history, world, rank)
    settings = [c.settings(3) for c in tr.dcams]
    with torch.no_grad():
        p = tr.params
        imgs = []
        screen = [ops.preprocess_gaussians_raw(p._xyz, p._features_dc, p._features_rest, p._scaling, p._rotation,
                                               p._opacity, rs) for rs in settings]
        stacked = tuple(torch.stack([s_[q] for s_ in screen]) for q in range(5))
        red, _ = tr._ex.exchange(*stacked, strategies, settings, world, rank, None, tr._peer)
        for k, st in enumerate(strategies):
            img = torch.zeros((3, H, W), device=dev)
            if st.local_rows() is not None:
                m2, rgb, co, radii, depths = red[k]
                img, *_ = ops.render_gaussians(m2, co, rgb, depths, radii, st.get_compute_locally(tr.tile_x, dev), settings[k])
                y0, y1 = st.local_pixel_rows(H)
                outside = torch.ones((H, W), dtype=torch.bool, device=dev)
                outside[y0:y1] = False
                assert (img[:, outside] == 0).all(), "non-local tiles must be exactly zero"
            dist.all_reduce(img)
            imgs.append(img.cpu().numpy())
    peer_bitexact = None
    if tr._peer is not None:  # 1b
        outs = []
        for peer in (tr._peer, None):
            leaves = [stacked[q].detach().clone().requires_grad_(True) for q in range(3)]
            (m2, c3, co, rad, dep), vs, _, _ = tr._ex.exchange_cat(leaves[0], leaves[1], leaves[2], stacked[3], stacked[4],
                                                                   strategies, settings, world, rank, None, peer)
            gen = torch.Generator(device=dev).manual_seed(7 + rank)
            up = [torch.randn(t.shape, device=dev, generator=gen) for t in (m2, c3, co)]
            ((m2 * up[0]).sum() + (c3 * up[1]).sum() + (co * up[2]).sum()).backward()
            outs.append(([m2.detach(), c3.detach(), co.detach(), rad, dep], [l.grad for l in leaves], vs))
        same = outs[0][2] == outs[1][2] and all(torch.equal(a, b) for a, b in zip(outs[0][0] + outs[0][1], outs[1][0] + outs[1][1]))
        flag = torch.tensor([1.0 if same else 0.0], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        peer_bitexact = bool(flag.item() > 0)
        log(f"[mgpu] bsz {B}: NVLink peer-memory exchange == all_to_all_single, forward rows and backward gradients: "
            f"{'bit-exact' if peer_bitexact else 'DIFFERENT'} ({outs[0][2][-1]} rows received on rank 0)")
    grads = _gather_grads(tr, world)
    losses = [torch.zeros((), device=dev) for _ in range(world)]
    dist.all_gather(losses, torch.tensor(loss, device=dev))
    res = {}
    if rank == 0:
        o = oracle
        T = tr.tile_y * tr.tile_x
        exp = {n: 0 for n in ("means3D", "scales", "rotations", "opacities", "shs")}
        tot_loss, img_err, img_bad = 0.0, 0.0, 0.0
        for k, cam in enumerate(cams):
            pre = o.preprocess_forward(scene["means3D"], scene["scales"], scene["rotations"], scene["shs"], scene["opacities"], cam)
            fwd = o.render_forward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                                   np.ones(T, np.uint8), (0, 0, 0))
            err = np.abs(imgs[k] - fwd["image"])
            img_err = max(img_err, float(err.max()))
            img_bad = max(img_bad, float((err > 1e-4 * np.abs(fwd["image"]) + 1e-5).mean()))
            st = strategies[k]
            dimg = np.zeros((3, H, W), np.float32)
            gtf = np.clip(gts[k].astype(np.float32) / np.float32(255), 0, 1)
            for li in range(len(st.gpu_ids)):
                y0, y1 = st.division_pos[li] * 16, min(st.division_pos[li + 1] * 16, H)
                l1, ss, g = o.loss(fwd["image"][:, y0:y1], gtf[:, y0:y1], H * W, 0.2)
                dimg[:, y0:y1] = g
                tot_loss += 0.8 * l1 + 0.2 * (1 - ss)
            rb = o.render_backward(H, W, pre["means2D"], pre["conic_opacity"], pre["rgb"], (0, 0, 0), fwd, dimg)
            pb = o.preprocess_backward(scene["means3D"], scene["scales"], scene["rotations"], scene["shs"],
                                       scene["opacities"], cam, pre["radii"], pre["clamped"], rb["means2D"],
                                       rb["conic_opacity"], rb["rgb"])
            for n in exp:
                exp[n] = exp[n] + pb[n]
        got_loss = float(sum(float(x) for x in losses))
        log(f"[mgpu] bsz {B} ({[len(s.gpu_ids) for s in strategies]} strips per view): assembled images max_abs_err "
            f"{img_err:.2e} (outside tol {img_bad:.1e}); loss sum over ranks {got_loss:.6f} vs oracle strip-wise {tot_loss:.6f}")
        worst, out = _compare(grads, _raw_param_grads(scene, exp), log, f"bsz {B}")
        ok = img_bad <= 2e-4 and abs(got_loss - tot_loss) <= 1e-4 * abs(tot_loss) and out <= MAX_OUTSIDE and peer_bitexact is not False
        res = {"ok": bool(ok), "strips_per_view": [len(s.gpu_ids) for s in strategies], "image_max_abs_err": img_err,
               "loss_rel_err": abs(got_loss - tot_loss) / abs(tot_loss), "grad_worst_rel": worst, "grad_outside_tol": out,
               "peer_exchange_bit_exact": peer_bitexact}
    return res, tr


def check(dev, rank, world, verbose=True):
    """All checks; collective (every rank of the default group calls it).  -> summary dict on rank 0 ({} elsewhere)."""
    from oracle.oracle import Oracle

    def log(msg):
        if verbose and rank == 0:
            print(msg, flush=True)

    # the other ranks wait in the next collective; torchrun's OMP_NUM_THREADS=1 default does not bind the oracle
    o = Oracle(np.float32, threads=max(1, min(32, (os.cpu_count() or 8) // 2))) if rank == 0 else None
    W, H, N = VIEW_W, VIEW_H, 30000
    scene = syn.make_scene(N - N % world, W, H, seed=21, radius_px=8.0)
    summary = {"scene": f"{N - N % world} Gaussians @ {W}x{H}, tolerance {RTOL:g} |ref| + {RTOL:g} rms(ref)", "views": {}}
    tr = None
    for B in sorted({world, 1, max(1, world // 2)}, reverse=True):
        if B != world and (H + 15) // 16 < 2 * (world // B):   # 13 tile rows cannot be cut into that many strips
            log(f"[mgpu] bsz {B}: skipped at world_size {world} (image too short for the strips)")
            continue
        res, tr_b = views_check(dev, rank, world, B, scene, log, o)
        if B == world:
            tr = tr_b
        if rank == 0:
            summary["views"][f"bsz_{B}"] = res

    # ---- 3. replicated-Gaussian gradient sync: fused sparse all-reduce == dense all-reduce -------------------
    from gs_b200 import grad_sync
    g = torch.Generator(device=dev).manual_seed(100 + rank)
    P2 = 20011
    shapes = [(P2, 3), (P2, 1, 3), (P2, 15, 3), (P2, 3), (P2, 4), (P2, 1)]
    touched = torch.rand((P2,), device=dev, generator=g) < 0.07     # each rank touches ~7 % of the Gaussians
    params_a, params_b = [], []
    for shp in shapes:
        grad = torch.randn(shp, device=dev, generator=g)
        grad[~touched] = 0
        pa, pb = torch.zeros(shp, device=dev), torch.zeros(shp, device=dev)
        pa.grad, pb.grad = grad.clone(), grad.clone()
        params_a.append(pa); params_b.append(pb)
    n_touched = grad_sync.sync_gradients_fused_sparse(params_a)
    grad_sync.sync_gradients_densely(params_b)
    same = all(torch.allclose(pa.grad, pb.grad, rtol=1e-6, atol=1e-6) for pa, pb in zip(params_a, params_b))
    flag = torch.tensor([1.0 if same else 0.0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    summary["sparse_grad_allreduce_equals_dense"] = bool(flag.item() > 0)
    log(f"[mgpu] fused sparse gradient all-reduce: {n_touched} of {P2} Gaussians touched, matches dense all-reduce: "
        f"{summary['sparse_grad_allreduce_equals_dense']}")

    # ---- 4. border-pixel exchange (row L1): ONE camera split over all ranks; strip losses must add up to the
    #         FULL-image loss and the gradients must equal the single-GPU full-image gradients -----------------
    tile_y = (H + 15) // 16
    if tile_y < 3 * world:  # 13 tile rows cannot be cut into `world` strips of >= 2 rows
        log(f"[mgpu] border exchange: skipped at world_size {world} (image too short for {world} strips)")
    else:
        cams = syn.make_batch_cameras(W, H, 1)
        gt0 = syn.make_gt_image(W, H, seed=50)
        tr2 = pipeline.Trainer(scene, cams, [torch.from_numpy(gt0).pin_memory()], dev, rank, world, border_exchange=True)
        loss2 = tr2.step(resident=False)
        l2 = [torch.zeros((), device=dev) for _ in range(world)]
        dist.all_gather(l2, torch.tensor(loss2, device=dev))
        g2 = _gather_grads(tr2, world)
        if rank == 0:
            ref2 = o.train_step(scene, cams[0], gt0)
            # each strip adds lambda*(1 - its partial ssim): the constant lambda appears once per strip
            got = float(sum(float(x) for x in l2)) - 0.2 * (world - 1)
            log(f"[mgpu] border exchange: strip losses sum to {got:.6f}, full-image oracle loss {ref2['loss']:.6f}")
            worst, out = _compare(g2, _raw_param_grads(scene, ref2["grads"]), log, "border exchange")
            summary["border_exchange"] = {"ok": bool(abs(got - ref2["loss"]) <= 1e-4 * abs(ref2["loss"]) and out <= MAX_OUTSIDE),
                                          "loss_rel_err": abs(got - ref2["loss"]) / abs(ref2["loss"]), "grad_worst_rel": worst}

    # ---- 5. timing feedback: an uneven division moves, and the step after the move is still the same function -------
    W5, H5 = 1600, 1072     # > 600 x 1000 and bsz < world: the reference's gate enables the feedback (division.py)
    cams5 = syn.make_batch_cameras(W5, H5, 1)
    sc5 = syn.make_scene(20000 - 20000 % world, W5, H5, seed=5, radius_px=20.0)
    sc5["means3D"][:, 1] = np.abs(sc5["means3D"][:, 1])      # everything in the lower half of the image: uneven rows
    gt5 = syn.make_gt_image(W5, H5, seed=9)
    tr5 = pipeline.Trainer(sc5, cams5, [torch.from_numpy(gt5).pin_memory()], dev, rank, world)
    first = None
    for it in range(6):
        l5 = tr5.step(resident=False)
        if it == 0:
            first = list(tr5._strategies[0].division_pos)
    last = list(tr5._strategies[0].division_pos)
    l5s = [torch.zeros((), device=dev) for _ in range(world)]
    dist.all_gather(l5s, torch.tensor(l5, device=dev))
    g5 = _gather_grads(tr5, world)
    if rank == 0:
        st = tr5._strategies[0]
        pre = o.preprocess_forward(sc5["means3D"], sc5["scales"], sc5["rotations"], sc5["shs"], sc5["opacities"], cams5[0])
        T5 = ((H5 + 15) // 16) * ((W5 + 15) // 16)
        fwd = o.render_forward(H5, W5, pre["means2D"], pre["conic_opacity"], pre["rgb"], pre["depths"], pre["radii"],
                               np.ones(T5, np.uint8), (0, 0, 0))
        dimg = np.zeros((3, H5, W5), np.float32)
        gtf = np.clip(gt5.astype(np.float32) / np.float32(255), 0, 1)
        tot = 0.0
        for li in range(len(st.gpu_ids)):
            y0, y1 = st.division_pos[li] * 16, min(st.division_pos[li + 1] * 16, H5)
            l1, ss, g = o.loss(fwd["image"][:, y0:y1], gtf[:, y0:y1], H5 * W5, 0.2)
            dimg[:, y0:y1] = g
            tot += 0.8 * l1 + 0.2 * (1 - ss)
        rb = o.render_backward(H5, W5, pre["means2D"], pre["conic_opacity"], pre["rgb"], (0, 0, 0), fwd, dimg)
        pb = o.preprocess_backward(sc5["means3D"], sc5["scales"], sc5["rotations"], sc5["shs"], sc5["opacities"], cams5[0],
                                   pre["radii"], pre["clamped"], rb["means2D"], rb["conic_opacity"], rb["rgb"])
        got = float(sum(float(x) for x in l5s))
        worst, out = _compare(g5, _raw_param_grads(sc5, pb), log, "after rebalancing")
        moved = first != last
        log(f"[mgpu] timing feedback: strips of the uneven view moved {first} -> {last} in {len(tr5.balance_log) - 1} "
            f"update(s); loss {got:.6f} vs oracle on the moved strips {tot:.6f}")
        summary["load_balance"] = {"ok": bool(moved and abs(got - tot) <= 1e-4 * abs(tot) and out <= MAX_OUTSIDE),
                                   "rows_before": first, "rows_after": last, "grad_worst_rel": worst}
    if rank == 0:
        oks = [v.get("ok", True) for v in summary["views"].values()] + [summary["sparse_grad_allreduce_equals_dense"]]
        oks += [summary[k]["ok"] for k in ("border_exchange", "load_balance") if k in summary]
        summary["ok"] = bool(all(oks))
        log(f"[mgpu] {'PASS' if summary['ok'] else 'FAIL'} world_size {world}")
    okf = torch.tensor([1.0 if (rank != 0 or summary.get("ok")) else 0.0], device=dev)
    dist.all_reduce(okf, op=dist.ReduceOp.MIN)
    del tr
    return summary if rank == 0 else {}


def main():
    sys.stdout.reconfigure(line_buffering=True)   # progress survives a timeout kill when stdout is a pipe
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    flags = int(os.environ.get("GS_B200_DEBUG_FLAGS", "0"))   # A/B switches of the library (include/grendel_gs_b200.h)
    if flags:
        from gs_b200 import _lib
        _lib.debug_set(flags)
        if rank == 0:
            print(f"[mgpu] GS_B200_DEBUG_FLAGS = {flags}", flush=True)
    summary = check(dev, rank, world, verbose=True)
    ok = torch.tensor([1.0 if (rank != 0 or summary.get("ok")) else 0.0], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if rank == 0:
        import json
        print("[mgpu] summary " + json.dumps(summary), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if ok.item() < 1:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
