"""8-bit image rows between the ranks of a strip division, for the image metrics (pipeline.Trainer.image_metrics).

The SSIM of a pixel reads the 11 x 11 neighbourhood around it, so the rank that owns a strip of a view needs the 5 rows on
each side of it: its window is image rows [max(0, y0 - 5), min(H, y1 + 5)) of the 8-bit render and ground truth, six
channels (render 0-2, ground truth 3-5).  exchange_halos fills the rows a rank does not own from the owners of the
neighbouring strips; gather_images assembles the whole 8-bit renders on rank 0.

Every rank holds every view's division (division.start_strategy), so all sizes are computed on the host and each call is
one all_to_all_single of uint8, with no size exchange.  all_to_all_single runs on the communicators the Trainer set up at
construction; batch_isend_irecv would open new point-to-point communicators lazily.  Strips are whole tile rows except the
last one of an image, which can be 1-15 rows tall: the strip above it then receives fewer than 5 rows, and the image ends
there.  Nothing here is CUDA-specific: the functions run on any device a process group serves (gloo on CPU tensors too).
"""
import torch
import torch.distributed as dist

HALO = 5      # rows of the SSIM window on each side of a pixel (ops.SSIM_HALO)
BLOCK_Y = 16


def window_rows(rows, image_height):
    """Local pixel rows (y0, y1) -> the window's image rows [max(0, y0 - 5), min(H, y1 + 5))."""
    return max(0, rows[0] - HALO), min(image_height, rows[1] + HALO)


def _strip(st, c, image_height):
    return st.division_pos[c] * BLOCK_Y, min(st.division_pos[c + 1] * BLOCK_Y, image_height)


def halo_plan(strategies, image_height):
    """-> [(view, source rank, destination rank, y0, y1)]: rows [y0, y1) of the view that the source owns and the
    destination's window needs.  Each strip sends its first min(5, rows) rows to the owner of the strip above and its
    last min(5, rows) rows to the owner of the strip below, in view order."""
    plan = []
    for v, st in enumerate(strategies):
        ids = st.gpu_ids
        for c in range(len(ids)):
            a, b = _strip(st, c, image_height)
            if c > 0:
                plan.append((v, ids[c], ids[c - 1], a, min(b, a + HALO)))
            if c + 1 < len(ids):
                plan.append((v, ids[c], ids[c + 1], max(a, b - HALO), b))
    return plan


def _all_to_all(send, recv_sizes, rank, world, group, device):
    """send[d]: flat uint8 tensors for rank d, in order; recv_sizes[s]: the byte counts expected from rank s.
    -> [per source: list of flat tensors of those sizes]."""
    in_splits = [sum(t.numel() for t in ts) for ts in send]
    out_splits = [sum(ns) for ns in recv_sizes]
    parts = [t for ts in send for t in ts]
    inp = torch.cat(parts) if parts else torch.empty((0,), dtype=torch.uint8, device=device)
    out = torch.empty((sum(out_splits),), dtype=torch.uint8, device=device)
    dist.all_to_all_single(out, inp, out_splits, in_splits, group=group)
    got, off = [], 0
    for ns in recv_sizes:
        mine = []
        for n in ns:
            mine.append(out[off:off + n])
            off += n
        got.append(mine)
    return got


def exchange_halos(windows, win_row0, strategies, image_height, image_width, rank, world, group, device):
    """windows[v]: this rank's (6, R, W) uint8 window of view v, holding image rows [win_row0[v], win_row0[v] + R) with
    the local strip's rows filled (None where the rank owns no strip of the view).  Fills the halo rows from the
    neighbouring strips' owners, in place: one all_to_all_single, none when no view is split."""
    plan = halo_plan(strategies, image_height)
    if not plan:
        return
    W = image_width
    send = [[] for _ in range(world)]
    recv = [[] for _ in range(world)]
    for v, src, dst, y0, y1 in plan:
        if src == rank:
            r0 = win_row0[v]
            send[dst].append(windows[v][:, y0 - r0:y1 - r0].reshape(-1))
        if dst == rank:
            recv[src].append((v, y0, y1))
    got = _all_to_all(send, [[6 * (y1 - y0) * W for _v, y0, y1 in ts] for ts in recv], rank, world, group, device)
    for src in range(world):
        for (v, y0, y1), flat in zip(recv[src], got[src]):
            r0 = win_row0[v]
            windows[v][:, y0 - r0:y1 - r0].copy_(flat.view(6, y1 - y0, W))


def gather_images(strips, strategies, image_height, image_width, rank, world, group, device):
    """strips[v]: this rank's (3, y1 - y0, W) uint8 rows of view v's 8-bit render (None where it owns no strip).
    -> on rank 0 (and at world size 1) the whole (3, H, W) renders in view order, copied to host memory (pinned when the
    device is a GPU, so the copies are asynchronous; they are complete once the current stream is synchronised); None on
    the other ranks.  Every other rank sends its strips to rank 0 in one all_to_all_single."""
    H, W, B = image_height, image_width, len(strategies)
    if world > 1:
        send = [[] for _ in range(world)]
        if rank != 0:
            send[0] = [strips[v].reshape(-1) for v in range(B) if strips[v] is not None]
        recv = [[] for _ in range(world)]
        if rank == 0:
            for v, st in enumerate(strategies):
                for c, gpu in enumerate(st.gpu_ids):
                    if gpu != 0:
                        a, b = _strip(st, c, H)
                        recv[gpu].append((v, a, b))
        got = _all_to_all(send, [[3 * (b - a) * W for _v, a, b in ts] for ts in recv], rank, world, group, device)
        if rank != 0:
            return None
    whole = torch.empty((B, 3, H, W), dtype=torch.uint8, device=device)
    for v, st in enumerate(strategies):
        if 0 in st.gpu_ids:
            a, b = _strip(st, st.gpu_ids.index(0), H)
            whole[v, :, a:b].copy_(strips[v])
    if world > 1:
        for src in range(world):
            for (v, a, b), flat in zip(recv[src], got[src]):
                whole[v, :, a:b].copy_(flat.view(3, b - a, W))
    on_gpu = torch.device(device).type == "cuda"
    host = torch.empty((B, 3, H, W), dtype=torch.uint8, pin_memory=on_gpu)
    host.copy_(whole, non_blocking=on_gpu)
    return list(host.unbind(0))
