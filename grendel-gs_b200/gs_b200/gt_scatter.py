"""The ground truth of each local strip of a batch (load_camera_from_cpu_to_all_gpu,
gaussian_renderer/loss_distribution.py:2395-2533): local_gt chooses where every strip's rows come from,
for the training step and for evaluation alike.

With --distributed_dataset_storage only ONE rank of the node holds the dataset (scatter_gt_strips): the first rank of
the node copies the uint8 rows the node needs from its (pinned) host memory to its GPU and sends every other rank
exactly the rows of its strips with one batch of point-to-point operations; the other ranks post the matching receives.
Without it every rank reads its own strips from its own copy of the images.

Strip rows follow get_coverage_y_min/max (loss_distribution.py:2321-2330): tile rows [l, r) -> pixel rows
[16 l, min(16 r, H)).
"""
import torch
import torch.distributed as dist

BLOCK_Y = 16


def coverage(row_l, row_r, image_height):
    return row_l * BLOCK_Y, min(row_r * BLOCK_Y, image_height)


def strip_tasks(strategies, world):
    """The gpuid2tasks of scatter_gt_strips for a batch's strip division: tasks[gpu] = [(batch position, tile row l,
    tile row r), ...] in position order, as division.start_strategy lists them."""
    tasks = [[] for _ in range(world)]
    for k, st in enumerate(strategies):
        for i, gpu in enumerate(st.gpu_ids):
            tasks[gpu].append((k, st.division_pos[i], st.division_pos[i + 1]))
    return tasks


def local_gt(gts, views, strategies, image_height, image_width, device, rank, world, group=None, *, scatter=False,
             cache=None, stream=None):
    """The ground truth of this rank's strip of every batch position.  gts: the set's uint8 (3,H,W) images by camera
    index (with scatter only rank 0's are read, and gts may be None elsewhere); views: the camera of each position of
    `strategies`, the batch's (or a span's) strip division.
    -> (pairs, host -> device bytes copied here, ready).  pairs[k] is None where position k has no local rows, else
    (tensor, row0): a (3, rows, W) uint8 tensor on `device` holding image rows [row0, row0 + rows).  The source:
      * scatter (a collective: every rank calls it, with local rows or not): the strip from rank 0, row0 = y0;
      * an image already on the device: read in place, row0 = 0;
      * a host image: its strip rows, row0 = y0.  A pinned image is copied by three channel copies; a pageable one,
        when `cache` is given, through a pinned copy of the strip kept in cache[(camera, y0, y1)].  Held-out images get
        no cache: their indices are not the training cameras'.
    stream: the copies go to this CUDA stream, and ready is the event they recorded (None when nothing was copied there);
    the consumer's stream waits on it.  Without a stream the copies go to the current stream."""
    if scatter:
        strips, h2d = scatter_gt_strips([gts[v] for v in views] if rank == 0 else image_width,
                                        strip_tasks(strategies, world), image_height, device, rank, world, group)
        return [(strips[k], st.local_pixel_rows(image_height)[0]) if k in strips else None
                for k, st in enumerate(strategies)], h2d, None
    pairs, h2d = [], 0
    with torch.cuda.stream(stream):
        for v, st in zip(views, strategies):
            rows = st.local_pixel_rows(image_height)
            if rows is None:
                pairs.append(None)
                continue
            g, (y0, y1) = gts[v], rows
            if g.is_cuda:
                pairs.append((g, 0))
                continue
            # the rows of one channel are contiguous in the image, so a strip is three asynchronous copies straight out
            # of a pinned image: no staging copy, and nothing to re-pin when the load balancer moves the strip boundaries
            # (a pinned staging strip per division cost several ms of cudaHostAlloc every time the strips of a 4K view
            # moved)
            if cache is not None and not g.is_pinned():
                key = (v, y0, y1)
                if key not in cache:
                    cache[key] = g[:, y0:y1, :].contiguous().pin_memory()
                d = cache[key].to(device, non_blocking=True)
            else:
                d = torch.empty((3, y1 - y0, image_width), dtype=torch.uint8, device=device)
                for c in range(3):
                    d[c].copy_(g[c, y0:y1, :], non_blocking=True)
            h2d += d.numel()
            pairs.append((d, y0))
        ready = None
        if stream is not None and h2d:
            ready = torch.cuda.Event()
            ready.record(stream)
    return pairs, h2d, ready


def scatter_gt_strips(gts_host, gpuid2tasks, image_height, device, rank, world, group=None, src=0):
    """gts_host: on rank `src` the list of (3,H,W) uint8 host tensors of the batch (ignored elsewhere);
    gpuid2tasks[gpu] = [(camera index, tile row l, tile row r), ...] (strip_tasks).
    -> ({camera index: (3, rows, W) uint8 tensor on `device`} for this rank's tasks, bytes copied host -> device here)."""
    mine, ops, h2d = {}, [], 0
    if rank == src:
        on_dev = {}
        for tasks in gpuid2tasks:
            for cam, l, r in tasks:
                if cam not in on_dev:  # the rows any rank of the node needs of this camera, copied once
                    lo = min(coverage(t[1], t[2], image_height)[0] for ts in gpuid2tasks for t in ts if t[0] == cam)
                    hi = max(coverage(t[1], t[2], image_height)[1] for ts in gpuid2tasks for t in ts if t[0] == cam)
                    g = gts_host[cam][:, lo:hi, :]
                    h2d += g.numel()
                    on_dev[cam] = (lo, g.to(device, non_blocking=True))
        keep = []   # sent tensors must outlive the requests
        for dst, tasks in enumerate(gpuid2tasks):
            for cam, l, r in tasks:
                y0, y1 = coverage(l, r, image_height)
                lo, t = on_dev[cam]
                strip = t[:, y0 - lo:y1 - lo, :].contiguous()
                if dst == rank:
                    mine[cam] = strip
                else:
                    keep.append(strip)
                    ops.append(dist.P2POp(dist.isend, strip, dst, group))
    else:
        width = None
        for cam, l, r in gpuid2tasks[rank]:
            y0, y1 = coverage(l, r, image_height)
            if width is None:
                width = _width(gts_host)
            buf = torch.empty((3, y1 - y0, width), dtype=torch.uint8, device=device)
            mine[cam] = buf
            ops.append(dist.P2POp(dist.irecv, buf, src, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return mine, h2d


def _width(hint):
    """Image width on a receiving rank: it knows the camera geometry, not the pixels."""
    if isinstance(hint, int):
        return hint
    return int(hint[0].shape[2])
