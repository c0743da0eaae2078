"""The reference's --zhx_time / --zhx_debug log files, written by the drop-in operators on logging iterations.

The reference hands every rasterizer call a `cuda_args` dict of strings (gaussian_renderer/__init__.py:510-539).  Its
CUDA extension appends, on logging iterations, to files in cuda_args["log_folder"] that analyze_statistic.py parses:
  gpu_time_ws=W_rk=R.log    --zhx_time: per-stage GPU times (parser :747-807, stage keys :1972-1991)
  n_contrib_ws=W_rk=R.log   --zhx_debug: per-tile list length / entries walked / entries blended (parser :843-962)
The parsers are the contract for the formats below.  Which numbers fill the n_contrib fields is documented in DESIGN.md
("Statistics logs"): the extension's source is not public, so the example lines in the parser pin some fields and the
rest are this project's choice.
"""
import os

import numpy as np


class LogRequest:
    """What one operator call has to log: built by request() from cuda_args, None when nothing is logged."""

    __slots__ = ("iteration", "time", "debug", "folder", "world_size", "global_rank", "local_rank")

    def __init__(self, cuda_args, time, debug):
        self.iteration = int(cuda_args["iteration"])
        self.time, self.debug = time, debug
        self.folder = str(cuda_args.get("log_folder", "."))
        self.world_size = str(cuda_args.get("world_size", "1"))
        self.global_rank = str(cuda_args.get("global_rank", "0"))
        self.local_rank = str(cuda_args.get("local_rank", "0"))

    def path(self, kind):
        return os.path.join(self.folder, f"{kind}_ws={self.world_size}_rk={self.global_rank}.log")


def request(cuda_args):
    """A LogRequest when this call logs, else None.  A call logs when mode is "train", int(iteration) % int(log_interval)
    == 1 (get_cuda_args_final has already moved the logging iteration into the batch, :514-520) and zhx_time or
    zhx_debug is "True".  Test mode passes iteration -1 and never logs; a dict without these keys never logs."""
    if not isinstance(cuda_args, dict) or cuda_args.get("mode") != "train":
        return None
    time, debug = cuda_args.get("zhx_time") == "True", cuda_args.get("zhx_debug") == "True"
    if not (time or debug):
        return None
    try:
        if int(cuda_args["iteration"]) % int(cuda_args["log_interval"]) != 1:
            return None
    except (KeyError, TypeError, ValueError, ZeroDivisionError):
        return None
    return LogRequest(cuda_args, time, debug)


def gpu_time_text(iteration, header, times):
    """One call's block of the gpu_time log: a header line `it=N, ...` (the parser reads the number up to the first comma
    and skips repeated headers of one iteration), then `<key>: <ms with 6 decimals> ms` per stage."""
    return f"it={int(iteration)}, {header}\n" + "".join(f"{k}: {float(v):.6f} ms\n" for k, v in times)


def n_contrib_text(iteration, local_rank, world_size, image_height, image_width, compute_locally, ranges, tile_stats):
    """The n_contrib log block of one render forward.  compute_locally (TY*TX) bool, ranges (TY*TX, 2) [start, end),
    tile_stats (TY*TX, 3) int64 as gs_render_forward_ts writes them; tile_x = TX = number of tile columns.
    One line per LOCAL tile in flattened order, then the summary line, which the parser attaches to the tile lines
    before it.  Returns "" when no tile is local: a summary without tile lines would fail the parser's assertion."""
    cl = np.asarray(compute_locally).reshape(-1).astype(bool)
    ranges = np.asarray(ranges).reshape(-1, 2).astype(np.int64)
    ts = np.asarray(tile_stats).reshape(-1, 3).astype(np.int64)
    tx = (int(image_width) + 15) // 16
    it = int(iteration)
    local = np.nonzero(cl)[0]
    if local.size == 0:
        return ""
    lines = []
    for t in local:
        n, walked, blended = (int(v) for v in ts[t])
        contrib = blended / 256.0
        lines.append(f"iteration: {it}, tile: ({t // tx}, {t % tx}), range: ({int(ranges[t, 1])}, {int(ranges[t, 0])}), "
                     f"num_rendered_this_tile: {n}, n_considered_per_pixel: {walked / 256.0:.6f}, "
                     f"n_contrib2loss_per_pixel: {contrib:.6f}, contrib2loss_ratio: {contrib / 256.0:.6f}\n")
    num_tiles = int(local.size)
    num_pixels = int(image_height) * int(image_width)
    R = int(ts[local, 0].sum())
    lines.append(f"iteration: {it}, local_rank: {int(local_rank)}, world_size: {int(world_size)}, num_tiles: {num_tiles}, "
                 f"num_pixels: {num_pixels}, num_rendered: {R}, global_ave_n_rendered_per_pix: {R / num_tiles:.6f}, "
                 f"global_ave_n_considered_per_pix: {int(ts[local, 1].sum()) / num_pixels:.6f}, "
                 f"global_ave_n_contrib2loss_per_pix: {int(ts[local, 2].sum()) / num_pixels:.6f}\n")
    return "".join(lines)


def append(path, text):
    if not text:
        return
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    with open(path, "a") as f:
        f.write(text)
