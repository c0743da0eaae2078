"""Pixel-wise workload division: tile-ROW strips of B images over W ranks.

Host-side restatement of /root/reference/gaussian_renderer/workload_division.py:
  division_pos_heuristic   :75-94    equal-cost split of a per-row cost vector (cumsum + searchsorted)
  start_strategy           :852-941  concatenate the B cameras' rows, split into W chunks, snap
                                     boundaries that fall within `border_divpos_coeff` rows of an image edge
  DivisionStrategy         :684-803  per-camera (gpu_ids, division_pos) + compute_locally mask
  StrategyHistory          :806-849, 944-998  per-camera running cost heuristic fed by measured times
Pure Python / CPU torch: every rank computes the same answer from the same inputs, no collective.
"""

import torch


def division_pos_heuristic(heuristic, world_size, right=True):
    """Split rows into world_size contiguous chunks of equal summed cost.
    heuristic: sequence of per-row costs.  Returns world_size+1 ascending row boundaries."""
    h = torch.as_tensor(heuristic, dtype=torch.float32).reshape(-1).cpu()
    n = h.numel()
    prefix = torch.cumsum(h, dim=0)
    per = prefix[-1] / world_size
    thr = torch.arange(1, world_size, dtype=torch.float32) * per
    idx = torch.searchsorted(prefix, thr, right=right).tolist()
    return [0] + [int(i) for i in idx] + [n]


class DivisionStrategy:
    """Which ranks render which tile rows of ONE camera."""

    def __init__(self, camera_uid, gpu_ids, division_pos, tile_y, global_rank):
        ws = len(gpu_ids)
        if ws <= 0 or len(division_pos) != ws + 1:
            raise ValueError("division_pos must have len(gpu_ids)+1 entries")
        if division_pos[0] != 0 or division_pos[-1] != tile_y:
            raise ValueError("division_pos must span [0, TILE_Y]")
        if any(b <= a for a, b in zip(division_pos, division_pos[1:])):
            raise ValueError("division_pos must be strictly ascending")
        self.camera_uid = camera_uid
        self.world_size = ws
        self.gpu_ids = list(gpu_ids)
        self.division_pos = [int(p) for p in division_pos]
        self.tile_y = tile_y
        self.rank = self.gpu_ids.index(global_rank) if global_rank in self.gpu_ids else -1

    def local_rows(self):
        """[row_l, row_r) tile rows owned by this rank, or None."""
        if self.rank < 0:
            return None
        return self.division_pos[self.rank], self.division_pos[self.rank + 1]

    def local_pixel_rows(self, image_height, block_y=16):
        """Pixel rows [y0, y1) of this rank's strip (loss_distribution.py:2321-2330)."""
        r = self.local_rows()
        if r is None:
            return None
        return r[0] * block_y, min(r[1] * block_y, image_height)

    def strategy_tensor(self, tile_x, device):
        """(world_size+1) int32 flattened tile-id boundaries for get_local2j_ids_bool."""
        return torch.tensor([p * tile_x for p in self.division_pos], dtype=torch.int32, device=device)

    def get_compute_locally(self, tile_x, device):
        r = self.local_rows()
        if r is None:
            return None
        m = torch.zeros((self.tile_y, tile_x), dtype=torch.bool, device=device)
        m[r[0]:r[1]] = True
        return m


class StrategyHistory:
    """Per-camera row-cost heuristic, initialised uniform and updated from measured times."""

    def __init__(self, camera_uids, tile_y, world_size):
        self.tile_y, self.world_size = tile_y, world_size
        self.accum_heuristic = {uid: torch.ones((tile_y,), dtype=torch.float32) for uid in camera_uids}
        self.history = []

    def update(self, strategies, gpu_camera_running_time, heuristic_decay=0.0):
        """gpu_camera_running_time[gpu][camera] in ms (workload_division.py:980-998): every row of a rank's
        strip is charged that rank's time divided by the strip height."""
        for cam_idx, s in enumerate(strategies):
            new = torch.zeros((self.tile_y,), dtype=torch.float32)
            for local_id, gpu in enumerate(s.gpu_ids):
                lo, hi = s.division_pos[local_id], s.division_pos[local_id + 1]
                new[lo:hi] = float(gpu_camera_running_time[gpu][cam_idx]) / (hi - lo)
            old = self.accum_heuristic[s.camera_uid]
            self.accum_heuristic[s.camera_uid] = new if heuristic_decay == 0 else old * heuristic_decay + new * (1 - heuristic_decay)
        self.history.append([[s.camera_uid, s.gpu_ids, s.division_pos] for s in strategies])


def running_time_of(stats_collector):
    """The cost the reference charges a (rank, camera) pair: forward + backward render time + 2 x loss time
    (workload_division.py:953-957); milliseconds."""
    return (float(stats_collector["forward_render_time"]) + float(stats_collector["backward_render_time"]) +
            2.0 * float(stats_collector.get("forward_loss_time", 0.0)))


def heuristics_update_enabled(iteration, world_size, bsz, image_height, image_width, adjust_strategy_warmup_iterations=-1,
                              no_heuristics_update=False):
    """finish_strategy_final's gate (workload_division.py:967-978): the row costs are only re-estimated after the warm-up,
    on more than one rank, and NOT when every rank can be handed whole images of at most 1080p (bsz >= world size) or the
    images are small (<= 600 x 1000) -- there the uniform split stays."""
    if iteration <= adjust_strategy_warmup_iterations or world_size == 1 or no_heuristics_update:
        return False
    if bsz >= world_size and (image_height <= 1080 or image_width <= 1920):
        return False
    if image_height <= 600 or image_width <= 1000:
        return False
    return True


def finish_strategy(history, strategies, gpu_camera_running_time, iteration, world_size, image_height, image_width,
                    heuristic_decay=0.0, adjust_strategy_warmup_iterations=-1, no_heuristics_update=False):
    """finish_strategy_final (workload_division.py:944-998) after the times have been all-gathered:
    gpu_camera_running_time[gpu][camera] in ms (-1 where the rank did not render the camera).  Returns True if the
    heuristic was updated (the next start_strategy then moves the strip boundaries)."""
    if not heuristics_update_enabled(iteration, world_size, len(strategies), image_height, image_width,
                                     adjust_strategy_warmup_iterations, no_heuristics_update):
        return False
    history.update(strategies, gpu_camera_running_time, heuristic_decay)
    return True


def start_strategy_whole_views(camera_uids, tile_y, world_size, global_rank):
    """The local-sampling division (workload_division.py:858-877): with k = B / world_size views per rank, batch position
    p is rendered whole -- tile rows [0, tile_y) -- by rank p // k.  It depends on positions only: camera_uids merely
    label the strategies (None where a rank does not know the camera), and no cost heuristic is read or updated.
    -> (strategies per camera, gpuid2tasks) as start_strategy."""
    B = len(camera_uids)
    if B % world_size:
        raise ValueError(f"local_sampling needs bsz divisible by world size (bsz {B}, world size {world_size})")
    per = B // world_size
    gpuid2tasks = [[] for _ in range(world_size)]
    strategies = []
    for idx, uid in enumerate(camera_uids):
        gpu = idx // per
        gpuid2tasks[gpu].append((idx, 0, tile_y))
        strategies.append(DivisionStrategy(uid, [gpu], [0, tile_y], tile_y, global_rank))
    return strategies, gpuid2tasks


def start_strategy(camera_uids, history, world_size, global_rank, border_divpos_coeff=1.0, local_sampling=False):
    """-> (strategies per camera, gpuid2tasks[gpu] = [(camera index, row_l, row_r), ...])."""
    tile_y = history.tile_y
    B = len(camera_uids)
    if local_sampling:
        return start_strategy_whole_views(camera_uids, tile_y, world_size, global_rank)
    gpuid2tasks = [[] for _ in range(world_size)]
    strategies = []
    cat = torch.cat([history.accum_heuristic[uid] for uid in camera_uids])
    pos = division_pos_heuristic(cat, world_size, right=True)
    for i in range(1, len(pos) - 1):  # snap to an image edge when closer than border_divpos_coeff rows
        rem = pos[i] % tile_y
        if rem + border_divpos_coeff >= tile_y:
            pos[i] = pos[i] // tile_y * tile_y + tile_y
        elif rem - border_divpos_coeff <= 0:
            pos[i] = pos[i] // tile_y * tile_y
    for i in range(len(pos) - 1):
        if not pos[i] + border_divpos_coeff < pos[i + 1]:
            raise ValueError(f"strip {i} is too thin: {pos}")
    for idx, uid in enumerate(camera_uids):
        off = idx * tile_y
        gpus, bounds = [], [0]
        for gpu in range(world_size):
            lo, hi = pos[gpu], pos[gpu + 1]
            if hi <= off or off + tile_y <= lo:
                continue
            l, r = max(lo, off) - off, min(hi, off + tile_y) - off
            gpus.append(gpu)
            bounds.append(r)
            gpuid2tasks[gpu].append((idx, l, r))
        strategies.append(DivisionStrategy(uid, gpus, bounds, tile_y, global_rank))
    return strategies, gpuid2tasks
