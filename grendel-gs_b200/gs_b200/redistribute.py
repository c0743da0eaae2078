"""Gaussian redistribution after densification (/root/reference/scene/gaussian_model.py:1247-1329,
redistribute_gaussians; all2all_gaussian_state :1073-1098): when the shards have grown unevenly
(min * threshold < max, :1247-1259) every Gaussian draws a destination rank (random_redistribute: uniform, :1243-1245)
and moves there together with its Adam moments.

The reference moves the six parameters and their twelve moment tensors with EIGHTEEN list all_to_alls (its fused
variant, implementation_2 :1200-1234, is disabled because it hung).  Here every Gaussian travels as ONE fused row --
59 parameter floats + 59 exp_avg + 59 exp_avg_sq -- in ONE all_to_all_single: a stable sort by destination gives the
send order (per destination: index order, exactly `state[destination == j]`), and the receive order is the
concatenation over source ranks (`torch.cat(state_from_gpuj)`), so the result is row for row what the reference builds.
Host-side torch ops (densification is host-side by decree, SURVEY.md 2 #7); the collective is the one exchange.py uses.
"""
import numpy as np
import torch
import torch.distributed as dist

from .densify import fresh_stats
from .exchange import all_to_all_single
from .optim import NAMES, group_params, moments, swap_rows


def fused_rows(tensors, order=None):
    """(P, ...) tensors -> (one (P, sum of widths) tensor whose row i is row i of every tensor, flattened and side by side,
    widths).  order: optional (P,) row indices, applied to the fused rows.  The one packing of a Gaussian's state into a
    row, for the redistribution's all-to-all and for model_io's PLY rows."""
    P = tensors[0].shape[0]
    widths = [int(np.prod(t.shape[1:])) if t.dim() > 1 else 1 for t in tensors]
    rows = torch.cat([t.reshape(P, w) for t, w in zip(tensors, widths)], dim=1)
    if order is not None:
        rows = rows.index_select(0, order)
    return rows.contiguous(), widths


def need_redistribute(n_local, group=None, threshold=7.0, first_after_densify=False):
    """gaussian_model.py:1247-1259: after the first densification, or when min * threshold < max over the ranks."""
    W = dist.get_world_size(group)
    if W == 1:
        return False, [int(n_local)]
    mine = torch.tensor([int(n_local)], dtype=torch.int64)
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    allc = torch.empty((W,), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(allc, mine.to(dev), group=group)
    counts = [int(v) for v in allc.cpu().tolist()]
    return bool(first_after_densify or min(counts) * threshold < max(counts)), counts


def redistribute(optimizer, destination=None, group=None, generator=None):
    """Moves every Gaussian (six parameters + Adam moments) to destination[i] with one collective.
    optimizer: the reference's six single-tensor groups.  destination: (P,) int64 ranks; default uniform random
    (get_destination_1).  -> dict of the six new parameters + "counts" (i2j_send_size, W x W) + the reset per-Gaussian
    statistics of :1300-1318."""
    W, me = dist.get_world_size(group), dist.get_rank(group)
    params = group_params(optimizer)
    P = params["xyz"].shape[0]
    dev = params["xyz"].device
    if destination is None:
        destination = torch.randint(0, W, (P,), device=dev, generator=generator)
    destination = destination.to(device=dev, dtype=torch.int64)
    if destination.shape != (P,) or (P and (int(destination.min()) < 0 or int(destination.max()) >= W)):
        raise ValueError("destination must hold one rank in [0, world size) per Gaussian")
    # counts: one all-gather + one read-back (the reference: bincount + all_gather_into_tensor + .cpu(), :1281-1292)
    local = torch.bincount(destination, minlength=W).to(torch.int32)
    i2j = torch.empty((W * W,), dtype=torch.int32, device=dev)
    dist.all_gather_into_tensor(i2j, local, group=group)
    i2j = i2j.reshape(W, W).cpu().numpy()
    send_splits, recv_splits = i2j[me].tolist(), i2j[:, me].tolist()
    # fused rows in send order
    state = {k: moments(optimizer, p) for k, p in params.items()}
    with torch.no_grad():
        tensors = [t for k in NAMES for t in (params[k].detach(),) + (state[k] or ())]
        order = torch.sort(destination, stable=True).indices
        send, widths = fused_rows(tensors, order)
        n_new = int(sum(recv_splits))
        recv = torch.empty((n_new, send.shape[1]), dtype=send.dtype, device=dev)
        all_to_all_single(recv, send, recv_splits, send_splits, group)
        del send
        parts = iter(torch.split(recv, widths, dim=1))
    new = {}
    for k in NAMES:
        shape = (n_new,) + tuple(params[k].shape[1:])
        take = lambda: next(parts).reshape(shape).contiguous()   # the next tensor's columns of the received rows
        new[k] = (take(), None if state[k] is None else (take(), take()))
    result = swap_rows(optimizer, new)
    result.update(fresh_stats(n_new, dev))
    result["send_to_gpui_cnt"] = torch.zeros((n_new, W), dtype=torch.int32, device=dev)
    result["counts"] = i2j.tolist()
    return result
