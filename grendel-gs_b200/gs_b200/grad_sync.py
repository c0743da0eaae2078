"""Gradient synchronisation for REPLICATED Gaussians (data parallelism without Gaussian sharding).

Restates /root/reference/scene/gaussian_model.py:1332-1439:
  sync_gradients_densely  (:1394-1407)  six all-reduces, one per parameter
  sync_gradients_sparsely (:1350-1391)  rows with non-zero _xyz.grad on any rank: mask all-reduce, then per
                                        parameter compact -> all-reduce -> scatter back
and provides the mode the reference leaves NotImplemented (:1438-1439, "fused_sparse"): the six gradients of
a touched Gaussian travel as ONE row of 11 + 3 K floats (K stored SH coefficients: 59 floats at degree 3), so a
step costs one byte-mask all-reduce(MAX) and ONE fp32 all-reduce(SUM) over NVLink instead of 1 + 6 collectives and
12 gather/scatter kernels.

(The live trainer shards Gaussians, so no gradient all-reduce is needed there -- SURVEY.md section 8e; this is row
L2 of section 8a, named by BASELINE.json's north_star.)
"""
import ctypes as C

import torch
import torch.distributed as dist

from . import _lib, ops

REST_FLOATS = (0, 9, 24, 45)  # features_rest floats per Gaussian at max_sh_degree 0..3 (scene/gaussian_model.py:150-156)


def _grads(params):
    g = []
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
        g.append(p.grad.contiguous())
    return g


def sync_gradients_densely(params, group=None):
    """One all-reduce(SUM) per parameter (gaussian_model.py:1394-1407)."""
    for g in _grads(params):
        dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group)


def sync_gradients_fused_sparse(params, group=None):
    """params: the six GaussianModel tensors in order (_xyz, _features_dc, _features_rest, _scaling, _rotation,
    _opacity), replicated on every rank, with .grad set.  On return every rank holds the summed gradients.
    Returns the number of Gaussians touched on any rank."""
    grads = _grads(params)
    P = grads[0].shape[0]
    widths = [g[0].numel() if P else 0 for g in grads]
    rest = widths[2]
    if P and (widths[:2] + widths[3:] != [3, 3, 3, 4, 1] or rest not in REST_FLOATS):
        raise ValueError(f"unexpected parameter layout {widths}; expected GaussianModel's [3,3,R,3,4,1] with R = 3 (K-1) "
                         f"in {REST_FLOATS}")
    dev = grads[0].device
    s = ops._stream()
    mask = torch.empty((max(P, 1),), dtype=torch.uint8, device=dev)
    _lib.call("gs_sparse_grad_mask", P, grads[0].data_ptr(), mask.data_ptr(), s)
    dist.all_reduce(mask, op=dist.ReduceOp.MAX, group=group)
    pos = torch.empty((max(P, 1),), dtype=torch.int32, device=dev)
    colstart = torch.empty((2,), dtype=torch.int32, device=dev)
    tb = _lib.query("gs_route_scan_temp_bytes", P, 1)
    temp = torch.empty((tb,), dtype=torch.uint8, device=dev)
    _lib.call("gs_route_scan", P, 1, mask.data_ptr(), pos.data_ptr(), colstart.data_ptr(), temp.data_ptr(), tb, s)
    n = int(colstart[1].item())  # host sync: sizes the one compacted buffer
    if n == 0:
        return 0
    rows = torch.empty((n, sum(widths)), dtype=torch.float32, device=dev)
    ptrs = (C.c_void_p * 6)(*[g.data_ptr() for g in grads])
    _lib.call("gs_sparse_grad_pack_rows", P, rest, mask.data_ptr(), pos.data_ptr(), ptrs, rows.data_ptr(), s)
    dist.all_reduce(rows, op=dist.ReduceOp.SUM, group=group)
    _lib.call("gs_sparse_grad_unpack_rows", P, rest, mask.data_ptr(), pos.data_ptr(), rows.data_ptr(), ptrs, s)
    for p, g in zip(params, grads):
        if p.grad.data_ptr() != g.data_ptr():
            p.grad.copy_(g)
    return n
