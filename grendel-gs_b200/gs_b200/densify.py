"""Densification step on top of gs_densify_select / gs_densify_gather: the effect of GaussianModel.densify_and_prune
(/root/reference/scene/gaussian_model.py:1005-1044 -> densify_and_clone :973-1003, densify_and_split :922-971,
densification_postfix :884-920, cat_tensors_to_optimizer :837-881, prune_points :816-835, _prune_optimizer :789-814) on
an optimizer with the reference's six single-tensor groups (optim.NAMES): three launches and one host read-back
instead of ~150 torch kernels and a dozen read-backs.

The optimizer is edited the way the reference edits it (optim.swap_rows): survivors keep their moments, new Gaussians
start at zero and "step" is untouched.  No CPU path.  The algorithm is checked on CPU against the reference's own run
(tests/test_densify_oracle.py) and on the device, decision for decision and bit for bit, against the reference's chain
of torch operations run on the same device (tests/test_densify_gpu.py).
"""
import ctypes as C

import torch

from . import _lib
from .ops import MAX_VIEWS
from .optim import NAMES, group_param, group_params, moments, swap_rows

KIND = {"xyz": 1, "scaling": 2}   # 0 copy, 1 position, 2 log-scale, 3 Adam moment (include/grendel_gs_b200.h)


def _as_rows(t):
    """(P, ...) tensor of 4- or 8-byte elements -> (tensor, number of 4-byte elements per row)."""
    if not t.is_cuda or not t.is_contiguous():
        raise TypeError("densification needs contiguous CUDA tensors (no CPU path)")
    if t.element_size() not in (4, 8):
        raise TypeError(f"unsupported element size {t.element_size()}")
    per_row = (t.numel() // max(t.shape[0], 1)) * (t.element_size() // 4)
    return t, per_row


def densify_and_prune(optimizer, xyz_gradient_accum, denom, max_grad, min_opacity, extent, percent_dense, max_screen_size,
                      send_to_gpui_cnt=None, noise=None):
    """-> dict with the six new parameters under the group names, the reset statistics ("xyz_gradient_accum", "denom",
    "max_radii2D", "sum_visible_count_in_one_batch"), "send_to_gpui_cnt" (if given) and "counts" = (kept, clones,
    children per copy, split-selected, new total).  `noise`: optional (>= 2 S, 3) standard-normal draws for the split
    (default: torch.randn on the device, like the reference's torch.normal)."""
    params = group_params(optimizer)
    P = params["xyz"].shape[0]
    dev = params["xyz"].device
    if P == 0:
        raise ValueError("no Gaussians")
    stream = torch.cuda.current_stream().cuda_stream
    accum = xyz_gradient_accum.reshape(-1).to(torch.float32).contiguous()
    den = denom.reshape(-1).to(torch.float32).contiguous()
    if accum.numel() != P or den.numel() != P:
        raise ValueError("xyz_gradient_accum / denom must have one entry per Gaussian")
    tb = _lib.query("gs_densify_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=dev)
    counts = (C.c_int32 * 6)()
    _lib.call("gs_densify_select", P, accum.data_ptr(), den.data_ptr(), params["scaling"].data_ptr(),
              params["opacity"].data_ptr(), C.c_float(max_grad), C.c_float(min_opacity), C.c_double(extent),
              C.c_double(percent_dense), 1 if max_screen_size else 0, temp.data_ptr(), tb, counts, stream)
    kept, clones, child1, child2, S, new_P = (int(c) for c in counts)
    if noise is None:
        noise = torch.randn((max(2 * S, 1), 3), dtype=torch.float32, device=dev)
    noise = noise.to(device=dev, dtype=torch.float32).contiguous()
    if noise.shape[0] < 2 * S or noise.shape[1] != 3:
        raise ValueError(f"noise must be (>= {2 * S}, 3)")
    # tensor table: parameters, their moments (if the optimizer has state), per-Gaussian bookkeeping
    src, dst, width, kind, outs = [], [], [], [], {}

    def add(name, t, k):
        t, w = _as_rows(t)
        o = torch.empty((new_P,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
        outs[name] = o
        if w == 0:   # _features_rest of a model stored at SH degree 0 (P,0,3): nothing to gather
            return
        src.append(t); dst.append(o); width.append(w); kind.append(k)

    state = {k: moments(optimizer, p) for k, p in params.items()}
    with torch.no_grad():
        for k in NAMES:
            add(k, params[k].detach(), KIND.get(k, 0))
            for j, t in enumerate(state[k] or ()):
                add((k, j), t, 3)
        if send_to_gpui_cnt is not None:
            add("send_to_gpui_cnt", send_to_gpui_cnt, 0)
        n = len(src)
        vp, i32 = C.c_void_p * n, C.c_int32 * n
        _lib.call("gs_densify_gather", P, S, new_P, n, vp(*[t.data_ptr() for t in src]), vp(*[t.data_ptr() for t in dst]),
                  i32(*width), i32(*kind), params["scaling"].data_ptr(), params["rotation"].data_ptr(), noise.data_ptr(),
                  temp.data_ptr(), stream)
    result = swap_rows(optimizer, {k: (outs[k], None if state[k] is None else (outs[k, 0], outs[k, 1])) for k in NAMES})
    result.update(fresh_stats(new_P, dev))          # densification_postfix :909-914
    if send_to_gpui_cnt is not None:
        result["send_to_gpui_cnt"] = outs["send_to_gpui_cnt"]
    result["counts"] = (kept, clones, child1, S, new_P)
    return result


def reset_opacity(optimizer):
    """GaussianModel.reset_opacity with replace_tensor_to_optimizer (scene/gaussian_model.py:555-561, :771-787), in
    place, one launch (gs_reset_opacity): every opacity logit o becomes inverse_sigmoid(min(sigmoid(o), 0.01)) and both
    Adam moments of the "opacity" group become zero, bit for bit as the reference's torch on the device; "step" is kept.
    The reference puts a NEW Parameter without a gradient into the group, so the optimizer step of that iteration skips
    the opacity; here the same parameter is kept and its .grad is set to None, which has that effect.
    -> the opacity parameter."""
    p = group_param(optimizer, "opacity")
    _check(p.data, "opacity", torch.float32, (None, 1))
    if not p.is_cuda:
        raise TypeError("reset_opacity needs a CUDA tensor (no CPU path)")
    m, v = moments(optimizer, p) or (None, None)
    if m is not None:
        for name, t in (("the opacity's first moment", m), ("the opacity's second moment", v)):
            _check(t, name, torch.float32, tuple(p.shape))
            if t.device != p.device:
                raise ValueError("the opacity moments must be on the parameter's device")
    with torch.cuda.device(p.device):
        _lib.call("gs_reset_opacity", p.shape[0], p.data.data_ptr(), m.data_ptr() if m is not None else None,
                  v.data_ptr() if v is not None else None, torch.cuda.current_stream(p.device).cuda_stream)
    p.grad = None
    return p


def _check(t, name, dtype, shape):
    """Refuse anything but a contiguous tensor of `dtype` and `shape` (None in `shape`: any size)."""
    if t is None:
        raise TypeError(f"{name} is None (no gradient was retained for this camera?)")
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(t).__name__}")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() != len(shape) or any(want is not None and got != want for got, want in zip(t.shape, shape)):
        raise ValueError(f"{name} must be {tuple('P' if d is None else d for d in shape)}, got {tuple(t.shape)}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def add_densification_stats(xyz_gradient_accum, denom, max_radii2D, means2D_grads, radii):
    """The densification statistics of one step, updated in place on the current stream by one launch with no host
    synchronisation (gs_densify_stats).  The reference's loop (densification.py:15-24 with
    GaussianModel.add_densification_stats, scene/gaussian_model.py:1046-1052), bit for bit: for each camera k in batch
    order, where radii[k] > 0,
        max_radii2D = torch.max(max_radii2D, radii[k]);  xyz_gradient_accum += norm(means2D_grads[k]);  denom += 1.
    xyz_gradient_accum, denom: (P, 1) float32; max_radii2D: (P,) float32 (the reference's layout, which
    densify_and_prune's reset statistics have).  means2D_grads: (B, P, 2) float32 or a list of B (P, 2) (each camera's
    means2D.grad); radii: (B, P) int32 or a list of B (P,).  1 <= B <= 64.  Nothing is made contiguous or converted here:
    other inputs are refused (ValueError / TypeError)."""
    if means2D_grads is None or radii is None:
        raise TypeError("means2D_grads and radii are required (no gradient was retained?)")
    grads =list(means2D_grads.unbind(0)) if isinstance(means2D_grads, torch.Tensor) else list(means2D_grads)
    rads = list(radii.unbind(0)) if isinstance(radii, torch.Tensor) else list(radii)
    B = len(grads)
    if not 1 <= B <= MAX_VIEWS:
        raise ValueError(f"between 1 and {MAX_VIEWS} views, got {B}")
    if len(rads) != B:
        raise ValueError(f"{B} gradient views but {len(rads)} radii views")
    P = xyz_gradient_accum.shape[0] if isinstance(xyz_gradient_accum, torch.Tensor) else None
    for name, t, shape in (("xyz_gradient_accum", xyz_gradient_accum, (P, 1)), ("denom", denom, (P, 1)),
                           ("max_radii2D", max_radii2D, (P,))):
        _check(t, name, torch.float32, shape)
    for k in range(B):
        _check(grads[k], f"means2D_grads[{k}]", torch.float32, (P, 2))
        _check(rads[k], f"radii[{k}]", torch.int32, (P,))
    dev = xyz_gradient_accum.device
    for t in [xyz_gradient_accum, denom, max_radii2D] + grads + rads:
        if not t.is_cuda:
            raise TypeError("add_densification_stats needs CUDA tensors (no CPU path)")
        if t.device != dev:
            raise ValueError("all tensors must be on one device")
    vp = C.c_void_p * B
    with torch.cuda.device(dev):
        _lib.call("gs_densify_stats", B, P, vp(*[t.data_ptr() for t in grads]), vp(*[t.data_ptr() for t in rads]),
                  xyz_gradient_accum.data_ptr(), denom.data_ptr(), max_radii2D.data_ptr(),
                  torch.cuda.current_stream(dev).cuda_stream)


def append_gaussians(optimizer, new_tensors):
    """cat_tensors_to_optimizer (/root/reference/scene/gaussian_model.py:837-881): rows appended to every parameter, their
    Adam moments start at zero, "step" is kept.  new_tensors: {group name: (n, ...) tensor}.  -> {name: new Parameter}."""
    new = {}
    for k in NAMES:
        old = group_param(optimizer, k)
        ext = new_tensors[k].to(device=old.device, dtype=old.dtype)
        m = moments(optimizer, old)
        new[k] = (torch.cat((old.detach(), ext), dim=0),
                  None if m is None else tuple(torch.cat((t, torch.zeros_like(ext)), dim=0) for t in m))
    return swap_rows(optimizer, new)


def fresh_stats(n, device):
    """The per-Gaussian densification statistics of n Gaussians right after the model changed (densification_postfix,
    scene/gaussian_model.py:909-914): all zero."""
    return {"xyz_gradient_accum": torch.zeros((n, 1), device=device), "denom": torch.zeros((n, 1), device=device),
            "max_radii2D": torch.zeros((n,), device=device),
            "sum_visible_count_in_one_batch": torch.zeros((n,), device=device)}
