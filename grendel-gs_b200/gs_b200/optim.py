"""Fused Adam for the Gaussian parameters: the optimizer step of /root/reference/train_internal.py:316-329
(`param.grad /= args.bsz` for all six parameters, then `gaussians.optimizer.step()`), ONE kernel launch per step.

Drop-in for the object the reference builds at scene/gaussian_model.py:257-292 (`torch.optim.Adam(l, lr=0.0,
eps=1e-15)`, six single-tensor groups with their own "lr" / "name"; "betas" / "eps" edited per group in sqrt lr-scale
mode, :295-312): same constructor, same `param_groups`, and the SAME state layout (`state[p]["step"]`, `["exp_avg"]`,
`["exp_avg_sq"]`) -- the reference's densification rewrites that state directly (`_prune_optimizer`,
`cat_tensors_to_optimizer`, `replace_tensor_to_optimizer`, gaussian_model.py:771-881) and checkpoints round-trip through
`state_dict()` / `load_state_dict()` of either class.  There is no CPU path: parameters must be CUDA fp32 tensors.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib

MAX_TENSORS = 8   # GS_ADAM_MAX_TENSORS

# the optimizer's groups in the reference's order (scene/gaussian_model.py:257-292): group name -> GaussianParams attribute
GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
          "scaling": "_scaling", "rotation": "_rotation"}
NAMES = tuple(GROUPS)


def group_param(optimizer, name):
    """The parameter of the optimizer's single-tensor group `name`; ValueError unless there is exactly one such group."""
    found = [g["params"] for g in optimizer.param_groups if g.get("name") == name]
    if len(found) != 1 or len(found[0]) != 1:
        raise ValueError(f"the optimizer needs the reference's single-tensor {name!r} group")
    return found[0][0]


def group_params(optimizer, ordered=False):
    """{name: parameter} of an optimizer with the reference's six single-tensor groups (NAMES) and no other; ValueError
    otherwise.  ordered: also in NAMES' order, as a state_dict numbers the groups by position."""
    got = [g.get("name") for g in optimizer.param_groups]
    if (got != list(NAMES)) if ordered else (len(got) != len(NAMES) or set(got) != set(NAMES)):
        raise ValueError(f"the optimizer must have the reference's six single-tensor groups {NAMES}"
                         f"{' in this order' if ordered else ''}, got {got}")
    return {k: group_param(optimizer, k) for k in NAMES}


def moments(optimizer, p):
    """(exp_avg, exp_avg_sq) of parameter p, or None before its first step."""
    st = optimizer.state.get(p)
    return (st["exp_avg"], st["exp_avg_sq"]) if st is not None and "exp_avg" in st else None


def swap_rows(optimizer, new):
    """Put new rows into the optimizer as the reference's densification does (_prune_optimizer,
    cat_tensors_to_optimizer, scene/gaussian_model.py:789-881).  new: {group name: (data, (exp_avg, exp_avg_sq) or None)}.
    Each group gets a NEW nn.Parameter over data; the old parameter's state entry moves to it with the moments replaced
    when given and every other key ("step") untouched.  -> {group name: new Parameter}."""
    groups = {g.get("name"): g for g in optimizer.param_groups}
    out = {}
    for name, (data, m) in new.items():
        p = out[name] = nn.Parameter(data)
        st = optimizer.state.pop(groups[name]["params"][0], None)
        if st is not None:
            if m is not None:
                st["exp_avg"], st["exp_avg_sq"] = m
            optimizer.state[p] = st
        groups[name]["params"][0] = p
    return out


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, grad_scale=1.0):
        if lr < 0.0 or eps < 0.0 or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("invalid Adam hyper-parameters")
        # the option keys torch.optim.Adam keeps in its groups, at the values this kernel implements: a state_dict
        # written here loads into torch.optim.Adam (load_state_dict REPLACES the groups by the saved ones) and back
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=0.0, amsgrad=False, maximize=False,
                                      foreach=None, capturable=False, differentiable=False, fused=None))
        self.grad_scale = float(grad_scale)

    @torch.no_grad()
    def step(self, closure=None, grad_scale=None):
        """grad_scale (default: the constructor's) multiplies every gradient inside the kernel -- pass 1/bsz instead of
        running `param.grad /= args.bsz` over the six tensors first."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        gs = self.grad_scale if grad_scale is None else float(grad_scale)
        todo = []
        for group in self.param_groups:
            b1, b2 = group["betas"]
            if group.get("weight_decay", 0.0) != 0.0 or group.get("amsgrad", False) or group.get("maximize", False):
                raise NotImplementedError("FusedAdam implements plain Adam only (weight_decay=0, amsgrad=False, maximize=False)"
                                          " -- what the reference configures, scene/gaussian_model.py:292")
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise TypeError("FusedAdam needs contiguous CUDA float32 parameters (no CPU path)")
                if p.grad.is_sparse:
                    raise RuntimeError("FusedAdam does not support sparse gradients")
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                st = self.state[p]
                if len(st) == 0:   # same lazy initialisation as torch.optim.Adam
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1
                m, v = st["exp_avg"], st["exp_avg_sq"]
                if m.shape != p.shape or v.shape != p.shape or not m.is_contiguous() or not v.is_contiguous():
                    raise RuntimeError("optimizer state does not match its parameter (shape / contiguity)")
                todo.append((p, g, m, v, float(group["lr"]), float(b1), float(b2), float(group["eps"]), int(st["step"])))
        stream = torch.cuda.current_stream().cuda_stream if todo else 0
        for i in range(0, len(todo), MAX_TENSORS):
            chunk = todo[i:i + MAX_TENSORS]
            n = len(chunk)
            vp, f64, i64 = C.c_void_p * n, C.c_double * n, C.c_int64 * n
            _lib.call("gs_adam_step", n, i64(*[c[0].numel() for c in chunk]), vp(*[c[0].data_ptr() for c in chunk]),
                      vp(*[c[1].data_ptr() for c in chunk]), vp(*[c[2].data_ptr() for c in chunk]),
                      vp(*[c[3].data_ptr() for c in chunk]), f64(*[c[4] for c in chunk]), f64(*[c[5] for c in chunk]),
                      f64(*[c[6] for c in chunk]), f64(*[c[7] for c in chunk]), i64(*[c[8] for c in chunk]),
                      C.c_float(gs), stream)
        return loss
