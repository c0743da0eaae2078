"""The reference's densification step restated in torch, operation for operation, on whatever device its inputs live on.

GaussianModel.densify_and_prune runs densify_and_clone, densification_postfix, densify_and_split (draws, children,
postfix, prune of the split originals) and the final opacity / world-size prune as a chain of torch operations on
the model's tensors (oracle/densify_oracle.py restates the same chain in numpy).  This module runs that chain with the
same operations -- boolean indexing, `cat`, `repeat`, `exp` / `log` / `sigmoid`, `bmm`, thresholds given as Python
doubles and compared with fp32 tensors, the split's scale divided by the Python scalar 0.8 N -- so on a CUDA device
it takes every decision and rounds every child exactly as the reference does when it trains there.  The normal draws
are an input (`noise`, (>= 2 S, 3)): `torch.normal(mean=0, std)` becomes `0 + std * noise`.

State: a dict of tensors, the six raw parameters under the group names, optional Adam moments under
"<name>.exp_avg" / "<name>.exp_avg_sq" (a group without them has no optimizer state, which the reference's
_prune_optimizer / cat_tensors_to_optimizer skip), optional per-Gaussian "send_to_gpui_cnt" and "row" (any per-Gaussian
int64 tensor carried like send_to_gpui_cnt: an arange gives every output row its source row).
"""
import numpy as np
import torch

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
CARRIED = ("send_to_gpui_cnt", "row")


def build_rotation(r):
    """(n, 4) raw quaternions (w, x, y, z) -> (n, 3, 3) rotation matrices of the normalised quaternions."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - w * z)
    R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y)
    R[:, 2, 1] = 2 * (y * z + w * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _postfix(st, new):
    """densification_postfix / cat_tensors_to_optimizer: parameters grow by `new`, moments (where present) by zeros."""
    for k in NAMES:
        st[k] = torch.cat((st[k], new[k]), dim=0)
        for m in (".exp_avg", ".exp_avg_sq"):
            if k + m in st:
                st[k + m] = torch.cat((st[k + m], torch.zeros_like(new[k])), dim=0)
    for k in CARRIED:
        if k in st:
            st[k] = torch.cat((st[k], new[k]), dim=0)


def _prune(st, mask):
    """prune_points / _prune_optimizer: keep the rows where mask is False."""
    valid = ~mask
    for k in list(st):
        st[k] = st[k][valid]


def densify_and_prune(state, noise, max_grad, min_opacity, extent, percent_dense, max_screen_size, N=2):
    """-> (new state, (clones, S = split-selected, pruned by the final prune, split mask over the input rows)).  `state`
    also holds "xyz_gradient_accum" and "denom" ((P, 1)); they are consumed, not returned."""
    st = {k: v for k, v in state.items() if k not in ("xyz_gradient_accum", "denom")}
    dev = st["xyz"].device
    P0 = st["xyz"].shape[0]
    grads = state["xyz_gradient_accum"] / state["denom"]
    grads[grads.isnan()] = 0.0
    # densify_and_clone
    sel = torch.where(torch.norm(grads, dim=-1) >= max_grad, True, False)
    sel = torch.logical_and(sel, torch.max(torch.exp(st["scaling"]), dim=1).values <= percent_dense * extent)
    new = {k: st[k][sel] for k in NAMES + CARRIED if k in st}
    _postfix(st, new)
    n_clone = int(sel.sum())
    # densify_and_split
    n_init = st["xyz"].shape[0]
    padded = torch.zeros((n_init,), device=dev)
    padded[: grads.shape[0]] = grads.squeeze(-1)
    sel = torch.where(padded >= max_grad, True, False)
    sel = torch.logical_and(sel, torch.max(torch.exp(st["scaling"]), dim=1).values > percent_dense * extent)
    S = int(sel.sum())
    split = sel[:P0].clone()
    stds = torch.exp(st["scaling"])[sel].repeat(N, 1)
    means = torch.zeros((stds.size(0), 3), device=dev)
    samples = means + stds * noise[: stds.size(0)]
    rots = build_rotation(st["rotation"][sel]).repeat(N, 1, 1)
    new = {"xyz": torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + st["xyz"][sel].repeat(N, 1),
           "scaling": torch.log(torch.exp(st["scaling"])[sel].repeat(N, 1) / (0.8 * N)),
           "rotation": st["rotation"][sel].repeat(N, 1),
           "f_dc": st["f_dc"][sel].repeat(N, 1, 1),
           "f_rest": st["f_rest"][sel].repeat(N, 1, 1),
           "opacity": st["opacity"][sel].repeat(N, 1)}
    for k in CARRIED:
        if k in st:
            new[k] = st[k][sel].repeat(N, 1)
    _postfix(st, new)
    _prune(st, torch.cat((sel, torch.zeros(N * S, device=dev, dtype=bool))))
    # final prune; max_radii2D is all zero after densification_postfix, so only the world-size test can act
    mask = (torch.sigmoid(st["opacity"]) < min_opacity).squeeze(-1)
    if max_screen_size:
        mask = torch.logical_or(mask, torch.exp(st["scaling"]).max(dim=1).values > 0.1 * extent)
    n_pruned = int(mask.sum())
    _prune(st, mask)
    return st, (n_clone, S, n_pruned, split)


def children_xyz_fp64(xyz, scaling, rotation, noise, N=2):
    """fp64 value of the split children's positions R(q) (s * z) + x of the Gaussians whose rows are given, from the
    same fp32 inputs: s = exp(log-scale) as the device computed it (`scaling` is that fp32 scale), q normalised, R and
    the products formed in fp64.  All arguments numpy; noise is (N S, 3).  -> (N S, 3) float64, copy-major."""
    x = np.tile(np.asarray(xyz, np.float64), (N, 1))
    s = np.tile(np.asarray(scaling, np.float64), (N, 1))
    q = np.tile(np.asarray(rotation, np.float64), (N, 1))
    q = q / np.sqrt((q * q).sum(axis=1, keepdims=True))
    w, a, b, c = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.stack([np.stack([1 - 2 * (b * b + c * c), 2 * (a * b - w * c), 2 * (a * c + w * b)], -1),
                  np.stack([2 * (a * b + w * c), 1 - 2 * (a * a + c * c), 2 * (b * c - w * a)], -1),
                  np.stack([2 * (a * c - w * b), 2 * (b * c + w * a), 1 - 2 * (a * a + b * b)], -1)], -2)
    return np.einsum("nij,nj->ni", R, s * np.asarray(noise, np.float64)[: x.shape[0]]) + x
