"""CPU: oracle/densify_oracle.py against tests/golden/densify.npz -- inputs and outputs of the REFERENCE's own
densify_and_prune (scene/gaussian_model.py:1005-1044 and the functions it calls) run on CPU tensors by
tests/golden/make_densify_golden.py."""
import os

import numpy as np
import pytest

from oracle import densify_oracle as do

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "densify.npz")


def load(case):
    z = np.load(GOLD)
    pre = f"c{case}."
    ins = {k[len(pre) + 3:]: z[k] for k in z.files if k.startswith(pre + "in.")}
    outs = {k[len(pre) + 4:]: z[k] for k in z.files if k.startswith(pre + "out.")}
    return ins, outs, z[pre + "noise"], z[pre + "scalars"]


def fused_emulation(st, noise, max_grad, min_opacity, extent, pd, screen):
    """numpy transcription of csrc/densify.cu (k_densify_flags -> one exclusive scan over five flag planes ->
    k_densify_gather): the select / scan / gather formulation must reproduce the reference's clone -> split -> prune ->
    prune sequence row for row.  Like the kernel, a child's scale is s times fl32(1 / 1.6) (torch's division by a
    Python scalar on CUDA; the CPU golden divides, which the rtol on `scaling` covers)."""
    F = np.float32
    P = st["xyz"].shape[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        grad = (st["xyz_gradient_accum"].reshape(-1).astype(F) / st["denom"].reshape(-1).astype(F)).astype(F)
    grad[np.isnan(grad)] = 0
    s = np.exp(st["scaling"].astype(F))
    smax = s.max(axis=1)
    dense_thr, big_thr = F(pd * extent), F(0.1 * extent)
    sel_clone = (np.abs(grad) >= F(max_grad)) & (smax <= dense_thr)
    sel_split = (grad >= F(max_grad)) & (smax > dense_thr)
    faint = (F(1) / (F(1) + np.exp(-st["opacity"].reshape(-1).astype(F)))).astype(F) < F(min_opacity)
    prune_orig = faint | (screen & (smax > big_thr))
    child_s = np.exp(np.log((s * (F(1) / F(1.6))).astype(F)).astype(F)).astype(F)
    prune_child = faint | (screen & (child_s.max(axis=1) > big_thr))
    planes = np.stack([~sel_split & ~prune_orig, sel_clone & ~prune_orig, sel_split & ~prune_child, sel_split & ~prune_child,
                       sel_split]).astype(np.int64)
    flat = planes.reshape(-1)
    pos = (np.cumsum(flat) - flat).reshape(5, P)
    new_P, S = int(pos[4, 0]), int(planes[4].sum())
    rank = pos[4] - new_P
    out = {}
    R = do.build_rotation(st["rotation"])
    for name, kind in [("xyz", "xyz"), ("f_dc", "copy"), ("f_rest", "copy"), ("opacity", "copy"), ("scaling", "scaling"),
                       ("rotation", "copy"), ("send_to_gpui_cnt", "copy")] + \
                      [(n + m, "moment") for n in do.NAMES for m in (".exp_avg", ".exp_avg_sq")]:
        src = st[name]
        dst = np.zeros((new_P,) + src.shape[1:], src.dtype)
        keep, clone, child = planes[0] == 1, planes[1] == 1, planes[2] == 1
        dst[pos[0][keep]] = src[keep]
        dst[pos[1][clone]] = 0 if kind == "moment" else src[clone]
        for copy, plane in ((0, 2), (1, 3)):
            if kind == "moment":
                val = 0
            elif kind == "scaling":
                val = np.log((np.exp(src[child].astype(F)) * (F(1) / F(1.6))).astype(F)).astype(F)
            elif kind == "xyz":
                z = noise[copy * S + rank[child]].astype(F)
                val = (np.einsum("nij,nj->ni", R[child], (s[child] * z).astype(F)) + src[child]).astype(F)
            else:
                val = src[child]
            dst[pos[plane][child]] = val
        out[name] = dst
    return out, (int(planes[0].sum()), int(planes[1].sum()), int(planes[2].sum()), S, new_P)


@pytest.mark.parametrize("case", [0, 1])
def test_select_scan_gather_formulation_equals_the_reference_sequence(case):
    ins, outs, noise, (max_grad, min_opacity, extent, pd, screen) = load(case)
    got, (n_keep, n_clone, n_child, S, new_P) = fused_emulation(ins, noise, float(max_grad), float(min_opacity), float(extent),
                                                                float(pd), bool(screen))
    assert new_P == outs["xyz"].shape[0] == n_keep + n_clone + 2 * n_child and S >= n_child
    for k, v in got.items():
        ref = outs[k]
        if k in ("xyz", "scaling"):
            np.testing.assert_allclose(v, ref, rtol=2e-6, atol=2e-6, err_msg=k)
        else:
            assert np.array_equal(v, ref), k


@pytest.mark.parametrize("case", [0, 1])
def test_densify_oracle_matches_the_reference_run(case):
    ins, outs, noise, (max_grad, min_opacity, extent, pd, screen) = load(case)
    got = do.densify_and_prune(ins, noise, float(max_grad), float(min_opacity), float(extent), float(pd), bool(screen))
    n_clone, n_split, n_pruned = got.pop("_counts")
    assert n_clone > 5 and n_split > 20 and n_pruned > 0           # every branch of the step is exercised
    assert got["xyz"].shape == outs["xyz"].shape
    for k, ref in outs.items():
        assert got[k].shape == ref.shape, k
        if k in ("xyz", "scaling"):   # split children: R(q) (s z) + x and log(s / 1.6): a few ulps between numpy and torch
            np.testing.assert_allclose(got[k], ref, rtol=2e-6, atol=2e-6, err_msg=k)
        else:                         # everything else is copied / zero-filled: exact
            assert np.array_equal(got[k], ref), k
    # moments of the new Gaussians are zero, those of the survivors are carried over
    P0 = ins["xyz"].shape[0]
    assert np.abs(got["f_rest.exp_avg"][: min(P0, 50)]).sum() > 0
    assert np.abs(got["f_rest.exp_avg"][-10:]).sum() == 0


@pytest.mark.parametrize("case", [0, 1])
def test_torch_restatement_matches_the_reference_run(case):
    """tests/densify_ref.py (the GPU tests' decision oracle) on CPU tensors against the reference's own CPU run: copied
    tensors bit for bit, children's positions and scales within the rtol above; children's fp64 positions agree too."""
    import torch
    import densify_ref as dr
    ins, outs, noise, (max_grad, min_opacity, extent, pd, screen) = load(case)
    st = {k: torch.from_numpy(v.copy()) for k, v in ins.items()}
    got, (n_clone, S, n_pruned, split_ref) = dr.densify_and_prune(st, torch.from_numpy(noise.copy()), float(max_grad),
                                                       float(min_opacity), float(extent), float(pd), 20 if screen else None)
    assert n_clone > 5 and S > 20 and n_pruned > 0
    assert set(got) == set(outs) - {"xyz_gradient_accum", "denom"}
    for k, v in got.items():
        v, ref = v.numpy(), outs[k]
        assert v.shape == ref.shape and v.dtype == ref.dtype, k
        if k in ("xyz", "scaling"):
            np.testing.assert_allclose(v, ref, rtol=2e-6, atol=2e-6, err_msg=k)
        else:
            assert np.array_equal(v, ref), k
    # the fp64 children: rows of the split Gaussians that survive the final prune, in the order of the children block
    s = np.exp(ins["scaling"])
    with np.errstate(divide="ignore", invalid="ignore"):
        grads = (ins["xyz_gradient_accum"] / ins["denom"]).reshape(-1)
        split = (np.nan_to_num(grads, nan=0.0) >= np.float32(max_grad)) & (s.max(axis=1) > np.float32(pd * extent))
    assert split.sum() == S and np.array_equal(split, split_ref.numpy())
    x64 = dr.children_xyz_fp64(ins["xyz"][split], s[split], ins["rotation"][split], noise[: 2 * S])
    # the golden case has no world-size prune of children (case 1) or prunes some: compare the children of case 1 only
    if not screen:
        kept = (1 / (1 + np.exp(-ins["opacity"][split].reshape(-1).astype(np.float64)))) >= min_opacity
        ref = outs["xyz"][-2 * int(kept.sum()):]
        np.testing.assert_allclose(ref, x64[np.tile(kept, 2)], rtol=2e-6, atol=2e-6)


def test_densify_select_takes_extent_and_percent_dense_as_doubles():
    """The reference's thresholds are fl32 of a double product (percent_dense * extent, 0.1 * extent): the binding
    must carry both scalars at full double precision, and a ctypes float argument converts exactly."""
    import ctypes
    from gs_b200 import _lib
    argtypes = _lib.SIGNATURES["gs_densify_select"][1]
    for j in (7, 8):
        assert issubclass(argtypes[j], ctypes.c_double)
        assert argtypes[j].from_param(0.1).value == 0.1                       # not rounded to fp32 on the way
        assert argtypes[j].from_param(ctypes.c_float(0.1)).value == float(np.float32(0.1))
        assert argtypes[j].from_param(ctypes.c_double(5.0)).value == 5.0
    lib = _lib.load()
    rc = lib.gs_densify_select(0, None, None, None, None, ctypes.c_float(0), ctypes.c_float(0), 10.0, 0.01, 0, None, 0,
                               None, None)
    assert rc == -1 and b"P" in lib.gs_last_error()
