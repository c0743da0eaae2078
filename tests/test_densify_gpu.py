"""-m gpu: gs_densify_select / gs_densify_gather (through gs_b200.densify.densify_and_prune) against the reference's
densification chain run on the same device (tests/densify_ref.py) on the constructed populations of
tests/densify_cases.py, with the same draws.

Decisions and everything that is copied must agree bit for bit: the counts, the order of the survivor / clone / child
rows (send_to_gpui_cnt carries unique 40-bit values, so its rows name their source), every copied parameter, the
survivors' Adam moments, zero moments for new Gaussians, the children's log-scales.  Children's positions are fp32 sums
in a different order (the kernel's FMA chain, the reference's bmm); both are measured against an fp64 evaluation from the
same fp32 inputs and the kernel may be at most twice as far from it as the reference, plus a few ulps of |x|."""
import ctypes as C

import numpy as np
import pytest
import torch

import densify_cases as dc
import densify_ref as dr

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = dc.NAMES


@pytest.fixture(scope="module")
def cases():
    return {c["name"]: c for c in dc.all_cases(DEV)}


def _optimizer(case):
    st = case["state"]
    params = {k: torch.nn.Parameter(torch.from_numpy(st[k]).to(DEV)) for k in NAMES}
    opt = torch.optim.Adam([{"params": [params[k]], "lr": 1e-3, "name": k} for k in NAMES], lr=0.0, eps=1e-15)
    for k in NAMES:
        if k + ".exp_avg" in st:
            opt.state[params[k]] = {"step": torch.tensor(7.0), "exp_avg": torch.from_numpy(st[k + ".exp_avg"]).to(DEV),
                                    "exp_avg_sq": torch.from_numpy(st[k + ".exp_avg_sq"]).to(DEV)}
    return opt


def run_kernel(case, use_noise=True):
    from gs_b200 import densify
    st = case["state"]
    opt = _optimizer(case)
    res = densify.densify_and_prune(opt, torch.from_numpy(st["xyz_gradient_accum"]).to(DEV),
                                    torch.from_numpy(st["denom"]).to(DEV), case["max_grad"], case["min_opacity"],
                                    case["extent"], case["pd"], 20 if case["screen"] else None,
                                    send_to_gpui_cnt=torch.from_numpy(st["send_to_gpui_cnt"]).to(DEV),
                                    noise=torch.from_numpy(case["noise"]).to(DEV) if use_noise else None)
    torch.cuda.synchronize()
    got = {"send_to_gpui_cnt": res["send_to_gpui_cnt"].cpu().numpy()}
    for k in NAMES:
        p = opt.param_groups[NAMES.index(k)]["params"][0]
        assert p is res[k] and p.requires_grad
        got[k] = p.detach().cpu().numpy()
        if p in opt.state:
            s = opt.state[p]
            assert float(s["step"]) == 7.0                        # step is untouched
            got[k + ".exp_avg"], got[k + ".exp_avg_sq"] = s["exp_avg"].cpu().numpy(), s["exp_avg_sq"].cpu().numpy()
    return got, res["counts"]


def run_ref(case):
    st = {k: torch.from_numpy(v).to(DEV) for k, v in case["state"].items()}
    P = st["xyz"].shape[0]
    st["row"] = torch.arange(P, device=DEV).reshape(P, 1)
    out, (n_clone, S, n_pruned, split) = dr.densify_and_prune(st, torch.from_numpy(case["noise"]).to(DEV),
                                                              case["max_grad"], case["min_opacity"], case["extent"],
                                                              case["pd"], 20 if case["screen"] else None)
    ref = {k: v.cpu().numpy() for k, v in out.items()}
    return ref, S, split.cpu().numpy()


def check_case(case, use_noise=True):
    """-> (worst kernel, worst reference) relative error of the children's positions against fp64."""
    got, (kept, clones, child, S, new_P) = run_kernel(case, use_noise)
    ref, S_ref, split = run_ref(case)
    name = case["name"]
    assert S == S_ref and new_P == ref["xyz"].shape[0], (name, (kept, clones, child, S, new_P), S_ref, ref["xyz"].shape)
    assert kept + clones + 2 * child == new_P
    assert set(got) == set(ref) - {"row"}, name
    # row order: send_to_gpui_cnt rows are unique, so equality says every output row came from the same source row
    assert np.array_equal(got["send_to_gpui_cnt"], ref["send_to_gpui_cnt"]), name
    for k, v in got.items():
        if k == "xyz":
            continue
        assert v.dtype == ref[k].dtype and v.shape == ref[k].shape, (name, k)
        assert np.array_equal(v.view(np.uint32) if v.dtype == np.float32 else v,
                              ref[k].view(np.uint32) if ref[k].dtype == np.float32 else ref[k]), (name, k)
        if k.endswith(".exp_avg") or k.endswith(".exp_avg_sq"):
            assert not v[kept:].any(), (name, k, "new Gaussians start with zero moments")
    assert np.array_equal(got["xyz"][: kept + clones], ref["xyz"][: kept + clones]), (name, "copied positions")
    if child == 0:
        return 0.0, 0.0
    # children: fp64 from the fp32 inputs
    st = case["state"]
    s32 = torch.exp(torch.from_numpy(st["scaling"]).to(DEV)).cpu().numpy()
    x64 = dr.children_xyz_fp64(st["xyz"][split], s32[split], st["rotation"][split], case["noise"][: 2 * S])
    rank = np.cumsum(split) - 1
    src = ref["row"][kept + clones:, 0]
    copy = np.repeat([0, 1], child)
    idx = copy * S + rank[src]
    want = x64[idx]
    z = np.asarray(case["noise"][idx], np.float64)
    x = np.asarray(st["xyz"][src], np.float64)
    scale = np.abs(x) + (np.abs(s32[src].astype(np.float64)) * np.abs(z)).sum(axis=1, keepdims=True)
    ek = np.abs(got["xyz"][kept + clones:] - want)
    er = np.abs(ref["xyz"][kept + clones:] - want)
    wk, wr = float((ek / scale).max()), float((er / scale).max())
    print(f"[parity] {name}: children xyz vs fp64: kernel worst_rel={wk:.2e} | device reference worst_rel={wr:.2e}")
    bar = 2.0 * wr * scale + 4.0 * np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)
    assert (ek <= bar).all(), (name, wk, wr)
    return wk, wr


def test_cases_populate_every_decision(cases):
    fam = {}
    for c in cases.values():
        fam.setdefault(c["family"], []).append(c["near"])
    print("[densify] near-threshold Gaussians per family:", {k: sum(v) for k, v in fam.items()})
    for f in ("grad", "dense", "dense_rounding", "big_orig", "big_child", "big_rounding", "opacity", "whole", "positions"):
        assert f in fam and sum(fam[f]) > 0, f
    # exact hits exist where the threshold was moved onto a reachable value
    labels = set(np.concatenate([c["label"] for c in cases.values()]).tolist())
    for tag in ("dense_shift0_at", "big_orig_cold0_at", "big_child0_at", "opacity0_at", "grad_at_pos_small",
                "grad_at_neg_large"):
        assert tag in labels, tag
    assert any(t.startswith("dense_new_at") or t.startswith("dense_old_at") for t in labels)
    assert any(t.startswith("big_new_at") or t.startswith("big_old_at") for t in labels)
    print("[densify] fl32(0.05) reachable by exp:", "dense_at" in labels)


@pytest.mark.parametrize("family", ["grad", "dense", "dense_rounding", "big_orig", "big_child", "big_rounding", "opacity",
                                    "whole", "positions", "shapes"])
def test_densify_matches_device_reference(cases, family):
    worst = [check_case(c) for c in cases.values() if c["family"] == family]
    assert worst
    print(f"[densify] {family}: {len(worst)} cases; children xyz worst_rel vs fp64: kernel "
          f"{max(w[0] for w in worst):.2e}, device reference {max(w[1] for w in worst):.2e}")


def test_whole_population_outcomes(cases):
    got, counts = run_kernel(cases["all_pruned"])
    assert counts[-1] == 0 and all(v.shape[0] == 0 for v in got.values())
    got, counts = run_kernel(cases["none_selected"], use_noise=False)     # S == 0: no draws at all
    assert counts[3] == 0 and counts[1] == 0 and counts[-1] == cases["none_selected"]["state"]["xyz"].shape[0]
    check_case(cases["none_selected"], use_noise=False)
    _, counts = run_kernel(cases["all_split"])
    P = cases["all_split"]["state"]["xyz"].shape[0]
    assert counts == (0, 0, P, P, 2 * P)


def test_densify_one_million_rows():
    """~1 M Gaussians: 45-float f_rest rows take the gather's element index past 2^25 per tensor."""
    c = dc.shape_case(dc.BIG_P, 7, 3)
    wk, wr = check_case(c)
    print(f"[densify] P={dc.BIG_P}: children xyz worst_rel kernel {wk:.2e}, device reference {wr:.2e}")


def test_gather_with_a_full_tensor_table(cases):
    """gs_densify_gather with the 24 tensors one launch takes: the 19 of a full optimizer and five more copied tensors
    of widths 1, 2 (int64), 5, 45 and 7."""
    from gs_b200 import _lib
    case = cases["interleaved"]
    st = case["state"]
    P = st["xyz"].shape[0]
    ref, S_ref, split = run_ref(case)
    src_rows = ref["row"][:, 0]
    d = {k: torch.from_numpy(v).to(DEV) for k, v in st.items()}
    rng = np.random.default_rng(5)
    extra = [rng.normal(size=(P, 1)).astype(np.float32), rng.integers(0, 1 << 50, size=(P, 1), dtype=np.int64),
             rng.normal(size=(P, 5)).astype(np.float32), rng.normal(size=(P, 15, 3)).astype(np.float32),
             rng.normal(size=(P, 7)).astype(np.float32)]
    table = [(k, d[k], {"xyz": 1, "scaling": 2}.get(k, 0)) for k in NAMES]
    table += [(k + m, d[k + m], 3) for k in NAMES for m in (".exp_avg", ".exp_avg_sq")]
    table += [("send_to_gpui_cnt", d["send_to_gpui_cnt"], 0)] + [(f"extra{i}", torch.from_numpy(e).to(DEV), 0)
                                                                for i, e in enumerate(extra)]
    assert len(table) == 24
    tb = _lib.query("gs_densify_temp_bytes", P)
    temp = torch.empty((tb,), dtype=torch.uint8, device=DEV)
    counts = (C.c_int32 * 6)()
    stream = torch.cuda.current_stream().cuda_stream
    _lib.call("gs_densify_select", P, d["xyz_gradient_accum"].data_ptr(), d["denom"].data_ptr(), d["scaling"].data_ptr(),
              d["opacity"].data_ptr(), C.c_float(case["max_grad"]), C.c_float(case["min_opacity"]),
              C.c_double(case["extent"]), C.c_double(case["pd"]), 1, temp.data_ptr(), tb, counts, stream)
    kept, clones, child, _, S, new_P = (int(v) for v in counts)
    assert S == S_ref and new_P == src_rows.size
    noise = torch.from_numpy(case["noise"]).to(DEV)
    outs = [torch.full((new_P,) + tuple(t.shape[1:]), -1, dtype=t.dtype, device=DEV) for _, t, _ in table]
    n = len(table)
    width = [t[0].numel() * t.element_size() // 4 for _, t, _ in table]
    _lib.call("gs_densify_gather", P, S, new_P, n, (C.c_void_p * n)(*[t.data_ptr() for _, t, _ in table]),
              (C.c_void_p * n)(*[o.data_ptr() for o in outs]), (C.c_int32 * n)(*width),
              (C.c_int32 * n)(*[k for _, _, k in table]), d["scaling"].data_ptr(), d["rotation"].data_ptr(),
              noise.data_ptr(), temp.data_ptr(), stream)
    torch.cuda.synchronize()
    for (name, t, kind), o in zip(table, outs):
        o, t = o.cpu().numpy(), t.cpu().numpy()
        if kind == 0:
            assert np.array_equal(o, t[src_rows]), name
        elif kind == 3:
            assert np.array_equal(o[:kept], t[src_rows[:kept]]) and not o[kept:].any(), name
        elif kind == 2:
            assert np.array_equal(o.view(np.uint32), ref["scaling"].view(np.uint32)), name
        else:
            np.testing.assert_allclose(o, ref["xyz"], rtol=1e-5, atol=1e-6, err_msg=name)
