"""CPU checks for models that store fewer SH coefficients (--sh_degree D < 3 in the reference: (D+1)^2 coefficients per
Gaussian, scene/gaussian_model.py:51-53, 150-156): the _sh preprocess entry points and the width-parameterised sparse
gradient rows refuse bad degrees, pointers and alignment before any launch, the raw-parameter operators refuse
inconsistent parameter shapes before any launch, and redistribution moves the (P,0,3) and (P,3,3) _features_rest tensors
of D = 0 and D = 1 models with their Adam moments."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from gs_b200 import build, _lib
    build.build()
    return _lib.load()


ARGS = r"""
import ctypes, json, sys
sys.path.insert(0, %(pkg)r)
from gs_b200 import _lib
lib = _lib.load()
FAKE = 1 << 20   # a 16-byte aligned address that is never dereferenced: no device is visible to this process
# the int arguments of each entry point in order, the index (among its pointers) of a 16-byte aligned one, and of the
# features_rest / dL_dfeatures_rest pointers (split forms)
FORMS = {"gs_preprocess_forward_sh": ("P sh max W H", 2, ()), "gs_preprocess_backward_sh": ("P sh max W H", 2, ()),
         "gs_preprocess_forward_raw_sh": ("P sh max W H", 4, (2,)),
         "gs_preprocess_backward_raw_sh": ("P sh max W H", 4, (2, 16)),
         "gs_preprocess_forward_batched_sh": ("B P sh max W H", 4, (2,)),
         "gs_preprocess_backward_batched_sh": ("B P sh max W H", 4, (2, 14))}

def call(name, ptr=None, **ints):
    names, _, _ = FORMS[name]
    vals = dict(dict(B=1, P=8, sh=1, max=2, W=16, H=16), **ints)
    ivals = [vals[n] for n in names.split()]
    args, k = [], 0
    argtypes = _lib.SIGNATURES[name][1]
    for j, t in enumerate(argtypes):
        if t is ctypes.c_int:
            args.append(ivals.pop(0))
        elif t is ctypes.c_float:
            args.append(1.0)
        elif j == len(argtypes) - 1:
            args.append(None)                     # stream
        else:
            args.append((ptr or {}).get(k, FAKE))
            k += 1
    return getattr(lib, name)(*args)

out = {}
for name, (names, aligned, rest) in FORMS.items():
    r = out[name] = {"active above stored": call(name, sh=2, max=1), "stored 4": call(name, sh=3, max=4),
                     "stored -1": call(name, sh=0, max=-1), "negative active": call(name, sh=-1),
                     "null pointer": call(name, ptr={0: None}), "misaligned": call(name, ptr={aligned: FAKE + 4}),
                     "valid": call(name), "valid, degree 0": call(name, sh=0, max=0)}
    for q, k in enumerate(rest):
        r[f"null rest {q}, stored 2"] = call(name, ptr={k: None})
        r[f"misaligned rest {q}, stored 2"] = call(name, ptr={k: FAKE + 4})
        r[f"null rest {q}, stored 0"] = call(name, sh=0, max=0, ptr={k: None})
        r[f"misaligned rest {q}, stored 0"] = call(name, sh=0, max=0, ptr={k: FAKE + 4})
VP = ctypes.c_void_p * 6
grads = VP(*[FAKE] * 6)
no_rest = VP(FAKE, FAKE, None, FAKE, FAKE, FAKE)
rows = {}
for name in ("gs_sparse_grad_pack_rows", "gs_sparse_grad_unpack_rows"):
    f = getattr(lib, name)
    rows[name] = {"rest 10": f(8, 10, FAKE, FAKE, grads, FAKE, None) if "unpack" not in name else
                  f(8, 10, FAKE, FAKE, FAKE, grads, None),
                  "null rest, rest 9": f(8, 9, FAKE, FAKE, no_rest, FAKE, None) if "unpack" not in name else
                  f(8, 9, FAKE, FAKE, FAKE, no_rest, None),
                  "null rest, rest 0": f(8, 0, FAKE, FAKE, no_rest, FAKE, None) if "unpack" not in name else
                  f(8, 0, FAKE, FAKE, FAKE, no_rest, None)}
print(json.dumps(dict(pre=out, rows=rows)))
"""


def test_sh_entry_point_argument_checks(lib):
    """0 <= sh_degree <= max_sh_degree <= 3, null and misaligned pointers, and the rest pointers: refused (GS_EINVAL)
    before any launch; a NULL or misaligned rest pointer is accepted only when the model stores degree 0 (it is never
    read then).  The calls run in a process that sees no device: a call that passes every check ends in GS_ECUDA."""
    code = ARGS % dict(pkg=os.path.join(ROOT, "grendel-gs_b200"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(res["pre"]) == 6
    for name, rc in res["pre"].items():
        for case in ("active above stored", "stored 4", "stored -1", "negative active", "null pointer", "misaligned"):
            assert rc[case] == -1, (name, case, rc[case])                # GS_EINVAL
        assert rc["valid"] == -2 and rc["valid, degree 0"] == -2, name   # GS_ECUDA: passed every check, no device
        for case, v in rc.items():
            if "rest" in case:
                assert v == (-2 if "stored 0" in case else -1), (name, case, v)
    for name, rc in res["rows"].items():
        assert rc == {"rest 10": -1, "null rest, rest 9": -1, "null rest, rest 0": -2}, (name, rc)


def test_header_declares_sh_entry_points():
    import re
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "grendel_gs_b200.h")).read(), flags=re.S)
    for form in ("forward", "backward", "forward_raw", "backward_raw", "forward_batched", "backward_batched"):
        old = re.search(r"\bgs_preprocess_" + form + r"\s*\(([^;]*?)\)\s*;", src, flags=re.S).group(1)
        new = re.search(r"\bgs_preprocess_" + form + r"_sh\s*\(([^;]*?)\)\s*;", src, flags=re.S).group(1)
        o = [p.strip() for p in old.split(",")]
        n = [p.strip() for p in new.split(",")]
        i = o.index("int sh_degree")
        assert n == o[:i + 1] + ["int max_sh_degree"] + o[i + 1:], form     # the same arguments + max_sh_degree


def test_scene_and_params_store_the_requested_degree():
    from gs_b200 import pipeline, synthetic as syn
    full = syn.make_scene(7, 64, 48, seed=3)
    for D in range(4):
        K = (D + 1) ** 2
        sc = syn.make_scene(7, 64, 48, seed=3, max_sh_degree=D)
        assert sc["shs"].shape == (7, K, 3) and np.array_equal(sc["shs"], full["shs"][:, :K])
        for k in ("means3D", "scales", "rotations", "opacities"):
            assert np.array_equal(sc[k], full[k])
        p = pipeline.GaussianParams(sc, "cpu", D)
        assert tuple(p._features_rest.shape) == (7, K - 1, 3) and p.max_sh_degree == p.active_sh_degree == D
        assert tuple(p.get_features.shape) == (7, K, 3)
    with pytest.raises(ValueError):
        pipeline.GaussianParams(syn.make_scene(7, 64, 48, max_sh_degree=1), "cpu")     # 4 coefficients, degree 3 asked
    with pytest.raises(ValueError):
        pipeline.GaussianParams(full, "cpu", 4)


def test_raw_operators_refuse_inconsistent_parameters_before_any_launch(monkeypatch):
    """preprocess_gaussians_raw and preprocess_gaussians_batched (one view and two) check _xyz, _scaling, _rotation and
    _opacity against the P rows of _xyz, and the features against P, before they read a camera or call the library: a
    ValueError for each mismatch, here with tensors on the host that could not be launched anyway."""
    from gs_b200 import _lib, ops, pipeline, synthetic as syn

    def forbid(*_a, **_k):
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "call", forbid)
    P, K = 5, 4
    good = [torch.zeros(P, 3), torch.zeros(P, 1, 3), torch.zeros(P, K - 1, 3), torch.zeros(P, 3), torch.zeros(P, 4),
            torch.zeros(P, 1)]
    rs = pipeline.DeviceCamera(syn.make_camera(16, 16), "cpu").settings(1)
    cases = [(0, (P, 4), "inconsistent"), (0, (P + 1, 3), "features"), (1, (P, 2, 3), "features"),
             (2, (P + 1, K - 1, 3), "features"), (3, (P - 1, 3), "inconsistent"), (3, (P, 4), "inconsistent"),
             (4, (P, 3), "inconsistent"), (4, (P + 1, 4), "inconsistent"), (5, (P + 1, 1), "inconsistent")]
    for q, shape, msg in cases:
        raw = list(good)
        raw[q] = torch.zeros(shape)
        with pytest.raises(ValueError, match=msg):
            ops.preprocess_gaussians_raw(*raw, rs)
        for B in (1, 2):
            with pytest.raises(ValueError, match=msg):
                ops.preprocess_gaussians_batched(*raw, torch.zeros(B, 40), 16, 16, 1)
    for B in (1, 2):   # consistent parameters pass the checks and are refused only for living on the host
        with pytest.raises(ValueError, match="CUDA tensor"):
            ops.preprocess_gaussians_batched(*good, torch.zeros(B, 40), 16, 16, 1)


def _redistribute_worker(rank, world, port, D, q):
    import torch.distributed as dist
    from gs_b200 import redistribute as rd
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    P = 40 + 29 * rank
    g = torch.Generator().manual_seed(300 + rank)
    shapes = {"xyz": (3,), "f_dc": (1, 3), "f_rest": ((D + 1) ** 2 - 1, 3), "opacity": (1,), "scaling": (3,),
              "rotation": (4,)}
    params = {k: torch.nn.Parameter(torch.randn((P,) + s, generator=g)) for k, s in shapes.items()}
    opt = torch.optim.Adam([{"params": [params[k]], "lr": 1e-3, "name": k} for k in rd.NAMES], lr=0.0, eps=1e-15)
    for k in rd.NAMES:
        params[k].grad = torch.randn(params[k].shape, generator=g)
    opt.step()
    before = {k: (params[k].detach().clone(), opt.state[params[k]]["exp_avg"].clone(),
                  opt.state[params[k]]["exp_avg_sq"].clone()) for k in rd.NAMES}
    dest = torch.randint(0, world, (P,), generator=g)
    res = rd.redistribute(opt, dest)
    ok = True
    for k in rd.NAMES:
        p_new = opt.param_groups[rd.NAMES.index(k)]["params"][0]
        st = opt.state[p_new]
        for q_, t in enumerate(before[k]):
            mine = [t[dest == j].contiguous() for j in range(world)]
            outs = [None] * world
            dist.all_gather_object(outs, mine)
            exp = torch.cat([outs[i][rank] for i in range(world)], dim=0)
            got = (p_new.detach(), st["exp_avg"], st["exp_avg_sq"])[q_]
            ok = ok and got.shape == exp.shape and torch.equal(got, exp)
        ok = ok and p_new is res[k] and tuple(p_new.shape[1:]) == shapes[k]
    n_new = res["xyz"].shape[0]
    for k in rd.NAMES:
        res[k].grad = torch.ones_like(res[k])
    opt.step()
    q.put((rank, bool(ok), n_new))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("D", [0, 1])
@pytest.mark.parametrize("world", [2, 3])
def test_redistribution_of_low_degree_models(world, D):
    """scene/gaussian_model.py:1073-1098 for a model stored at SH degree 0 (_features_rest (P,0,3)) or 1 ((P,3,3)): every
    tensor, the empty ones included, arrives row for row as the per-tensor exchanges of the reference build it."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29750 + 10 * D + world
    procs = [ctx.Process(target=_redistribute_worker, args=(r, world, port, D, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res), res
    assert sum(n for *_, n in res) == sum(40 + 29 * r for r in range(world))
