"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/grendel_gs_b200.h declares, and the ctypes table mirrors the header (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "grendel_gs_b200.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"GS_API[^;(]*?\b(gs_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from gs_b200 import build, _lib
    build.build()
    return _lib.load()


def test_header_declares_the_whole_hot_path():
    names = declared_symbols()
    for must in ("gs_preprocess_forward", "gs_preprocess_backward", "gs_render_count", "gs_render_forward",
                 "gs_render_backward", "gs_get_local2j_ids_bool", "gs_get_block_xy", "gs_loss_forward",
                 "gs_loss_backward", "gs_route_scan", "gs_xchg_route", "gs_xchg_pack", "gs_xchg_unpack", "gs_xchg_pack_grad", "gs_xchg_scatter_grad", "gs_sparse_grad_pack", "gs_preprocess_forward_batched", "gs_profile_read"):
        assert must in names


def test_library_exports_every_declared_symbol(lib):
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in the header but not exported"


def test_ctypes_table_matches_header(lib):
    from gs_b200 import _lib
    assert sorted(_lib.SIGNATURES) == declared_symbols()
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name, (_, argtypes) in _lib.SIGNATURES.items():
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", src, flags=re.S)
        assert m, name
        params = m.group(1).strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(argtypes), f"{name}: header has {n} parameters, ctypes table {len(argtypes)}"


def test_constants_and_version(lib):
    a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert lib.gs_get_block_xy(ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)) == 0
    assert (a.value, b.value, c.value) == (16, 16, 256)
    assert b"sm_90a" in lib.gs_version()
    # argument validation happens before any CUDA call
    assert lib.gs_get_block_xy(None, None, None) != 0
    assert b"null" in lib.gs_last_error().lower()


def test_argument_errors_are_reported_not_crashed(lib):
    """Every entry point validates its arguments before the first CUDA call and reports through the return code +
    gs_last_error() (the reference side sees a Python exception, never a crash or an exit): exercised here, without a GPU,
    on the entry points added for batches, the peer exchange, Adam and densification."""
    from gs_b200 import _lib
    i32, vp = ctypes.c_int32, ctypes.c_void_p
    R = ctypes.c_int64(0)
    one = (i32 * 2)(0, 0)
    bad = [
        ("gs_render_count_batched", (0, one, 16, 16, None, None, None, None, None, None, None, None, None, None, 0, ctypes.byref(R), None)),
        ("gs_render_count_batched", (65, one, 16, 16, None, None, None, None, None, None, None, None, None, None, 0, ctypes.byref(R), None)),
        ("gs_render_count_batched", (1, (i32 * 2)(3, 5), 16, 16, None, None, None, None, None, None, None, None, None, None, 0, ctypes.byref(R), None)),
        ("gs_render_count_launch", (2, None, 4, 16, 16, None, None, None, None, None, None, None, None, None, None, 0, ctypes.byref(vp()), None)),
        ("gs_render_count_launch", (1, None, 4, 16, 16, None, None, None, None, None, None, None, None, None, None, 0, None, None)),
        ("gs_render_count_read", (None, ctypes.byref(R), None)),
        ("gs_render_count_read", (ctypes.cast(ctypes.byref(R), vp), ctypes.byref(R), None)),   # not a ticket of the library
        ("gs_render_backward_batched", (0, 0, 0, 16, 16, None, None, None, None, None, None, None, None, None, 0, None, None, None, None)),
        ("gs_loss_forward_batched", (1, 16, 16, None, None, None, None, None, 0, None)),
        ("gs_xr_pack_dev", (0, 4, 2, 16, 16, None, None, None, None, None, None, None, None, None, None, 0, None, 64, None)),
        ("gs_xr_pull_grad", (1, 4, 17, 16, 16, None, None, None, None, None, None, None, 64, None, None, None, None)),
        ("gs_peer_alloc", (0, None, None)),
        ("gs_peer_open", (None, None)),
        ("gs_adam_step", (9, None, None, None, None, None, None, None, None, None, None, ctypes.c_float(1.0), None)),
        ("gs_adam_step", (1, None, None, None, None, None, None, None, None, None, None, ctypes.c_float(1.0), None)),
        ("gs_densify_select", (0, None, None, None, None, ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(1), ctypes.c_float(0.01), 0, None, 0, None, None)),
        ("gs_densify_gather", (4, 0, 4, 25, None, None, None, None, None, None, None, None, None)),
    ]
    for name, args in bad:
        rc = getattr(lib, name)(*args)
        assert rc == -1, (name, rc)                       # GS_EINVAL
        assert len(lib.gs_last_error()) > 10, name
        with pytest.raises(_lib.GsError):
            _lib.call(name, *args)
    assert lib.gs_debug_set(0) == 0 and lib.gs_debug_set(0) == 0
    assert lib.gs_adam_step(0, None, None, None, None, None, None, None, None, None, None, ctypes.c_float(1.0), None) == 0


PREPROCESS_ARGS = r"""
import ctypes, json, sys
sys.path.insert(0, %(pkg)r)
from gs_b200 import _lib
lib = _lib.load()
FAKE = 1 << 20   # a 16-byte aligned address that is never dereferenced: no device is visible to this process
# the int arguments of each entry point in order, and the index (among its pointers) of a 16-byte aligned one
FORMS = {"gs_preprocess_forward": ("P sh W H", 2), "gs_preprocess_backward": ("P sh W H", 2),
         "gs_preprocess_forward_raw": ("P sh W H", 4), "gs_preprocess_backward_raw": ("P sh W H", 4),
         "gs_preprocess_forward_batched": ("B P sh W H", 4), "gs_preprocess_backward_batched": ("B P sh W H", 4)}

def call(name, ptr=None, **ints):
    names, _ = FORMS[name]
    vals = dict(dict(B=1, P=8, sh=3, W=16, H=16), **ints)
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
for name, (names, aligned) in FORMS.items():
    r = out[name] = {"negative P": call(name, P=-1), "sh_degree 4": call(name, sh=4),
                     "null pointer": call(name, ptr={0: None}), "misaligned": call(name, ptr={aligned: FAKE + 4}),
                     "P 0, null pointers": call(name, P=0, ptr={k: None for k in range(40)}),
                     "P 0, no image": call(name, P=0, W=0), "valid": call(name)}
    if "batched" in name:
        r["B 0"], r["B 65"] = call(name, B=0), call(name, B=65)
print(json.dumps(out))
"""


def test_preprocess_argument_checks(lib):
    """The six preprocess entry points refuse bad sizes, pointers and alignment before any launch.  The calls run in a
    process that sees no device, so a check that stops working ends in a launch error and never touches one."""
    import json
    import subprocess
    import sys
    code = PREPROCESS_ARGS % dict(pkg=os.path.join(ROOT, "grendel-gs_b200"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(out) == 6
    for name, rc in out.items():
        for case in ("negative P", "sh_degree 4", "null pointer", "misaligned") + (("B 0", "B 65") * ("batched" in name)):
            assert rc[case] == -1, (name, case, rc[case])              # GS_EINVAL
        assert rc["P 0, null pointers"] == 0, name                      # GS_OK: nothing to do
        assert rc["valid"] == -2, name                                  # GS_ECUDA: passed every check, no device
        # gs_preprocess_forward has always refused an empty image, even with P == 0; the others accept it
        assert rc["P 0, no image"] == (-1 if name == "gs_preprocess_forward" else 0), name


LOSS_ARGS = r"""
import ctypes, json, sys
sys.path.insert(0, %(pkg)r)
from gs_b200 import _lib
lib = _lib.load()
FAKE = 1 << 20   # an address that is never dereferenced: no device is visible to this process
H, W = 64, 16

def call(rows, gts=None, B=None, temp_bytes=None):
    B = len(rows) if B is None else B
    flat = (ctypes.c_int32 * max(4, 4 * len(rows)))(*[v for r in rows for v in r])
    g = (ctypes.c_void_p * max(1, len(rows)))(*(gts if gts is not None else [FAKE] * len(rows)))
    tb = lib.gs_loss_temp_bytes_batched(len(rows), flat, W) if temp_bytes is None else temp_bytes
    f = lib.gs_loss_forward_batched(B, H, W, flat, FAKE, g, FAKE, FAKE, tb, None)
    b = lib.gs_loss_backward_batched(B, H, W, flat, FAKE, g, FAKE, FAKE, FAKE, FAKE, None)
    return [f, b]

ok = (0, 32, 5, 27)
maps = 1024 + 9 * 32 * W * 4
print(json.dumps({
    "B 0": call([ok], B=0), "B 65": call([ok] * 65),
    "row0 < 0": call([(-1, 32, 0, 32)]), "row1 > H": call([(0, H + 1, 0, H)]), "row1 < row0": call([(9, 8, 8, 8)]),
    "c0 < row0": call([(8, 32, 7, 32)]), "c1 > row1": call([(0, 32, 0, 33)]), "c1 < c0": call([(0, 32, 20, 19)]),
    "null gt": call([(0, 0, 0, 0), ok], gts=[None, None]), "null gt, second view": call([ok, ok], gts=[FAKE, None]),
    "one byte short": call([ok], temp_bytes=maps - 1),
    "valid": call([ok], temp_bytes=maps), "valid, empty view without gt": call([(0, 0, 0, 0), ok], gts=[None, FAKE]),
}))
"""


def test_loss_argument_checks(lib):
    """gs_loss_{forward,backward}_batched refuse bad view counts, rows and ground-truth pointers before any launch, and
    the forward a workspace one byte short of the header and maps.  The calls run in a process that sees no device, so
    a check that stops working ends in a launch error and never touches one."""
    import json
    import subprocess
    import sys
    code = LOSS_ARGS % dict(pkg=os.path.join(ROOT, "grendel-gs_b200"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    for case in ("B 0", "B 65", "row0 < 0", "row1 > H", "row1 < row0", "c0 < row0", "c1 > row1", "c1 < c0", "null gt",
                 "null gt, second view"):
        assert out[case] == [-1, -1], (case, out[case])                   # GS_EINVAL, forward and backward
    assert out["one byte short"][0] == -3                                  # GS_ENOMEM; the backward takes no size
    for case in ("valid", "valid, empty view without gt"):
        assert out[case] == [-2, -2], (case, out[case])                   # GS_ECUDA: passed every check, no device


def test_dropin_package_exports_reference_names():
    import diff_gaussian_rasterization as d
    from simple_knn._C import distCUDA2  # noqa: F401
    # the gsplat stub is opt-in (shims/): it must not shadow a real gsplat install on the package path (ADVICE r1)
    import importlib.util
    assert not os.path.exists(os.path.join(os.path.dirname(os.path.dirname(d.__file__)), "gsplat"))
    spec = importlib.util.spec_from_file_location("gsplat_stub", os.path.join(os.path.dirname(os.path.dirname(d.__file__)),
                                                                              "shims", "gsplat", "__init__.py"))
    gsplat = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gsplat)
    assert d._C.get_block_XY() == (16, 16, 256)
    for n in ("GaussianRasterizationSettings", "GaussianRasterizer"):
        assert hasattr(d, n)
    for n in ("get_local2j_ids_bool", "get_local2j_ids_bool_adjust_mode6", "get_block_XY"):
        assert hasattr(d._C, n)
    fields = d.GaussianRasterizationSettings._fields
    assert fields == ("image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
                      "projmatrix", "sh_degree", "campos", "prefiltered", "debug")
    for n in ("rasterization", "fully_fused_projection", "spherical_harmonics", "isect_tiles", "isect_offset_encode",
              "rasterize_to_pixels"):
        assert hasattr(gsplat, n)


def test_operator_refuses_cpu_tensors():
    """No CPU fallback: CPU tensors are rejected instead of silently computed elsewhere."""
    import torch
    import diff_gaussian_rasterization as d
    rs = d.GaussianRasterizationSettings(16, 16, 1.0, 1.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3,
                                         torch.zeros(3), False, False)
    r = d.GaussianRasterizer(raster_settings=rs)
    with pytest.raises(ValueError):
        r.preprocess_gaussians(torch.zeros(4, 3), torch.ones(4, 3), torch.ones(4, 4), torch.zeros(4, 16, 3),
                               torch.ones(4, 1), {})
