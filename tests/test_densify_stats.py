"""CPU: argument checks of gs_densify_stats (C ABI) and of gs_b200.densify.add_densification_stats.

The C-ABI calls run in a process that sees no device, so a check that stops working ends in a launch error (GS_ECUDA)
and never touches one.  The wrapper checks shapes, dtypes and contiguity before the device, so they are covered here
with CPU tensors, which it then refuses for being on the CPU."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CABI_ARGS = r"""
import ctypes, json, sys
sys.path.insert(0, %(pkg)r)
from gs_b200 import _lib
lib = _lib.load()
FAKE = 1 << 20   # a 16-byte aligned address that is never dereferenced: no device is visible to this process
vp = ctypes.c_void_p

def call(B=2, P=8, grads=None, radii=None, table_len=None, accum=FAKE, denom=FAKE, maxr=FAKE, no_tables=False):
    n = B if table_len is None else table_len
    g = (vp * max(n, 1))(*(grads or [FAKE + 64 * k for k in range(n)]))
    r = (vp * max(n, 1))(*(radii or [FAKE + 4096 + 64 * k for k in range(n)]))
    if no_tables:
        g = r = None
    return lib.gs_densify_stats(B, P, g, r, accum, denom, maxr, None)

out = {
    "B 0": call(B=0, table_len=1), "B 65": call(B=65), "B -1": call(B=-1, table_len=1), "P -1": call(P=-1),
    "null tables": call(no_tables=True), "null gradient entry": call(grads=[FAKE, None]),
    "null radii entry": call(radii=[None, FAKE]),
    "null accum": call(accum=None), "null denom": call(denom=None), "null max": call(maxr=None),
    "gradient 4 bytes off": call(grads=[FAKE, FAKE + 4]), "gradient 2 bytes off": call(grads=[FAKE + 2, FAKE]),
    "radii 2 bytes off": call(radii=[FAKE, FAKE + 2]),
    "accum 2 bytes off": call(accum=FAKE + 2), "denom 1 byte off": call(denom=FAKE + 1), "max 2 bytes off": call(maxr=FAKE + 2),
    "P 0": call(P=0), "valid": call(), "valid, 64 views": call(B=64), "valid, odd 4-byte outputs": call(accum=FAKE + 4),
}
out["error text"] = (lib.gs_densify_stats(0, 8, None, None, None, None, None, None), lib.gs_last_error().decode())
print(json.dumps(out))
"""


def test_cabi_refuses_before_any_launch():
    from gs_b200 import build
    build.build()
    code = CABI_ARGS % dict(pkg=os.path.join(ROOT, "grendel-gs_b200"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    for case in ("B 0", "B 65", "B -1", "P -1", "null tables", "null gradient entry", "null radii entry", "null accum",
                 "null denom", "null max", "gradient 4 bytes off", "gradient 2 bytes off", "radii 2 bytes off",
                 "accum 2 bytes off", "denom 1 byte off", "max 2 bytes off"):
        assert out[case] == -1, (case, out[case])                       # GS_EINVAL
    assert out["P 0"] == 0                                               # GS_OK: nothing to launch
    for case in ("valid", "valid, 64 views", "valid, odd 4-byte outputs"):
        assert out[case] == -2, (case, out[case])                       # GS_ECUDA: passed every check, no device
    rc, text = out["error text"]
    assert rc == -1 and "num_views" in text


def _inputs(B=3, P=10):
    return ((torch.zeros((P, 1)), torch.zeros((P, 1)), torch.zeros((P,))), torch.zeros((B, P, 2)),
            torch.ones((B, P), dtype=torch.int32))


@pytest.mark.parametrize("case", [
    "B 0", "B 65", "radii views != gradient views", "P mismatch between views", "P mismatch with the statistics",
    "gradients (P, 3)", "float64 gradients", "int64 radii", "float16 statistics", "accum (P,)", "max (P, 1)",
    "non-contiguous gradients", "non-contiguous accum", "None gradient", "None gradients", "CPU tensors",
    "statistics not tensors",
])
def test_wrapper_refuses(case):
    from gs_b200 import densify
    (a, d, m), g, r = _inputs()
    P = a.shape[0]
    exc = ValueError
    if case == "B 0":
        g, r = g[:0], r[:0]
    elif case == "B 65":
        g, r = g[[0] * 65], r[[0] * 65]
    elif case == "radii views != gradient views":
        r = r[:2]
    elif case == "P mismatch between views":
        g = [g[0], g[1][:-1], g[2]]
    elif case == "P mismatch with the statistics":
        g, r = g[:, :-1], r[:, :-1]
    elif case == "gradients (P, 3)":
        g = torch.zeros((3, P, 3))
    elif case == "float64 gradients":
        g, exc = g.double(), TypeError
    elif case == "int64 radii":
        r, exc = r.long(), TypeError
    elif case == "float16 statistics":
        d, exc = d.half(), TypeError
    elif case == "accum (P,)":
        a = a.reshape(-1)
    elif case == "max (P, 1)":
        m = m.reshape(-1, 1)
    elif case == "non-contiguous gradients":
        g = g.transpose(1, 2).contiguous().transpose(1, 2)
    elif case == "non-contiguous accum":
        a = torch.zeros((P, 2))[:, :1]
    elif case == "None gradient":
        g, exc = [g[0], None, g[2]], TypeError
    elif case == "None gradients":
        g, exc = None, TypeError
    elif case == "CPU tensors":
        exc = TypeError                      # well-formed, but on the CPU: there is no CPU path
    elif case == "statistics not tensors":
        a, exc = a.numpy(), TypeError
    with pytest.raises(exc):
        densify.add_densification_stats(a, d, m, g, r)
    assert not a.any() if isinstance(a, torch.Tensor) else True
