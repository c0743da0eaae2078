"""CPU checks of the --zhx_time / --zhx_debug logs (gs_b200.statlog, ops._gpu_time): the files the formatters write from
known numbers parse, with the reference's own analyze_statistic.py parsers, back to those numbers; the logging rule of
cuda_args; the profiler's state around a logging call; and gs_render_forward{,_batched}_ts refusing a misaligned
tile_stats pointer before any launch."""
import ast
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

from gs_b200 import ops, statlog

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANALYZE = "/root/reference/analyze_statistic.py"

# the stage keys analyze_statistic.py sums per iteration (:1972-1991)
GPU_FORWARD = ["10 preprocess time", "24 updateDistributedStatLocally.updateTileTouched time", "30 InclusiveSum time",
               "40 duplicateWithKeys time", "50 SortPairs time", "60 identifyTileRanges time", "70 render time",
               "81 sum_n_render time", "82 sum_n_consider time", "83 sum_n_contrib time"]
GPU_BACKWARD = ["b10 render time", "b20 preprocess time"]


@pytest.fixture(scope="module")
def parsers():
    """The reference's two log parsers and their helpers, loaded with ast: the module itself imports matplotlib."""
    if not os.path.exists(ANALYZE):
        pytest.skip("the reference checkout is not present")
    with warnings.catch_warnings():   # the module's regex literals are not raw strings
        warnings.simplefilter("ignore", SyntaxWarning)
        tree = ast.parse(open(ANALYZE).read())
    want = {"extract_json_from_gpu_time_log", "extract_json_from_n_contrib_log", "get_number_prefix",
            "get_number_tuple_prefix"}
    mod = ast.Module(body=[n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want], type_ignores=[])
    ns = {"os": os, "json": json}
    exec(compile(mod, ANALYZE, "exec"), ns)
    assert want <= set(ns)
    return ns


def cuda_args(folder, **kw):
    a = dict(mode="train", world_size="2", global_rank="1", local_rank="1", log_folder=str(folder), log_interval="250",
             iteration="1", zhx_debug="False", zhx_time="False", stats_collector={})
    a.update(kw)
    return a


def test_stage_keys_are_the_analyzer_columns():
    keys = [k for call in ("preprocess forward", "render forward", "render backward", "preprocess backward")
            for k, _ in ops.REFERENCE_STAGE_KEYS[call]]
    assert keys == GPU_FORWARD + GPU_BACKWARD
    if os.path.exists(ANALYZE):
        src = open(ANALYZE).read()
        for k in keys:
            assert f'"{k}"' in src, k
    t = ops.reference_stage_times("render forward", {"70 render": (1.5, 1), "50 SortPairs": (0.25, 2)})
    d = dict(t)
    assert d["70 render time"] == 1.5 and d["50 SortPairs time"] == 0.25 and d["40 duplicateWithKeys time"] == 0.0
    assert d["81 sum_n_render time"] == d["82 sum_n_consider time"] == d["83 sum_n_contrib time"] == 0.0


def test_gpu_time_log_parses_back(parsers, tmp_path):
    log = statlog.request(cuda_args(tmp_path, zhx_time="True"))
    path = log.path("gpu_time")
    assert os.path.basename(path) == "gpu_time_ws=2_rk=1.log"
    blocks = [(1, "preprocess forward", [("10 preprocess time", 0.291950)]),
              (1, "render forward", [(k, 0.125 * (j + 1)) for j, k in enumerate(GPU_FORWARD[1:])]),
              (1, "render backward", [("b10 render time", 3.0)]),
              (1, "preprocess backward", [("b20 preprocess time", 1e-7)]),     # printed with 6 decimals: 0.000000
              (251, "preprocess forward", [("10 preprocess time", 12.5)])]
    for it, call, times in blocks:
        statlog.append(path, statlog.gpu_time_text(it, f"rk=1, ws=2, {call}", times))
    got = parsers["extract_json_from_gpu_time_log"](path)
    want = [{"iteration": 1, "10 preprocess time": 0.29195, "b10 render time": 3.0, "b20 preprocess time": 0.0,
             **{k: 0.125 * (j + 1) for j, k in enumerate(GPU_FORWARD[1:])}},
            {"iteration": 251, "10 preprocess time": 12.5}]
    assert got == want


def test_n_contrib_log_parses_back(parsers, tmp_path):
    H, W = 40, 50                         # 3 x 4 tiles, ragged on both edges
    T = 12
    cl = np.array([0, 1, 1, 0, 1, 1, 1, 0, 0, 1, 0, 1], bool)
    rng = np.random.default_rng(3)
    n = np.where(cl, rng.integers(0, 300, T), 0)
    n[5] = 0                              # an empty local tile: range (0, 0)
    ends = np.cumsum(n)
    ranges = np.stack([ends - n, ends], 1)
    ranges[n == 0] = 0
    walked = np.where(cl, rng.integers(0, 256 * 300, T), 0)
    blended = np.where(cl, rng.integers(0, 256 * 50, T), 0)
    walked[5] = blended[5] = 0
    ts = np.stack([n, walked, blended], 1).astype(np.int64)
    log = statlog.request(cuda_args(tmp_path, zhx_debug="True"))
    path = log.path("n_contrib")
    assert os.path.basename(path) == "n_contrib_ws=2_rk=1.log"
    for it in (1, 251):
        statlog.append(path, statlog.n_contrib_text(it, log.local_rank, log.world_size, H, W, cl, ranges, ts))
    statlog.append(path, statlog.n_contrib_text(501, 1, 2, H, W, np.zeros(T, bool), ranges, ts))   # nothing local
    got = parsers["extract_json_from_n_contrib_log"](path)
    assert [b["iteration"] for b in got] == [1, 251]
    local = np.nonzero(cl)[0]
    R = int(n.sum())
    for b in got:
        assert len(b["data"]) == local.size
        for d, t in zip(b["data"], local):
            assert d["iteration"] == b["iteration"]
            assert d["tile"] == (int(t) // 4, int(t) % 4)
            assert d["range"] == (int(ranges[t, 1]), int(ranges[t, 0]))
            assert d["num_rendered_this_tile"] == n[t]
            assert d["n_considered_per_pixel"] == round(walked[t] / 256, 6)
            assert d["n_contrib2loss_per_pixel"] == round(blended[t] / 256, 6)
        assert b["stats"] == {"iteration": b["iteration"], "local_rank": 1, "world_size": 2, "num_tiles": int(local.size),
                              "num_pixels": H * W, "num_rendered": R,
                              "global_ave_n_rendered_per_pix": round(R / local.size, 6),
                              "global_ave_n_considered_per_pix": round(int(walked.sum()) / (H * W), 6),
                              "global_ave_n_contrib2loss_per_pix": round(int(blended.sum()) / (H * W), 6)}


def test_n_contrib_line_reproduces_the_parser_example():
    """The example tile line above the parser (analyze_statistic.py:917): 138 entries, range (1639, 1501), every entry
    walked by all 256 pixels, 19824 blends."""
    ts = np.array([[138, 138 * 256, 19824]], np.int64)
    text = statlog.n_contrib_text(1, 0, 1, 16, 16, np.ones(1, bool), np.array([[1501, 1639]]), ts)
    assert text.splitlines()[0] == ("iteration: 1, tile: (0, 0), range: (1639, 1501), num_rendered_this_tile: 138, "
                                    "n_considered_per_pixel: 138.000000, n_contrib2loss_per_pixel: 77.437500, "
                                    "contrib2loss_ratio: 0.302490")


def test_logging_rule(tmp_path):
    on = dict(zhx_time="True", zhx_debug="True")
    r = statlog.request(cuda_args(tmp_path, **on))
    assert r is not None and r.time and r.debug and r.iteration == 1
    assert statlog.request(cuda_args(tmp_path, iteration="251", zhx_time="True")).time
    for off in (dict(iteration="2"), dict(iteration="250"), dict(mode="test", iteration="-1"), dict(mode="test"),
                dict(zhx_time="False", zhx_debug="False"), dict(zhx_time="true", zhx_debug="1")):
        assert statlog.request(cuda_args(tmp_path, **{**on, **off})) is None, off
    r = statlog.request(cuda_args(tmp_path, zhx_debug="True"))
    assert r.debug and not r.time
    for a in (None, {}, {"stats_collector": {}}, dict(mode="train", zhx_time="True")):
        assert statlog.request(a) is None


@pytest.fixture(scope="module")
def lib():
    from gs_b200 import build, _lib
    build.build()
    return _lib.load()


def test_gpu_time_restores_the_profiler(lib, tmp_path):
    """A logging call switches the profiler on for its own launches and back to the state it found; the times a caller
    had collected survive into that caller's next read; a call that does not log touches nothing."""
    from gs_b200 import _lib
    log = statlog.request(cuda_args(tmp_path, zhx_time="True"))
    path = log.path("gpu_time")
    assert not _lib.PROFILE_ON
    with ops._gpu_time(None, "render forward"):
        assert not _lib.PROFILE_ON
    with ops._gpu_time(statlog.request(cuda_args(tmp_path, zhx_debug="True")), "render forward"):
        assert not _lib.PROFILE_ON
    assert not os.path.exists(path)
    with ops._gpu_time(log, "render forward"):
        assert _lib.PROFILE_ON
    assert not _lib.PROFILE_ON
    text = open(path).read().splitlines()
    assert text[0].startswith("it=1,") and len(text) == 1 + len(GPU_FORWARD) - 1
    _lib.profile_enable(True)
    try:
        _lib.profile_carry({"70 render": (2.0, 1)})            # stands for the caller's own records
        with ops._gpu_time(log, "render backward"):
            assert _lib.PROFILE_ON
        assert _lib.PROFILE_ON
        assert _lib.profile_read() == {"70 render": (2.0, 1)}
    finally:
        _lib.profile_enable(False)


TS_ARGS = r"""
import ctypes, json, sys
sys.path.insert(0, %(pkg)r)
from gs_b200 import _lib
lib = _lib.load()
FAKE = 1 << 20   # an address that is never dereferenced: no device is visible to this process
vs = (ctypes.c_int32 * 2)(0, 4)

def call(name, ts, R=0):
    # means2D .. sort_temp, sort_temp_bytes, ranges .. stats, tile_stats, seg_ws, seg_ws_bytes, stream
    args = [FAKE] * 12 + [1 << 30] + [FAKE] * 5 + [ts] + [FAKE, 1 << 30, None]
    if name == "gs_render_forward_ts":
        return lib.gs_render_forward_ts(4, R, 32, 32, *args)
    return lib.gs_render_forward_batched_ts(1, vs, R, 32, 32, *args)

out = {}
for name in ("gs_render_forward_ts", "gs_render_forward_batched_ts"):
    out[name] = {"misaligned": call(name, FAKE + 4), "misaligned, R > 0": call(name, FAKE + 12, R=5),
                 "aligned": call(name, FAKE + 8), "null": call(name, None)}
print(json.dumps(out))
"""


def test_tile_stats_pointer_checks(lib):
    """gs_render_forward{,_batched}_ts refuse a tile_stats pointer that is not 8-byte aligned before any launch (GS_EINVAL)
    and accept NULL or an aligned one.  The calls run in a process that sees no device, so a check that stops working
    ends in a launch error and never touches one."""
    code = TS_ARGS % dict(pkg=os.path.join(ROOT, "grendel-gs_b200"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    for name, rc in out.items():
        assert rc["misaligned"] == -1 and rc["misaligned, R > 0"] == -1, (name, rc)   # GS_EINVAL
        assert rc["aligned"] == -2 and rc["null"] == -2, (name, rc)                   # GS_ECUDA: passed every check
