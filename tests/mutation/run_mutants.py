"""Mutation runner for the kernels of catalogue.py: which deliberately wrong kernel does the suite let through?

    python tests/mutation/run_mutants.py --build            # no GPU needed: nvcc cross-compiles
    python tests/mutation/run_mutants.py --run [--jobs N]   # on an H100; writes the kill matrix (JSON)
    python tests/mutation/run_mutants.py --merge a.json,b.json --out m.json   # combine runs (and earlier merged matrices)

--build copies csrc/ (with include/) once per mutant of catalogue.py into tests/mutation/build/<id>/ (git-ignored), applies that one
mutant (its original snippet must occur exactly once), compiles only the mutated .cu with the flags of
gs_b200/build.py (ARCH, COMMON, PER_FILE) and links it with the unmutated objects of the other sources into
build/<id>/libgrendel_gs_b200.so.  The unmutated library is built the same way into build/base/.  lib/ and the
package's own build directory are never touched.

--run runs the unmutated library first: it must pass the whole selection, or the run stops.  Then, for each mutant,
one pytest child process runs the test files of catalogue.SELECTION for its source file with GS_B200_LIB pointing at
the mutant's library (gs_b200/_lib.py loads that file instead of lib/).  Inside a child this module is loaded as a
pytest plugin: after a file's first failing test the rest of that file is skipped, since one failure decides the
file's verdict.  Every child is waited for (and killed at --timeout); nothing is left running.

The JSON holds, per mutant, the first failing test of every selected file (null = the mutant survived that file),
whether the files that existed before the mutation tests killed it, and whether the whole selection does.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(ROOT, "grendel-gs_b200")
CSRC = os.path.join(PKG, "csrc")
BUILD = os.path.join(HERE, "build")
LIBNAME = "libgrendel_gs_b200.so"

# ---- pytest plugin (active only in the child processes, which set GS_MUTATION_REPORT) ----------------------------------
_failed = {}      # test file -> first failing node id
_counts = {}      # test file -> {outcome: n}


def _file_of(nodeid):
    return nodeid.split("::", 1)[0]


def pytest_runtest_setup(item):
    if os.environ.get("GS_MUTATION_REPORT") and _file_of(item.nodeid) in _failed:
        import pytest
        pytest.skip("an earlier test of this file already failed on this library")


def pytest_runtest_logreport(report):
    if not os.environ.get("GS_MUTATION_REPORT"):
        return
    f = _file_of(report.nodeid)
    c = _counts.setdefault(f, {})
    if report.failed:
        _failed.setdefault(f, report.nodeid)
        c["failed"] = c.get("failed", 0) + 1
    elif report.when == "call" or report.skipped:
        key = "passed" if report.passed else "skipped"
        c[key] = c.get(key, 0) + 1


def pytest_sessionfinish(session, exitstatus):
    path = os.environ.get("GS_MUTATION_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(failed=_failed, counts=_counts, exitstatus=int(exitstatus)), f)


# ---- build --------------------------------------------------------------------------------------------------------------
def _catalogue():
    sys.path.insert(0, HERE)
    import catalogue
    return catalogue


def _edits(m):
    orig = m.original if isinstance(m.original, tuple) else (m.original,)
    repl = m.replacement if isinstance(m.replacement, tuple) else (m.replacement,)
    assert len(orig) == len(repl), m.id
    return list(zip(orig, repl))


def mutate(m, text):
    """The source text with mutant m applied; raises unless every original snippet occurs exactly once."""
    for orig, repl in _edits(m):
        n = text.count(orig)
        if n != 1:
            raise SystemExit(f"{m.id}: snippet occurs {n} times in {m.file} (must be exactly once): {orig!r}")
        text = text.replace(orig, repl)
    return text


def _bld():
    sys.path.insert(0, PKG)
    from gs_b200 import build as b
    return b


def _copy_sources(d):
    """csrc/ and include/ under d in the repository's layout (common.cuh includes ../../include/...); returns csrc."""
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(d, "include"))
    shutil.copytree(CSRC, os.path.join(d, "pkg", "csrc"))
    return os.path.join(d, "pkg", "csrc")


def _compile(b, src_dir, name, obj):
    cmd = [b.nvcc(), *b.ARCH, *b.COMMON, *b.PER_FILE.get(name, []), "-c", os.path.join(src_dir, name), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src_dir}/{name}:\n{r.stderr[-4000:]}")


def _link(b, objs, out):
    tmp = out + f".tmp{os.getpid()}"
    r = subprocess.run([b.nvcc(), *b.ARCH, "-shared", "-o", tmp, *objs, "-cudart", "static"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed for {out}:\n{r.stderr[-4000:]}")
    os.replace(tmp, out)


def build_all(cat, ids, jobs):
    b = _bld()
    sources = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    # every snippet is checked before anything is compiled
    texts = {}
    for m in cat.MUTANTS:
        if m.id in ids:
            with open(os.path.join(CSRC, m.file)) as f:
                texts[m.id] = mutate(m, f.read())
    base = os.path.join(BUILD, "base")
    shutil.rmtree(base, ignore_errors=True)
    base_src = _copy_sources(base)
    t0 = time.time()
    with ThreadPoolExecutor(max_workers=jobs) as ex:
        list(ex.map(lambda s: _compile(b, base_src, s, os.path.join(base, s.replace(".cu", ".o"))), sources))
    _link(b, [os.path.join(base, s.replace(".cu", ".o")) for s in sources], os.path.join(base, LIBNAME))
    print(f"[build] base: {len(sources)} sources in {time.time() - t0:.0f} s", flush=True)

    def one(m):
        d = os.path.join(BUILD, m.id)
        shutil.rmtree(d, ignore_errors=True)
        src = _copy_sources(d)
        with open(os.path.join(src, m.file), "w") as f:
            f.write(texts[m.id])
        obj = os.path.join(d, m.file.replace(".cu", ".o"))
        _compile(b, src, m.file, obj)
        objs = [obj if s == m.file else os.path.join(base, s.replace(".cu", ".o")) for s in sources]
        _link(b, objs, os.path.join(d, LIBNAME))
        return m.id

    t0 = time.time()
    todo = [m for m in cat.MUTANTS if m.id in ids]
    with ThreadPoolExecutor(max_workers=jobs) as ex:
        for mid in ex.map(one, todo):
            print(f"[build] {mid} ok", flush=True)
    print(f"[build] {len(todo)} mutants in {time.time() - t0:.0f} s", flush=True)


# ---- run ----------------------------------------------------------------------------------------------------------------
def run_child(lib, files, timeout, extra):
    """One pytest process over `files` with GS_B200_LIB=lib; returns (report dict, seconds)."""
    fd, report = tempfile.mkstemp(prefix="gs_mutation_", suffix=".json")
    os.close(fd)
    env = dict(os.environ, GS_B200_LIB=lib, GS_MUTATION_REPORT=report,
               PYTHONPATH=os.pathsep.join([HERE] + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep) if p]))
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "run_mutants", "-p", "no:cacheprovider",
           *extra, *files]
    t0 = time.time()
    try:
        r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)
        out = r.stdout[-3000:]
        with open(report) as f:
            rep = json.load(f)
    except subprocess.TimeoutExpired:   # subprocess.run killed and reaped the child
        rep, out = dict(failed={f: "timeout" for f in files}, counts={}, exitstatus=-1), "timeout"
    except (OSError, ValueError):       # the child died before writing its report
        rep = dict(failed={f: "no report" for f in files}, counts={}, exitstatus=-2)
    finally:
        if os.path.exists(report):
            os.remove(report)
    rep["tail"] = out
    return rep, time.time() - t0


def _summary(cat, rows):
    live = [r for r in rows if not r["equivalent"]]
    files = sorted({r["file"] for r in rows})
    return dict(
        mutants=len(rows), equivalent=len(rows) - len(live),
        killed_before={f: sum(r["killed_before"] for r in live if r["file"] == f) for f in files},
        killed_after={f: sum(r["killed"] for r in live if r["file"] == f) for f in files},
        total={f: sum(r["file"] == f for r in live) for f in files},
        survived_before=[r["id"] for r in live if not r["killed_before"]],
        survivors=[r["id"] for r in live if not r["killed"]])


def merge(cat, paths, out_path):
    """One kill matrix from runs over parts of the selection (e.g. --before-only, then --after-only): a mutant's
    verdicts per file are combined, killed_before comes from the BEFORE files alone.  A path may also be an earlier
    merged matrix: its runs and rows are carried over as they are."""
    rows, runs = {}, []
    for p in paths:
        with open(p) as f:
            d = json.load(f)
        runs += d["runs"] if "runs" in d else [dict(baseline=d["baseline"], summary=d["summary"])]
        for r in d["mutants"]:
            row = rows.setdefault(r["id"], dict(r, killed_by={}, seconds=0.0))
            row["killed_by"].update(r["killed_by"])
            row["seconds"] = round(row["seconds"] + r["seconds"], 1)
    for row in rows.values():
        row["equivalent"] = cat.EQUIVALENT.get(row["id"])   # the catalogue's current verdict
        before = set(cat.SELECTION[row["file"]]["BEFORE"])
        row["killed_before"] = any(v for f, v in row["killed_by"].items() if f in before)
        row["killed"] = any(row["killed_by"].values())
    order = {m.id: i for i, m in enumerate(cat.MUTANTS)}
    result = dict(runs=runs, mutants=sorted(rows.values(), key=lambda r: order[r["id"]]))
    result["summary"] = _summary(cat, result["mutants"])
    with open(out_path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["summary"]))


def run_all(cat, ids, jobs, timeout, out_path, extra, part=None):
    """part: None (the whole selection), "BEFORE" or "AFTER" (that half only)."""
    sel = {k: [f for h in ("BEFORE", "AFTER") if part in (None, h) for f in v[h]] for k, v in cat.SELECTION.items()}
    todo = [m for m in cat.MUTANTS if m.id in ids]
    all_files = sorted({f for m in todo for f in sel[m.file]})
    for f in all_files:
        if not os.path.exists(os.path.join(ROOT, f)):
            raise SystemExit(f"selected test file missing: {f}")
    base_lib = os.path.join(BUILD, "base", LIBNAME)
    for p in [base_lib] + [os.path.join(BUILD, i, LIBNAME) for i in ids]:
        if not os.path.exists(p):
            raise SystemExit(f"{p} missing: run --build first")
    t_start = time.time()
    rep, dt = run_child(base_lib, all_files, timeout, extra)
    base_counts = rep["counts"]
    print(f"[run] baseline: {dt:.0f} s, failed {rep['failed']}, counts {base_counts}", flush=True)
    if rep["failed"] or rep["exitstatus"] != 0:
        print(rep["tail"])
        raise SystemExit("the unmutated library does not pass the selection")
    result = dict(baseline=dict(files=all_files, seconds=round(dt, 1), counts=base_counts), mutants=[])

    def one(m):
        files = sel[m.file]
        r, t = run_child(os.path.join(BUILD, m.id, LIBNAME), files, timeout, extra)
        before = set(cat.SELECTION[m.file]["BEFORE"])
        killed_by = {f: r["failed"].get(f) for f in files}
        row = dict(id=m.id, file=m.file, models=m.models, equivalent=cat.EQUIVALENT.get(m.id),
                   killed_before=any(killed_by[f] for f in files if f in before),
                   killed=any(killed_by.values()), killed_by=killed_by, seconds=round(t, 1))
        print(f"[run] {m.id} {'KILLED' if row['killed'] else 'SURVIVED'} (before: "
              f"{'killed' if row['killed_before'] else 'survived'}) {t:.0f} s {killed_by}", flush=True)
        return row

    with ThreadPoolExecutor(max_workers=jobs) as ex:
        result["mutants"] = list(ex.map(one, todo))
    result["summary"] = dict(_summary(cat, result["mutants"]), jobs=jobs, wall_seconds=round(time.time() - t_start, 1))
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["summary"]))
    return result


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--build", action="store_true", help="build the baseline and every mutant (no GPU needed)")
    ap.add_argument("--run", action="store_true", help="run the selection against the baseline and every mutant")
    ap.add_argument("--only", default="", help="comma-separated mutant ids (default: all)")
    ap.add_argument("--jobs", type=int, default=min(8, os.cpu_count() or 1),
                    help="parallel compilations (--build) or pytest children sharing the GPU (--run)")
    ap.add_argument("--timeout", type=float, default=1200.0, help="seconds per pytest child")
    ap.add_argument("--out", default=os.path.join(BUILD, "kill_matrix.json"))
    ap.add_argument("--part", choices=("BEFORE", "AFTER"), help="run only that half of the selection")
    ap.add_argument("--merge", default="", help="comma-separated kill matrices to combine into --out (runs nothing)")
    ap.add_argument("--list", action="store_true", help="print the catalogue and check every snippet")
    args, extra = ap.parse_known_args()
    cat = _catalogue()
    ids = [m.id for m in cat.MUTANTS]
    assert len(set(ids)) == len(ids), "duplicate mutant ids"
    if args.only:
        want = args.only.split(",")
        unknown = set(want) - set(ids)
        if unknown:
            raise SystemExit(f"unknown mutant ids: {sorted(unknown)}")
        ids = [i for i in ids if i in want]
    if args.list:
        for m in cat.MUTANTS:
            with open(os.path.join(CSRC, m.file)) as f:
                mutate(m, f.read())
            print(f"{m.id} {m.file:14s} {m.models}")
    if args.build:
        build_all(cat, set(ids), args.jobs)
    if args.run:
        run_all(cat, ids, args.jobs, args.timeout, args.out, extra, args.part)
    if args.merge:
        merge(cat, args.merge.split(","), args.out)
    if not (args.build or args.run or args.list or args.merge):
        ap.print_help()


if __name__ == "__main__":
    main()
