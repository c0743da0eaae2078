"""Builds lib/libgrendel_gs_b200.so from csrc/*.cu with nvcc for sm_90a (cross-compiles without a GPU).

The library has no torch dependency: it is a plain CUDA + C-ABI shared object (include/grendel_gs_b200.h)
that the Python host side binds with ctypes.  The built .so stays in-tree (git-ignored) under lib/.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
OBJDIR = os.path.join(PKG, "build")
LIB = os.path.join(LIBDIR, "libgrendel_gs_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "--expt-relaxed-constexpr", "-Xptxas", "-v"]
# translation units whose fp32 chain must match the oracle op for op (tile indices bit-exact)
PER_FILE = {"preprocess.cu": ["-fmad=false"]}


def nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(PKG, "..", "include", "grendel_gs_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defs=(), variant=None):
    """Compile every .cu for sm_90a and link the shared library. Returns the library path.
    defs / variant: tuning builds -- extra -D flags, linked as lib/libgrendel_gs_b200.<variant>.so (selected at run time
    with GS_B200_LIB=<path>; A/B of compile-time parameters in one device call)."""
    lib_out, objdir = LIB, OBJDIR
    if variant:
        lib_out = os.path.join(LIBDIR, f"libgrendel_gs_b200.{variant}.so")
        objdir = os.path.join(PKG, "build", variant)
        force = True
    if not force and not is_stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(objdir, exist_ok=True)
    cc = nvcc()
    logs = {}

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [cc, *ARCH, *COMMON, *PER_FILE.get(src, []), *defs, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs[src] = r.stderr
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    tmp_out = lib_out + f".tmp{os.getpid()}"   # linked beside the target and renamed: a reader never sees half a library
    cmd = [cc, *ARCH, "-shared", "-o", tmp_out, *objs, "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp_out, lib_out)
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        for k in sorted(logs):
            f.write(f"==== {k}\n{logs[k]}\n")
    if verbose:
        for k in sorted(logs):
            print(f"==== {k}\n{logs[k]}")
    return lib_out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
