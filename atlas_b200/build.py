"""In-tree build of `lib/libatlas_b200.so` with nvcc for sm_90a (H100; no JIT cache: the library is built next to the
sources by `__graft_entry__.build()`).  Every .cu under csrc/ is compiled to an object file in
parallel (only the stale ones), then linked into one shared library."""
import glob
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
OBJ_DIR = os.path.join(LIB_DIR, "obj")
LIB = os.path.join(LIB_DIR, "libatlas_b200.so")

NVCC_FLAGS = [
    "-Xcompiler", "-fPIC", "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
]
LINK_FLAGS = ["-shared", "-Xcompiler", "-fPIC", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _headers():
    deps = glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh"))
    deps.append(os.path.join(os.path.dirname(HERE), "include", "atlas_b200.h"))
    return deps


def _obj(src):
    return os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library.  Returns the library path."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdrs = _headers()
    todo = [s for s in sources() if force or _stale(_obj(s), [s] + hdrs)]
    logs = []

    def compile_one(src):
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", _obj(src), src]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
        return res.stderr

    if todo:
        with ThreadPoolExecutor(max_workers=min(len(todo), os.cpu_count() or 4)) as pool:
            logs = list(pool.map(compile_one, todo))
    objs = [_obj(s) for s in sources()]
    if todo or _stale(LIB, objs):
        cmd = [_nvcc()] + LINK_FLAGS + ["-o", LIB] + objs
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("link failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose:
        print("\n".join(logs))
    return LIB


if __name__ == "__main__":
    import sys

    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
