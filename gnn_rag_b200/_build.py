"""Build libgnnrag_b200.so in-tree with nvcc for sm_90a (no torch headers, plain C ABI).

The .so and the objects are build products (git-ignored).  ``build()`` is a no-op when
the library is newer than every source file.  Each ``csrc/*.cu`` is compiled to its own object (in parallel,
only when it or a header changed) under ``build/`` and the objects are linked into the shared library."""
import glob
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.path.join(HERE, "libgnnrag_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
OBJ_DIR = os.path.join(HERE, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _headers():
    return glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(INCLUDE, "*.h"))


def _deps():
    return sources() + _headers()


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(p) > t for p in _deps())


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libgnnrag_b200.so")
    return nvcc


def _compile_one(nvcc, src, obj, verbose):
    cmd = [nvcc] + NVCC_FLAGS + ["-I", INCLUDE, "-c", "-o", obj, src]
    if verbose:
        print(" ".join(cmd))
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed on %s:\n%s%s" % (os.path.basename(src), res.stdout, res.stderr))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdr_t = max([os.path.getmtime(p) for p in _headers()] + [os.path.getmtime(__file__)])
    jobs, objs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_t):
            jobs.append((src, obj))
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4) or 1) as ex:
        for f in [ex.submit(_compile_one, nvcc, s, o, verbose) for s, o in jobs]:
            f.result()
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH + ".tmp"] + objs
    if verbose:
        print(" ".join(cmd))
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc link failed:\n" + res.stdout + res.stderr)
    os.replace(LIB_PATH + ".tmp", LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    import sys
    print(build(force="--incremental" not in sys.argv, verbose=True))
