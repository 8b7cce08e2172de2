"""Build libcogview_b200.so in-tree with nvcc for sm_90a (no torch dependency in the library).

    python -m cogview_b200.csrc.build [--force] [--verbose]

Objects are compiled in parallel and cached by source mtime; the shared library lands next to this
file (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
LIB = os.path.join(HERE, "libcogview_b200.so")
OBJ_DIR = os.path.join(HERE, "build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", os.path.join(ROOT, "include"),
]


def sources():
    return sorted(f for f in os.listdir(HERE) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(ROOT, "include", "cogview_b200.h"))
    return max(os.path.getmtime(h) for h in hs)


def _compile(src, force, verbose):
    obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
    spath = os.path.join(HERE, src)
    if not force and os.path.exists(obj):
        if os.path.getmtime(obj) >= max(os.path.getmtime(spath), _headers_mtime()):
            return obj, None
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", spath, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, (r.stdout + r.stderr)


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    objs = [o for o, _ in results]
    rebuilt = [log for _, log in results if log is not None]
    if verbose:
        for log in rebuilt:
            sys.stderr.write(log)
    if rebuilt or not os.path.exists(LIB) or force:
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
