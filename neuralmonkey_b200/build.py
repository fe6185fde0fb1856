"""In-tree build of libnmb200.so (sm_90a, H100) with plain nvcc.

The shared library is written next to this file (git-ignored), so the package
is importable from the repository tree.  `python -m neuralmonkey_b200.build`
rebuilds what is out of date; `--force` rebuilds everything.
"""
import concurrent.futures
import os
import shutil
import subprocess
import sys
from typing import List

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
OBJ_DIR = os.path.join(PKG_DIR, "build")
LIB_PATH = os.path.join(PKG_DIR, "libnmb200.so")
HEADER = os.path.join(os.path.dirname(PKG_DIR), "include", "nmb200.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libnmb200.so")
    return nvcc


def sources() -> List[str]:
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime() -> float:
    deps = [HEADER] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)
                       if f.endswith((".cuh", ".h"))]
    return max(os.path.getmtime(d) for d in deps)


def _compile(src: str, force: bool) -> str:
    obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
    src_path = os.path.join(CSRC, src)
    newest = max(os.path.getmtime(src_path), _deps_mtime())
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= newest:
        return obj
    cmd = [_nvcc()] + NVCC_FLAGS + ["-c", src_path, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed for {}:\n{}\n{}".format(
            src, res.stdout, res.stderr))
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every csrc/*.cu for sm_90a and link libnmb200.so."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = sources()
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as pool:
        objs = list(pool.map(lambda s: _compile(s, force), srcs))
    need_link = (force or not os.path.exists(LIB_PATH)
                 or any(os.path.getmtime(o) > os.path.getmtime(LIB_PATH)
                        for o in objs))
    if need_link:
        # link beside the target and rename: a reader (or a snapshot of the tree) never sees half a library
        tmp_path = LIB_PATH + ".tmp.{}".format(os.getpid())
        cmd = [_nvcc(), "-shared", "-o", tmp_path] + objs + [
            "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            if os.path.exists(tmp_path):
                os.remove(tmp_path)
            raise RuntimeError("link failed:\n{}\n{}".format(
                res.stdout, res.stderr))
        os.replace(tmp_path, LIB_PATH)
        if verbose:
            print("linked", LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
