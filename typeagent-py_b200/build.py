"""Build libtavec.so (the C-ABI CUDA library) in-tree for sm_90a (H100).

    python typeagent-py_b200/build.py [--force]

nvcc cross-compiles without a GPU.  The library is written next to this file so that it
travels to the GPU box with the repo snapshot.  cudart is linked statically: the library
shares the CUDA primary context (and stream/event handles) with whatever else is in the
process (e.g. torch), but not a libcudart.so.
"""

from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libtavec.so")
STAMP = os.path.join(HERE, ".libtavec.stamp")
SOURCES = ["tav_api.cu", "tav_scan.cu", "tav_mma.cu", "tav_group.cu", "tav_sort.cu", "tav_merge_range.cu",
           "tav_compact.cu", "tav_multi.cu", "tav_leaders.cu"]
HEADERS = ["tav_common.cuh", "tav_internal.h", "tav_ptx.cuh", "../../include/tavec.h"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xptxas=-v",
    "-Xcompiler", "-fPIC,-O3,-Wall",
    "-shared", "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    for name in SOURCES + HEADERS + [os.path.basename(__file__)]:
        path = os.path.join(CSRC, name) if name != os.path.basename(__file__) else __file__
        with open(path, "rb") as f:
            h.update(name.encode() + b"\0" + f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


HOST_LIB = os.path.join(HERE, "libtavhost.so")
HOST_SRC = os.path.join(CSRC, "tav_pyhost.c")


def build_host_helper(force: bool = False) -> str | None:
    """libtavhost.so: a CPython-API helper of the Python host layer (list[int] -> int64 buffer).  Optional:
    without it (no Python.h, no gcc) `vectorbase.py` converts through array('q'), 14 us slower."""
    import sysconfig

    if not force and os.path.exists(HOST_LIB) and os.path.getmtime(HOST_LIB) >= os.path.getmtime(HOST_SRC):
        return HOST_LIB
    include = sysconfig.get_paths()["include"]
    if not os.path.exists(os.path.join(include, "Python.h")):
        return None
    cmd = [os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-Wall", f"-I{include}", "-o", HOST_LIB, HOST_SRC]
    try:
        proc = subprocess.run(cmd, capture_output=True, text=True)
    except OSError:
        return None
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        return None
    return HOST_LIB


def build(force: bool = False, verbose: bool = False) -> str:
    build_host_helper(force)
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == digest:
                return LIB
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB, *[os.path.join(CSRC, s) for s in SOURCES]]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed ({proc.returncode}): {' '.join(cmd)}")
    with open(os.path.join(HERE, "build_ptxas.log"), "w") as f:
        f.write(proc.stdout + proc.stderr)
    with open(STAMP, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
