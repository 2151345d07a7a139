"""Builds libmvsmpl.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m mvsmplfitting_b200.build [--force]
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
OUT = os.path.join(_HERE, "libmvsmpl.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def source_files():
    return sorted(sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(_HERE, "..", "include", "*.h")))


def source_hash() -> str:
    """sha256 over every source the library is compiled from (file names + contents): the build id.  It is compiled into
    the library (-DMVS_BUILD_ID, exported by mvs_build_id()) so that a stale libmvsmpl.so can be told from a fresh one
    (__graft_entry__.smoke and tests/test_abi.py compare the two)."""
    import hashlib
    h = hashlib.sha256()
    for p in source_files():
        h.update(os.path.basename(p).encode())
        h.update(open(p, "rb").read())
    return h.hexdigest()[:16]


def built_id() -> str | None:
    """the build id inside the existing libmvsmpl.so, read from the file (never dlopen a library that may be rebuilt next)"""
    if not os.path.exists(OUT):
        return None
    blob = open(OUT, "rb").read()
    i = blob.find(b"MVS_BUILD_ID=")
    if i < 0:
        return None
    j = blob.find(b"\0", i)
    return blob[i + len(b"MVS_BUILD_ID="):j].decode(errors="replace")


def needs_build() -> bool:
    return built_id() != source_hash()


def build_debug() -> str:
    """libmvsmpl_dbg.so with -DMVS_PHASE_DBG (per-phase clock stamps in frame_step_kernel); profiling scripts only"""
    out = os.path.join(_HERE, "libmvsmpl_dbg.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-DMVS_PHASE_DBG", '-DMVS_BUILD_ID="%s-dbg"' % source_hash(), "-o", out] + sources() + ["-lcuda"])
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    cmd = [nvcc] + NVCC_FLAGS + ['-DMVS_BUILD_ID="%s"' % source_hash()] + (["-Xptxas", "-v"] if verbose else []) + \
        ["-o", OUT] + sources() + ["-lcuda"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    if "--debug" in sys.argv:
        print(build_debug())
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
