"""Build the sm_90a shared library in-tree (``lib/libflmr_maxsim.so``).

nvcc cross-compiles without a GPU; the resulting .so is git-ignored but travels to the GPU box
with the repository snapshot.  Used by ``__graft_entry__.build()`` and lazily by ``_cabi`` when the
library is missing or older than its sources.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libflmr_maxsim.so")
SOURCES = [os.path.join(CSRC, "flmr_maxsim.cu")]
HEADERS = sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(PKG_DIR, "..", "include", "flmr_maxsim.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
]


def find_nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libflmr_maxsim.so")
    return nvcc


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.exists(f) and os.path.getmtime(f) > t for f in SOURCES + HEADERS)


DEBUG_LIB_PATH = os.path.join(LIB_DIR, "libflmr_maxsim_debug.so")


def build(force: bool = False, verbose: bool = False, debug: bool = False) -> str:
    """Compile the library if missing/stale; returns its path.

    ``debug=True`` builds ``libflmr_maxsim_debug.so`` with ``-DFLMR_DEBUG``: the timing-experiment
    instantiation of the scan kernel and the ``FLMR_DEBUG_MODE`` / ``FLMR_LANE_RBQ`` / ``FLMR_NUM_CTAS`` /
    ``FLMR_ARGMAX_SIMT`` environment knobs exist only there (tools/ select it with ``FLMR_MAXSIM_LIB``);
    the release library reads no environment variables."""
    if debug:
        return _compile(DEBUG_LIB_PATH, ["-DFLMR_DEBUG"], verbose)
    if not force and not is_stale():
        return LIB_PATH
    return _compile(LIB_PATH, [], verbose)


def _compile(out_path: str, extra: list, verbose: bool) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    tmp = out_path + ".tmp.%d" % os.getpid()
    cmd = [find_nvcc(), *NVCC_FLAGS, *extra, "-o", tmp, *SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (proc.stdout, proc.stderr))
    if verbose:
        print(proc.stderr)
    os.replace(tmp, out_path)
    return out_path


if __name__ == "__main__":
    import sys
    print(build(force=True, verbose=True, debug="--debug" in sys.argv))
