"""Builds opendwm_b200/libdwm_b200.so (sm_90a) in-tree with nvcc.

Usage: python -m opendwm_b200.build [--debug-wait] [--force]

The shared library is the C-ABI boundary declared in include/dwm_b200.h.  It is
built in-tree (git-ignored) so that it travels to the GPU box with the repo
snapshot.  nvcc cross-compiles without a GPU.
"""
import argparse
import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libdwm_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
    "-std=c++17", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(
        os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_digest(extra):
    h = hashlib.sha256()
    for root in (CSRC, INCLUDE):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(f.encode())
                    h.update(fh.read())
    h.update(" ".join(extra).encode())
    return h.hexdigest()


def _compile(src, obj, flags, log):
    cmd = ["nvcc", *flags, "-I", INCLUDE, "-c", src, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError(
            "nvcc failed for {}:\n{}".format(src, res.stdout + res.stderr))
    return obj


def build(debug_wait=False, force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    flags = list(NVCC_FLAGS)
    if debug_wait:
        flags.append("-DDWM_BOUNDED_WAIT")
    digest = _deps_digest(flags)
    stamp = os.path.join(BUILD, "stamp")
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        with open(stamp) as f:
            if f.read().strip() == digest:
                return LIB

    srcs = _sources()
    objs = []
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        futs = []
        for s in srcs:
            base = os.path.splitext(os.path.basename(s))[0]
            obj = os.path.join(BUILD, base + ".o")
            log = os.path.join(BUILD, base + ".log")
            futs.append(ex.submit(_compile, s, obj, flags, log))
        for f in futs:
            objs.append(f.result())
    cmd = ["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
           "-o", LIB, *objs]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    with open(stamp, "w") as f:
        f.write(digest)
    if verbose:
        for s in srcs:
            base = os.path.splitext(os.path.basename(s))[0]
            with open(os.path.join(BUILD, base + ".log")) as f:
                sys.stdout.write(f.read())
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--debug-wait", action="store_true",
                    help="bounded mbarrier spins that trap instead of hanging")
    ap.add_argument("--force", action="store_true")
    ap.add_argument("-v", "--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.debug_wait, a.force, a.verbose))
