"""Build libdib_b200.so (the C-ABI library of include/dib_b200.h) in-tree with nvcc for the H100 (sm_90a).

The .so is a build product (git-ignored).  No torch headers are involved: the library is plain CUDA C++ behind an
extern "C" surface.

Every translation unit is compiled to its own object (in parallel, cached by content hash under csrc/_obj/) and the
objects are linked into a temporary file that is renamed over the library, all under an fcntl lock, so that N ranks
importing the package at once cannot interleave writes.  The source stamp hashes file CONTENTS under relative names:
the same tree at another path matches.  A stale prebuilt library is never used silently.
"""
import fcntl
import hashlib
import os
import shutil
import subprocess
import sys
import warnings
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
OBJ_DIR = os.path.join(CSRC, "_obj")
LIB_PATH = os.path.join(PKG_DIR, "libdib_b200.so")
STAMP = LIB_PATH + ".srchash"
HEADERS = [os.path.join(PKG_DIR, "..", "include", h) for h in ("dib_b200.h", "dib_b200_test_hooks.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _headers():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + HEADERS


def _digest(paths, extra=b""):
    h = hashlib.sha256()
    for f in paths:
        if not os.path.isfile(f):
            continue
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode() + b"\0" + fh.read() + b"\0")
    h.update(" ".join(NVCC_FLAGS).encode() + extra)
    return h.hexdigest()


def _hash():
    with open(__file__, "rb") as fh:
        me = fh.read()
    return _digest(_sources() + _headers(), hashlib.sha256(me).digest())


def nvcc_path():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _stamp_matches(want):
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == want


def _compile_one(nvcc, src, hdr_digest, verbose):
    key = _digest([src], hdr_digest.encode())[:24]
    obj = os.path.join(OBJ_DIR, os.path.basename(src) + "." + key + ".o")
    if os.path.exists(obj):
        return obj, ""
    for old in os.listdir(OBJ_DIR):                      # drop stale objects of this source
        if old.startswith(os.path.basename(src) + "."):
            os.unlink(os.path.join(OBJ_DIR, old))
    tmp = obj + f".tmp{os.getpid()}"
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", tmp, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed on {os.path.basename(src)}:\n" + res.stdout + res.stderr)
    os.replace(tmp, obj)
    return obj, res.stderr


def build_library(force=False, verbose=False):
    """Compile if the sources changed (or force).  Returns the library path."""
    want = _hash()
    if not force and _stamp_matches(want):
        return LIB_PATH
    nvcc = nvcc_path()
    if nvcc is None:
        if os.path.exists(LIB_PATH):
            warnings.warn("libdib_b200.so does not match the csrc/ sources and nvcc is not available to rebuild it: "
                          "using the prebuilt library AS IS", RuntimeWarning)
            return LIB_PATH
        raise RuntimeError("nvcc not found and no prebuilt libdib_b200.so")
    os.makedirs(OBJ_DIR, exist_ok=True)
    with open(os.path.join(PKG_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and _stamp_matches(want):       # another rank built it while we waited
                return LIB_PATH
            if force:
                for old in os.listdir(OBJ_DIR):
                    os.unlink(os.path.join(OBJ_DIR, old))
            hdr = _digest(_headers())
            srcs = _sources()
            with ThreadPoolExecutor(max_workers=min(len(srcs), os.cpu_count() or 4)) as ex:
                outs = list(ex.map(lambda s: _compile_one(nvcc, s, hdr, verbose), srcs))
            tmp = LIB_PATH + f".tmp{os.getpid()}"
            res = subprocess.run([nvcc] + NVCC_FLAGS[:2] + ["-shared", "-o", tmp] + [o for o, _ in outs],
                                 capture_output=True, text=True)
            if res.returncode != 0:
                raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
            os.replace(tmp, LIB_PATH)
            if verbose:
                print("".join(log for _, log in outs))
            with open(STAMP + ".tmp", "w") as fh:
                fh.write(want)
            os.replace(STAMP + ".tmp", STAMP)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB_PATH


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
