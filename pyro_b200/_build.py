"""Build the native library in-tree with nvcc for sm_90a (H100).

``libpyro_b200.so`` (the C-ABI of include/pyro_b200.h; pure CUDA runtime, no torch types) and
``libpyro_b200_hostcheck.so`` (test-only CPU build of the element functors and the NUTS core).
Objects go to ``build/``; the shared objects sit next to this file (git-ignored), so the package is
importable from the source tree.  Staleness is decided by a content hash of the sources (file times
do not survive a copy of the tree), stored next to each library.
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(ROOT, "build")
LIB = os.path.join(HERE, "libpyro_b200.so")
HOSTCHECK = os.path.join(HERE, "libpyro_b200_hostcheck.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                     "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets"]
HOST_ONLY = {"hostcheck.cu"}


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; cannot build libpyro_b200.so")
    return exe


def _files():
    hdrs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    hdrs += [os.path.join(ROOT, "include", f) for f in sorted(os.listdir(os.path.join(ROOT, "include")))]
    srcs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")]
    return hdrs, srcs


def _hash(paths, extra=""):
    h = hashlib.sha256(extra.encode())
    for p in paths:
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stamp_ok(lib, digest):
    stamp = lib + ".hash"
    if not (os.path.exists(lib) and os.path.exists(stamp)):
        return False
    with open(stamp) as f:
        return f.read().strip() == digest


def _write_stamp(lib, digest):
    with open(lib + ".hash", "w") as f:
        f.write(digest)


def _run(cmd, what):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("%s failed:\n%s\n%s\n%s" % (what, " ".join(cmd), r.stdout, r.stderr))


def build(force=False, verbose=False):
    hdrs, srcs = _files()
    dev_srcs = [s for s in srcs if os.path.basename(s) not in HOST_ONLY]
    dev_digest = _hash(hdrs + dev_srcs, " ".join(NVCC_FLAGS))
    if force or not _stamp_ok(LIB, dev_digest):
        os.makedirs(BUILD, exist_ok=True)
        hdr_digest = _hash(hdrs, " ".join(NVCC_FLAGS))
        jobs, objs = [], []
        for src in dev_srcs:
            obj = os.path.join(BUILD, os.path.basename(src)[:-3] + ".o")
            objs.append(obj)
            d = _hash([src], hdr_digest)
            if force or not _stamp_ok(obj, d):
                jobs.append((src, obj, d))
        if verbose:
            print("[pyro_b200] compiling %d CUDA sources for sm_90a" % len(jobs), file=sys.stderr)

        def one(job):
            src, obj, d = job
            _run([_nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj], "nvcc " + os.path.basename(src))
            _write_stamp(obj, d)

        if jobs:
            with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
                list(ex.map(one, jobs))
        _run([_nvcc()] + ARCH + ["-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                                  "-o", LIB] + objs + ["-lcudart"], "link libpyro_b200.so")
        _write_stamp(LIB, dev_digest)
    host_srcs = [s for s in srcs if os.path.basename(s) in HOST_ONLY]
    host_digest = _hash(hdrs + host_srcs, "hostcheck")
    if force or not _stamp_ok(HOSTCHECK, host_digest):
        _run([_nvcc(), "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
              "-Wno-deprecated-gpu-targets"] + host_srcs + ["-o", HOSTCHECK], "hostcheck build")
        _write_stamp(HOSTCHECK, host_digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
