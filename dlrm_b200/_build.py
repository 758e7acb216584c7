"""Build libdlrm_b200.so in-tree with nvcc for sm_90a (H100).  The library is built ahead of time by
`__graft_entry__.build()` and loaded from the tree, so a run needs no compiler and no JIT cache."""
import glob
import hashlib
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdlrm_b200.so")
STAMP = os.path.join(LIBDIR, "libdlrm_b200.stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "--use_fast_math=false",
]
NVCC_FLAGS = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _digest():
    """Hash of the sources' CONTENTS and names -- not of their absolute paths: a library built once must count as
    fresh in any copy of the tree (a path-dependent digest would make every first process of a copied tree rebuild
    the library, all ranks of a torchrun at once)."""
    h = hashlib.sha256()
    for f in sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [
            os.path.join(os.path.dirname(HERE), "include", "dlrm_b200.h")]:
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def is_fresh():
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == _digest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into lib/libdlrm_b200.so.  Returns the path."""
    if not force and is_fresh():
        return LIB
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libdlrm_b200.so")
    os.makedirs(LIBDIR, exist_ok=True)
    # One builder at a time (the ranks of a torchrun all arrive here together): an exclusive lock, a re-check once it
    # is held, output to a private file that is renamed into place -- nobody ever maps a half-written library.
    import fcntl

    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and is_fresh():
                return LIB
            tmp = LIB + ".tmp.%d" % os.getpid()
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + sources()
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
            if verbose:
                print(r.stderr)
            os.replace(tmp, LIB)
            with open(STAMP + ".tmp", "w") as fh:
                fh.write(_digest())
            os.replace(STAMP + ".tmp", STAMP)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
