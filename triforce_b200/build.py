"""Builds libtriforce_b200.so (sm_90a, H100) in-tree with nvcc, and the C oracle helpers are not part of it.

    python -m triforce_b200.build            # build if stale
    python -m triforce_b200.build --force
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libtriforce_b200.so")
STAMP = os.path.join(LIB_DIR, "build.stamp")

SOURCES = ["abi.cu", "retrieval_build.cu", "verify_attn.cu", "decoder_ops.cu", "sampling.cu", "skinny_gemm.cu", "stream_linear.cu", "tree_attn_tc.cu", "allreduce.cu", "loop_graph.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--use_fast_math=false",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "--extended-lambda",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=...)")


def _fingerprint() -> str:
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + ["../../include/triforce_b200.h"]
    for f in files:
        p = os.path.normpath(os.path.join(CSRC, f))
        if os.path.isfile(p):
            h.update(f.encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    h.update((" ".join(NVCC_FLAGS) + os.environ.get("TF_EXTRA_NVCC_FLAGS", "")).encode())
    return h.hexdigest()


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() != _fingerprint()


def build(force: bool = False, verbose: bool = True) -> str:
    """Builds under an exclusive file lock into per-process temporaries and renames the finished library into place, so that
    concurrent callers (torchrun ranks, pytest-xdist workers) never load a half-written .so."""
    if not force and not is_stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    import fcntl
    with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():  # another process finished the build while we waited
                return LIB_PATH
            return _build_locked(verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose: bool) -> str:
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"] + os.environ.get("TF_EXTRA_NVCC_FLAGS", "").split()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIB_DIR, src.replace(".cu", f".{os.getpid()}.o"))
        cmd = [_nvcc(), *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src} ====\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(LIB_DIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    if failed:
        for o in objs:
            if os.path.exists(o):
                os.remove(o)
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed; see triforce_b200/lib/build.log")
    # default static cudart: the library is self-contained next to torch's own runtime (streams are driver handles)
    tmp_lib = LIB_PATH + f".{os.getpid()}.tmp"
    subprocess.check_call([_nvcc(), "-shared", "-o", tmp_lib, *objs])
    os.replace(tmp_lib, LIB_PATH)
    for o in objs:
        os.remove(o)
    with open(STAMP + ".tmp", "w") as f:
        f.write(_fingerprint())
    os.replace(STAMP + ".tmp", STAMP)
    if verbose:
        print(f"[triforce_b200] built {LIB_PATH}")
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
