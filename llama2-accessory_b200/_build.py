"""Build libb200decode.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

Staleness is decided by a content hash of the sources (file times do not survive the copy to the GPU box), and the
build is serialised with a file lock so that the ranks of a multi-process launch never compile concurrently."""
import fcntl
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = ["api.cu", "gemv.cu", "gemv1.cu", "mega1.cu", "mega2.cu", "attn.cu", "prefill.cu", "moe.cu", "sample.cu", "pack.cpp"]
HDR = ["common.cuh", "gemv_core.cuh", "gemv1_core.cuh", "ll.cuh"]
OUT = os.path.join(HERE, "libb200decode.so")
STAMP = OUT + ".srchash"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-shared"]


def _source_hash():
    h = hashlib.sha256()
    files = [os.path.join(HERE, "csrc", f) for f in SRC + HDR]
    files.append(os.path.join(os.path.dirname(HERE), "include", "b200_decode.h"))
    for f in files:
        h.update(os.path.basename(f).encode())
        h.update(open(f, "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _stale():
    if not os.path.isfile(OUT) or not os.path.isfile(STAMP):
        return True
    return open(STAMP).read().strip() != _source_hash()


def build(force=False, verbose=False):
    if not force and not _stale():
        return OUT
    with open(os.path.join(HERE, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not _stale():  # another process built it while we waited
                return OUT
            nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
            if not os.path.isfile(nvcc):
                nvcc = "nvcc"
            tmp = OUT + f".tmp{os.getpid()}"
            cmd = [nvcc] + FLAGS + ["-o", tmp] + [os.path.join(HERE, "csrc", f) for f in SRC]
            if verbose:
                print(" ".join(cmd))
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
            os.replace(tmp, OUT)
            with open(STAMP, "w") as f:
                f.write(_source_hash())
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose=True))
