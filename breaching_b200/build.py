"""Build the sm_90a (H100) shared library in-tree (``breaching_b200/lib/libbreaching_b200.so``).

nvcc cross-compiles without a GPU.  The library is a build product and git-ignored.  Usage:
``python -m breaching_b200.build [--force]``.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libbreaching_b200.so")
SOURCES = ["engine.cu", "igemm_simt.cu", "igemm_tc.cu", "layers.cu", "objective.cu", "tokens.cu", "analysis.cu", "linear_small.cu", "stem_cols.cu", "augment.cu", "lbfgs.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math=false",
    "-Xcompiler", "-fPIC,-O3,-Wall", "-Xptxas", "-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _source_hash():
    """Content hash of everything the library is built from (mtimes do not survive copying the tree to another machine)."""
    import hashlib

    h = hashlib.sha256()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(HERE, "..", "include", "breaching_b200.h")]
    for path in files:
        h.update(os.path.basename(path).encode())
        with open(path, "rb") as handle:
            h.update(handle.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


STAMP = os.path.join(LIBDIR, "build.stamp")


def needs_build():
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as handle:
        return handle.read().strip() != _source_hash()


def build(force=False, verbose=False):
    """Idempotent and safe under concurrent callers (one process per GPU all call it): file lock + atomic rename."""
    import fcntl

    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not needs_build():  # another process built it while we waited
            return LIB
        objs = []
        flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
        for src in SOURCES:
            obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
            cmd = [_nvcc(), *flags, "-c", os.path.join(CSRC, src), "-o", obj]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if verbose or res.returncode != 0:
                sys.stderr.write(res.stdout + res.stderr)
            if res.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src}")
            with open(obj + ".ptxas.log", "w") as handle:
                handle.write(res.stderr)
            objs.append(obj)
        tmp = LIB + f".tmp{os.getpid()}"
        cmd = [_nvcc(), "-shared", "-o", tmp, *objs, "-lcudart", "-lcuda"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError("link failed")
        os.replace(tmp, LIB)
        with open(STAMP, "w") as handle:
            handle.write(_source_hash())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
