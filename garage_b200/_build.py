"""In-tree build of libgarage_ec.so (sm_90a only; nvcc cross-compiles without a GPU)."""
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
SO = os.path.join(PKG, "libgarage_ec.so")
SOURCES = ["garage_ec.cu"]
DEPS = ["garage_ec.cu", "rs_kernels.cuh", "clay_kernels.cuh", "sse_kernels.cuh", "gf256.h", "gf256_tables.inc", "blake2b.h"]


def nvcc_path():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def nvcc_cmd(out=SO, extra=()):
    return [
        nvcc_path(), "-O3", "-std=c++17",
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-lineinfo", "-Xcompiler", "-fPIC,-O3", "-shared",
        "-I", os.path.join(ROOT, "include"),
        *extra,
        "-o", out,
        *[os.path.join(CSRC, s) for s in SOURCES],
    ]


def stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, d) for d in DEPS] + [os.path.join(ROOT, "include", "garage_ec.h")]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def _multi_rank():
    return int(os.environ.get("WORLD_SIZE", "1")) > 1


def _wait_for(path, seconds=600):
    import time

    t0 = time.time()
    while not os.path.exists(path):
        if time.time() - t0 > seconds:
            raise RuntimeError("timed out waiting for %s to be built by local rank 0" % path)
        time.sleep(0.5)
    return path


def build(force=False, verbose=False):
    """Compile the CUDA extension if sources are newer than the .so (or force).  Under
    torchrun only local rank 0 ever compiles, and only when the library is missing (a stale
    mtime after the snapshot copy must not make 8 ranks race on one output file)."""
    if not force:
        if os.path.exists(SO) and (_multi_rank() or not stale()):
            return SO
        if _multi_rank() and int(os.environ.get("LOCAL_RANK", "0")) != 0:
            return _wait_for(SO)
    if not all(os.path.exists(os.path.join(CSRC, d)) for d in DEPS):
        raise RuntimeError("garage_b200/csrc sources missing")
    tmp = SO + ".tmp%d" % os.getpid()
    cmd = nvcc_cmd(out=tmp, extra=("-Xptxas", "-v") if verbose else ())
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    os.replace(tmp, SO)  # atomic: a concurrent loader never sees a half-written library
    if verbose:
        print(r.stderr)
    return SO


BM_SO = os.path.join(PKG, "libgarage_block.so")
BM_SOURCES = [os.path.join(CSRC, "block_manager.cpp"), os.path.join(CSRC, "shard_wire.cpp"), os.path.join(CSRC, "placement.cpp")]
BM_DEPS = BM_SOURCES + [os.path.join(ROOT, "include", "garage_block_manager.h"), os.path.join(ROOT, "include", "garage_ec.h"),
                        os.path.join(ROOT, "include", "garage_shard_wire.h"), os.path.join(ROOT, "include", "garage_placement.h"),
                        os.path.join(CSRC, "blake2b.h")]


def build_block_manager(force=False):
    """C++ host mirror of BlockManager (libgarage_block.so): plain g++, links only the C ABI."""
    build(force=False)
    if not force and os.path.exists(BM_SO):
        fresh = (all(os.path.getmtime(d) <= os.path.getmtime(BM_SO) for d in BM_DEPS if os.path.exists(d))
                 and os.path.getmtime(SO) <= os.path.getmtime(BM_SO))
        if fresh or _multi_rank():
            return BM_SO
    if not force and _multi_rank() and int(os.environ.get("LOCAL_RANK", "0")) != 0:
        return _wait_for(BM_SO)
    cxx = os.environ.get("CXX") or shutil.which("g++") or "g++"
    cmd = [cxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-Wall", "-Wextra",
           "-I", os.path.join(ROOT, "include"), *BM_SOURCES, "-L", PKG, "-lgarage_ec",
           "-Wl,-rpath,$ORIGIN", "-o", BM_SO + ".tmp%d" % os.getpid()]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    os.replace(cmd[-1], BM_SO)
    return BM_SO


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_block_manager(force="--force" in sys.argv))
