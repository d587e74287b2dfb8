"""Builds warpx_b200/libpic_b200.so (CUDA kernels + C ABI) for sm_90a (H100), in-tree, with nvcc.  The digest of the
sources and flags it was built from is kept in warpx_b200/build/libpic_b200.so.sha256."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpic_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
         "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
# The fluid kernels restate the reference's arithmetic operation by operation: no multiply-add contraction there.
FILE_FLAGS = {"fluid.cu": ["-fmad=false"]}


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def digest():
    """SHA-256 over everything the library is built from: the CUDA sources, the C header and the nvcc flags."""
    import hashlib
    h = hashlib.sha256(" ".join([NVCC] + FLAGS + sorted(str(v) for v in FILE_FLAGS.items())).encode())
    deps = sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(HERE, "..", "include", "pic_b200.h")]
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stamp(lib):
    return os.path.join(os.path.dirname(lib), "build", os.path.basename(lib) + ".sha256")


def stale(lib=LIB):
    """True when lib is missing or was built from other sources or flags.  Compares contents, not modification times,
    so that a copied or re-checked-out tree whose library is current is used as it is."""
    try:
        with open(_stamp(lib)) as f:
            return not os.path.exists(lib) or f.read().strip() != digest()
    except OSError:
        return True


def build(force=False, verbose=False, extra=(), lib=LIB):
    """Compile every translation unit and link lib (default: in-tree); object files go to build/ beside it."""
    if not force and not stale(lib):
        return lib
    objdir = os.path.dirname(_stamp(lib))
    os.makedirs(objdir, exist_ok=True)
    want = digest()
    procs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + FLAGS + FILE_FLAGS.get(os.path.basename(src), []) + list(extra) + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    ok = True
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or (verbose and out):
            sys.stderr.write(out.decode())
        ok = ok and p.returncode == 0
    if not ok:
        raise RuntimeError("nvcc failed")
    tmp = lib + ".tmp.%d" % os.getpid()            # link beside the target, then rename: never a half-written library
    cmd = [NVCC, "-shared"] + ARCH + ["-o", tmp] + objs + ["-lcudart"]
    subprocess.run(cmd, check=True)
    os.replace(tmp, lib)
    with open(_stamp(lib), "w") as f:
        f.write(want + "\n")
    return lib


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True,
          extra=["-Xptxas", "-v"] if "--ptxas" in sys.argv else [])
    print(LIB)
