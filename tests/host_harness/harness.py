"""TEST INFRASTRUCTURE -- the host harness: the product's CUDA sources executed on the host, for a container
without a GPU.  Four builds, all into tests/host_harness/_build/, none of them part of the product:

  lib()           the thin kernels of lwfa.cu / charge.cu / nci.cu: `__host__ __device__` bodies behind a launch
                  macro; -DPIC_HOST_HARNESS turns the launches into host loops over the same thread ids (nvcc,
                  host code only);
  simt()          deposit_runs.cu and gather_push_tile.cu, unmodified, under the SIMT emulator of simt_host.h
                  (g++; every CUDA thread a cooperative fiber, warp collectives as lock-step exchanges);
  host_library()  EVERY file of warpx_b200/csrc -- kernels, argument builders, the C++ step driver -- through the
                  launch-syntax transformer of cuda2host.py and the same emulator: the product's C ABI on the host;
                  host_simulation_class() drives it with warpx_b200.engine.Simulation, run_ranks() runs several
                  "ranks" as threads over the NCCL stand-in of fake_nccl.cpp.

They check indexing, lane roles, step sequence and arithmetic against the oracle; they prove nothing about races,
launch geometry, device memory or speed -- the `-m gpu` tests do that through the real library -- and they are
never imported by the product package."""
import ctypes as C
import os
import subprocess

from warpx_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "warpx_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libpic_lwfa_host.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SRCS = ["lwfa.cu", "charge.cu", "nci.cu", "runtime.cu"]
PROBES = [os.path.join(HERE, "shape_probe.cu")]
_LIB = None


def build():
    deps = [os.path.join(CSRC, f) for f in SRCS + ["lwfa_body.cuh", "harness_launch.cuh", "pic_common.cuh"]] + \
           [os.path.join(ROOT, "include", "pic_b200.h")] + PROBES
    if os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cmd = [NVCC, "-DPIC_HOST_HARNESS", "-O2", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC",
           "-Xcompiler", "-ffp-contract=off", "--fmad=false", "--expt-relaxed-constexpr",
           "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", OUT] + \
          ["-I", CSRC] + [os.path.join(CSRC, f) for f in SRCS] + PROBES + ["-lcudart"]
    subprocess.run(cmd, check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return OUT


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    L = C.CDLL(build())
    fabp, soap, gp = C.POINTER(abi.pic_fab), C.POINTER(abi.pic_soa), C.POINTER(abi.pic_geom)
    bp, lp, jp = C.POINTER(abi.pic_boundaries), C.POINTER(abi.pic_laser_antenna), C.POINTER(abi.pic_plasma_injector)
    dp, ip, vp = abi.c_double_p, abi.c_int_p, C.c_void_p
    for name, (res, args) in abi.LWFA_SIGNATURES(fabp, soap, gp, bp, lp, jp, dp, ip, vp).items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L.pic_host_shape.restype, L.pic_host_shape.argtypes = C.c_int, [C.c_int, C.c_double, dp]
    L.pic_host_shifted_shape.restype, L.pic_host_shifted_shape.argtypes = C.c_int, [C.c_int, C.c_double, C.c_int, dp]
    L.pic_set_error_mode.argtypes = [C.c_int]
    L.pic_last_error.restype = C.c_char_p
    L.pic_set_error_mode(abi.PIC_ERR_RETURN)
    _LIB = L
    return L


# --------------------------------------------------------------------------------------------
# SIMT emulation of the warp-level kernels (simt_host.h): the kernel SOURCE of csrc/deposit_runs.cu
# compiled by g++ with every CUDA thread as a cooperative fiber.
# --------------------------------------------------------------------------------------------
SIMT_OUT = os.path.join(HERE, "_build", "libpic_simt.so")
_SIMT = None


def build_simt():
    deps = [os.path.join(HERE, "simt_host.h"), os.path.join(HERE, "simt_deposit.cpp"), os.path.join(HERE, "simt_gather.cpp"),
            os.path.join(ROOT, "include", "pic_b200.h")] + \
           [os.path.join(CSRC, f) for f in ("deposit_runs.cu", "deposit_common.cuh", "pic_common.cuh", "runtime.cu",
                                            "gather_push_tile.cu", "gather_common.cuh", "bins.cuh")]
    if os.path.exists(SIMT_OUT) and all(os.path.getmtime(d) <= os.path.getmtime(SIMT_OUT) for d in deps):
        return SIMT_OUT
    os.makedirs(os.path.dirname(SIMT_OUT), exist_ok=True)
    cuda = os.path.dirname(os.path.dirname(NVCC))
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-DPIC_SIMT_HOST", "-include",
           os.path.join(HERE, "simt_host.h"), "-x", "c++", "-I", os.path.join(cuda, "include"), "-I", CSRC,
           "-ffp-contract=off", "-Wno-attributes", "-Wno-unknown-pragmas",
           os.path.join(HERE, "simt_deposit.cpp"), os.path.join(HERE, "simt_gather.cpp"), os.path.join(CSRC, "runtime.cu"),
           "-o", SIMT_OUT,
           "-L", os.path.join(cuda, "lib64"), "-lcudart"]
    subprocess.run(cmd, check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return SIMT_OUT


def simt():
    global _SIMT
    if _SIMT is not None:
        return _SIMT
    L = C.CDLL(build_simt())
    fabp, soap = C.POINTER(abi.pic_fab), C.POINTER(abi.pic_soa)
    L.simt_deposit_runs.restype = C.c_int
    L.simt_deposit_runs.argtypes = [soap, C.c_long, C.c_long, fabp, abi.c_double_p, abi.c_double_p, abi.c_int_p,
                                    C.c_double, C.c_double, C.c_double, C.c_int, C.c_int]
    L.simt_gather_push.restype = C.c_int
    L.simt_gather_push.argtypes = [soap, fabp, fabp, abi.c_double_p, abi.c_double_p, abi.c_int_p, C.c_double, C.c_double,
                                   C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(abi.pic_bins), C.c_int]
    _SIMT = L
    return L


# --------------------------------------------------------------------------------------------
# The WHOLE library on the host: every file of warpx_b200/csrc (kernels, argument builders, the C++ step
# driver engine.cu) compiled by g++ against the SIMT emulator, through the source transformer of cuda2host.py
# (kernel<<<...>>>(...) -> SIMT_LAUNCH).  "Device" memory is host memory.  Same C ABI as the product library.
# --------------------------------------------------------------------------------------------
HOST_OUT = os.path.join(HERE, "_build", "libpic_host.so")
_HOST = None


def build_host_library():
    from . import cuda2host
    src_dir = os.path.join(HERE, "_build", "host_src")
    srcs = cuda2host.transform_tree(CSRC, src_dir)
    deps = srcs + [os.path.join(src_dir, f) for f in os.listdir(src_dir) if f.endswith(".cuh")] + \
        [os.path.join(HERE, "simt_host.h"), os.path.join(ROOT, "include", "pic_b200.h")]
    if os.path.exists(HOST_OUT) and all(os.path.getmtime(d) <= os.path.getmtime(HOST_OUT) for d in deps):
        return HOST_OUT
    cuda = os.path.dirname(os.path.dirname(NVCC))
    common = ["/usr/bin/g++", "-std=c++17", "-O1", "-fPIC", "-DPIC_SIMT_HOST", "-DPIC_HOST_HARNESS", "-include",
              os.path.join(HERE, "simt_host.h"), "-I", os.path.join(cuda, "include"), "-I", src_dir,
              "-ffp-contract=off", "-Wno-attributes", "-Wno-unknown-pragmas"]
    import concurrent.futures
    objs = [s[:-4] + ".o" for s in srcs]

    def one(so):
        src, obj = so
        if os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(d) for d in deps if not d.endswith(".cpp") or d == src):
            return
        subprocess.run(common + ["-c", src, "-o", obj], check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        list(ex.map(one, zip(srcs, objs)))
    subprocess.run(["/usr/bin/g++", "-shared", "-o", HOST_OUT] + objs + ["-L", os.path.join(cuda, "lib64"), "-lcudart", "-ldl"],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return HOST_OUT


def host_library():
    """The product's C ABI, executed on the host (ctypes signatures of warpx_b200.lib.bind)."""
    global _HOST
    if _HOST is None:
        from warpx_b200 import lib as piclib
        # PIC_HOST_LIBRARY: a differently built copy (e.g. -fsanitize=address, see tools/host_asan.sh)
        L = piclib.bind(C.CDLL(os.environ.get("PIC_HOST_LIBRARY") or build_host_library()))
        L.pic_set_error_mode(abi.PIC_ERR_RETURN)
        _HOST = L
    return _HOST


def host_simulation_class():
    """warpx_b200.engine.Simulation driving the host library: CPU tensors hold the "device" arrays, there are no
    streams.  Single rank, C++ step driver."""
    import torch
    from warpx_b200.engine import Simulation

    class HostSimulation(Simulation):
        def _backend(self, device):
            return torch, host_library(), torch.device("cpu")

        @property
        def stream(self):
            return None

        def _sync(self):
            pass

    return HostSimulation


# --------------------------------------------------------------------------------------------
# Several "ranks" on the host: threads of this process, each with its own engine instance of the host library,
# exchanging through fake_nccl.cpp (selected with PIC_NCCL_LIBRARY) -- the multi-rank paths of the C++ step driver
# (NCCL halo sweeps, particle migration, slabs along a non-periodic axis) without a GPU.
# --------------------------------------------------------------------------------------------
FAKE_NCCL = os.path.join(HERE, "_build", "libpic_fake_nccl.so")


def _build_nccl_standin(out, defines):
    src = os.path.join(HERE, "fake_nccl.cpp")
    if not os.path.exists(out) or os.path.getmtime(src) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        tmp = "%s.tmp.%d" % (out, os.getpid())
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-pthread"] + defines +
                       ["-o", tmp, src, "-ldl"], check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        os.replace(tmp, out)
    return out


def build_fake_nccl():
    return _build_nccl_standin(FAKE_NCCL, [])


# The same stand-in over DEVICE buffers (-DPIC_STANDIN_DEVICE): ranks as threads of one process driving the real
# library on one GPU, each on its own stream (tests/test_gpu_multirank.py).
DEVICE_NCCL = os.path.join(HERE, "_build", "libpic_standin_nccl_device.so")


def build_device_nccl():
    return _build_nccl_standin(DEVICE_NCCL, ["-DPIC_STANDIN_DEVICE"])


class ThreadDist:
    """The few torch.distributed calls warpx_b200.engine.Simulation makes, between threads."""

    class ReduceOp:
        SUM, MAX = "sum", "max"

    class _Shared:
        def __init__(self, world):
            import threading
            self.world = world
            self.barrier = threading.Barrier(world)
            self.slots = [None] * world

    def __init__(self, shared, rank):
        self.shared, self.rank = shared, rank

    def get_rank(self):
        return self.rank

    def get_world_size(self):
        return self.shared.world

    def barrier(self):
        self.shared.barrier.wait()

    def broadcast(self, tensor, src):
        sh = self.shared
        if self.rank == src:
            sh.slots[src] = tensor.clone()
        sh.barrier.wait()
        if self.rank != src:
            tensor.copy_(sh.slots[src])
        sh.barrier.wait()

    def all_reduce(self, tensor, op=None):
        import torch
        sh = self.shared
        sh.slots[self.rank] = tensor.clone()
        sh.barrier.wait()
        stack = torch.stack(sh.slots)
        res = stack.max(dim=0).values if op == self.ReduceOp.MAX else stack.sum(dim=0)
        sh.barrier.wait()
        tensor.copy_(res)


def run_ranks(world, fn):
    """fn(rank, dist) on `world` threads; returns the list of results (re-raises the first exception)."""
    import threading
    os.environ["PIC_NCCL_LIBRARY"] = build_fake_nccl()
    host_library()                       # build / load once, before the threads start
    shared = ThreadDist._Shared(world)
    out, err = [None] * world, [None] * world

    def target(r):
        try:
            out[r] = fn(r, ThreadDist(shared, r))
        except BaseException as e:       # noqa: BLE001 -- reported to the caller below
            err[r] = e
            shared.barrier.abort()
    threads = [threading.Thread(target=target, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in err:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    for e in err:
        if e is not None:
            raise e
    return out
