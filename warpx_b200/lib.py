"""Loader of the C-ABI shared library (warpx_b200/libpic_b200.so).

There is no CPU fallback: if the library is missing, or was built from other sources, it is built with nvcc (sm_90a
cross-compiles without a GPU); if that fails, or a kernel is requested without a CUDA device, the call raises.
"""
import ctypes as C
import os

from . import abi, build as _build

_LIB = None


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.LIB
    if not os.path.exists(path) or (os.path.isdir(_build.CSRC) and os.path.exists(_build.NVCC) and _build.stale()):
        path = _rebuild()
    _LIB = bind(C.CDLL(path))
    _LIB.pic_apply_env_defaults()
    return _LIB


def _rebuild():
    """Build the library from the current sources: in-tree when the package directory is writable, otherwise (a
    read-only install) into a per-user directory under the system's temporary directory, never into the tree."""
    import fcntl
    import tempfile
    if os.access(_build.HERE, os.W_OK):
        where, target = _build.HERE, _build.LIB
    else:
        where = os.path.join(tempfile.gettempdir(), "warpx_b200-%d" % os.getuid(), _build.digest()[:16])
        os.makedirs(where, exist_ok=True)
        target = os.path.join(where, os.path.basename(_build.LIB))
    # one process per GPU: only one rank compiles, the others wait for the lock and find the library fresh
    with open(os.path.join(where, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build.build(lib=target)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def bind(L):
    """Declare argtypes / restype of every entry point of include/pic_b200.h on the loaded library."""
    fabp, soap, stp, gp, bp = (C.POINTER(abi.pic_fab), C.POINTER(abi.pic_soa),
                               C.POINTER(abi.pic_stencil), C.POINTER(abi.pic_geom),
                               C.POINTER(abi.pic_bins))
    dp, ip, vp = abi.c_double_p, abi.c_int_p, C.c_void_p
    escp = C.POINTER(abi.pic_escape_list)
    bndp, lasp, injp = (C.POINTER(abi.pic_boundaries), C.POINTER(abi.pic_laser_antenna),
                        C.POINTER(abi.pic_plasma_injector))
    sig = {
        "pic_set_error_mode": (None, [C.c_int]),
        "pic_last_error": (C.c_char_p, []),
        "pic_version": (C.c_char_p, []),
        "pic_apply_env_defaults": (None, []),
        "pic_launch_count": (C.c_long, []),
        "pic_set_deposit_mode": (None, [C.c_int]),
        "pic_set_gather_mode": (None, [C.c_int]),
        "pic_set_fdtd_mode": (None, [C.c_int]),
        "pic_fdtd_bulk_launches": (C.c_long, []),
        "pic_evolve_b": (C.c_int, [fabp, fabp, stp, C.c_double, vp]),
        "pic_evolve_e": (C.c_int, [fabp, fabp, fabp, stp, C.c_double, vp]),
        "pic_gather_push": (C.c_int, [soap, C.c_long, C.c_long, fabp, fabp, dp, dp, ip, C.c_double,
                                      C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, bp, escp, vp]),
        "pic_particles_wrap_listed": (C.c_int, [soap, gp, escp, vp]),
        "pic_deposit_esirkepov": (C.c_int, [soap, C.c_long, C.c_long, fabp, dp, dp, ip, C.c_double,
                                            C.c_double, C.c_double, C.c_int, bp, vp]),
        "pic_fill_boundary_local": (C.c_int, [fabp, C.c_int, C.c_int, gp, vp]),
        "pic_sum_boundary_local": (C.c_int, [fabp, C.c_int, C.c_int, gp, vp]),
        "pic_boundary_local_multi": (C.c_int, [fabp, C.c_int, C.c_int, C.c_int, C.c_int, gp, vp]),
        "pic_apply_filter": (C.c_int, [fabp, fabp, ip, vp]),
        "pic_apply_filter_multi": (C.c_int, [fabp, fabp, C.c_int, ip, vp]),
        "pic_halo_slab_count": (C.c_long, [fabp, C.c_int, C.c_int, C.c_int]),
        "pic_halo_pack": (C.c_int, [fabp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]),
        "pic_halo_unpack": (C.c_int, [fabp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]),
        "pic_particles_wrap_periodic": (C.c_int, [soap, gp, vp]),
        "pic_particles_classify": (C.c_int, [soap, gp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp]),
        "pic_particles_classify_listed": (C.c_int, [soap, gp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, escp, vp]),
        "pic_migrate_note_appended": (C.c_int, [vp, escp, vp]),
        "pic_engine_listed_sweeps": (C.c_long, []),
        "pic_engine_fused_sum_exchanges": (C.c_long, []),
        "pic_halo_pack_multi": (C.c_int, [fabp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]),
        "pic_halo_unpack_multi": (C.c_int, [fabp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]),
        "pic_migrate_message_doubles": (C.c_long, [C.c_int]),
        "pic_migrate_workspace_bytes": (C.c_long, [C.c_int]),
        "pic_migrate_pack": (C.c_int, [soap, vp, vp, C.c_int, vp, vp]),
        "pic_migrate_unpack": (C.c_int, [soap, vp, vp, vp, vp, vp, C.c_int, C.c_long, vp, vp, vp]),
        "pic_bins_count": (C.c_long, [ip, ip, ip]),
        "pic_sort_workspace_bytes": (C.c_long, [C.c_long, C.c_long]),
        "pic_sort_particles_by_cell": (C.c_int, [soap, soap, gp, bp, vp, vp]),
        "pic_sum_squares_unique": (C.c_int, [fabp, gp, vp, vp]),
        "pic_particle_energy": (C.c_int, [soap, C.c_double, vp, vp]),
        "pic_engine_create": (vp, [gp, ip, ip, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                                   C.c_int, ip]),
        "pic_engine_destroy": (None, [vp]),
        "pic_engine_dt": (C.c_double, [vp]),
        "pic_engine_guards": (None, [vp, ip]),
        "pic_engine_enable_timing": (C.c_int, [vp, C.c_int]),
        "pic_engine_stage_count": (C.c_int, []),
        "pic_engine_stage_name": (C.c_char_p, [C.c_int]),
        "pic_engine_stage_ms": (C.c_int, [vp, dp, C.POINTER(C.c_long)]),
        "pic_engine_set_fields": (C.c_int, [vp, fabp]),
        "pic_engine_add_species": (C.c_int, [vp, C.c_double, C.c_double, soap, soap, C.c_long, vp, ip, vp, vp]),
        "pic_engine_set_comm": (C.c_int, [vp, vp, ip]),
        "pic_comm_unique_id": (C.c_int, [C.POINTER(C.c_ubyte)]),
        "pic_comm_create": (vp, [C.POINTER(C.c_ubyte), C.c_int, C.c_int]),
        "pic_comm_destroy": (None, [vp]),
        "pic_engine_species_buffer": (C.c_int, [vp, C.c_int, C.POINTER(C.c_long)]),
        "pic_engine_evolve": (C.c_int, [vp, C.c_int, C.c_int, vp]),
        "pic_engine_set_boundaries": (C.c_int, [vp, bndp]),
        "pic_engine_set_moving_window": (C.c_int, [vp, C.c_int, C.c_double]),
        "pic_engine_set_boost": (C.c_int, [vp, C.c_double, C.c_double]),
        "pic_engine_redistribute": (C.c_int, [vp, vp]),
        "pic_halo_copy": (C.c_int, [vp, fabp, C.c_int, ip, vp]),
        "pic_halo_add": (C.c_int, [vp, fabp, C.c_int, ip, ip, vp]),
        "pic_engine_set_nci_corrector": (C.c_int, [vp, dp, dp]),
        "pic_engine_set_injector": (C.c_int, [vp, C.c_int, injp]),
        "pic_engine_add_laser": (C.c_int, [vp, lasp, soap, C.c_long]),
        "pic_engine_laser_np": (C.c_long, [vp, C.c_int]),
        "pic_engine_time": (C.c_double, [vp]),
        "pic_engine_set_step": (C.c_int, [vp, C.c_long, C.c_double]),
        "pic_engine_prob_domain": (None, [vp, dp]),
    }
    sig.update(abi.LWFA_SIGNATURES(fabp, soap, gp, bndp, lasp, injp, dp, ip, vp))
    sig.update(abi.FLUID_SIGNATURES(fabp, dp, vp))
    for name, (res, args) in sig.items():
        fn = getattr(L, name)      # AttributeError if include/pic_b200.h and the library disagree
        fn.restype = res
        fn.argtypes = args
    L._declared = sorted(sig)
    return L


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("warpx_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return torch


def check(rc, L=None):
    if rc != 0:
        L = L or lib()
        raise RuntimeError("pic_b200: " + L.pic_last_error().decode())
