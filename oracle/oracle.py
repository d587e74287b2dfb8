"""TEST INFRASTRUCTURE -- Python face of the CPU oracle (oracle/pic_oracle.cpp).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product package (warpx_b200/) never does.

Two builds exist (oracle/Makefile):
  * ``restated``  -- leaf arithmetic restated by hand (oracle/libpic_oracle.so);
  * ``reference`` -- leaf arithmetic = the reference's own headers compiled verbatim
                     (oracle/_ref/libpic_oracle_ref.so, built only where WARPX_REFERENCE_DIR names a WarpX
                     source tree; tests/golden/reference_leaves.json records what it computes).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
from warpx_b200 import abi  # noqa: E402  (declarations only)

_LIBS = {}


def build(ref=True):
    """Compile the oracle (and, where WARPX_REFERENCE_DIR names a WarpX source tree, the reference-leaf variant)."""
    subprocess.run(["make", "-s", "-C", _HERE], check=True)
    src = os.environ.get("WARPX_REFERENCE_DIR")
    if ref and src and os.path.isdir(os.path.join(src, "Source")):
        subprocess.run(["make", "-s", "-C", _HERE, "ref", "REF=" + os.path.abspath(src)], check=True)


def have_ref():
    return os.path.exists(os.path.join(_HERE, "_ref", "libpic_oracle_ref.so"))


def lib(kind="restated"):
    if kind in _LIBS:
        return _LIBS[kind]
    path = os.path.join(_HERE, "libpic_oracle.so" if kind == "restated"
                        else os.path.join("_ref", "libpic_oracle_ref.so"))
    if not os.path.exists(path):
        if kind == "restated":
            build(ref=False)
        else:
            raise FileNotFoundError(path)
    L = C.CDLL(path)
    dp, ip, vp = abi.c_double_p, abi.c_int_p, C.c_void_p
    fabp, soap, stp, gp = (C.POINTER(abi.pic_fab), C.POINTER(abi.pic_soa),
                           C.POINTER(abi.pic_stencil), C.POINTER(abi.pic_geom))
    sig = {
        "orc_leaf_name": (C.c_char_p, []),
        "orc_shape": (C.c_int, [C.c_int, C.c_double, dp]),
        "orc_shifted_shape": (C.c_int, [C.c_int, C.c_double, C.c_int, dp]),
        "orc_push_momentum": (None, [C.c_int, dp, dp, C.c_double, C.c_double, C.c_double]),
        "orc_update_position": (None, [dp, dp, C.c_double]),
        "orc_stencil_coefs": (None, [C.c_int, dp, stp]),
        "orc_max_dt": (C.c_double, [C.c_int, dp]),
        "orc_evolve_b": (C.c_int, [fabp, fabp, stp, C.c_double]),
        "orc_evolve_e": (C.c_int, [fabp, fabp, fabp, stp, C.c_double]),
        "orc_gather_push": (C.c_int, [soap, C.c_long, C.c_long, fabp, fabp, dp, dp, ip, C.c_double,
                                      C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int]),
        "orc_deposit_esirkepov": (C.c_int, [soap, C.c_long, C.c_long, fabp, dp, dp, ip, C.c_double,
                                            C.c_double, C.c_double, C.c_int]),
        "orc_fill_boundary": (None, [fabp, C.c_int, ip, gp]),
        "orc_sum_boundary": (None, [fabp, C.c_int, ip, ip, gp]),
        "orc_wrap_periodic": (None, [soap, gp]),
        "orc_sum_squares_unique": (C.c_double, [fabp, C.c_int, gp]),
        "orc_checksum_cell_centered": (C.c_double, [fabp, ip, ip]),
        "orc_sim_create": (vp, [ip, dp, dp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
                                C.c_double, ip, C.c_int, ip]),
        "orc_apply_filter": (None, [fabp, fabp, ip]),
        "orc_filter_stencil": (None, [C.c_int, dp]),
        "orc_sim_destroy": (None, [vp]),
        "orc_sim_dt": (C.c_double, [vp]),
        "orc_sim_guards": (None, [vp, ip]),
        "orc_sim_nboxes": (C.c_int, [vp]),
        "orc_sim_add_species": (C.c_int, [vp, C.c_double, C.c_double, C.c_long] + [dp] * 7),
        "orc_sim_evolve": (None, [vp, C.c_int, C.c_int]),
        "orc_sim_np": (C.c_long, [vp, C.c_int]),
        "orc_sim_get_particles": (None, [vp, C.c_int, C.c_int, dp]),
        "orc_sim_box_np": (C.c_long, [vp, C.c_int, C.c_int]),
        "orc_sim_fab": (None, [vp, C.c_int, C.c_int, fabp]),
        "orc_sim_checksum_field": (C.c_double, [vp, C.c_int]),
        "orc_sim_field_energy": (None, [vp, dp]),
        "orc_sim_timers": (None, [vp, dp]),
        "orc_sim_set_boundaries": (C.c_int, [vp, C.POINTER(abi.pic_boundaries)]),
        "orc_sim_set_moving_window": (C.c_int, [vp, C.c_int, C.c_double]),
        "orc_sim_add_plasma": (C.c_int, [vp, C.c_double, C.c_double, C.POINTER(abi.pic_plasma_injector)]),
        "orc_sim_add_laser": (C.c_int, [vp, C.POINTER(abi.pic_laser_antenna)]),
        "orc_sim_laser_np": (C.c_long, [vp, C.c_int]),
        "orc_sim_get_laser_particles": (None, [vp, C.c_int, C.c_int, dp]),
        "orc_sim_laser_info": (None, [vp, C.c_int, dp]),
        "orc_sim_get_z_inj": (None, [vp, C.c_int, dp]),
        "orc_sim_time": (C.c_double, [vp]),
        "orc_sim_prob_domain": (None, [vp, dp]),
        "orc_apply_pec_field": (None, [fabp, C.c_int, gp, C.POINTER(abi.pic_boundaries), ip]),
        "orc_apply_pec_current": (None, [fabp, gp, C.POINTER(abi.pic_boundaries)]),
        "orc_shift_fab": (None, [fabp, gp, C.c_int, C.c_int, C.c_double]),
        "orc_antenna_push": (None, [C.POINTER(abi.pic_laser_antenna), dp, soap, C.c_double, C.c_double]),
        "orc_add_plasma": (C.c_long, [C.POINTER(abi.pic_plasma_injector), gp, dp, dp, dp, dp, dp, dp, C.c_long,
                                      C.c_double, dp]),
        "orc_sim_set_boost": (C.c_int, [vp, C.c_double, C.c_double]),
        "orc_sim_set_nci_corrector": (C.c_int, [vp, dp, dp]),
        "orc_nci_table_index": (C.c_int, [C.c_double, C.c_int]),
        "orc_nci_godfrey_stencil": (None, [dp, dp, C.c_int, C.c_int, C.c_double, dp]),
        "orc_apply_nci_filter": (None, [C.POINTER(abi.pic_fab), C.POINTER(abi.pic_fab), dp, ip, ip]),
        "orc_apply_particle_boundaries": (None, [soap, gp, C.POINTER(abi.pic_boundaries), C.c_char_p]),
        "orc_antenna_particles": (C.c_long, [C.POINTER(abi.pic_laser_antenna), dp, dp, dp, dp, dp, dp, dp, C.c_long]),
        "orc_sim_rho_checksum": (C.c_double, [vp]),
        "orc_deposit_charge": (C.c_int, [soap, fabp, dp, dp, ip, C.c_double, C.c_int]),
        "orc_apply_pec_rho": (None, [fabp, gp, C.POINTER(abi.pic_boundaries)]),
        "orc_particle_energy": (None, [soap, C.c_double, dp]),
        "orc_sim_particle_energy": (None, [vp, C.c_int, dp]),
        "orc_num_threads": (C.c_int, []),
        "orc_set_num_threads": (None, [C.c_int]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _LIBS[kind] = L
    return L


def _dp(a):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(abi.c_double_p)


# --------------------------------------------------------------------------------------------
# Host-side containers used by the stage-level oracle calls (numpy owns the memory)
# --------------------------------------------------------------------------------------------
class HostFab:
    """One field component on the cell box [box_lo, box_hi]; numpy array indexed [k, j, i]."""

    def __init__(self, box_lo, box_hi, ng, stag, data=None):
        self.desc = abi.make_fab(None, box_lo, box_hi, ng, stag)
        self.a = np.zeros(self.desc.shape) if data is None else np.ascontiguousarray(data, dtype=np.float64)
        assert self.a.shape == self.desc.shape
        self.desc.p = self.a.ctypes.data

    def valid(self):
        return self.a[self.desc.valid_slices()]


def fab_array(descs):
    arr = (abi.pic_fab * len(descs))()
    for n, d in enumerate(descs):
        arr[n] = d.desc if hasattr(d, "desc") else d
    return arr


class HostParticles:
    """SoA in PIdx order x y z w ux uy uz."""
    NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")

    def __init__(self, **kw):
        self.np = len(kw["x"])
        for n in self.NAMES:
            setattr(self, n, np.ascontiguousarray(kw[n], dtype=np.float64).copy())
        self.soa = abi.pic_soa()
        for n in self.NAMES:
            setattr(self.soa, n, getattr(self, n).ctypes.data)
        self.soa.idcpu = None
        self.soa.np = self.np

    def copy(self):
        return HostParticles(**{n: getattr(self, n) for n in self.NAMES})


# --------------------------------------------------------------------------------------------
# Whole-loop driver
# --------------------------------------------------------------------------------------------
class OracleSim:
    """Single-level periodic explicit-FDTD PIC run == WarpX::Evolve restated (pic_oracle.cpp)."""

    def __init__(self, n_cell, prob_lo, prob_hi, nox, galerkin=1, pusher=abi.PUSHER_BORIS,
                 solver=abi.SOLVER_YEE, cfl=1.0, dt=0.0, nb=(1, 1, 1), kind="restated",
                 use_filter=False, filter_npass=(1, 1, 1)):
        self.L = lib(kind)
        self.h = self.L.orc_sim_create(abi.int3(n_cell), abi.dbl3(prob_lo), abi.dbl3(prob_hi), nox,
                                       galerkin, pusher, solver, cfl, dt, abi.int3(nb),
                                       1 if use_filter else 0, abi.int3(filter_npass))
        if not self.h:
            raise ValueError("bad oracle configuration")
        self.n_cell = tuple(n_cell)
        self.nspecies = 0
        self.dt = self.L.orc_sim_dt(self.h)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_sim_destroy(self.h)
            self.h = None

    def guards(self):
        out = (C.c_int * 12)()
        self.L.orc_sim_guards(self.h, out)
        v = list(out)
        return {"ng_EB": v[0:3], "ng_J": v[3:6], "ng_FG": v[6:9], "ng_FS": v[9:12]}

    def add_species(self, q, m, x, y, z, w, ux, uy, uz):
        arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (x, y, z, w, ux, uy, uz)]
        self.nspecies += 1
        return self.L.orc_sim_add_species(self.h, q, m, len(arrs[0]), *[_dp(a) for a in arrs])

    # ---- laser-wakefield additions (single box; configure before adding particles) ----
    def set_boundaries(self, bnd):
        rc = self.L.orc_sim_set_boundaries(self.h, C.byref(bnd))
        if rc:
            raise ValueError("orc_sim_set_boundaries: %d" % rc)

    def set_moving_window(self, direction, v_over_c):
        rc = self.L.orc_sim_set_moving_window(self.h, direction, v_over_c)
        if rc:
            raise ValueError("orc_sim_set_moving_window: %d" % rc)

    def set_boost(self, gamma_boost):
        """warpx.gamma_boost, boost_direction = z; injectors and antennas added later take it over."""
        rc = self.L.orc_sim_set_boost(self.h, gamma_boost, abi.beta_of_gamma(gamma_boost))
        if rc:
            raise ValueError("orc_sim_set_boost: call before adding species / lasers")

    def set_nci_corrector(self, stencil_exeybz, stencil_bxbyez):
        """particles.use_fdtd_nci_corr with the two z stencils (m_stencil_2 of the reference's filters)."""
        rc = self.L.orc_sim_set_nci_corrector(self.h, (C.c_double * 5)(*stencil_exeybz), (C.c_double * 5)(*stencil_bxbyez))
        if rc:
            raise ValueError("orc_sim_set_nci_corrector: call before adding species")

    def add_plasma(self, q, m, injector):
        self.nspecies += 1
        return self.L.orc_sim_add_plasma(self.h, q, m, C.byref(injector))

    def add_laser(self, laser):
        return self.L.orc_sim_add_laser(self.h, C.byref(laser))

    def laser_particles(self, il):
        n = self.L.orc_sim_laser_np(self.h, il)
        out = {}
        for c, name in enumerate(HostParticles.NAMES):
            a = np.empty(n)
            self.L.orc_sim_get_laser_particles(self.h, il, c, _dp(a))
            out[name] = a
        return out

    def laser_info(self, il):
        out = (C.c_double * 4)()
        self.L.orc_sim_laser_info(self.h, il, out)
        return dict(zip(("S_X", "S_Y", "mobility", "weight"), list(out)))

    def z_at_injection(self, isp):
        a = np.empty(self.L.orc_sim_np(self.h, isp))
        self.L.orc_sim_get_z_inj(self.h, isp, _dp(a))
        return a

    def time(self):
        return self.L.orc_sim_time(self.h)

    def prob_domain(self):
        out = (C.c_double * 6)()
        self.L.orc_sim_prob_domain(self.h, out)
        return list(out[0:3]), list(out[3:6])

    def evolve(self, nsteps, synchronize_last=True):
        self.L.orc_sim_evolve(self.h, nsteps, 1 if synchronize_last else 0)

    def particles(self, isp):
        n = self.L.orc_sim_np(self.h, isp)
        out = {}
        for c, name in enumerate(HostParticles.NAMES):
            a = np.empty(n)
            self.L.orc_sim_get_particles(self.h, isp, c, _dp(a))
            out[name] = a
        return out

    def fab(self, comp, ibox=0):
        """(descriptor, numpy view [k,j,i]) of component comp (0..8 = Ex..jz) of box ibox."""
        d = abi.pic_fab()
        self.L.orc_sim_fab(self.h, ibox, comp, C.byref(d))
        buf = (C.c_double * d.size).from_address(d.p)
        return d, np.frombuffer(buf, dtype=np.float64).reshape(d.shape)

    def checksum_field(self, comp):
        return self.L.orc_sim_checksum_field(self.h, comp)

    def field_energy(self):
        out = (C.c_double * 2)()
        self.L.orc_sim_field_energy(self.h, out)
        return out[0], out[1]

    def rho_checksum(self):
        """Checksum of the cell-centred `rho` diagnostic (all containers; single box)."""
        return self.L.orc_sim_rho_checksum(self.h)

    def particle_energy(self, isp):
        out = (C.c_double * 2)()
        self.L.orc_sim_particle_energy(self.h, isp, out)
        return out[0], out[1]

    def timers(self):
        out = (C.c_double * 5)()
        self.L.orc_sim_timers(self.h, out)
        return dict(zip(("push", "deposit", "fdtd", "halo", "other"), list(out)))
