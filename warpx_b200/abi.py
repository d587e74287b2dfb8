"""ctypes mirror of include/pic_b200.h (the C ABI).  Pure declarations: no compute, no CUDA."""
import ctypes as C

import numpy as np

c_double_p = C.POINTER(C.c_double)
c_int_p = C.POINTER(C.c_int)


class pic_fab(C.Structure):
    _fields_ = [("p", C.c_void_p), ("lo", C.c_int * 3), ("hi", C.c_int * 3),
                ("ng", C.c_int * 3), ("stag", C.c_int * 3)]

    @property
    def shape(self):  # numpy (z, y, x) shape of the allocated region
        return tuple(self.hi[d] - self.lo[d] + 1 for d in (2, 1, 0))

    @property
    def size(self):
        return int(np.prod(self.shape))

    def valid_slices(self):
        """numpy slices (z, y, x) of the valid region inside the allocated array."""
        return tuple(slice(self.ng[d], self.hi[d] - self.lo[d] + 1 - self.ng[d]) for d in (2, 1, 0))


class pic_soa(C.Structure):
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("z", C.c_void_p), ("w", C.c_void_p),
                ("ux", C.c_void_p), ("uy", C.c_void_p), ("uz", C.c_void_p),
                ("idcpu", C.c_void_p), ("np", C.c_long)]


class pic_stencil(C.Structure):
    _fields_ = [("algo", C.c_int), ("cx", C.c_double * 5), ("cy", C.c_double * 5),
                ("cz", C.c_double * 5)]


class pic_bins(C.Structure):
    _fields_ = [("cell_start", C.c_void_p), ("box_lo", C.c_int * 3), ("box_hi", C.c_int * 3),
                ("tile", C.c_int * 3), ("np_binned", C.c_long)]


class pic_escape_list(C.Structure):
    _fields_ = [("idx", C.c_void_p), ("count", C.c_void_p), ("capacity", C.c_int),
                ("lo", C.c_double * 3), ("hi", C.c_double * 3)]


class pic_geom(C.Structure):
    _fields_ = [("n_cell", C.c_int * 3), ("prob_lo", C.c_double * 3), ("prob_hi", C.c_double * 3),
                ("periodic", C.c_int * 3)]


class pic_boundaries(C.Structure):
    _fields_ = [("field_lo", C.c_int * 3), ("field_hi", C.c_int * 3),
                ("particle_lo", C.c_int * 3), ("particle_hi", C.c_int * 3)]


class pic_laser_antenna(C.Structure):
    _fields_ = [("position", C.c_double * 3), ("nvec", C.c_double * 3), ("p_X", C.c_double * 3),
                ("wavelength", C.c_double), ("e_max", C.c_double), ("waist", C.c_double),
                ("duration", C.c_double), ("t_peak", C.c_double), ("focal_distance", C.c_double),
                ("phi0", C.c_double), ("gamma_boost", C.c_double), ("beta_boost", C.c_double)]


class pic_plasma_injector(C.Structure):
    _fields_ = [("ppc", C.c_int * 3), ("bound_lo", C.c_double * 3), ("bound_hi", C.c_double * 3),
                ("density", C.c_double), ("do_continuous_injection", C.c_int),
                ("gamma_boost", C.c_double), ("beta_boost", C.c_double)]


class pic_gaussian_beam(C.Structure):
    _fields_ = [("x_m", C.c_double * 3), ("rms", C.c_double * 3), ("cut", C.c_double * 3),
                ("bound_lo", C.c_double * 3), ("bound_hi", C.c_double * 3), ("q_tot", C.c_double),
                ("npart", C.c_long), ("do_symmetrize", C.c_int), ("symmetrization_order", C.c_int),
                ("do_focusing", C.c_int), ("focal_distance", C.c_double),
                ("u_m", C.c_double * 3), ("u_th", C.c_double * 3), ("seed", C.c_uint64),
                ("gamma_boost", C.c_double), ("beta_boost", C.c_double)]


class pic_coulomb_collision(C.Structure):
    _fields_ = [("q1", C.c_double), ("m1", C.c_double), ("q2", C.c_double), ("m2", C.c_double),
                ("coulomb_log", C.c_double), ("seed", C.c_uint64), ("collision_index", C.c_int),
                ("same_species", C.c_int)]


class pic_fusion_collision(C.Structure):
    _fields_ = [("q1", C.c_double), ("m1", C.c_double), ("q2", C.c_double), ("m2", C.c_double),
                ("mA", C.c_double), ("mB", C.c_double), ("type", C.c_int), ("fusion_multiplier", C.c_double),
                ("fusion_probability_threshold", C.c_double), ("fusion_probability_target_value", C.c_double),
                ("seed", C.c_uint64), ("collision_index", C.c_int), ("same_species", C.c_int)]


class pic_flux_injector(C.Structure):
    _fields_ = [("num_ppc", C.c_double), ("surface_flux_pos", C.c_double), ("normal_axis", C.c_int),
                ("direction", C.c_int), ("flux", C.c_double), ("tmin", C.c_double), ("tmax", C.c_double),
                ("bound_lo", C.c_double * 3), ("bound_hi", C.c_double * 3), ("u_m", C.c_double * 3),
                ("u_th", C.c_double * 3), ("seed", C.c_uint64)]


FUSION_DT_NHE4, FUSION_DD_PT, FUSION_DD_NHE3, FUSION_PB_3HE4 = 0, 1, 2, 3
SPENT_ID = 0xFFFFFFFFFFFFFFFF          # PIC_SPENT_ID: a reactant whose weight a fusion used up

FIELD_PERIODIC, FIELD_PEC = 0, 1
PARTICLE_PERIODIC, PARTICLE_ABSORBING, PARTICLE_REFLECTING = 0, 1, 2
_FIELD_BC = {"periodic": FIELD_PERIODIC, "pec": FIELD_PEC}
_PARTICLE_BC = {"periodic": PARTICLE_PERIODIC, "absorbing": PARTICLE_ABSORBING, "reflecting": PARTICLE_REFLECTING}


def make_boundaries(field_lo, field_hi, particle_lo=None, particle_hi=None):
    """boundary.field_lo/hi and boundary.particle_lo/hi by name; particles default to periodic on
    periodic field faces and absorbing elsewhere (Source/Utils/WarpXUtil.cpp:470-540)."""
    b = pic_boundaries()
    for d in range(3):
        b.field_lo[d], b.field_hi[d] = _FIELD_BC[field_lo[d]], _FIELD_BC[field_hi[d]]
        dflt_lo = "periodic" if field_lo[d] == "periodic" else "absorbing"
        dflt_hi = "periodic" if field_hi[d] == "periodic" else "absorbing"
        b.particle_lo[d] = _PARTICLE_BC[particle_lo[d] if particle_lo else dflt_lo]
        b.particle_hi[d] = _PARTICLE_BC[particle_hi[d] if particle_hi else dflt_hi]
    return b


def beta_of_gamma(gamma_boost):
    """ReadBoostedFrameParameters (Source/Utils/WarpXUtil.cpp:114-121)."""
    import math
    return math.sqrt(1.0 - 1.0 / gamma_boost ** 2.0) if gamma_boost > 1.0 else 0.0


def make_laser(position, direction, polarization, wavelength, e_max, waist, duration, t_peak,
               focal_distance, phi0=0.0, gamma_boost=1.0):
    a = pic_laser_antenna()
    a.gamma_boost, a.beta_boost = float(gamma_boost), beta_of_gamma(gamma_boost)
    for d in range(3):
        a.position[d], a.nvec[d], a.p_X[d] = float(position[d]), float(direction[d]), float(polarization[d])
    a.wavelength, a.e_max, a.waist, a.duration = float(wavelength), float(e_max), float(waist), float(duration)
    a.t_peak, a.focal_distance, a.phi0 = float(t_peak), float(focal_distance), float(phi0)
    return a


def make_injector(ppc, bound_lo, bound_hi, density, do_continuous_injection=False, gamma_boost=1.0):
    inj = pic_plasma_injector()
    inj.gamma_boost, inj.beta_boost = float(gamma_boost), beta_of_gamma(gamma_boost)
    for d in range(3):
        inj.ppc[d] = int(ppc[d])
        inj.bound_lo[d], inj.bound_hi[d] = float(bound_lo[d]), float(bound_hi[d])
    inj.density = float(density)
    inj.do_continuous_injection = 1 if do_continuous_injection else 0
    return inj


DBL_MAX = 1.7976931348623157e308

_AXES = {"x": 0, "y": 1, "z": 2}


def make_flux_injector(num_particles_per_cell, surface_flux_pos, flux_normal_axis, flux_direction, flux=1.0,
                       u_m=(0.0, 0.0, 0.0), u_th=(0.0, 0.0, 0.0), bound_lo=(-np.inf,) * 3, bound_hi=(np.inf,) * 3,
                       flux_tmin=-1.0, flux_tmax=-1.0, seed=0):
    """<species>.injection_style = NFluxPerCell by the deck's names: num_particles_per_cell (real), surface_flux_pos,
    flux_normal_axis ("x", "y", "z" or 0..2), flux_direction (+1 / -1), flux (flux_profile = constant, or a
    parse_flux_function that is a constant), u_m = (ux_m, uy_m, uz_m) and u_th = (ux_th, uy_th, uz_th) in units of c
    (momentum_distribution_type = gaussianflux), bound_lo/hi = xmin..zmax, flux_tmin / flux_tmax (< 0: unset); seed
    keys the injector's random streams."""
    f = pic_flux_injector()
    f.num_ppc, f.surface_flux_pos = float(num_particles_per_cell), float(surface_flux_pos)
    f.normal_axis = _AXES[flux_normal_axis.lower()] if isinstance(flux_normal_axis, str) else int(flux_normal_axis)
    f.direction, f.flux = int(flux_direction), float(flux)
    f.tmin, f.tmax = float(flux_tmin), float(flux_tmax)
    for d in range(3):
        f.bound_lo[d], f.bound_hi[d] = float(bound_lo[d]), float(bound_hi[d])
        f.u_m[d], f.u_th[d] = float(u_m[d]), float(u_th[d])
    f.seed = int(seed)
    return f


def make_gaussian_beam(x_m, rms, npart, q_tot, u_m=(0.0, 0.0, 0.0), u_th=(0.0, 0.0, 0.0), cut=(DBL_MAX,) * 3,
                       bound_lo=(-np.inf,) * 3, bound_hi=(np.inf,) * 3, do_symmetrize=False, symmetrization_order=4,
                       focal_distance=None, seed=0, gamma_boost=1.0, do_backward_propagation=False):
    """<species>.injection_style = "gaussian_beam" by the deck's names: x_m = (x_m, y_m, z_m), rms = (x_rms, y_rms,
    z_rms), cut = (x_cut, y_cut, z_cut) in units of rms, bound_lo/hi = xmin..zmax, u_m / u_th in units of c,
    focal_distance set = do_focusing.  do_backward_propagation is refused: no deck of the project uses it."""
    if do_backward_propagation:
        raise NotImplementedError("gaussian_beam: do_backward_propagation is not supported")
    b = pic_gaussian_beam()
    for d in range(3):
        b.x_m[d], b.rms[d], b.cut[d] = float(x_m[d]), float(rms[d]), float(cut[d])
        b.bound_lo[d], b.bound_hi[d] = float(bound_lo[d]), float(bound_hi[d])
        b.u_m[d], b.u_th[d] = float(u_m[d]), float(u_th[d])
    b.npart, b.q_tot = int(npart), float(q_tot)
    b.do_symmetrize, b.symmetrization_order = (1 if do_symmetrize else 0), int(symmetrization_order)
    b.do_focusing = 0 if focal_distance is None else 1
    b.focal_distance = 0.0 if focal_distance is None else float(focal_distance)
    b.seed = int(seed)
    b.gamma_boost, b.beta_boost = float(gamma_boost), beta_of_gamma(gamma_boost)
    return b


def LWFA_SIGNATURES(fabp, soap, gp, bp, lp, jp, dp, ip, vp):
    """ctypes signatures of the non-periodic-domain entry points of include/pic_b200.h."""
    return {
        "pic_apply_pec_field": (C.c_int, [fabp, C.c_int, gp, bp, ip, vp]),
        "pic_apply_pec_current": (C.c_int, [fabp, gp, bp, vp]),
        "pic_shift_fab": (C.c_int, [fabp, vp, gp, C.c_int, C.c_int, C.c_double, vp]),
        "pic_laser_antenna_info": (C.c_int, [lp, dp, dp]),
        "pic_laser_antenna_particles": (C.c_long, [lp, dp, dp, dp, vp, vp, vp, vp, C.c_long]),
        "pic_laser_antenna_push": (C.c_int, [lp, dp, soap, C.c_double, C.c_double, vp]),
        "pic_add_plasma": (C.c_long, [jp, gp, dp, ip, ip, dp, dp, soap, C.c_long, C.c_uint64, C.c_double, vp]),
        "pic_add_gaussian_beam": (C.c_long, [C.POINTER(pic_gaussian_beam), C.c_double, gp, dp, dp, soap, C.c_long,
                                             C.c_double, vp]),
        "pic_philox4x64": (C.c_int, [C.c_uint64, C.c_long, C.c_long, vp, vp]),
        "pic_gaussian_beam_normals": (C.c_int, [C.c_uint64, C.c_long, C.c_long, vp, vp]),
        "pic_particles_owned_weights": (C.c_int, [soap, dp, dp, vp, vp]),
        "pic_deposit_charge": (C.c_int, [soap, C.c_long, C.c_long, fabp, dp, dp, ip, C.c_double, C.c_int, vp]),
        "pic_apply_pec_rho": (C.c_int, [fabp, gp, bp, vp]),
        "pic_particles_boundary_workspace_ints": (C.c_long, [C.c_int]),
        "pic_particles_boundary_mark": (C.c_int, [soap, gp, bp, vp, C.c_int, vp]),
        "pic_particles_boundary_compact": (C.c_int, [soap, vp, C.c_int, C.c_int, vp]),
        "pic_nci_godfrey_table_index": (C.c_int, [C.c_double, C.c_int]),
        "pic_nci_godfrey_stencil": (None, [dp, dp, C.c_int, C.c_int, C.c_double, dp]),
        "pic_apply_nci_filter": (C.c_int, [fabp, fabp, dp, ip, ip, C.c_int, vp]),
    }


def COLLISION_SIGNATURES(soap, bp, gp, vp):
    """ctypes signatures of the binary-collision entry points of include/pic_b200.h."""
    return {
        "pic_collide_pairwise_coulomb": (C.c_int, [C.POINTER(pic_coulomb_collision), soap, bp, vp, soap, bp, vp, gp,
                                                   C.c_double, C.c_long, vp, vp, vp, vp]),
        "pic_engine_add_collision": (C.c_int, [vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_uint64]),
        "pic_fusion_workspace_bytes": (C.c_long, [C.c_long, C.c_long]),
        "pic_collide_nuclear_fusion": (C.c_int, [C.POINTER(pic_fusion_collision), soap, bp, vp, soap, bp, vp, gp,
                                                 C.c_double, C.c_long, vp, vp, vp, C.c_long, vp, vp]),
        "pic_fusion_create_products": (C.c_int, [C.POINTER(pic_fusion_collision), soap, bp, soap, bp, gp, C.c_long, vp,
                                                 C.c_long, soap, C.c_long, C.c_uint64, soap, C.c_long, C.c_uint64,
                                                 C.POINTER(C.c_long), vp]),
        "pic_particles_mark_spent": (C.c_int, [soap, vp, C.c_int, vp]),
        "pic_engine_species_next_id": (C.c_uint64, [vp, C.c_int]),
        "pic_engine_set_species_next_id": (C.c_int, [vp, C.c_int, C.c_uint64]),
        "pic_engine_set_species_flags": (C.c_int, [vp, C.c_int, C.c_int, C.c_int]),
        "pic_engine_add_fusion": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double,
                                            C.c_double, C.c_int, C.c_uint64]),
    }


def FLUX_SIGNATURES(soap, gp, ip, vp):
    """ctypes signatures of the flux-injection entry points of include/pic_b200.h."""
    fp = C.POINTER(pic_flux_injector)
    return {
        "pic_flux_workspace_bytes": (C.c_long, [fp, gp]),
        "pic_add_flux_particles": (C.c_long, [fp, C.c_int, gp, ip, ip, C.c_long, C.c_double, C.c_double, soap, C.c_long,
                                              C.c_uint64, C.POINTER(C.c_uint64), vp, C.c_long, vp]),
        "pic_engine_add_flux_injector": (C.c_int, [vp, C.c_int, fp]),
    }


def FLUID_SIGNATURES(fabp, dp, vp):
    """ctypes signatures of the fluid-species entry points of include/pic_b200.h (a fluid state is 4 pic_fab)."""
    return {
        "pic_fluid_gather_push": (C.c_int, [fabp, fabp, fabp, C.c_double, C.c_double, C.c_double, vp]),
        "pic_fluid_advect": (C.c_int, [fabp, fabp, dp, C.c_double, vp, vp]),
        "pic_fluid_deposit_current": (C.c_int, [fabp, fabp, C.c_double, vp]),
        "pic_fluid_deposit_charge": (C.c_int, [fabp, fabp, C.c_double, vp]),
        "pic_engine_add_fluid_species": (C.c_int, [vp, C.c_double, C.c_double, fabp, fabp]),
        "pic_engine_fluid_state": (C.c_int, [vp, C.c_int]),
    }


SOLVER_YEE, SOLVER_CKC, SOLVER_NONE = 0, 1, 2
PIC_ERR_ABORT, PIC_ERR_RETURN = 0, 1
PUSHER_BORIS, PUSHER_VAY, PUSHER_HC = 0, 1, 2
# pic_set_deposit_mode / pic_set_gather_mode (include/pic_b200.h)
PIC_DEPOSIT_RUNS, PIC_DEPOSIT_TILE, PIC_DEPOSIT_RUNS2, PIC_DEPOSIT_RUNS_SLOTRED = 0, 1, 2, 3
PIC_DEPOSIT_RUNS2_SLOTRED, PIC_DEPOSIT_RUNS4, PIC_DEPOSIT_RUNS4_SLOTRED = 4, 5, 6
PIC_DEPOSIT_CELLS, PIC_DEPOSIT_CELLS2, PIC_DEPOSIT_CELLS2_WIDE = 7, 8, 9
PIC_DEPOSIT_CELLS3, PIC_DEPOSIT_CELLS3_WIDE = 10, 11
PIC_DEPOSIT_RUNS_SLAB = 12
PIC_GATHER_TILE, PIC_GATHER_PAIRS, PIC_GATHER_PAIRS_WIDE, PIC_GATHER_PAIRS_192 = 0, 1, 2, 3

# Yee staggering of WarpX (Source/WarpX.cpp:2117-2125): 1 = nodal.  Order Ex Ey Ez Bx By Bz jx jy jz.
YEE_STAG = ((0, 1, 1), (1, 0, 1), (1, 1, 0),
            (1, 0, 0), (0, 1, 0), (0, 0, 1),
            (0, 1, 1), (1, 0, 1), (1, 1, 0))
COMP_NAMES = ("Ex", "Ey", "Ez", "Bx", "By", "Bz", "jx", "jy", "jz")


def make_fab(ptr, box_lo, box_hi, ng, stag):
    """Descriptor of one component on the cell box [box_lo, box_hi] (inclusive)."""
    f = pic_fab()
    f.p = ptr
    for d in range(3):
        f.stag[d] = stag[d]
        f.ng[d] = ng[d]
        f.lo[d] = box_lo[d] - ng[d]
        f.hi[d] = box_hi[d] + stag[d] + ng[d]
    return f


def make_geom(n_cell, prob_lo, prob_hi, periodic=(1, 1, 1)):
    g = pic_geom()
    for d in range(3):
        g.n_cell[d] = int(n_cell[d])
        g.prob_lo[d] = float(prob_lo[d])
        g.prob_hi[d] = float(prob_hi[d])
        g.periodic[d] = int(periodic[d])
    return g


def int3(v):
    return (C.c_int * 3)(*[int(a) for a in v])


def dbl3(v):
    return (C.c_double * 3)(*[float(a) for a in v])


def dbl4(v):
    return (C.c_double * 4)(*[float(a) for a in v])
