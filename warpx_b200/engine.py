"""Host side of the reference's explicit EM-PIC step (single level, FDTD): the Simulation object.

The step itself -- WarpX::Evolve, OneStep_nosub, SyncCurrent, Synchronize, HandleParticlesAtBoundaries -- runs in
the library's C++ step driver; the header of csrc/engine.cu maps each of its functions to the reference's.  Every
stage is a call through the C ABI (include/pic_b200.h) into hand-written sm_90a kernels.  PyTorch only owns device
memory and the stream; with several ranks torch.distributed broadcasts the id of the driver's NCCL communicator.
There is no CPU path: constructing a Simulation without a CUDA device raises.
"""
import ctypes as C
import math
import weakref

import numpy as np

from . import abi, parallel
from .lib import check as _check_rc, lib, require_cuda

_error_source = None      # the library whose pic_last_error() a failed call reports (the one the last Simulation loaded)


def check(rc):
    if rc != 0:
        _check_rc(rc, _error_source)


C_LIGHT = 299792458.0
EP0 = 8.8541878128e-12
MU0 = 1.25663706212e-06


def stencil_coefficients(solver, dx):
    """FiniteDifferenceSolver ctor (FieldSolver/FiniteDifferenceSolver/FiniteDifferenceSolver.cpp:30-103):
    Yee CartesianYeeAlgorithm.H:30-42, CKC CartesianCKCAlgorithm.H:31-101 (Cowan 2013)."""
    st = abi.pic_stencil()
    st.algo = solver
    inv = [1.0 / d for d in dx]
    for n in range(5):
        st.cx[n] = st.cy[n] = st.cz[n] = 0.0
    st.cx[0], st.cy[0], st.cz[0] = inv
    if solver == abi.SOLVER_CKC:
        delta = max(inv)
        rx, ry, rz = ((v / delta) * (v / delta) for v in inv)
        beta = 0.125 * (1.0 - rx * ry * rz / (ry * rz + rz * rx + rx * ry))
        irf = 1.0 / (ry * rz + rz * rx + rx * ry)
        gx = ry * rz * (0.0625 - 0.125 * ry * rz * irf)
        gy = rx * rz * (0.0625 - 0.125 * rx * rz * irf)
        gz = rx * ry * (0.0625 - 0.125 * rx * ry * irf)
        st.cx[1] = (1.0 - 2.0 * ry * beta - 2.0 * rz * beta - 4.0 * gx) * inv[0]
        st.cy[1] = (1.0 - 2.0 * rx * beta - 2.0 * rz * beta - 4.0 * gy) * inv[1]
        st.cz[1] = (1.0 - 2.0 * rx * beta - 2.0 * ry * beta - 4.0 * gz) * inv[2]
        st.cx[2], st.cx[3], st.cx[4] = ry * beta * inv[0], rz * beta * inv[0], gx * inv[0]
        st.cy[2], st.cy[3], st.cy[4] = rz * beta * inv[1], rx * beta * inv[1], gy * inv[1]
        st.cz[2], st.cz[3], st.cz[4] = rx * beta * inv[2], ry * beta * inv[2], gz * inv[2]
    return st


def max_dt(solver, dx):
    """WarpX::ComputeDt (Evolve/WarpXComputeDt.cpp:56-95): Yee CartesianYeeAlgorithm.H:48-56,
    CKC CartesianCKCAlgorithm.H:107-118."""
    if solver == abi.SOLVER_YEE:
        return 1.0 / (math.sqrt(sum(1.0 / (d * d) for d in dx)) * C_LIGHT)
    return min(dx) / C_LIGHT


def nci_godfrey_stencils(lib, lines, cdtodz, galerkin=True):
    """The two z stencils of Godfrey's NCI corrector (WarpX::InitNCICorrector, Source/Initialization/
    WarpXInitData.cpp:858-890 -> NCIGodfreyFilter::ComputeStencils): `lines` holds lines of the reference's
    coefficient tables keyed like tests/golden/nci_godfrey_lines.json ({"galerkin_Ex_Ey_Bz": {"99": [4 numbers],
    ...}, ..., "_provenance": {"tab_length": 101}}); the tables are the caller's data, not part of this package.
    Returns (stencil_exeybz, stencil_bxbyez), each 5 numbers with coefficient 0 halved."""
    tab_length = int(lines["_provenance"]["tab_length"])
    index = lib.pic_nci_godfrey_table_index(cdtodz, tab_length)
    out = []
    for which in ("Ex_Ey_Bz", "Bx_By_Ez"):
        table = lines[("galerkin_" if galerkin else "momentum_") + which]
        if str(index) not in table or str(index + 1) not in table:
            raise KeyError("nci_godfrey_stencils: the table lines %d, %d (c dt / dz = %g) were not supplied" % (index, index + 1, cdtodz))
        st = (C.c_double * 5)()
        lib.pic_nci_godfrey_stencil(abi.dbl4(table[str(index)]), abi.dbl4(table[str(index + 1)]), index, tab_length, cdtodz, st)
        out.append(list(st))
    return tuple(out)


def guard_cells(nox, dt, dx, use_filter=False, filter_npass=(1, 1, 1), do_moving_window=False, use_nci=False):
    """guardCellManager::Init (Parallelization/GuardCellManager.cpp:62-172, 310-343) for: no MR,
    not safe_guard_cells, FDTD solver; use_nci: the NCI corrector's 4 extra cells along z (:87-90,319-330).  Returns also ng_depos_J (:165) -- ng_J itself
    grows by stencil_length-1 = npass when the bilinear filter is on (:169-172); a moving window needs
    at least 2 guard cells everywhere (:103-115, one level)."""
    ng_EB, ng_J, ng_FG, ng_FS, ng_depos_J = [], [], [], [], []
    for d in range(3):
        ngt = nox
        ng = ngt + 1 if ngt % 2 else ngt
        if use_nci and d == 2:
            ng = ngt + 4 + ((ngt + 4) % 2)
        ngj0 = ngt
        if do_moving_window:
            ng, ngj0 = max(ng, 2), max(ngj0, 2)
        ngj = ngj0 + int(math.ceil(C_LIGHT * 0.5 * dt / dx[d]))
        fs = 1
        ng = max(ng, fs)
        fg = min((nox + 1) // 2, ng)
        if use_nci and d == 2:
            fg = min(fg + 4, ng)
        fg = max(fg, fs)
        ng_depos_J.append(ngj)
        if use_filter:
            ngj += filter_npass[d]
        ng_EB.append(ng); ng_J.append(ngj); ng_FG.append(fg); ng_FS.append(fs)
    return dict(ng_EB=ng_EB, ng_J=ng_J, ng_FG=ng_FG, ng_FS=ng_FS, ng_depos_J=ng_depos_J)


def shared_comm(L, dist, torch, device):
    """The ONE private NCCL communicator of this process (csrc/comm.cu), created on first use and reused by every
    Simulation: rank 0 draws the 128-byte id, torch.distributed broadcasts it.  Kept on the `dist` object; release it
    with release_comm(dist) on every rank at the same point of the program (after a barrier), before
    torch.distributed.destroy_process_group()."""
    comm = getattr(dist, "_pic_comm", None)
    if comm:
        return comm
    rank, world = dist.get_rank(), dist.get_world_size()
    ident = torch.zeros(128, dtype=torch.uint8, device=device)
    if rank == 0:
        raw = (C.c_ubyte * 128)()
        check(L.pic_comm_unique_id(raw))
        ident.copy_(torch.tensor(list(raw), dtype=torch.uint8))
    dist.broadcast(ident, 0)
    raw = (C.c_ubyte * 128)(*ident.cpu().tolist())
    comm = L.pic_comm_create(raw, world, rank)
    if not comm:
        raise RuntimeError(L.pic_last_error().decode())
    dist._pic_comm, dist._pic_comm_lib = comm, L
    return comm


def release_comm(dist):
    """Destroy the process's private communicator (collective in effect: call on every rank, engines closed)."""
    comm = getattr(dist, "_pic_comm", None)
    if comm:
        dist._pic_comm_lib.pic_comm_destroy(comm)
        dist._pic_comm = None


class Species:
    NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")

    def __init__(self, sim, name, q, m, arrays, capacity, ids=None, species_type=None):
        t = sim.torch
        self.sim, self.name, self.q, self.m = weakref.proxy(sim), name, q, m
        self.species_type = canonical_species_type(species_type) if species_type is not None else None
        self.np = len(arrays["x"])
        self.capacity = max(capacity, self.np)
        # two SoA buffers: the counting sort permutes from one into the other
        self.buf = [t.empty((7, self.capacity), dtype=t.float64, device=sim.device) for _ in range(2)]
        # 64-bit particle id (the reference's idcpu): rank in the upper bits, local index below
        self.ids = [t.empty(self.capacity, dtype=t.int64, device=sim.device) for _ in range(2)]
        if ids is None:
            self.ids[0][:self.np] = t.arange(self.np, dtype=t.int64, device=sim.device) + (sim.rank << 40)
        else:               # restart: the ids a checkpoint carries
            self.ids[0][:self.np].copy_(t.from_numpy(np.ascontiguousarray(ids, dtype=np.int64)))
        self.cur = 0
        for n, name_ in enumerate(self.NAMES):
            a = arrays[name_]
            src = a if isinstance(a, t.Tensor) else t.from_numpy(np.ascontiguousarray(a, dtype=np.float64))
            self.buf[0][n, :self.np].copy_(src, non_blocking=True)
        self.cell_start = None    # cell-sort scratch of the C++ driver (Simulation._register_species), none without bins
        self.work = None
        self.do_not_push = self.do_not_deposit = False     # Simulation.set_species_flags

    def soa(self, which=None):
        b = self.buf[self.cur if which is None else which]
        s = abi.pic_soa()
        for n, name in enumerate(self.NAMES):
            setattr(s, name, b[n].data_ptr())
        s.idcpu = self.ids[self.cur if which is None else which].data_ptr()
        s.np = self.np
        return s

    def id_array(self):
        return self.ids[self.cur][:self.np]

    def array(self, name):
        return self.buf[self.cur][self.NAMES.index(name), :self.np]


# <species>.species_type -> (charge [C], mass [kg]): Source/Particles/SpeciesPhysicalProperties.cpp, with its aliases
Q_E, M_P, M_U = 1.602176634e-19, 1.67262192369e-27, 1.66053906660e-27    # PhysConst::q_e, m_p, m_u
_SPECIES_ALIASES = {"protium": "hydrogen1", "deuterium": "hydrogen2", "tritium": "hydrogen3"}
SPECIES_PROPERTIES = {
    "neutron": (0.0, 1.0013784193052508 * M_P),
    "proton": (Q_E, M_P),
    "hydrogen1": (1 * Q_E, 1.00782503223 * M_U),
    "hydrogen2": (1 * Q_E, 2.01410177812 * M_U),
    "hydrogen3": (1 * Q_E, 3.0160492779 * M_U),
    "helium3": (2 * Q_E, 3.0160293201 * M_U),
    "helium4": (2 * Q_E, 4.00260325413 * M_U),
    "boron11": (5 * Q_E, 11.00930536 * M_U),
}


def canonical_species_type(name):
    """The table's name of a species_type (aliases resolved); unknown names are refused."""
    k = _SPECIES_ALIASES.get(str(name).lower(), str(name).lower())
    if k not in SPECIES_PROPERTIES:
        raise ValueError("unknown species_type %r (known: %s)" % (name, ", ".join(sorted(set(SPECIES_PROPERTIES) | set(_SPECIES_ALIASES)))))
    return k


def species_charge_mass(species_type):
    """(q, m) of a species_type, as <species>.species_type sets them."""
    return SPECIES_PROPERTIES[canonical_species_type(species_type)]


def nuclear_fusion_type(reactants, products):
    """BinaryCollisionUtils::get_nuclear_fusion_type (BinaryCollisionUtils.cpp:40-123) for the two-product reactions
    and proton-boron: the abi.FUSION_* of the reactants' and products' species types; other combinations are refused."""
    r, p = sorted(reactants), sorted(products)
    if r == ["boron11", "hydrogen1"]:                  # :104-116
        if p != ["helium4"]:
            raise ValueError("proton-boron fusion: exactly one product species, of type helium4")
        return abi.FUSION_PB_3HE4
    if r == ["hydrogen2", "hydrogen3"]:
        if p != ["helium4", "neutron"]:
            raise ValueError("deuterium-tritium fusion: the products must be of type neutron and helium4")
        return abi.FUSION_DT_NHE4
    if r == ["hydrogen2", "hydrogen2"]:
        if p == ["helium3", "neutron"]:
            return abi.FUSION_DD_NHE3
        if p == ["hydrogen1", "hydrogen3"]:
            return abi.FUSION_DD_PT
        raise ValueError("deuterium-deuterium fusion: the products must be of type helium3 and neutron, or hydrogen3 and "
                         "hydrogen1")
    raise NotImplementedError("nuclear fusion between species of type %s and %s is not supported (D + T, D + D and "
                              "p + B11 only)" % tuple(reactants))


class FluidSpecies:
    """A cold relativistic fluid (WarpXFluidContainer): two states of four all-nodal components N, NUx, NUy, NUz
    with 2 guard nodes; the advection writes one from the other, `cur` names the current one."""
    NAMES = ("N", "NUx", "NUy", "NUz")
    NG = (2, 2, 2)

    def __init__(self, sim, name, q, m):
        t = sim.torch
        self.name, self.q, self.m = name, float(q), float(m)
        self.data, self.fabs = [], []
        for _ in range(2):
            descs, arrs = [], []
            for _c in range(4):
                d = abi.make_fab(None, sim.box_lo, sim.box_hi, self.NG, (1, 1, 1))
                a = t.zeros(d.shape, dtype=t.float64, device=sim.device)
                d.p = a.data_ptr()
                descs.append(d)
                arrs.append(a)
            self.data.append(arrs)
            self.fabs.append((abi.pic_fab * 4)(*descs))
        self.cur = 0

    def state(self, which=None):
        return self.fabs[self.cur if which is None else which]


class Simulation:
    def __init__(self, n_cell, prob_lo, prob_hi, nox, galerkin=1, pusher=abi.PUSHER_BORIS,
                 solver=abi.SOLVER_YEE, cfl=1.0, dt=None, dist=None, sort_interval=4,
                 tile=(8, 8, 8), use_bins=True, device=None,
                 use_filter=False, filter_npass=(1, 1, 1), boundaries=None, moving_window=None, nb=None,
                 gamma_boost=1.0, nci_stencils=None):
        """boundaries: abi.pic_boundaries (boundary.field_lo/hi, boundary.particle_lo/hi; default all
        periodic); moving_window: (direction, v/c) == warpx.do_moving_window / moving_window_dir /
        moving_window_v; nb: brick grid (default parallel.brick_grid(world); a moving window needs slabs
        along its direction, e.g. (1, 1, world)); use_bins=False: no cell sort, the order-agnostic kernels.
        solver=abi.SOLVER_NONE (algo.maxwell_solver = none): the fields are never updated, the particles are gathered
        and pushed without depositing; it needs an explicit dt and takes no filter, antenna, NCI corrector or fluid."""
        global _error_source
        if solver == abi.SOLVER_NONE and not dt:
            raise ValueError("algo.maxwell_solver = none needs an explicit dt")
        self.torch, self.L, self.device = self._backend(device)
        _error_source = self.L
        t = self.torch
        self.L.pic_set_error_mode(abi.PIC_ERR_RETURN)   # Python raises instead of abort()
        self.dist = dist
        self.rank = dist.get_rank() if dist is not None else 0
        self.world = dist.get_world_size() if dist is not None else 1
        self.n_cell = tuple(int(v) for v in n_cell)
        self.prob_lo, self.prob_hi = tuple(prob_lo), tuple(prob_hi)
        self.geom = abi.make_geom(n_cell, prob_lo, prob_hi)
        self.dx = [(prob_hi[d] - prob_lo[d]) / n_cell[d] for d in range(3)]     # amrex::Geometry::CellSize
        self.dinv = [1.0 / v for v in self.dx]                                   # WarpX::InvCellSize
        self.nox, self.galerkin, self.pusher, self.solver = nox, galerkin, pusher, solver
        self.dt = dt if dt else cfl * max_dt(solver, self.dx)
        self.use_filter, self.filter_npass = bool(use_filter), tuple(int(v) for v in filter_npass)
        self.boundaries, self.moving_window = boundaries, moving_window
        # warpx.gamma_boost with boost_direction = z; prob_lo / prob_hi are boosted-frame values already
        # (ConvertLabParamsToBoost, Source/Utils/WarpXUtil.cpp:180-262)
        self.gamma_boost, self.beta_boost = float(gamma_boost), abi.beta_of_gamma(gamma_boost)
        if boundaries is not None:
            for d in range(3):
                self.geom.periodic[d] = 1 if boundaries.field_lo[d] == abi.FIELD_PERIODIC else 0
        self.nonperiodic = not all(self.geom.periodic[d] for d in range(3))
        # particles.use_fdtd_nci_corr: (stencil_exeybz, stencil_bxbyez) from nci_godfrey_stencils
        self.nci_stencils = nci_stencils
        self.lasers = []
        self.time = 0.0
        g = guard_cells(nox, self.dt, self.dx, self.use_filter, self.filter_npass, moving_window is not None,
                        nci_stencils is not None)
        self.ng_EB, self.ng_J, self.ng_FG, self.ng_FS = g["ng_EB"], g["ng_J"], g["ng_FG"], g["ng_FS"]
        self.dec = parallel.Decomposition(self.n_cell, tuple(nb) if nb is not None else parallel.brick_grid(self.world),
                                          self.rank)
        self.box_lo, self.box_hi = self.dec.box_lo, self.dec.box_hi
        self.sort_interval, self.tile, self.use_bins = sort_interval, tuple(tile), use_bins
        # fields: Ex Ey Ez Bx By Bz jx jy jz, AMReX-shaped (valid + guards), Fortran order
        self.data, descs = [], []
        for c in range(9):
            ng = self.ng_EB if c < 6 else self.ng_J
            d = abi.make_fab(None, self.box_lo, self.box_hi, ng, abi.YEE_STAG[c])
            a = t.zeros(d.shape, dtype=t.float64, device=self.device)
            d.p = a.data_ptr()
            self.data.append(a)
            descs.append(d)
        self.fab = descs
        self.species = []
        self.fluids = []
        self.is_synchronized = True
        self.istep = 0
        self._scratch = t.zeros(8, dtype=t.float64, device=self.device)
        # The step sequence runs in the library's C++ driver (csrc/engine.cu); with several ranks it
        # exchanges guard cells and particles over its own NCCL communicator (csrc/comm.cu; the
        # 128-byte id is broadcast through torch.distributed, the only thing torch transports).
        self.comm = None
        self.native = self.L.pic_engine_create(C.byref(self.geom), abi.int3(self.box_lo), abi.int3(self.box_hi),
                                               nox, galerkin, pusher, solver, cfl, self.dt, sort_interval,
                                               1 if self.use_filter else 0, abi.int3(self.filter_npass))
        if not self.native:
            raise RuntimeError("pic_b200: " + self.L.pic_last_error().decode())
        self.collisions = []
        self.flux_injectors = []
        if boundaries is not None:
            check(self.L.pic_engine_set_boundaries(self.native, C.byref(boundaries)))
        if moving_window is not None:
            check(self.L.pic_engine_set_moving_window(self.native, int(moving_window[0]), float(moving_window[1])))
        if self.gamma_boost > 1.0:
            check(self.L.pic_engine_set_boost(self.native, self.gamma_boost, self.beta_boost))
        if nci_stencils is not None:
            check(self.L.pic_engine_set_nci_corrector(self.native, (C.c_double * 5)(*nci_stencils[0]),
                                                      (C.c_double * 5)(*nci_stencils[1])))
        g12 = (C.c_int * 12)()
        self.L.pic_engine_guards(self.native, g12)
        assert list(g12) == self.ng_EB + self.ng_J + self.ng_FG + self.ng_FS
        assert self.L.pic_engine_dt(self.native) == self.dt
        if self.world > 1:
            self._sync()
            self.comm = shared_comm(self.L, dist, t, self.device)
            check(self.L.pic_engine_set_comm(self.native, self.comm, abi.int3(self.dec.nb)))
        check(self.L.pic_engine_set_fields(self.native, (abi.pic_fab * 9)(*self.fab)))

    def close(self):
        """Destroy the C++ driver of this run (device scratch, events).  The NCCL communicator is the process's shared
        one (shared_comm) and outlives the Simulation.  Idempotent; __del__ calls it."""
        native, self.native = getattr(self, "native", None), None
        if native:
            try:
                self._sync()
            except Exception:            # interpreter shutdown
                pass
            self.L.pic_engine_destroy(native)
        self.comm = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _backend(self, device):
        """(torch, library, device) of this run: a CUDA device and the nvcc-built library -- there is no CPU
        fallback.  (tests/host_harness overrides this hook to run the SAME sources, compiled by g++ against its
        SIMT emulator, for the CPU test-suite of a container without a GPU; nothing in the package does.)"""
        t = require_cuda()
        return t, lib(), (t.device("cuda", t.cuda.current_device()) if device is None else device)

    def _sync(self):
        self.torch.cuda.synchronize()

    def enable_stage_timing(self, on=True):
        """CUDA events (on the launching stream) around every stage, recorded inside pic_engine_evolve
        (pic_engine_enable_timing; switching on resets the sums); read with stage_ms()."""
        check(self.L.pic_engine_enable_timing(self.native, 1 if on else 0))

    def stage_ms(self):
        """{stage: (average milliseconds per call, calls)} of every timed stage (synchronises)."""
        n = self.L.pic_engine_stage_count()
        ms, calls = (C.c_double * n)(), (C.c_long * n)()
        check(self.L.pic_engine_stage_ms(self.native, ms, calls))
        return {self.L.pic_engine_stage_name(k).decode(): (ms[k] / calls[k], int(calls[k])) for k in range(n) if calls[k]}

    # ------------------------------------------------------------------------------------
    @property
    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def add_species(self, name, q, m, x, y, z, w, ux, uy, uz, capacity_factor=None, ids=None, species_type=None,
                    capacity=None):
        """Particles must lie inside this rank's box (use workloads.* with box_lo/box_hi).  ids: 64-bit particle ids
        (default: rank << 40 | index).  species_type: <species>.species_type (see SPECIES_PROPERTIES), which
        add_fusion reads.  capacity: entries of every particle array (default len(x) * capacity_factor); a species that
        receives fusion products needs room for them."""
        if capacity_factor is None:
            capacity_factor = 1.0 if self.world == 1 else 1.25
        if self.fluids:
            raise NotImplementedError("runs with fluid species take no particle species")
        arrays = dict(x=x, y=y, z=z, w=w, ux=ux, uy=uy, uz=uz)
        cap = int(len(x) * capacity_factor) + (0 if self.world == 1 else 65536) if capacity is None else int(capacity)
        sp = Species(self, name, q, m, arrays, cap, ids=ids, species_type=species_type)
        self._register_species(sp)
        return sp

    def add_empty_species(self, name, capacity, species_type=None, q=None, m=None):
        """A species without particles and room for `capacity` (e.g. the products of a fusion).  q and m default to
        those of species_type."""
        if species_type is not None:
            dq, dm = species_charge_mass(species_type)
            q, m = dq if q is None else q, dm if m is None else m
        if q is None or m is None:
            raise ValueError("add_empty_species: give species_type or q and m")
        empty = np.empty(0)
        return self.add_species(name, q, m, empty, empty, empty, empty, empty, empty, empty, species_type=species_type,
                                capacity=int(capacity))

    def add_plasma_species(self, name, q, m, injector, capacity, species_type=None):
        """A species created on the device by its plasma injector (PhysicalParticleContainer::InitData ->
        AddPlasma over the whole domain, PhysicalParticleContainer.cpp:450-454,855-922); with
        injector.do_continuous_injection the moving window keeps refilling the uncovered slab.
        capacity: entries of every particle array (the run must never exceed it).  species_type: as for add_species."""
        injector.gamma_boost, injector.beta_boost = self.gamma_boost, self.beta_boost
        empty = np.empty(0)
        sp = Species(self, name, q, m, {k: empty for k in Species.NAMES}, int(capacity), species_type=species_type)
        soa = sp.soa(0)
        # ids = creation index in the order a single box would create the particles (k slowest): the
        # ranks below this one come first when the bricks are slabs along z
        first_id = 0
        for r in range(self.rank):
            other = parallel.Decomposition(self.n_cell, self.dec.nb, r)
            cnt = self.L.pic_add_plasma(C.byref(injector), C.byref(self.geom), abi.dbl3(self.dx), abi.int3(other.box_lo),
                                        abi.int3(other.box_hi), abi.dbl3(self.prob_lo), abi.dbl3(self.prob_hi), None, 0, 0,
                                        0.0, None)
            if cnt < 0:
                raise RuntimeError("pic_b200: " + self.L.pic_last_error().decode())
            first_id += cnt
        n = self.L.pic_add_plasma(C.byref(injector), C.byref(self.geom), abi.dbl3(self.dx), abi.int3(self.box_lo),
                                  abi.int3(self.box_hi), abi.dbl3(self.prob_lo), abi.dbl3(self.prob_hi), C.byref(soa),
                                  sp.capacity, first_id, 0.0, self.stream)
        if n < 0:
            raise RuntimeError("pic_b200: " + self.L.pic_last_error().decode())
        sp.np = int(n)
        self._register_species(sp)
        check(self.L.pic_engine_set_injector(self.native, len(self.species) - 1, C.byref(injector)))
        return sp

    def add_beam_species(self, name, q, m, beam, capacity, species_type=None):
        """A Gaussian beam (abi.pic_gaussian_beam, <species>.injection_style = "gaussian_beam") created on the device by
        pic_add_gaussian_beam (PhysicalParticleContainer::AddGaussianBeam + InitData, PhysicalParticleContainer.cpp:
        450-454,503-677), in the lab frame or mapped into this run's boosted frame at the current time.  Each rank keeps
        the particles of its own brick; ids are creation indices, the same on any decomposition.  A beam is created
        once and never refilled.  capacity: entries of every particle array (the run must never exceed it).  species_type:
        as for add_species."""
        beam.gamma_boost, beam.beta_boost = self.gamma_boost, self.beta_boost
        empty = np.empty(0)
        sp = Species(self, name, q, m, {k: empty for k in Species.NAMES}, int(capacity), species_type=species_type)
        soa = sp.soa(0)
        # this brick's half-open share of the domain; the domain's own faces are open (the library drops or wraps there)
        own_lo = [self.prob_lo[d] + self.dx[d] * self.box_lo[d] if self.box_lo[d] > 0 else -math.inf for d in range(3)]
        own_hi = [self.prob_lo[d] + self.dx[d] * (self.box_hi[d] + 1) if self.box_hi[d] < self.n_cell[d] - 1 else math.inf
                  for d in range(3)]
        n = self.L.pic_add_gaussian_beam(C.byref(beam), q, C.byref(self.geom), abi.dbl3(own_lo), abi.dbl3(own_hi),
                                         C.byref(soa), sp.capacity, self.time, self.stream)
        if n < 0:
            raise RuntimeError("pic_b200: " + self.L.pic_last_error().decode())
        sp.np = int(n)
        self._register_species(sp)
        return sp

    def add_fluid_species(self, name, q, m, density, momentum):
        """fluids.species_names / <species>.*: a cold relativistic fluid (WarpXFluidContainer), initialised like InitData
        (Source/Fluids/WarpXFluidContainer.cpp:166-254) in the lab frame over this rank's valid nodes, at
        x = prob_lo + i dx: N = n, NU = n u c.  density(x, y, z) -> n [m^-3] and momentum(x, y, z) -> (ux, uy, uz) in
        units of c are evaluated here on the host in float64, on numpy arrays of node coordinates.  One rank, periodic
        domains without a moving window or boost, no particle species or antennas; other runs are refused before
        anything is allocated."""
        if self.nonperiodic:
            raise NotImplementedError("fluid species: every face must be periodic")
        if self.moving_window is not None:
            raise NotImplementedError("fluid species: moving windows are not supported")
        if self.gamma_boost > 1.0:
            raise NotImplementedError("fluid species: boosted frames are not supported")
        if self.world > 1:
            raise NotImplementedError("fluid species: one rank only")
        if self.species or self.lasers:
            raise NotImplementedError("fluid species: runs with particle species or antennas are not supported")
        coords = [self.prob_lo[d] + np.arange(self.box_lo[d], self.box_hi[d] + 2) * self.dx[d] for d in range(3)]
        Z, Y, X = np.meshgrid(coords[2], coords[1], coords[0], indexing="ij")
        n = np.broadcast_to(np.asarray(density(X, Y, Z), dtype=np.float64), X.shape)
        u = [np.broadcast_to(np.asarray(v, dtype=np.float64), X.shape) for v in momentum(X, Y, Z)]
        fl = FluidSpecies(self, name, q, m)
        vs = fl.fabs[0][0].valid_slices()
        vals = (n, n * (u[0] * C_LIGHT), n * (u[1] * C_LIGHT), n * (u[2] * C_LIGHT))
        for c in range(4):
            fl.data[0][c][vs].copy_(self.torch.from_numpy(np.array(vals[c], dtype=np.float64)))
        check(self.L.pic_engine_add_fluid_species(self.native, fl.q, fl.m, fl.fabs[0], fl.fabs[1]))
        self.fluids.append(fl)
        return fl

    def fluid_numpy(self, i):
        """(descriptor, {"N", "NUx", "NUy", "NUz": numpy array [k, j, i], guards included}) of fluid species i."""
        fl = self.fluids[i]
        return fl.state()[0], {name: fl.data[fl.cur][c].cpu().numpy() for c, name in enumerate(FluidSpecies.NAMES)}

    def add_laser(self, laser):
        """lasers.names / <laser>.*: a Gaussian antenna (LaserParticleContainer ctor + InitData,
        LaserParticleContainer.cpp:84-270,369-560).  The antenna particles are generated on the host like
        the reference does and uploaded once."""
        t = self.torch
        laser.gamma_boost, laser.beta_boost = self.gamma_boost, self.beta_boost
        dxa, lo, hi = abi.dbl3(self.dx), abi.dbl3(self.prob_lo), abi.dbl3(self.prob_hi)
        n = self.L.pic_laser_antenna_particles(C.byref(laser), dxa, lo, hi, None, None, None, None, 0)
        host = np.zeros((7, max(n, 1)))
        if n > 0:
            got = self.L.pic_laser_antenna_particles(C.byref(laser), dxa, lo, hi, host[0].ctypes.data, host[1].ctypes.data,
                                                     host[2].ctypes.data, host[3].ctypes.data, n)
            assert got == n
        buf = t.from_numpy(host).to(self.device)
        ids = t.arange(max(n, 1), dtype=t.int64, device=self.device)
        soa = abi.pic_soa()
        for k, name in enumerate(Species.NAMES):
            setattr(soa, name, buf[k].data_ptr())
        soa.idcpu = ids.data_ptr()
        soa.np = n
        check(self.L.pic_engine_add_laser(self.native, C.byref(laser), C.byref(soa), max(n, 1)))
        self.lasers.append(dict(laser=laser, buf=buf, ids=ids, np=n))
        return len(self.lasers) - 1

    def add_collision(self, species1, species2, coulomb_log=-1.0, ndt=1, seed=0):
        """One entry of collisions.collision_names with <name>.type = pairwisecoulomb: <name>.species = species1
        species2 (Species objects, names or indices; the same species twice is an intra-species collision),
        <name>.CoulombLog (<= 0: computed per pair from the cell's Debye length) and <name>.ndt.  seed keys the
        collision's random streams (warpx.random_seed): a run's result depends on the particles by id, the seed, the
        collision's position in the list, the step and the cell, not on their storage order.  One rank only.  A restarted run registers
        its collisions again, in the same order.  Returns the collision's index."""
        isp = [self._species_index(v) for v in (species1, species2)]
        check(self.L.pic_engine_add_collision(self.native, isp[0], isp[1], float(coulomb_log), int(ndt), int(seed)))
        self.collisions.append(dict(species=tuple(isp), coulomb_log=float(coulomb_log), ndt=int(ndt), seed=int(seed)))
        return len(self.collisions) - 1

    def add_fusion(self, species1, species2, products, multiplier=1.0, probability_threshold=0.02,
                   probability_target_value=0.002, ndt=1, seed=0):
        """One entry of collisions.collision_names with <name>.type = nuclearfusion: <name>.species = species1 species2
        (the same species twice: D + D within one species), <name>.product_species = products (two species, in the
        order the products are written; one helium4 species for proton-boron), <name>.fusion_multiplier,
        fusion_probability_threshold, fusion_probability_target_value and ndt.  The reaction follows from the species
        types, as get_nuclear_fusion_type infers it: D + T -> n + He4, D + D -> n + He3 or p + T, p + B11 -> 3 He4 (six
        alphas of weight w / 2 per event, three at each reactant's position).  Products appear at their
        reactants' positions; reactants whose weight is used up leave the run at the end of the step.  It shares the
        collision index, the schedule and the determinism of add_collision.  One rank only.  Returns the index."""
        isp = [self._species_index(v) for v in (species1, species2)]
        if len(products) not in (1, 2):
            raise ValueError("add_fusion: a fusion takes one or two product species")
        ipr = [self._species_index(v) for v in products]
        types = [self.species[i].species_type for i in isp + ipr]
        if any(v is None for v in types):
            raise ValueError("add_fusion: every reactant and product needs a species_type")
        ftype = nuclear_fusion_type(types[:2], types[2:])
        ipr_b = ipr[1] if len(ipr) == 2 else -1
        check(self.L.pic_engine_add_fusion(self.native, isp[0], isp[1], ipr[0], ipr_b, ftype, float(multiplier),
                                           float(probability_threshold), float(probability_target_value), int(ndt),
                                           int(seed)))
        self.collisions.append(dict(species=tuple(isp), products=tuple(ipr), type=ftype, multiplier=float(multiplier),
                                    probability_threshold=float(probability_threshold),
                                    probability_target_value=float(probability_target_value), ndt=int(ndt),
                                    seed=int(seed)))
        return len(self.collisions) - 1

    def add_flux_injection(self, species, injector):
        """A source of particles through a plane for species (a Species object, name or index): injector is an
        abi.pic_flux_injector from abi.make_flux_injector and stands for <species>.injection_style = NFluxPerCell with
        <species>.num_particles_per_cell, surface_flux_pos, flux_normal_axis, flux_direction, flux_tmin, flux_tmax,
        xmin..zmax, flux_profile = constant with <species>.flux (or a constant parse_flux_function) and
        momentum_distribution_type = gaussianflux with ux_m..uz_m, ux_th..uz_th.  Every step then injects
        int(num_particles_per_cell + Random) particles per plane cell, weighted by flux dt, before the step's particle
        boundaries and migration (PhysicalParticleContainer::AddPlasmaFlux).  The species needs the capacity for what
        the run injects.  Lab frame only: runs with a moving window or a boosted frame are refused.  The injector's
        index (the order of these calls) is part of its random streams; a restarted run registers its injectors
        again, in the same order.  Returns the index."""
        if self.moving_window is not None or self.gamma_boost > 1.0:
            raise NotImplementedError("flux injection: lab-frame runs without a moving window only")
        isp = self._species_index(species)
        check(self.L.pic_engine_add_flux_injector(self.native, isp, C.byref(injector)))
        self.flux_injectors.append((isp, injector))
        return len(self.flux_injectors) - 1

    def set_species_flags(self, species, do_not_push=False, do_not_deposit=False):
        """<species>.do_not_push / <species>.do_not_deposit of a species (a Species object, name or index), also one that
        read_checkpoint restored (checkpoints do not carry the flags).  do_not_push: the species' positions and momenta
        keep their bits while it is still sorted, collided, fused and wrapped; do_not_deposit: it is pushed but adds
        nothing to J or to rho_numpy().  Immobile targets, test species and diagnostics-only species use them."""
        isp = self._species_index(species)
        check(self.L.pic_engine_set_species_flags(self.native, isp, 1 if do_not_push else 0, 1 if do_not_deposit else 0))
        sp = self.species[isp]
        sp.do_not_push, sp.do_not_deposit = bool(do_not_push), bool(do_not_deposit)

    def species_next_id(self, isp):
        """The id the next particle species isp creates receives (its id counter)."""
        return int(self.L.pic_engine_species_next_id(self.native, int(isp)))

    def set_species_next_id(self, isp, next_id):
        """Restart: continue species isp's id counter from a checkpoint."""
        check(self.L.pic_engine_set_species_next_id(self.native, int(isp), int(next_id)))

    def _species_index(self, v):
        if isinstance(v, (int, np.integer)):
            return int(v)
        for i, sp in enumerate(self.species):
            if sp is v or (isinstance(v, str) and sp.name == v):
                return i
        raise ValueError("add_collision: no species %r" % (v,))

    def laser_numpy(self, il, sort_by_id=True):
        la = self.lasers[il]
        n = int(self.L.pic_engine_laser_np(self.native, il))
        out = {name: la["buf"][k, :n].cpu().numpy() for k, name in enumerate(Species.NAMES)}
        out["id"] = la["ids"][:n].cpu().numpy()
        if sort_by_id:
            order = np.argsort(out["id"], kind="stable")
            out = {k: v[order] for k, v in out.items()}
        return out

    def _register_species(self, sp):
        """Append sp and hand it to the C++ driver.  With use_bins the driver gets the cell-sort scratch and sorts the
        particles at once; without, it keeps no bins, never sorts and runs the order-agnostic kernels."""
        self.species.append(sp)
        cell_start = work = None
        if self.use_bins:
            t = self.torch
            nb = self.L.pic_bins_count(abi.int3(self.box_lo), abi.int3(self.box_hi), abi.int3(self.tile))
            sp.cell_start = t.empty(nb + 1, dtype=t.int32, device=self.device)
            sp.work = t.empty(self.L.pic_sort_workspace_bytes(sp.capacity, nb), dtype=t.uint8, device=self.device)
            cell_start, work = sp.cell_start.data_ptr(), sp.work.data_ptr()
        a, b = sp.soa(0), sp.soa(1)
        check(self.L.pic_engine_add_species(self.native, sp.q, sp.m, C.byref(a), C.byref(b), sp.capacity, cell_start,
                                            abi.int3(self.tile), work, self.stream))
        self._sync_from_native()

    def _sync_from_native(self):
        """Mirror the C++ driver's view (current buffer, count) into the Python objects."""
        for isp, sp in enumerate(self.species):
            n = C.c_long()
            sp.cur = self.L.pic_engine_species_buffer(self.native, isp, C.byref(n))
            sp.np = n.value

    def lower_corner(self, ng):
        """WarpX::LowerCorner of the box grown by ng (Source/WarpX.cpp:2851-2874; RealBox lo =
        prob_lo + index*dx) and lbound of that box."""
        lo = [self.box_lo[d] - ng[d] for d in range(3)]
        xyzmin = [self.prob_lo[d] + self.dx[d] * lo[d] for d in range(3)]
        return abi.dbl3(xyzmin), abi.int3(lo)

    def Evolve(self, numsteps, synchronize_last=True):
        """WarpX::Evolve: numsteps steps of the C++ driver (pic_engine_evolve), then its view mirrored here."""
        check(self.L.pic_engine_evolve(self.native, numsteps, 1 if synchronize_last else 0, self.stream))
        self.istep += numsteps
        self.is_synchronized = bool(synchronize_last)
        self._sync_from_native()
        for i, fl in enumerate(self.fluids):
            fl.cur = self.L.pic_engine_fluid_state(self.native, i)
        # the moving window translates the problem domain; t_new
        dom = (C.c_double * 6)()
        self.L.pic_engine_prob_domain(self.native, dom)
        self.prob_lo, self.prob_hi = tuple(dom[0:3]), tuple(dom[3:6])
        for d in range(3):
            self.geom.prob_lo[d], self.geom.prob_hi[d] = dom[d], dom[3 + d]
        self.time = self.L.pic_engine_time(self.native)

    def set_step(self, istep, time):
        """Restart: continue counting steps (cell-sort cadence) and time from a checkpoint."""
        self.istep, self.time = int(istep), float(time)
        check(self.L.pic_engine_set_step(self.native, int(istep), float(time)))

    # ---- diagnostics -------------------------------------------------------------------
    def field_energy(self):
        """FieldEnergy reduced diagnostic (Diagnostics/ReducedDiags/FieldEnergy.cpp:120-144):
        (E energy, B energy) in J, summed over ranks."""
        t = self.torch
        out = self._scratch
        for c in range(6):
            check(self.L.pic_sum_squares_unique(C.byref(self.fab[c]), C.byref(self.geom),
                                                out[c:c + 1].data_ptr(), self.stream))
        e2b2 = t.stack([out[0:3].sum(), out[3:6].sum()])
        if self.dist is not None and self.world > 1:
            self.dist.all_reduce(e2b2)
        dV = self.dx[0] * self.dx[1] * self.dx[2]
        v = e2b2.cpu().numpy()
        return 0.5 * v[0] * EP0 * dV, 0.5 * v[1] / MU0 * dV

    def particle_energy(self):
        """ParticleEnergy reduced diagnostic (Diagnostics/ReducedDiags/ParticleEnergy.cpp:86-170):
        per species (total kinetic energy [J], sum of weights), summed over ranks."""
        t = self.torch
        out = t.zeros((max(len(self.species), 1), 2), dtype=t.float64, device=self.device)
        for isp, sp in enumerate(self.species):
            soa = sp.soa()
            check(self.L.pic_particle_energy(C.byref(soa), sp.m, out[isp].data_ptr(), self.stream))
        if self.dist is not None and self.world > 1:
            self.dist.all_reduce(out)
        v = out.cpu().numpy()
        return [(float(v[i, 0]), float(v[i, 1])) for i in range(len(self.species))]

    def particle_number(self):
        """ParticleNumber reduced diagnostic (Diagnostics/ReducedDiags/ParticleNumber.cpp): per species (number of
        macroparticles, sum of weights), summed over ranks."""
        out = []
        for sp in self.species:
            w = sp.array("w")
            n, ws = sp.np, float(w.sum().item()) if sp.np else 0.0
            if self.dist is not None and self.world > 1:
                tt = self.torch.tensor([float(n), ws], dtype=self.torch.float64, device=self.device)
                self.dist.all_reduce(tt)
                n, ws = int(tt[0].item()), float(tt[1].item())
            out.append((int(n), ws))
        return out

    def rho_numpy(self):
        """The `rho` diagnostic of a plotfile (Diagnostics/ComputeDiagFunctors/RhoFunctor.cpp:35-81): every
        container (species without do_not_deposit, then laser antennas) deposits its charge on a nodal array with ng_depos_rho guard
        cells and applies the PEC / reflecting image charge, the containers are added, then
        WarpX::ApplyFilterandSumBoundaryRho (Parallelization/WarpXComm.cpp:1552-1568).  Returns
        (descriptor, numpy array [k, j, i]).  One rank."""
        if self.world > 1:
            raise NotImplementedError("rho diagnostic: one rank")
        t = self.torch
        base = max(self.nox, 2) if self.moving_window is not None else self.nox
        ng = max(base + 1 + int(math.ceil(C_LIGHT * self.dt / self.dx[d])) for d in range(3))   # GuardCellManager.cpp:130-165

        def make(ngv):
            d = abi.make_fab(None, self.box_lo, self.box_hi, ngv, (1, 1, 1))
            a = t.zeros(d.shape, dtype=t.float64, device=self.device)
            d.p = a.data_ptr()
            return d, a

        rho_d, rho = make((ng,) * 3)
        one_d, one = make((ng,) * 3)
        xyzmin, lo = self.lower_corner((ng,) * 3)
        containers = [(sp.soa(), sp.q) for sp in self.species if not sp.do_not_deposit]   # MultiParticleContainer.cpp:576,598
        for il, la in enumerate(self.lasers):
            soa = abi.pic_soa()
            for k, name in enumerate(Species.NAMES):
                setattr(soa, name, la["buf"][k].data_ptr())
            soa.idcpu, soa.np = la["ids"].data_ptr(), int(self.L.pic_engine_laser_np(self.native, il))
            containers.append((soa, 1.0))                                  # LaserParticleContainer: charge = 1
        for soa, q in containers:
            one.zero_()
            check(self.L.pic_deposit_charge(C.byref(soa), 0, soa.np, C.byref(one_d), abi.dbl3(self.dinv), xyzmin, lo, q,
                                            self.nox, self.stream))
            if self.nonperiodic:
                check(self.L.pic_apply_pec_rho(C.byref(one_d), C.byref(self.geom), C.byref(self.boundaries), self.stream))
            rho += one
        for fl in self.fluids:                                             # RhoFunctor.cpp:47-51
            check(self.L.pic_fluid_deposit_charge(C.byref(fl.state()[0]), C.byref(rho_d), fl.q, self.stream))
        work_d, work, ngw = rho_d, rho, [ng] * 3
        if self.use_filter:
            ngw = [ng + self.filter_npass[d] for d in range(3)]
            work_d, work = make(ngw)
            check(self.L.pic_apply_filter(C.byref(rho_d), C.byref(work_d), abi.int3(self.filter_npass), self.stream))
        allper = abi.make_geom(self.n_cell, self.prob_lo, self.prob_hi)      # the refresh after the sum covers every guard
        for dim in range(3):
            if self.geom.periodic[dim]:
                check(self.L.pic_sum_boundary_local(C.byref(work_d), dim, ngw[dim], C.byref(self.geom), self.stream))
        for dim in range(3):
            if self.geom.periodic[dim]:
                check(self.L.pic_fill_boundary_local(C.byref(work_d), dim, ngw[dim], C.byref(allper), self.stream))
        if self.use_filter:
            n = self.filter_npass
            rho.copy_(work[n[2]:work.shape[0] - n[2], n[1]:work.shape[1] - n[1], n[0]:work.shape[2] - n[0]])
        return rho_d, rho.cpu().numpy()

    def total_particles(self):
        n = sum(sp.np for sp in self.species)
        if self.dist is not None and self.world > 1:
            tt = self.torch.tensor([n], dtype=self.torch.int64, device=self.device)
            self.dist.all_reduce(tt)
            n = int(tt.item())
        return n

    def set_field(self, comp, values):
        """Overwrite component comp (0..8 = Ex..jz), guards included, with a host array shaped like
        field_numpy(comp)[1] (e.g. warpx.E/B_ext_grid_init_style = parse_*_ext_grid_function at start-up)."""
        a = np.ascontiguousarray(values, dtype=np.float64)
        assert a.shape == tuple(self.data[comp].shape)
        self.data[comp].copy_(self.torch.from_numpy(a))

    def field_numpy(self, comp):
        """(descriptor, numpy array [k, j, i]) of component comp (0..8 = Ex..jz)."""
        return self.fab[comp], self.data[comp].cpu().numpy()

    def species_numpy(self, isp, sort_by_id=False):
        sp = self.species[isp]
        out = {n: sp.array(n).cpu().numpy() for n in Species.NAMES}
        out["id"] = sp.id_array().cpu().numpy()
        if sort_by_id:
            order = np.argsort(out["id"], kind="stable")
            out = {k: v[order] for k, v in out.items()}
        return out
