"""Deterministic initial conditions for the benchmark / parity configurations (host side, numpy).

These restate what the reference's plasma injector produces for the decks named in
BASELINE.json so that the oracle and the CUDA engine start from bit-identical arrays:

* positions: ``NUniformPerCell`` regular lattice, ``InjectorPositionRegular::getPositionUnitBox``
  (Source/Initialization/InjectorPosition.H:67-108) and ``getCellCoords``
  (Source/Particles/PhysicalParticleContainer.cpp:151-173): ``pos = lo + (i + r) * dx``;
* weights: ``w = n * dx*dy*dz / ppc`` (Source/Particles/AddPlasmaUtilities.H:73-77,
  PhysicalParticleContainer.cpp:1275-1288);
* momenta: ``u = (gamma*beta) * c`` (PhysicalParticleContainer.cpp:1271-1273).

Where the reference draws random numbers from AMReX's stream (config 2's thermal momenta, config 4's Gaussian beam),
a counter-based Philox4x64-10 generator keyed by a seed replaces it (philox_normal, beam_normals), so that every
decomposition, the oracle and the device see the same draws.  AMReX's own stream is not reproduced.
"""
import numpy as np

# CODATA 2018, Source/ablastr/constant.H:44-54
C = 299792458.0
EP0 = 8.8541878128e-12
MU0 = 1.25663706212e-06
Q_E = 1.602176634e-19
M_E = 9.1093837015e-31


def lattice_positions(n_cell, prob_lo, prob_hi, ppc, box_lo=None, box_hi=None):
    """Cell-major regular lattice (cell index i fastest, then j, k; particle-in-cell slowest
    varying inside a cell like the reference's i_part loop).  Returns x, y, z (float64)."""
    n_cell = np.asarray(n_cell)
    lo = np.zeros(3, dtype=int) if box_lo is None else np.asarray(box_lo)
    hi = n_cell - 1 if box_hi is None else np.asarray(box_hi)
    dx = (np.asarray(prob_hi, dtype=np.float64) - np.asarray(prob_lo, dtype=np.float64)) / n_cell
    nx, ny, nz = (int(v) for v in ppc)
    # i_part -> (ix, iy, iz) exactly as InjectorPosition.H:99-102
    ip = np.arange(nx * ny * nz)
    ixp = ip // (ny * nz)
    izp = (ip - ixp * (ny * nz)) // ny
    iyp = (ip - ixp * (ny * nz)) - ny * izp
    r = [(0.5 + ixp) / nx, (0.5 + iyp) / ny, (0.5 + izp) / nz]
    idx = [np.arange(lo[d], hi[d] + 1) for d in range(3)]
    K, J, I = np.meshgrid(idx[2], idx[1], idx[0], indexing="ij")   # i fastest
    cells = [I.ravel(), J.ravel(), K.ravel()]
    out = []
    for d in range(3):
        # (ncell, ppc) -> flattened with the in-cell index fastest
        p = prob_lo[d] + (cells[d][:, None] + r[d][None, :]) * dx[d]
        out.append(np.ascontiguousarray(p.ravel()))
    return out


def langmuir_3d(n=64, ppc=(1, 1, 1), lx=40.0e-6, n0=2.0e24, epsilon=0.01):
    """Config 1: Examples/Tests/langmuir/inputs_base_3d (two species, analytic momenta)."""
    prob_lo, prob_hi = (-lx / 2,) * 3, (lx / 2,) * 3
    n_cell = (n, n, n)
    x, y, z = lattice_positions(n_cell, prob_lo, prob_hi, ppc)
    dx = lx / n
    wp = np.sqrt(2.0 * n0 * Q_E ** 2 / (EP0 * M_E))   # inputs_base_3d:8
    kp = wp / C
    k = 2.0 * 2.0 * np.pi / lx
    a = epsilon * k / kp
    ux = a * np.sin(k * x) * np.cos(k * y) * np.cos(k * z)
    uy = a * np.cos(k * x) * np.sin(k * y) * np.cos(k * z)
    uz = a * np.cos(k * x) * np.cos(k * y) * np.sin(k * z)
    w = np.full_like(x, n0 * dx ** 3 / (ppc[0] * ppc[1] * ppc[2]))
    species = [
        dict(name="electrons", q=-Q_E, m=M_E, x=x, y=y, z=z, w=w, ux=ux * C, uy=uy * C, uz=uz * C),
        dict(name="positrons", q=Q_E, m=M_E, x=x.copy(), y=y.copy(), z=z.copy(), w=w.copy(),
             ux=-ux * C, uy=-uy * C, uz=-uz * C),
    ]
    return dict(n_cell=n_cell, prob_lo=prob_lo, prob_hi=prob_hi, species=species,
                analytic=dict(k=k, wp=wp, epsilon=epsilon))


def langmuir_fluid_3d(n=64, lx=40.0e-6, n0=2.0e24, epsilon=0.01):
    """Examples/Tests/langmuir_fluids/inputs_test_3d_langmuir_fluid: electron and positron cold fluids of density n0
    with the Langmuir wave's momenta, periodic, Yee, cfl 1, 40 steps.  Each fluid: name, q, m, density(x, y, z) and
    momentum(x, y, z) -> (ux, uy, uz) in units of c, for Simulation.add_fluid_species."""
    wp = np.sqrt(2.0 * n0 * Q_E ** 2 / (EP0 * M_E))   # the deck's my_constants
    kp = wp / C
    k = 2.0 * 2.0 * np.pi / lx
    a = epsilon * k / kp

    def density(x, y, z):
        return np.full(np.shape(x), n0)

    def momentum(sign):
        return lambda x, y, z: (sign * a * np.sin(k * x) * np.cos(k * y) * np.cos(k * z),
                                sign * a * np.cos(k * x) * np.sin(k * y) * np.cos(k * z),
                                sign * a * np.cos(k * x) * np.cos(k * y) * np.sin(k * z))

    fluids = [dict(name="electrons", q=-Q_E, m=M_E, density=density, momentum=momentum(1.0)),
              dict(name="positrons", q=Q_E, m=M_E, density=density, momentum=momentum(-1.0))]
    return dict(n_cell=(n, n, n), prob_lo=(-lx / 2,) * 3, prob_hi=(lx / 2,) * 3, fluids=fluids, max_step=40,
                analytic=dict(k=k, wp=np.sqrt(2.0 * n0 * Q_E ** 2 / (EP0 * M_E)), epsilon=epsilon))


def philox_normal(seed, first_id, count, ncomp=3):
    """Counter-based N(0,1) numbers: particle `id` always gets the same values, independent of how
    the domain is decomposed (SURVEY.md section 8d, config 2).  numpy Philox4x64 keyed by `seed`,
    advanced to the particle id (one 4x64 block = 4 uint64 -> 2 Box-Muller pairs per particle)."""
    out = np.empty((count, ncomp))
    chunk = 1 << 22                      # bounded temporaries for the 10^8-particle configurations
    for b in range(0, count, chunk):
        n = min(chunk, count - b)
        bg = np.random.Philox(key=seed)
        bg.advance(int(first_id) + b)    # one counter increment (4 x uint64) per particle
        raw = bg.random_raw(4 * n).reshape(n, 4)
        u = (raw >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)   # [0,1)
        u1 = 1.0 - u[:, 0:2]             # (0,1]
        r = np.sqrt(-2.0 * np.log(u1))
        th = 2.0 * np.pi * u[:, 2:4]
        g = (r[:, 0] * np.cos(th[:, 0]), r[:, 0] * np.sin(th[:, 0]), r[:, 1] * np.cos(th[:, 1]))
        for c in range(ncomp):
            out[b:b + n, c] = g[c]
    return out


def philox_blocks(seed, first_block, nblocks):
    """Raw Philox4x64-10 words, shape (nblocks, 4): block j = numpy Philox(key=seed) after advance(j)."""
    bg = np.random.Philox(key=seed)
    bg.advance(int(first_block))
    return bg.random_raw(4 * int(nblocks)).reshape(int(nblocks), 4)


def beam_normals(seed, first_draw, count):
    """The 8 N(0,1) numbers of each Gaussian-beam draw (pic_add_gaussian_beam), shape (count, 8): draw i takes
    blocks 2i and 2i+1 and turns each into two Box-Muller pairs exactly as philox_normal does (53-bit uniforms,
    u1 = 1 - u): (r0 cos th0, r0 sin th0, r1 cos th1, r1 sin th1).  Columns 0-5 are x, y, z, ux, uy, uz."""
    raw = philox_blocks(seed, 2 * int(first_draw), 2 * int(count)).reshape(int(count), 2, 4)
    u = (raw >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)
    r = np.sqrt(-2.0 * np.log(1.0 - u[:, :, 0:2]))
    th = 2.0 * np.pi * u[:, :, 2:4]
    g = np.stack((r[:, :, 0] * np.cos(th[:, :, 0]), r[:, :, 0] * np.sin(th[:, :, 0]),
                  r[:, :, 1] * np.cos(th[:, :, 1]), r[:, :, 1] * np.sin(th[:, :, 1])), axis=2)
    return np.ascontiguousarray(g.reshape(int(count), 8))


def uniform_plasma_3d(n=256, ppc=(2, 2, 2), lx=40.0e-6, density=1.0e25, u_th=0.01,
                      seed=20240923, box_lo=None, box_hi=None, perturbation=0.0, n_cell=None):
    """Config 2 / 3 / 5: Examples/Physics_applications/uniform_plasma/inputs_base_3d scaled up:
    electrons only, thermal u/c ~ N(0, u_th^2) per component from a counter-based generator so
    that every decomposition sees the same particles.  `perturbation` adds the (non-chaotic)
    Langmuir mode of config 1 on top."""
    n_cell = (n, n, n) if n_cell is None else tuple(n_cell)
    lxs = tuple(float(v) for v in lx) if np.ndim(lx) else (float(lx),) * 3   # per-axis box length
    prob_lo, prob_hi = tuple(-0.5 * v for v in lxs), tuple(0.5 * v for v in lxs)
    lx = lxs[0]
    lo = np.zeros(3, dtype=int) if box_lo is None else np.asarray(box_lo)
    hi = np.asarray(n_cell) - 1 if box_hi is None else np.asarray(box_hi)
    x, y, z = lattice_positions(n_cell, prob_lo, prob_hi, ppc, lo, hi)
    nppc = ppc[0] * ppc[1] * ppc[2]
    dxs = [lxs[d] / n_cell[d] for d in range(3)]
    w = np.full_like(x, density * dxs[0] * dxs[1] * dxs[2] / nppc)
    # global particle id = global cell number * nppc + in-cell index  (decomposition independent)
    idx = [np.arange(lo[d], hi[d] + 1) for d in range(3)]
    K, J, I = np.meshgrid(idx[2], idx[1], idx[0], indexing="ij")
    gcell = (I + n_cell[0] * (J + n_cell[1] * K)).ravel().astype(np.int64)
    u = np.empty((gcell.size * nppc, 3))
    if box_lo is None and box_hi is None:
        u[:] = philox_normal(seed, 0, gcell.size * nppc)
    else:
        # rows of consecutive cells along i are consecutive ids
        ni = hi[0] - lo[0] + 1
        rows = gcell.reshape(-1, ni)[:, 0]
        for r, first_cell in enumerate(rows):
            u[r * ni * nppc:(r + 1) * ni * nppc] = philox_normal(seed, int(first_cell) * nppc, ni * nppc)
    u *= u_th * C
    if perturbation:
        k = 2.0 * 2.0 * np.pi / lx
        wp = np.sqrt(density * Q_E ** 2 / (EP0 * M_E))
        a = perturbation * k / (wp / C) * C
        u[:, 0] += a * np.sin(k * x) * np.cos(k * y) * np.cos(k * z)
        u[:, 1] += a * np.cos(k * x) * np.sin(k * y) * np.cos(k * z)
        u[:, 2] += a * np.cos(k * x) * np.cos(k * y) * np.sin(k * z)
    species = [dict(name="electrons", q=-Q_E, m=M_E, x=x, y=y, z=z, w=w,
                    ux=np.ascontiguousarray(u[:, 0]), uy=np.ascontiguousarray(u[:, 1]),
                    uz=np.ascontiguousarray(u[:, 2]))]
    return dict(n_cell=n_cell, prob_lo=prob_lo, prob_hi=prob_hi, species=species)


def _random_per_cell(seed, n_cell, prob_lo, prob_hi, ppc):
    """NRandomPerCell: ppc positions uniform inside every cell (cell i fastest, then j, k; the particles of a cell
    consecutive).  Particle p takes Philox4x64-10 block p of `seed` (philox_blocks), words 0-2 as 53-bit uniforms."""
    n_cell = np.asarray(n_cell)
    dx = (np.asarray(prob_hi, dtype=np.float64) - np.asarray(prob_lo, dtype=np.float64)) / n_cell
    ncell = int(np.prod(n_cell))
    K, J, I = np.meshgrid(*[np.arange(n_cell[d]) for d in (2, 1, 0)], indexing="ij")
    cells = [np.repeat(a.ravel(), ppc) for a in (I, J, K)]
    u = (philox_blocks(seed, 0, ncell * ppc)[:, :3] >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)
    return [np.ascontiguousarray(prob_lo[d] + (cells[d] + u[:, d]) * dx[d]) for d in range(3)]


def _collision_species(name, q, m, seed, n_cell, prob_lo, prob_hi, ppc, density, u_th, u_m=(0.0, 0.0, 0.0)):
    """momentum_distribution_type = "gaussian": u = (u_m + u_th N(0, 1)) c per component (philox_normal of seed + 1)"""
    x, y, z = _random_per_cell(seed, n_cell, prob_lo, prob_hi, ppc)
    dV = np.prod((np.asarray(prob_hi) - np.asarray(prob_lo)) / np.asarray(n_cell))
    g = philox_normal(seed + 1, 0, len(x))
    u = [np.ascontiguousarray((u_m[d] + u_th[d] * g[:, d]) * C) for d in range(3)]
    return dict(name=name, q=q, m=m, x=x, y=y, z=z, w=np.full(len(x), density * dV / ppc), ux=u[0], uy=u[1], uz=u[2])


def collision_xyz_3d(n=8, ppc=200, seed=2034958209):
    """Examples/Tests/collision/inputs_test_3d_collision_xyz: electrons and ions (mass 5 m_e, the deck's value) at
    1e21 m^-3, 200 random particles per cell each, electrons drifting along x; algo.maxwell_solver = none, dt =
    1.224744871e-07, 150 steps; electron-ion, electron-electron and ion-ion collisions with CoulombLog 15.9 every 10
    steps.  n: cells per axis (the deck's 8; other values keep its cell size); seed: warpx.random_seed."""
    lx = 4.154046151855669e2 * n / 8
    n_cell, prob_lo, prob_hi = (n,) * 3, (0.0,) * 3, (lx,) * 3
    ue, ui = 0.044237441120300, 0.006256118919701
    species = [_collision_species("electron", -Q_E, M_E, seed, n_cell, prob_lo, prob_hi, ppc, 1.0e21, (ue,) * 3, (ue, 0, 0)),
               _collision_species("ion", Q_E, 4.554691780000000e-30, seed + 2, n_cell, prob_lo, prob_hi, ppc, 1.0e21,
                                  (ui,) * 3)]
    collisions = [dict(species=(0, 1), coulomb_log=15.9, ndt=10, seed=seed),
                  dict(species=(0, 0), coulomb_log=15.9, ndt=10, seed=seed),
                  dict(species=(1, 1), coulomb_log=15.9, ndt=10, seed=seed)]
    # analysis_collision_3d.py: <ux_e - ux_i>/c ~ a exp(b step) at steps 0, 10, ..., 150, mean error < 0.001
    return dict(n_cell=n_cell, prob_lo=prob_lo, prob_hi=prob_hi, dt=1.224744871e-07, max_step=150, species=species,
                collisions=collisions, analysis=dict(a=0.041817463099883, b=-0.083851393560288, tolerance=0.001))


def collision_iso_3d(n=8, ppc=1000, seed=1):
    """Examples/Tests/collision/inputs_test_3d_collision_iso: electrons at 1.116e28 m^-3, 1000 random particles per
    cell, anisotropic temperature (u_th 0.0033163 c along x, 0.0031592 c across); algo.maxwell_solver = none, dt =
    1.4e-17, 100 steps (stop_time 1.4e-15); electron-electron collisions with CoulombLog 2 every step."""
    lx = 4.0e-6 * n / 8
    n_cell, prob_lo, prob_hi = (n,) * 3, (0.0,) * 3, (lx,) * 3
    u_th = (0.0033163331635535603, 0.00315918518549115, 0.00315918518549115)
    species = [_collision_species("electron", -Q_E, M_E, seed, n_cell, prob_lo, prob_hi, ppc, 1.116e28, u_th)]
    return dict(n_cell=n_cell, prob_lo=prob_lo, prob_hi=prob_hi, dt=1.4e-17, max_step=100, species=species,
                collisions=[dict(species=(0, 0), coulomb_log=2.0, ndt=1, seed=seed)],
                analysis=dict(T_par=5.62, T_per=5.1, ne=1.116e28, coulomb_log=2.0, tolerance=0.05))


def laser_acceleration_3d(n_cell=(32, 32, 256), max_step=100, solver=0, pusher=0):
    """Config 4's deterministic ancestor: Examples/Physics_applications/laser_acceleration/
    inputs_base_3d (test_3d_laser_acceleration): Yee, Boris, order 3, bilinear filter on (WarpX
    default), z moving window at c with PEC walls, Gaussian laser antenna, electrons at rest on the
    NUniformPerCell lattice with continuous injection.  Returns the deck as plain data; the
    particles are created by the injector (oracle / engine), not here."""
    inf = float("inf")
    return dict(
        n_cell=tuple(n_cell), prob_lo=(-30.e-6, -30.e-6, -56.e-6), prob_hi=(30.e-6, 30.e-6, 12.e-6),
        field_lo=("periodic", "periodic", "pec"), field_hi=("periodic", "periodic", "pec"),
        nox=3, use_filter=True, cfl=1.0, moving_window_dir=2, moving_window_v=1.0, max_step=max_step,
        solver=solver, pusher=pusher,      # 0 = Yee / Boris (the deck); 1 = CKC / Vay (BASELINE.json config 4)
        species=[dict(name="electrons", q=-Q_E, m=M_E, ppc=(1, 1, 1),
                      bound_lo=(-20.e-6, -20.e-6, 0.0), bound_hi=(20.e-6, 20.e-6, inf),
                      density=2.e23, do_continuous_injection=True)],
        lasers=[dict(name="laser1", position=(0., 0., 9.e-6), direction=(0., 0., 1.),
                     polarization=(0., 1., 0.), e_max=16.e12, waist=5.e-6, duration=15.e-15,
                     t_peak=30.e-15, focal_distance=100.e-6, wavelength=0.8e-6)],
        region_of_interest=(12.0e-6, 13.0e-6))


def boosted_domain(prob_lo, prob_hi, gamma_boost, moving_window_v=None, direction=2):
    """ConvertLabParamsToBoost (Source/Utils/WarpXUtil.cpp:180-262): geometry.prob_lo / prob_hi along the
    boost direction are lab-frame values in the deck; WarpX multiplies them by
    1 / (gamma (1 - beta beta_window)), beta_window = moving_window_v / c when the window moves along the
    boost, else beta."""
    from . import abi
    beta = abi.beta_of_gamma(gamma_boost)
    beta_window = beta if moving_window_v is None else moving_window_v
    convert_factor = 1.0 / (gamma_boost * (1 - beta * beta_window))
    lo, hi = list(prob_lo), list(prob_hi)
    lo[direction] *= convert_factor
    hi[direction] *= convert_factor
    return tuple(lo), tuple(hi)


def max_step_boost_accelerator(zmax_plasma, zmin_domain_boost, gamma_boost, moving_window_v, dt):
    """WarpX::computeMaxStepBoostAccelerator (Source/Initialization/WarpXInitData.cpp:820-859):
    warpx.zmax_plasma_to_compute_max_step -> the step at which the lower end of the (boosted, moving)
    domain passes the upper end of the plasma."""
    from . import abi
    beta = abi.beta_of_gamma(gamma_boost)
    len_plasma_boost = zmax_plasma / gamma_boost
    v_plasma_boost = -beta * C
    interaction_time_boost = (len_plasma_boost - zmin_domain_boost) / (moving_window_v * C - v_plasma_boost)
    return int(interaction_time_boost / dt)


def laser_acceleration_boosted_3d(n_cell=(16, 16, 128), max_step=60, gamma_boost=10.0, density=1.e23,
                                  use_fdtd_nci_corr=False, beam=False):
    """BASELINE.json config 4 in the small: Examples/Tests/boosted_diags/
    inputs_test_3d_laser_acceleration_btd (CKC, Vay, order 3, bilinear filter, z moving window at c, PEC in
    z, Gaussian antenna, electrons + ions at rest in the lab with continuous injection, gamma_boost = 10)
    without the back-transformed diagnostics, on a grid fine enough for omega_p dt < 1 (the regression deck
    itself runs at omega_p dt = 4.4).  prob_lo / prob_hi below are the boosted-frame values; everything under
    species / lasers / beams is lab-frame, as in the deck.  beam=True adds the deck's witness beam under
    "beams" (keyword arguments of abi.make_gaussian_beam plus name, q, m): its draws come from the
    counter-based generator of beam_normals, not AMReX's, so the deck's own checksums stay out of reach."""
    M_P = 1.67262192369e-27
    lo, hi = boosted_domain((-128.e-6, -128.e-6, -40.e-6), (128.e-6, 128.e-6, 0.0), gamma_boost, 1.0)
    bounds = dict(bound_lo=(-120.e-6, -120.e-6, 0.0), bound_hi=(120.e-6, 120.e-6, .003))
    extra = {}
    if beam:
        extra["beams"] = [dict(name="beam", q=-Q_E, m=M_E, x_m=(0.0, 0.0, -20.e-6), rms=(1.e-6, 1.e-6, .2e-6),
                               npart=1000, q_tot=-1.e-14, u_m=(0.0, 0.0, 200000.), u_th=(.2, .2, 20.))]
    return dict(**extra,
        n_cell=tuple(n_cell), prob_lo=lo, prob_hi=hi, gamma_boost=gamma_boost,
        field_lo=("periodic", "periodic", "pec"), field_hi=("periodic", "periodic", "pec"),
        nox=3, use_filter=True, cfl=1.0, moving_window_dir=2, moving_window_v=1.0, max_step=max_step,
        solver=1, pusher=1, use_fdtd_nci_corr=bool(use_fdtd_nci_corr),      # particles.use_fdtd_nci_corr = 1 in the deck
        species=[dict(name="electrons", q=-Q_E, m=M_E, ppc=(1, 1, 1), density=density,
                      do_continuous_injection=True, **bounds),
                 dict(name="ions", q=Q_E, m=M_P, ppc=(1, 1, 1), density=density,
                      do_continuous_injection=True, **bounds)],
        lasers=[dict(name="laser1", position=(0., 0., -0.1e-6), direction=(0., 0., 1.),
                     polarization=(0., 1., 0.), e_max=2.e12, waist=45.e-6, duration=20.e-15,
                     t_peak=40.e-15, focal_distance=0.5e-3, wavelength=0.81e-6)])


def staggered_coordinates(fab, prob_lo, dx):
    """x, y, z (numpy, broadcastable to the fab's [k, j, i] array) of every ALLOCATED point of a
    component, as WarpX::ComputeExternalFieldOnGridUsingParser evaluates them
    (Source/Initialization/WarpXInitData.cpp:1140-1147): index * dx + prob_lo + (1 - nodal) * dx / 2."""
    out = []
    for d in range(3):
        idx = np.arange(fab.lo[d], fab.hi[d] + 1, dtype=np.float64)
        fac = (1.0 - fab.stag[d]) * dx[d] * 0.5
        c = idx * dx[d] + prob_lo[d] + fac
        shape = [1, 1, 1]
        shape[2 - d] = len(c)
        out.append(c.reshape(shape))
    return out


def pec_field_3d():
    """Examples/Tests/pec/inputs_test_3d_pec_field: a wave packet between two PEC walls (no particles),
    125 steps at cfl 0.9; initial Ey / Bx from warpx.E/B_ext_grid_init_style = parse_*_ext_grid_function."""
    z1, z2, wavelength = -2.e-6, 2.e-6, 1.e-6

    def ey(x, y, z):
        return ((1.e5 * np.sin(2 * np.pi * (z) / wavelength)) * (z < z2) * (z > z1)) + 0.0 * (x + y)

    def bx(x, y, z):
        return (((-1.e5 * np.sin(2 * np.pi * (z) / wavelength)) / C)) * (z < z2) * (z > z1) + 0.0 * (x + y)

    return dict(n_cell=(32, 32, 256), prob_lo=(-8.e-6, -8.e-6, -4.e-6), prob_hi=(8.e-6, 8.e-6, 4.e-6),
                field_lo=("periodic", "periodic", "pec"), field_hi=("periodic", "periodic", "pec"),
                nox=1, use_filter=True, cfl=0.9, max_step=125, init_fields={1: ey, 3: bx}, species=[])


def pec_particle_3d():
    """Examples/Tests/pec/inputs_test_3d_pec_particle: two heavy particles 2 nm from a PEC wall in x
    (order 3, Vay pusher, bilinear filter, cfl 0.9, 20 steps)."""
    M_P = 1.67262192369e-27          # ablastr/constant.H:54
    pos = (31.998e-6, 0.0, 0.0)
    one = lambda v: np.array([v], dtype=np.float64)   # noqa: E731
    species = [
        dict(name="electron", q=-Q_E, m=M_P, x=one(pos[0]), y=one(pos[1]), z=one(pos[2]), w=one(1.0),
             ux=one(0.0), uy=one(0.0), uz=one(0.0)),
        dict(name="proton", q=Q_E, m=M_P, x=one(pos[0]), y=one(pos[1]), z=one(pos[2]), w=one(1.0),
             ux=one(0.0), uy=one(-2.0 * C), uz=one(0.0)),
    ]
    return dict(n_cell=(128, 64, 64), prob_lo=(-32.e-6,) * 3, prob_hi=(32.e-6,) * 3,
                field_lo=("pec", "periodic", "periodic"), field_hi=("pec", "periodic", "periodic"),
                nox=3, use_filter=True, cfl=0.9, max_step=20, pusher=1, species=species, mass=M_P)


def laser_injection_3d():
    """Examples/Tests/laser_injection/inputs_test_3d_laser_injection: a Gaussian antenna radiating into
    vacuum between PEC walls, moving window at c, order 1, no filter, 20 steps (no plasma)."""
    return dict(
        n_cell=(32, 32, 240), prob_lo=(-20.e-6, -20.e-6, -12.e-6), prob_hi=(20.e-6, 20.e-6, 12.e-6),
        field_lo=("periodic", "periodic", "pec"), field_hi=("periodic", "periodic", "pec"),
        nox=1, use_filter=False, cfl=1.0, moving_window_dir=2, moving_window_v=1.0, max_step=20,
        solver=0, pusher=0, species=[],
        lasers=[dict(name="laser1", position=(0., 0., 9.e-6), direction=(0., 0., 1.), polarization=(0., 1., 0.),
                     e_max=4.e12, waist=5.e-6, duration=15.e-15, t_peak=30.e-15, focal_distance=100.e-6,
                     wavelength=0.8e-6)])


def particle_boundaries_3d():
    """Examples/Tests/boundaries/inputs_test_3d_particle_boundaries: neutral particles flying into
    reflecting (x), absorbing (y) and periodic (z) faces of a 16^3 box, 8 steps, order 1."""
    c = C
    arr = lambda *v: np.array(v, dtype=np.float64)   # noqa: E731
    z2, z3 = arr(0., 0.), arr(0., 0., 0.)
    species = [
        dict(name="reflecting_particles", q=0.0, m=M_E, x=arr(-0.9, 0.91), y=z2, z=z2, w=arr(1., 1.),
             ux=arr(-0.9, 0.91) * c, uy=z2, uz=z2),
        dict(name="absorbing_particles", q=0.0, m=M_E, x=z3, y=arr(-0.92, 0.93, 0.), z=z3, w=arr(1., 1., 1.),
             ux=z3, uy=arr(-0.92, 0.93, 0.) * c, uz=z3),
        dict(name="periodic_particles", q=0.0, m=M_E, x=z2, y=z2, z=arr(-0.94, 0.95), w=arr(1., 1.),
             ux=z2, uy=z2, uz=arr(-0.94, 0.95) * c),
    ]
    return dict(n_cell=(16, 16, 16), prob_lo=(-1.0,) * 3, prob_hi=(1.0,) * 3,
                field_lo=("pec", "pec", "periodic"), field_hi=("pec", "pec", "periodic"),
                particle_lo=("reflecting", "absorbing", "periodic"), particle_hi=("reflecting", "absorbing", "periodic"),
                nox=1, use_filter=True, cfl=1.0, max_step=8, species=species)


# ---- the reference's 3D nuclear fusion decks (Examples/Tests/nuclear_fusion/inputs_test_3d_*) ----------------------
M_U = 1.66053906660e-27
_FUSION_MASS = {"hydrogen1": 1.00782503223 * M_U, "hydrogen2": 2.01410177812 * M_U, "hydrogen3": 3.0160492779 * M_U,
                "helium3": 3.0160293201 * M_U, "helium4": 4.00260325413 * M_U, "boron11": 11.00930536 * M_U,
                "neutron": 1.0013784193052508 * 1.67262192369e-27}
_FUSION_CHARGE = {"hydrogen1": 1, "hydrogen2": 1, "hydrogen3": 1, "helium3": 2, "helium4": 2, "boron11": 5, "neutron": 0}


def _fusion_species(name, species_type, seed, geom, ppc, density, u):
    """NRandomPerCell species of a fusion deck, not pushed and not depositing: density(x, y, z) [m^-3] and u(x, y, z) ->
    (ux, uy, uz) in units of c, evaluated at the particles' positions; w = density dV / ppc."""
    x, y, z = _random_per_cell(seed, geom[0], geom[1], geom[2], ppc)
    dV = np.prod((np.asarray(geom[2]) - np.asarray(geom[1])) / np.asarray(geom[0]))
    ux, uy, uz = (np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), x.shape) * C) for v in u(x, y, z))
    w = np.ascontiguousarray(np.broadcast_to(np.asarray(density(x, y, z), dtype=np.float64), x.shape) * dV / ppc)
    return dict(name=name, species_type=species_type, q=_FUSION_CHARGE[species_type] * Q_E, m=_FUSION_MASS[species_type],
                x=x, y=y, z=z, w=w, ux=ux, uy=uy, uz=uz, do_not_push=True, do_not_deposit=True)


def _merge(name, a, b):
    """<species>.injection_sources: the particles of two sources in one species"""
    out = dict(a, name=name)
    for k in ("x", "y", "z", "w", "ux", "uy", "uz"):
        out[k] = np.concatenate([a[k], b[k]])
    return out


def _product(name, species_type, capacity):
    return dict(name=name, species_type=species_type, capacity=int(capacity), do_not_push=True, do_not_deposit=True)


def _thermal(seed, theta):
    """maxwell_boltzmann with theta (InjectorMomentumBoltzmann, no drift): per component N(0, sqrt(theta)) in units of c"""
    def u(x, y, z):
        g = philox_normal(seed, 0, len(x))
        return tuple(np.sqrt(theta) * g[:, d] for d in range(3))
    return u


def _two_product_deck(reaction, scale, seed):
    """inputs_test_3d_deuterium_tritium_fusion ("dt") and inputs_test_3d_deuterium_deuterium_fusion ("dd")"""
    geom = ((8, 8, 16), (0.0, 0.0, 0.0), (8.0, 8.0, 16.0))
    ncell = 8 * 8 * 16
    keV = 1.e3 * Q_E
    E_step = 22. * keV
    m_d, m_t = _FUSION_MASS["hydrogen2"], _FUSION_MASS["hydrogen3"]
    n1 = max(int(10000 * scale), 2)
    if reaction == "dt":
        m_r = m_d * m_t / (m_d + m_t)
        r2, m2 = "hydrogen3", m_t
        uz1 = lambda x, y, z: (0.0, 0.0, np.sqrt(2 * m_r * E_step * np.floor(z) ** 2) / (m_d * C))
        uz2 = lambda x, y, z: (0.0, 0.0, -np.sqrt(2 * m_r * E_step * np.floor(z) ** 2) / (m_t * C))
        prods = ("helium4", "neutron")
    else:
        r2, m2 = "hydrogen2", m_d
        uz1 = lambda x, y, z: (0.0, 0.0, np.sqrt(m_d * E_step * np.floor(z) ** 2) / (m_d * C))
        uz2 = lambda x, y, z: (0.0, 0.0, -np.sqrt(m_d * E_step * np.floor(z) ** 2) / (m_d * C))
        prods = ("helium3", "neutron")
    one = lambda x, y, z: 1.0
    species = [_fusion_species("reactant1_1", "hydrogen2", seed, geom, n1, one, uz1),
               _fusion_species("reactant2_1", r2, seed + 2, geom, n1, one, uz2),
               _product("product1_1", prods[0], 2 * n1 * ncell), _product("product2_1", prods[1], 2 * n1 * ncell)]
    fusions = [dict(species=(0, 1), products=(2, 3), multiplier=1e50, threshold=0.02, target=0.002)]
    sets = [dict(reactants=(0, 1), products=(2, 3), pairs_per_cell=n1, densities=(1.0, 1.0), target=0.002)]
    if reaction == "dt":
        bg, beam = 1.e26, 1.e20
        nh, nl, n2 = max(int(100 * scale), 1), max(int(900 * scale), 1), max(int(100 * scale), 1)
        high = _fusion_species("d2", "hydrogen2", seed + 4, geom, nh, lambda x, y, z: 10. * bg, lambda x, y, z: (0., 0., 0.))
        low = _fusion_species("d2", "hydrogen2", seed + 6, geom, nl, lambda x, y, z: 10. / 9. * beam,
                              lambda x, y, z: (0.0, 0.0, np.sqrt(2 * m_d * E_step * np.floor(z) ** 2) / (m_d * C)))
        species += [_merge("reactant1_2", high, low),
                    _fusion_species("reactant2_2", "hydrogen3", seed + 8, geom, n2, lambda x, y, z: bg,
                                    lambda x, y, z: (0., 0., 0.)),
                    _product("product1_2", "helium4", 2 * (nh + nl) * ncell),
                    _product("product2_2", "neutron", 2 * (nh + nl) * ncell)]
        fusions.append(dict(species=(4, 5), products=(6, 7), multiplier=1e15, threshold=0.02, target=0.02))
        # each injection source weighs its own particles: the beam is 900 particles per cell at 10/9 beam_dens
        sets.append(dict(reactants=(4, 5), products=(6, 7), pairs_per_cell=nl, densities=(10. / 9. * beam, bg),
                         target=0.02, beam_only=True))
    return dict(n_cell=geom[0], prob_lo=geom[1], prob_hi=geom[2], nox=1, cfl=1.0, max_step=1, seed=seed,
                species=species, fusions=fusions,
                analysis=dict(reaction=reaction, E_step=E_step, sets=sets, tol=1e-12, energy_tol=1e-8,
                              isotropy=0.03, xy_isotropy=0.05, rho_tol=2e-11))


def fusion_dt_3d(scale=1.0, seed=4):
    """Examples/Tests/nuclear_fusion/inputs_test_3d_deuterium_tritium_fusion: 8 x 8 x 16 cells of 1 m, order 1, Yee with
    cfl 1, one step; every species is not pushed and does not deposit.  Set 1: 10 000 D + 10 000 T per cell at momenta
    constant per z slice (E* = 22 keV floor(z)^2), fusion_multiplier 1e50.  Set 2: D of two injection sources (100 at
    rest at 1e27 m^-3 and 900 of a beam at 1.1e20 m^-3 per cell) on 100 T at rest at 1e26 m^-3, multiplier 1e15, target
    value 0.02.  scale multiplies the particles per cell (1 is the deck)."""
    return _two_product_deck("dt", scale, seed)


def fusion_dd_3d(scale=1.0, seed=5):
    """Examples/Tests/nuclear_fusion/inputs_test_3d_deuterium_deuterium_fusion: set 1 of the D-T deck with two deuterium
    species in head-on beams (E* = 22 keV floor(z)^2) fusing into He3 + n."""
    return _two_product_deck("dd", scale, seed)


def fusion_dd_intraspecies_3d(scale=1.0, seed=1034958209):
    """Examples/Tests/nuclear_fusion/inputs_test_3d_deuterium_deuterium_fusion_intraspecies: 8^3 cells over
    [-1 mm, 1 mm]^3, Yee with cfl 1, 10 steps; 10 000 deuterons per cell at 1e26 m^-3 with a gaussian thermal
    spread of 0.003265007901313691 c per component, D + D -> He3 + n within the species with multiplier 1e10.  The
    analysis reads <sigma v> from the neutrons' ParticleNumber history: 2.603e-18 cm^3/s within 2 %."""
    geom = ((8, 8, 8), (-1e-3,) * 3, (1e-3,) * 3)
    n = max(int(10000 * scale), 2)
    u_th = 0.003265007901313691
    def u(x, y, z):
        g = philox_normal(seed + 1, 0, len(x))
        return tuple(u_th * g[:, d] for d in range(3))
    d = _fusion_species("deuterium", "hydrogen2", seed, geom, n, lambda x, y, z: 1e26, u)
    species = [d, _product("helium3", "helium3", 2 * len(d["x"])), _product("neutron", "neutron", 2 * len(d["x"]))]
    # The deck uses shape order 3; no species is pushed or deposits, so the order does not enter the result, and 8 cells
    # per axis are too few for the guard cells of order 3 in this engine's periodic exchange: order 1.
    return dict(n_cell=geom[0], prob_lo=geom[1], prob_hi=geom[2], nox=1, cfl=1.0, max_step=10, seed=seed,
                species=species, fusions=[dict(species=(0, 0), products=(1, 2), multiplier=1e10, threshold=0.02,
                                               target=0.002)],
                analysis=dict(density=1e26, volume=(2e-3) ** 3, sigma_v=2.603e-18, tolerance=0.02))


def proton_boron_3d(scale=1.0, seed=6):
    """Examples/Tests/nuclear_fusion/inputs_test_3d_proton_boron_fusion: 8 x 8 x 16 cells of 1 m, order 1, Yee with cfl
    1, one step, five p + B11 -> 3 alpha sets, every species not pushed and not depositing:
      1. 10 000 p + 10 000 B per cell in head-on beams (E* = 22 keV floor(z)^2), multiplier 1e50;
      2. 1000 p per cell (a tenth, where y - floor(y) < 0.1, at rest at 1e27 m^-3, the rest a beam at 1.1e20 m^-3 with
         E = 22 keV floor(z)^2) on 100 B at rest at 1e26 m^-3, multiplier 1e15, target value 0.02;
      3. 600 p at 1e28 and 1000 B at 5e28 m^-3, Maxwellian at 44 keV, multiplier 1e15;
      4. 100 p at 1e35 m^-3 with 550 keV on 100 B at rest at 1 m^-3, multiplier 1e21: every boron is used up;
      5. set 4 with fusion_probability_threshold 1e123: borons remain.
    scale multiplies the particles per cell (1 is the deck: about 24 M particles)."""
    geom = ((8, 8, 16), (0.0, 0.0, 0.0), (8.0, 8.0, 16.0))
    ncell = 8 * 8 * 16
    keV = 1.e3 * Q_E
    E_step = 22. * keV
    m_h, m_b = _FUSION_MASS["hydrogen1"], _FUSION_MASS["boron11"]
    m_r = m_h * m_b / (m_h + m_b)
    s = lambda n: max(int(n * scale), 1)
    at_rest = lambda x, y, z: (0., 0., 0.)
    bg, beam, T = 1.e26, 1.e20, 44. * keV
    E4 = 550 * keV
    p4 = lambda x, y, z: (0., 0., np.sqrt(2 * m_h * E4) / (m_h * C))
    specs = [
        (("proton1", "hydrogen1", s(10000), lambda x, y, z: 1.0,
          lambda x, y, z: (0., 0., np.sqrt(2 * m_r * E_step * np.floor(z) ** 2) / (m_h * C))),
         ("boron1", "boron11", s(10000), lambda x, y, z: 1.0,
          lambda x, y, z: (0., 0., -np.sqrt(2 * m_r * E_step * np.floor(z) ** 2) / (m_b * C))), 1e50, 0.02, 0.002),
        (("proton2", "hydrogen1", s(1000), lambda x, y, z: np.where(y - np.floor(y) < 0.1, 10. * bg, 10. / 9. * beam),
          lambda x, y, z: (0., 0., np.where(y - np.floor(y) < 0.1, 0.,
                                            np.sqrt(2 * m_h * E_step * np.floor(z) ** 2) / (m_h * C)))),
         ("boron2", "boron11", s(100), lambda x, y, z: bg, at_rest), 1e15, 0.02, 0.02),
        (("proton3", "hydrogen1", s(600), lambda x, y, z: 1e28, _thermal(seed + 101, T / (m_h * C * C))),
         ("boron3", "boron11", s(1000), lambda x, y, z: 5e28, _thermal(seed + 103, T / (m_b * C * C))), 1e15, 0.02, 0.002),
        (("proton4", "hydrogen1", s(100), lambda x, y, z: 1e35, p4), ("boron4", "boron11", s(100), lambda x, y, z: 1.0,
                                                                      at_rest), 1e21, 0.02, 0.002),
        (("proton5", "hydrogen1", s(100), lambda x, y, z: 1e35, p4), ("boron5", "boron11", s(100), lambda x, y, z: 1.0,
                                                                      at_rest), 1e21, 1e123, 0.002),
    ]
    species, fusions, sets = [], [], []
    for k, (p, b, mult, thr, target) in enumerate(specs):
        i = len(species)
        species.append(_fusion_species(p[0], p[1], seed + 10 * k, geom, p[2], p[3], p[4]))
        species.append(_fusion_species(b[0], b[1], seed + 10 * k + 2, geom, b[2], b[3], b[4]))
        species.append(_product("alpha%d" % (k + 1), "helium4", 6 * max(p[2], b[2]) * ncell))
        fusions.append(dict(species=(i, i + 1), products=(i + 2,), multiplier=mult, threshold=thr, target=target))
        sets.append(dict(reactants=(i, i + 1), products=(i + 2,), pairs_per_cell=max(p[2], b[2]), target=target))
    sets[0]["densities"] = (1.0, 1.0)
    sets[1].update(densities=(beam, bg), pairs_per_cell=int(round(0.9 * s(1000))), beam_only=True)
    return dict(n_cell=geom[0], prob_lo=geom[1], prob_hi=geom[2], nox=1, cfl=1.0, max_step=1, seed=seed,
                species=species, fusions=fusions,
                analysis=dict(reaction="pb", E_step=E_step, sets=sets, tol=1e-12, energy_tol=1e-8, isotropy=0.03,
                              thermal_isotropy=0.1, xy_isotropy=0.05, thermal=dict(T_keV=44.0, n_p=1e28, n_b=5e28,
                                                                                    tolerance=0.2), rho_tol=2e-11))


# ---- the reference's 3D flux-injection deck (Examples/Tests/flux_injection/inputs_test_3d_flux_injection) ------------
M_P = 1.67262192369e-27


def flux_injection_3d(n=16, ppc=100.0, max_step=2, seed=7):
    """Examples/Tests/flux_injection/inputs_test_3d_flux_injection: n^3 cells over [-4, 4]^3 m, periodic,
    algo.maxwell_solver = none with warpx.const_dt = 7e-9, shape order 3, max_step steps; four empty species fed through
    planes (injection_style = NFluxPerCell, num_particles_per_cell = ppc, flux 1 m^-2 s^-1, gaussianflux momenta with
    u_th = 0.1 on every axis): electrons through y = -4 towards +y with uy_m = 0.07, protons through x = +4 towards -x
    with ux_m = 0.05, "negative" electrons through z = -4 towards +z with uz_m = -0.07, "negative" protons through
    z = +4 towards -z with uz_m = -0.05.  Each species gets the capacity of max_step full injections.  The analysis
    (analysis_flux_injection_3d.py) histograms the momenta of each species against N_tot = flux 64 m^2 t_max times a
    Gaussian (transverse, within 0.07 of the peak) or a Gaussian-flux distribution (normal, within 0.05)."""
    th = (0.1, 0.1, 0.1)
    cap = int(max_step * n * n * (int(ppc) + 1))
    sources = [("electron", -Q_E, M_E, "y", -4.0, +1, (0.0, 0.07, 0.0)),
               ("proton", Q_E, M_P, "x", 4.0, -1, (0.05, 0.0, 0.0)),
               ("electron_negative", -Q_E, M_E, "z", -4.0, +1, (0.0, 0.0, -0.07)),
               ("proton_negative", Q_E, M_P, "z", 4.0, -1, (0.0, 0.0, -0.05))]
    species = [dict(name=name, q=q, m=m, capacity=cap,
                    flux=dict(num_particles_per_cell=ppc, surface_flux_pos=pos, flux_normal_axis=axis,
                              flux_direction=direction, flux=1.0, u_m=u_m, u_th=th, seed=seed))
               for name, q, m, axis, pos, direction, u_m in sources]
    return dict(n_cell=(n, n, n), prob_lo=(-4.0, -4.0, -4.0), prob_hi=(4.0, 4.0, 4.0), nox=3, dt=7e-9, max_step=max_step,
                species=species, analysis=dict(flux=1.0, emission_surface=8 * 8, hist_bins=50, hist_range=(-0.5, 0.5),
                                               gaussian_tol=0.07, flux_tol=0.05))
