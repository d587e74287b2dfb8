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
