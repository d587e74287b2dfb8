"""Seeded particle sets for the deposition and gather parity tests, and the numpy restatement of how the kernels
classify their particles (tests/test_particle_sets.py checks with it that every set contains what it is meant to).

Every set is a ParticleSet: arrays x y z w ux uy uz in the engine's bin order (8^3 supercells, cells x-fastest inside,
bins.cuh::bin_of_cell), the cell_start table of the sort that produced that order (the particles may have moved since),
and the geometry.  Positions are "pushed": the deposition takes x as the new position and x - v dt as the old one.
Weights are drawn log-uniformly over 1e-3 .. 1e3 times the lattice weight, so a kernel that takes the weight of
another particle or record slot gives a wrong number.  Every particle lies inside the valid box or on its upper face
(x == prob_hi: pushed, not yet wrapped), or one ulp below its lower face; its old position at most one cell away.
The tests therefore allocate J with nox + 2 guard cells and E / B with 4: every set stays inside the documented
preconditions, and a kernel error shows up as a wrong number, never as an access outside the arrays.

    steady          oracle-evolved thermal plasma, sorted as the engine sorts, then 3 more oracle steps
    poisson         Poisson(8) cell counts plus cells with 0, 1, 31, 32, 33 and 600 particles
    faces           particles exactly on cell, supercell and box faces and one ulp below them, x == prob_hi
    crowded_movers  one supercell with 240 particles changing cell diagonally (1920 queued sub-particles),
                    movers across supercell faces
    scrambled_rows  a 16-ppc supercell whose particles alternate rows after the sort (isolated rows), every other
                    supercell shifted by one supercell after the sort (leavers)
    sparse1/31/33   1, 31 or 33 particles, all in one cell of one supercell
A suffix "+offset" puts the same particles into a brick at box_lo = (64, 32, 96) of a larger domain."""
import functools

import numpy as np

from warpx_b200 import workloads

NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")
TILE = 8
SETS = ("steady", "poisson", "faces", "crowded_movers", "scrambled_rows", "sparse1", "sparse31", "sparse33")
OFFSET_BOX_LO = (64, 32, 96)
DENSITY = 1.0e25
DX_BENCH = 40.0e-6 / 256          # the benchmark's cell size
DX_EXACT = 2.0 ** -23             # a power of two: face coordinates and grid coordinates are exact


class ParticleSet:
    def __init__(self, name, n, dx, p, cell_start, dt, prob_lo=None, box_lo=(0, 0, 0)):
        self.name, self.n, self.dx, self.p, self.cell_start, self.dt = name, tuple(n), tuple(dx), p, cell_start, dt
        self.box_lo = tuple(box_lo)
        # domain: centred on the origin for box_lo = 0, else the brick sits at box_lo of a domain with prob_lo < 0
        self.prob_lo = tuple(prob_lo) if prob_lo is not None else tuple(-0.5 * n[d] * dx[d] for d in range(3))
        self.origin = tuple(self.prob_lo[d] + self.box_lo[d] * dx[d] for d in range(3))      # lower corner of the box
        self.prob_hi = tuple(self.origin[d] + n[d] * dx[d] for d in range(3))                # upper corner of the box
        self.q, self.m = -workloads.Q_E, workloads.M_E
        self.np = len(p["x"])
        self.np_binned = self.np

    @property
    def box_hi(self):
        return tuple(self.box_lo[d] + self.n[d] - 1 for d in range(3))

    @property
    def dinv(self):
        return [1.0 / v for v in self.dx]

    def arrays(self):
        return {k: self.p[k].copy() for k in NAMES}

    def corner(self, ng):
        """xyzmin and lo of arrays with ng guard cells (helpers.lower_corner)."""
        lo = [self.box_lo[d] - ng[d] for d in range(3)]
        return [self.prob_lo[d] + self.dx[d] * lo[d] for d in range(3)], lo


def host_bins(x, y, z, origin, dx, n, tile):
    """pic_bins on the host: the supercell-major bin of every particle (bins.cuh::bin_of_cell), a stable sort by bin
    and the cell_start table -- what the device counting sort produces.  origin = lower corner of the box."""
    b = bin_of(x, y, z, origin, dx, n, tile)
    order = np.argsort(b, kind="stable")
    n, tile = np.asarray(n), np.asarray(tile)
    nbins = int(np.prod((n + tile - 1) // tile) * np.prod(tile))
    cell_start = np.searchsorted(b[order], np.arange(nbins + 1)).astype(np.int32)
    return order, cell_start


def bin_of(x, y, z, origin, dx, n, tile=(TILE,) * 3):
    n, tile = np.asarray(n), np.asarray(tile)
    nt = (n + tile - 1) // tile
    cell = [np.clip(np.floor((v - origin[d]) / dx[d]).astype(np.int64), 0, n[d] - 1) for d, v in enumerate((x, y, z))]
    t = [cell[d] // tile[d] for d in range(3)]
    li = [cell[d] - t[d] * tile[d] for d in range(3)]
    tid = t[0] + nt[0] * (t[1] + nt[1] * t[2])
    return tid * int(np.prod(tile)) + li[0] + tile[0] * (li[1] + tile[1] * li[2])


def log_weights(rng, count, dx):
    w_lattice = DENSITY * dx[0] * dx[1] * dx[2] / 8
    return w_lattice * 10.0 ** rng.uniform(-3.0, 3.0, count)


def cfl_dt(dx):
    return 0.95 / (np.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)


def u_of_v(v):
    """Momentum per mass u = gamma v of the velocities v (rows of 3 components)."""
    v = np.asarray(v, dtype=np.float64)
    return v / np.sqrt(1.0 - np.sum(v * v, axis=-1, keepdims=True) / workloads.C ** 2)


def _finish(name, n, dx, pos, u, rng, dt, sort_pos=None):
    """Weights, bin order of the positions `sort_pos` (default: the positions themselves), the set."""
    origin = [-0.5 * n[d] * dx[d] for d in range(3)]
    sort_pos = pos if sort_pos is None else sort_pos
    order, cell_start = host_bins(*sort_pos, origin, dx, n, (TILE,) * 3)
    p = {k: np.ascontiguousarray(v[order]) for k, v in zip(("x", "y", "z"), pos)}
    for c, k in enumerate(("ux", "uy", "uz")):
        p[k] = np.ascontiguousarray(u[order, c])
    p["w"] = log_weights(rng, len(order), dx)
    return ParticleSet(name, n, dx, p, cell_start, dt)


def _uniform_in_cells(rng, counts, n, dx):
    """counts[k, j, i] particles at random positions inside cell (i, j, k) of a box centred on the origin."""
    cells = np.repeat(np.arange(counts.size), counts.ravel())
    i, j, k = cells % n[0], (cells // n[0]) % n[1], cells // (n[0] * n[1])
    return [-0.5 * n[d] * dx[d] + (c + rng.uniform(0.0, 1.0, cells.size)) * dx[d] for d, c in enumerate((i, j, k))]


def steady_state(n=(16, 16, 8), u_th=0.05, steps=24, after_sort=3, nox=3, dx=DX_BENCH):
    """Particles of a thermal plasma after `steps` oracle steps, sorted into the engine's bin order, then `after_sort`
    more steps.  Returns (workload, dt, particles, cell_start of the sort)."""
    from oracle import oracle
    lx = tuple(dx * v for v in n)
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=(2, 2, 2), u_th=u_th, lx=lx)
    s = wl["species"][0]
    sim = oracle.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox)
    sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.evolve(steps)
    p = sim.particles(0)
    order, cell_start = host_bins(p["x"], p["y"], p["z"], wl["prob_lo"], (dx,) * 3, n, (TILE,) * 3)
    sim2 = oracle.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox)
    sim2.add_species(s["q"], s["m"], *[p[k][order] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
    sim2.evolve(after_sort)
    return wl, sim2.dt, sim2.particles(0), cell_start


def steady(seed=1, n=(16, 16, 8)):
    dx = (DX_BENCH,) * 3
    wl, dt, p, cell_start = steady_state(n=n)
    q = {k: np.ascontiguousarray(p[k]) for k in NAMES}
    q["w"] = log_weights(np.random.default_rng(seed), len(q["x"]), dx)
    return ParticleSet("steady", n, dx, q, cell_start, dt)


# cells (i, j, k) of the poisson set with chosen counts: supercell corners empty, a run longer than a warp's span
POISSON_CHOSEN = {(8, 0, 0): 0, (7, 7, 7): 0, (0, 15, 7): 0, (5, 5, 5): 1, (9, 3, 2): 31, (10, 3, 2): 32, (11, 3, 2): 33,
                  (3, 2, 1): 600}


def poisson(seed=2):
    n, dx = (16, 16, 8), (DX_EXACT,) * 3
    rng = np.random.default_rng(seed)
    counts = rng.poisson(8, (n[2], n[1], n[0]))
    for (i, j, k), c in POISSON_CHOSEN.items():
        counts[k, j, i] = c
    pos = _uniform_in_cells(rng, counts, n, dx)
    u = rng.normal(0.0, 0.02 * workloads.C, (len(pos[0]), 3))
    return _finish("poisson", n, dx, pos, u, rng, cfl_dt(dx))


def faces(seed=3):
    """Coordinates drawn per axis from: a cell face, a supercell face, a box face (0 and n), one ulp below any of
    those, or a random interior point.  dx is a power of two, so a face coordinate is exact and so is its grid
    coordinate.  A third of the particles are at rest (old position == new position, on the face)."""
    n, dx = (16, 16, 16), (DX_EXACT,) * 3
    rng = np.random.default_rng(seed)
    count = 3000
    pos = []
    for d in range(3):
        lo = -0.5 * n[d] * dx[d]
        choices = np.array([0, 1, 3, TILE - 1, TILE, TILE + 1, n[d] - 1, n[d]])
        face = rng.choice(choices[choices <= n[d]], count)
        v = lo + face * dx[d]
        kind = rng.integers(0, 3, count)                    # 0 on the face, 1 one ulp below, 2 interior
        v = np.where(kind == 1, np.nextafter(v, -np.inf), v)
        interior = lo + rng.uniform(0.0, n[d], count) * dx[d]
        v = np.where(kind == 2, interior, v)
        pos.append(v)
    u = rng.normal(0.0, 0.05 * workloads.C, (count, 3))
    u[rng.uniform(size=count) < 1.0 / 3.0] = 0.0
    return _finish("faces", n, dx, pos, u, rng, cfl_dt(dx))


CROWDED_SUPERCELL = (1, 0, 0)


def crowded_movers(seed=4):
    """2 particles per cell at rest-ish, plus 240 particles in supercell CROWDED_SUPERCELL that changed cell along x,
    y and z this step (old position in the cell (i-1, j-1, k-1), inside the supercell: 8 queued sub-particles each),
    plus 120 particles that crossed a supercell face (their old cell is in the neighbouring supercell)."""
    n, dx = (16, 16, 8), (DX_EXACT,) * 3
    rng = np.random.default_rng(seed)
    dt = cfl_dt(dx)
    base = _uniform_in_cells(rng, np.full((n[2], n[1], n[0]), 2), n, dx)
    u_base = rng.normal(0.0, 0.001 * workloads.C, (len(base[0]), 3))
    lo = [-0.5 * n[d] * dx[d] for d in range(3)]
    # diagonal movers: new position 0.05..0.2 cell above the lower faces, moved 0.3 cell per axis this step
    m = 240
    cells = [TILE * CROWDED_SUPERCELL[d] + rng.integers(1, TILE, m) for d in range(3)]
    mov = [lo[d] + (cells[d] + rng.uniform(0.05, 0.2, m)) * dx[d] for d in range(3)]
    u_mov = u_of_v(np.stack([0.3 * dx[d] / dt * np.ones(m) for d in range(3)], axis=1))
    # supercell-face crossers: new cell = first cell of a supercell along one axis, old cell in the supercell below
    c = 120
    axis = rng.choice([d for d in range(3) if n[d] > TILE], c)
    cr = [lo[d] + rng.uniform(0.0, n[d], c) * dx[d] for d in range(3)]
    v = np.zeros((c, 3))
    for d in range(3):
        sel = axis == d
        first = TILE * rng.integers(1, n[d] // TILE, sel.sum())       # a supercell face inside the box
        cr[d][sel] = lo[d] + (first + rng.uniform(0.05, 0.2, sel.sum())) * dx[d]
        v[sel, d] = 0.3 * dx[d] / dt
    u_cr = u_of_v(v)
    pos = [np.concatenate([base[d], mov[d], cr[d]]) for d in range(3)]
    u = np.concatenate([u_base, u_mov, u_cr])
    return _finish("crowded_movers", n, dx, pos, u, rng, dt)


SCRAMBLED_SUPERCELL = (0, 0, 0)


def scrambled_rows(seed=5):
    """16 particles per cell in supercell SCRAMBLED_SUPERCELL, 3 elsewhere, sorted; then every other particle of the
    dense supercell (in bin order) moves to the neighbouring row of cells in y (inside the supercell): every particle
    there differs in row from both lane neighbours.  Every particle of the other supercells moves by one
    supercell along x (wrapped inside the box): all of them left their supercell since the sort."""
    n, dx = (16, 16, 8), (DX_EXACT,) * 3
    rng = np.random.default_rng(seed)
    counts = np.full((n[2], n[1], n[0]), 3)
    sx, sy, sz = (TILE * v for v in SCRAMBLED_SUPERCELL)
    counts[sz:sz + TILE, sy:sy + TILE, sx:sx + TILE] = 16
    pos = _uniform_in_cells(rng, counts, n, dx)
    u = rng.normal(0.0, 0.02 * workloads.C, (len(pos[0]), 3))
    lo = [-0.5 * n[d] * dx[d] for d in range(3)]
    order, cell_start = host_bins(*pos, lo, dx, n, (TILE,) * 3)
    pos = [v[order] for v in pos]
    u = u[order]
    cell = [np.floor((pos[d] - lo[d]) / dx[d]).astype(np.int64) for d in range(3)]
    dense = (cell[0] // TILE == SCRAMBLED_SUPERCELL[0]) & (cell[1] // TILE == SCRAMBLED_SUPERCELL[1]) & \
            (cell[2] // TILE == SCRAMBLED_SUPERCELL[2])
    odd = dense & (np.cumsum(dense) % 2 == 0)
    step = np.where(cell[1] % TILE == TILE - 1, -1.0, 1.0)
    pos[1] = np.where(odd, pos[1] + step * dx[1], pos[1])
    lx = n[0] * dx[0]
    shifted = pos[0] + TILE * dx[0]
    shifted = np.where(shifted >= lo[0] + lx, shifted - lx, shifted)
    pos[0] = np.where(dense, pos[0], shifted)
    p = {k: np.ascontiguousarray(v) for k, v in zip(("x", "y", "z"), pos)}
    for c, k in enumerate(("ux", "uy", "uz")):
        p[k] = np.ascontiguousarray(u[:, c])
    p["w"] = log_weights(rng, len(p["x"]), dx)
    return ParticleSet("scrambled_rows", n, dx, p, cell_start, cfl_dt(dx))


SPARSE_CELL = (9, 10, 3)


def sparse(count, seed=6):
    n, dx = (16, 16, 8), (DX_EXACT,) * 3
    rng = np.random.default_rng(seed + count)
    counts = np.zeros((n[2], n[1], n[0]), dtype=np.int64)
    counts[SPARSE_CELL[2], SPARSE_CELL[1], SPARSE_CELL[0]] = count
    pos = _uniform_in_cells(rng, counts, n, dx)
    u = rng.normal(0.0, 0.1 * workloads.C, (count, 3))
    return _finish("sparse%d" % count, n, dx, pos, u, rng, cfl_dt(dx))


def moved_to_offset_box(s, box_lo=OFFSET_BOX_LO):
    """The same particles in the brick at box_lo of a domain whose lower corner is negative (twice the brick's
    position away from the origin): positions translated, bins unchanged (they are relative to box_lo)."""
    prob_lo = tuple(-2.0 * box_lo[d] * s.dx[d] for d in range(3))
    p = s.arrays()
    for d, k in enumerate(("x", "y", "z")):
        p[k] = p[k] + (prob_lo[d] + box_lo[d] * s.dx[d] - s.origin[d])
    return ParticleSet(s.name + "+offset", s.n, s.dx, p, s.cell_start, s.dt, prob_lo=prob_lo, box_lo=box_lo)


@functools.lru_cache(maxsize=None)
def get(name):
    """The set `name` of SETS, with an optional "+offset" suffix (built once per process; use .arrays() for copies)."""
    if name.endswith("+offset"):
        return moved_to_offset_box(get(name[:-len("+offset")]))
    if name.startswith("sparse"):
        return sparse(int(name[len("sparse"):]))
    return {"steady": steady, "poisson": poisson, "faces": faces, "crowded_movers": crowded_movers,
            "scrambled_rows": scrambled_rows}[name]()


# ---------------------------------------------------------------------------------------------------------------------
# What the kernels see: the classifications of deposit_runs.cu, deposit_cells.cu and gather_push_tile.cu restated
# ---------------------------------------------------------------------------------------------------------------------
def grid_positions(s, ng, relative_time=None):
    """New and old positions in grid units of arrays with ng guard cells (pic_common.cuh deposit_coords), per axis."""
    dt = s.dt
    relative_time = -0.5 * dt if relative_time is None else relative_time
    tshift = relative_time + 0.5 * dt
    xyzmin, _ = s.corner(ng)
    u = [s.p[k] for k in ("ux", "uy", "uz")]
    inv_c2 = 1.0 / (workloads.C * workloads.C)
    gaminv = 1.0 / np.sqrt(1.0 + u[0] * u[0] * inv_c2 + u[1] * u[1] * inv_c2 + u[2] * u[2] * inv_c2)
    new, old = [], []
    for d, k in enumerate(("x", "y", "z")):
        xn = ((s.p[k] - xyzmin[d]) + tshift * u[d] * gaminv) * s.dinv[d]
        new.append(xn)
        old.append(xn - dt * s.dinv[d] * u[d] * gaminv)
    return new, old


def shape_index(x, nox):
    """Cell index of the shape factor of order nox (ShapeFactors.H): floor for odd orders, nearest node for even."""
    return np.floor(x + (0.5 if nox % 2 == 0 else 0.0)).astype(np.int64)


def quiet_kernel_events(s, nox, ng):
    """deposit_quiet_kernel's view of the particles: movers (changed cell), lone strays (the `lone` rule on the keys of
    a chunk of 32) and register-window jumps (flush_all) over warps of 16 chunks."""
    new, old = grid_positions(s, ng)
    inew = [shape_index(v, nox) for v in new]
    iold = [np.floor(v).astype(np.int64) if nox == 1 else shape_index(v, nox) for v in old]
    moved = (inew[0] != iold[0]) | (inew[1] != iold[1]) | (inew[2] != iold[2])
    key = np.where(moved, -1, inew[0] + 1024 * (inew[1] + 1024 * inew[2]))
    lones = jumps = 0
    cur = -1
    for base in range(0, s.np, 32):
        if base % 512 == 0:
            cur = -1                     # a new warp
        k = key[base:base + 32]
        nval = len(k)
        for lane in range(nval):
            prev = k[lane - 1] if lane > 0 else None
            if lane > 0 and k[lane] == prev:
                continue                 # not a run head
            nxt = k[lane + 1] if lane + 1 < nval else None
            if 0 < lane < nval - 1 and k[lane] >= 0 and prev >= 0 and nxt >= 0 and k[lane] != prev and \
                    k[lane] != nxt and (nxt == prev or nxt == prev + 1):
                lones += 1
                continue
            if k[lane] < 0:
                continue
            if k[lane] != cur:
                if cur >= 0 and k[lane] != cur + 1:
                    jumps += 1
                cur = k[lane]
    return {"movers": int(moved.sum()), "lones": lones, "jumps": jumps}


def cells_kernel_queue(s, nox, ng):
    """deposit_cells_kernel's view: per supercell the sub-particles `enqueue` requests for the particles that are not
    quiet in their bin's cell (2 per direction of change), and the particles that reach outside the supercell (listed)."""
    new, old = grid_positions(s, ng)
    inew = [np.floor(v).astype(np.int64) for v in new]
    sh = [np.floor(old[d]).astype(np.int64) - inew[d] for d in range(3)]
    nt = [(s.n[d] + TILE - 1) // TILE for d in range(3)]
    binid = np.repeat(np.arange(len(s.cell_start) - 1), np.diff(s.cell_start))
    sc = binid // TILE ** 3
    lc = [binid % TILE, (binid // TILE) % TILE, (binid // TILE ** 2) % TILE]
    sc_xyz = [sc % nt[0], (sc // nt[0]) % nt[1], sc // (nt[0] * nt[1])]
    inside = np.ones(s.np, dtype=bool)
    t = []
    for d in range(3):
        td = inew[d] + np.minimum(sh[d], 0) - ng[d] - TILE * sc_xyz[d]
        t.append(td)
        inside &= (np.abs(sh[d]) <= 1) & (td >= 0) & (td + (sh[d] != 0) < TILE)
    simple = inside & (sh[0] == 0) & (sh[1] == 0) & (sh[2] == 0) & (t[0] == lc[0]) & (t[1] == lc[1]) & (t[2] == lc[2])
    nq = np.where(inside & ~simple, (1 + (sh[0] != 0)) * (1 + (sh[1] != 0)) * (1 + (sh[2] != 0)), 0)
    queued = np.bincount(sc, weights=nq, minlength=int(np.prod(nt))).astype(np.int64)
    return {"queued": queued, "listed": int((~inside).sum())}


def gather_tile_events(s, ng):
    """gather_push_tile_kernel's view: per supercell the particles whose (y, z) row differs from both lane neighbours
    (deferred to the CTA-local list), and the particles outside the supercell of their bin (global stray list)."""
    xyzmin, lo = s.corner(ng)
    ci = [lo[d] + ((s.p[k] - xyzmin[d]) * s.dinv[d]).astype(np.int64) for d, k in enumerate(("x", "y", "z"))]
    nt = [(s.n[d] + TILE - 1) // TILE for d in range(3)]
    isolated = np.zeros(int(np.prod(nt)), dtype=np.int64)
    leavers = 0
    for t in range(int(np.prod(nt))):
        b, e = int(s.cell_start[t * TILE ** 3]), int(s.cell_start[(t + 1) * TILE ** 3])
        if b >= e:
            continue
        tc = (t % nt[0], (t // nt[0]) % nt[1], t // (nt[0] * nt[1]))
        t0 = [s.box_lo[d] + tc[d] * TILE for d in range(3)]
        sl = slice(b, e)
        in_tile = np.ones(e - b, dtype=bool)
        for d in range(3):
            in_tile &= (ci[d][sl] >= t0[d]) & (ci[d][sl] < t0[d] + TILE)
        leavers += int((~in_tile).sum())
        idx = np.arange(e - b)
        lane = idx % 32
        row = np.where(in_tile, ci[1][sl] * 65536 + ci[2][sl], -1 - lane)
        prev = np.concatenate([[0], row[:-1]])
        nxt = np.concatenate([row[1:], [0]])
        last = (lane == 31) | (idx == e - b - 1)
        iso = ~((lane > 0) & (row == prev)) & ~(~last & (row == nxt))
        isolated[t] = int((iso & in_tile).sum())
    return {"isolated": isolated, "leavers": leavers}


def on_faces(s):
    """Per axis: particles exactly on a cell face, one ulp below one, and exactly on the box's upper face."""
    out = {}
    for d, k in enumerate(("x", "y", "z")):
        g = (s.p[k] - s.origin[d]) / s.dx[d]
        on = g == np.round(g)
        up = np.nextafter(s.p[k], np.inf)
        g_up = (up - s.origin[d]) / s.dx[d]
        below = ~on & (g_up == np.round(g_up))
        out[k] = {"on": int(on.sum()), "below": int(below.sum()), "prob_hi": int((s.p[k] == s.prob_hi[d]).sum()),
                  "supercell": int((on & (np.round(g) % TILE == 0) & (g > 0) & (g < s.n[d])).sum())}
    return out


def reach(s, shape, ng, nox):
    """Nodes of arrays with ng guard cells (numpy shape (z, y, x)) that some particle's Esirkepov stencil may touch: for
    every particle the box from its lower (old or new) cell - 3 to its upper cell + 4, a superset of the N+3 nodes of
    orders 1..4 (with the one-cell shift of the old stencil)."""
    new, old = grid_positions(s, ng)
    diff = np.zeros(tuple(v + 1 for v in shape), dtype=np.int64)
    lo, hi = [], []
    for d in (2, 1, 0):
        a = np.floor(np.minimum(new[d], old[d])).astype(np.int64) - 3
        b = np.floor(np.maximum(new[d], old[d])).astype(np.int64) + 5        # exclusive
        lim = shape[2 - d]
        lo.append(np.clip(a, 0, lim))
        hi.append(np.clip(b, 0, lim))
    for corner in range(8):
        idx = tuple(hi[a] if (corner >> a) & 1 else lo[a] for a in range(3))
        sign = -1 if bin(corner).count("1") % 2 else 1
        np.add.at(diff, idx, sign)
    return np.cumsum(np.cumsum(np.cumsum(diff, 0), 1), 2)[:shape[0], :shape[1], :shape[2]] > 0
