"""CPU tests (-m "not gpu"): the multi-rank paths of the C++ step driver on the host.  The "ranks" are threads of
this process, each with its own engine instance of the host library (tests/host_harness: every csrc file compiled
by g++ against the SIMT emulator); the eight NCCL entry points the driver binds at run time resolve to
tests/host_harness/fake_nccl.cpp (PIC_NCCL_LIBRARY).  Checked against the single-box oracle: guard-cell sweeps and
particle migration between bricks, and -- never exercised on a device so far -- slabs along a non-periodic axis
with PEC walls, the moving window pulling planes from the next slab, continuous injection on the top slab with
global ids, and the antenna replicated on every rank.  TEST INFRASTRUCTURE; no product code runs this way."""
import numpy as np
import pytest

from warpx_b200 import abi, parallel, workloads


pytestmark = pytest.mark.timeout(900)


@pytest.fixture(scope="module")
def hh():
    from host_harness import harness
    return harness


def _gather_fields(res, osim, world):
    """max |rank value - oracle value| per component over the valid points of every brick, and the oracle's scale."""
    err, scale = [], []
    for c in range(9):
        od, oa = osim.fab(c)
        worst = 0.0
        for r in range(world):
            (d, a), (blo, bhi) = res[r]["fields"][c], res[r]["box"]
            sl = tuple(slice(od.ng[2 - ax] + blo[2 - ax], od.ng[2 - ax] + bhi[2 - ax] + 1 + abi.YEE_STAG[c][2 - ax])
                       for ax in range(3))
            worst = max(worst, float(np.max(np.abs(a[d.valid_slices()] - oa[sl]))))
        err.append(worst)
        scale.append(float(np.max(np.abs(oa))))
    return err, scale


def test_two_bricks_periodic_loop_matches_oracle(orc, hh):
    """Config 1 in the small (16^3 Langmuir wave) on two bricks: NCCL halo sweeps (FillBoundary / SumBoundary) and
    particle migration of the C++ driver, 8 steps, against the single-box oracle; particle count conserved."""
    HS = hh.host_simulation_class()
    n, world = 16, 2
    full = workloads.langmuir_3d(n=n)

    def rank_fn(rank, dist):
        dec = parallel.Decomposition((n, n, n), parallel.brick_grid(world), rank)
        sim = HS(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=1, dist=dist, sort_interval=4)
        for s in full["species"]:
            cell = [np.floor((s[k] - full["prob_lo"][d]) / sim.dx[d]).astype(int) for d, k in enumerate("xyz")]
            m = np.ones(len(s["x"]), dtype=bool)
            for d in range(3):
                m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
            sim.add_species(s["name"], s["q"], s["m"], *[s[k][m] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
        n0 = sim.total_particles()
        sim.Evolve(8)
        assert sim.total_particles() == n0 == 2 * n ** 3
        return dict(fields={c: sim.field_numpy(c) for c in range(9)}, box=(sim.box_lo, sim.box_hi))

    res = hh.run_ranks(world, rank_fn)
    osim = orc.OracleSim(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=1)
    for s in full["species"]:
        osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    osim.evolve(8)
    err, scale = _gather_fields(res, osim, world)
    for c in (0, 1, 2, 6, 7, 8):             # B is round-off in this electrostatic mode
        assert err[c] <= 1e-10 * scale[c], abi.COMP_NAMES[c]


def test_eight_bricks_order3_thermal_loop_matches_oracle(orc, hh):
    """2 x 2 x 2 bricks of 8^3 cells, order 3, bilinear filter, thermal particles at u_th = 0.3 c (every brick trades
    particles with its face, edge and corner neighbours): 6 steps against the single-box oracle."""
    HS = hh.host_simulation_class()
    n, world, nsteps = 16, 8, 6
    full = workloads.uniform_plasma_3d(n=n, ppc=(2, 1, 1), u_th=0.3, perturbation=0.01)
    s = full["species"][0]

    def rank_fn(rank, dist):
        dec = parallel.Decomposition((n, n, n), parallel.brick_grid(world), rank)
        sim = HS(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=3, dist=dist, sort_interval=4, use_filter=True)
        cell = [np.floor((s[k] - full["prob_lo"][d]) / sim.dx[d]).astype(int) for d, k in enumerate("xyz")]
        m = np.ones(len(s["x"]), dtype=bool)
        for d in range(3):
            m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
        sim.add_species(s["name"], s["q"], s["m"], *[s[k][m] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
        n0, mine = sim.total_particles(), sim.species[0].np
        sim.Evolve(nsteps)
        assert sim.total_particles() == n0
        return dict(fields={c: sim.field_numpy(c) for c in range(9)}, box=(sim.box_lo, sim.box_hi),
                    moved=sim.species[0].np != mine)

    swept = hh.host_library().pic_engine_listed_sweeps()
    res = hh.run_ranks(world, rank_fn)
    assert any(r["moved"] for r in res)
    # the migration classified from the push's list of brick leavers (3 axis sweeps x 6 steps x 8 ranks), not by sweeping
    assert hh.host_library().pic_engine_listed_sweeps() - swept == 3 * nsteps * world
    osim = orc.OracleSim(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=3, use_filter=True)
    osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    osim.evolve(nsteps)
    err, scale = _gather_fields(res, osim, world)
    for c in range(9):
        assert err[c] <= 1e-11 * scale[c], abi.COMP_NAMES[c]


def test_two_wide_bricks_order3_fused_current_exchange_matches_oracle(orc, hh):
    """Two bricks of 16^3 cells, order 3, bilinear filter, u_th = 0.3 c: wide enough for the fused SumBoundary +
    refresh of J (halo mode 2: one exchange per axis instead of two) -- 6 steps against the single-box oracle, and the
    fused exchange really ran (one per step and rank)."""
    HS = hh.host_simulation_class()
    n_cell, world, nsteps = (32, 16, 16), 2, 6
    full = workloads.uniform_plasma_3d(n_cell=n_cell, ppc=(2, 1, 1), u_th=0.3, lx=(4e-6, 2e-6, 2e-6), perturbation=0.01)
    s = full["species"][0]

    def rank_fn(rank, dist):
        dec = parallel.Decomposition(n_cell, parallel.brick_grid(world), rank)
        sim = HS(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=3, dist=dist, sort_interval=4, use_filter=True)
        cell = [np.floor((s[k] - full["prob_lo"][d]) / sim.dx[d]).astype(int) for d, k in enumerate("xyz")]
        m = np.ones(len(s["x"]), dtype=bool)
        for d in range(3):
            m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
        sim.add_species(s["name"], s["q"], s["m"], *[s[k][m] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
        n0 = sim.total_particles()
        sim.Evolve(nsteps)
        assert sim.total_particles() == n0
        return dict(fields={c: sim.field_numpy(c) for c in range(9)}, box=(sim.box_lo, sim.box_hi))

    assert parallel.brick_grid(world) == (2, 1, 1)
    before = hh.host_library().pic_engine_fused_sum_exchanges()
    res = hh.run_ranks(world, rank_fn)
    assert hh.host_library().pic_engine_fused_sum_exchanges() - before == nsteps * world
    osim = orc.OracleSim(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=3, use_filter=True)
    osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    osim.evolve(nsteps)
    err, scale = _gather_fields(res, osim, world)
    for c in range(9):
        assert err[c] <= 1e-11 * scale[c], abi.COMP_NAMES[c]


@pytest.mark.parametrize("world", [4])
def test_z_slabs_with_moving_window_match_oracle(orc, hh, world):
    """The laser-acceleration deck in the small (12 x 12 x 64, order 3, filter, PEC z, moving window at c, antenna,
    continuous injection) on slabs along z: every field and every electron (by id) against the single-box oracle."""
    from test_oracle import make_lwfa_oracle
    HS = hh.host_simulation_class()
    nsteps = 10
    wl = workloads.laser_acceleration_3d(n_cell=(12, 12, 64), max_step=nsteps)

    def rank_fn(rank, dist):
        sim = HS(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"], dist=dist, use_filter=True,
                 sort_interval=4, nb=(1, 1, world), boundaries=abi.make_boundaries(wl["field_lo"], wl["field_hi"]),
                 moving_window=(wl["moving_window_dir"], wl["moving_window_v"]))
        sp = wl["species"][0]
        sim.add_plasma_species(sp["name"], sp["q"], sp["m"],
                               abi.make_injector(sp["ppc"], sp["bound_lo"], sp["bound_hi"], sp["density"], True),
                               capacity=12 * 12 * 200)
        la = wl["lasers"][0]
        sim.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"], la["e_max"],
                                     la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
        sim.Evolve(nsteps)
        return dict(fields={c: sim.field_numpy(c) for c in range(9)}, box=(sim.box_lo, sim.box_hi),
                    parts=sim.species_numpy(0, sort_by_id=False), dz=sim.dx[2], prob=(sim.prob_lo, sim.prob_hi))

    res = hh.run_ranks(world, rank_fn)
    osim = make_lwfa_oracle(orc, wl)
    osim.evolve(nsteps)
    plo, phi = osim.prob_domain()
    assert res[0]["prob"][0] == pytest.approx(plo, rel=0, abs=1e-20) and res[-1]["prob"][1] == pytest.approx(phi, rel=0, abs=1e-20)
    err, scale = _gather_fields(res, osim, world)
    for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):
        s = max(scale[c] for c in group)
        assert s > 0
        for c in group:
            assert err[c] <= 1e-11 * s, abi.COMP_NAMES[c]
    B = osim.particles(0)
    ids = np.concatenate([res[r]["parts"]["id"] for r in range(world)])
    order = np.argsort(ids)
    assert np.array_equal(ids[order], np.arange(len(B["x"])))          # global ids: every electron exactly once
    assert sum(len(res[r]["parts"]["x"]) > 0 for r in range(world)) >= 2    # the plasma straddles a slab boundary: migration
    for k in ("x", "y", "z"):
        a = np.concatenate([res[r]["parts"][k] for r in range(world)])[order]
        assert np.max(np.abs(a - B[k])) / res[0]["dz"] <= 1e-10, k
    for k in ("ux", "uy", "uz"):
        a = np.concatenate([res[r]["parts"][k] for r in range(world)])[order]
        assert np.max(np.abs(a - B[k])) / workloads.C <= 1e-10, k


def test_boosted_frame_z_slabs_match_oracle(orc, hh):
    """BASELINE.json configs[3] in the small (laser acceleration in the boosted frame, gamma = 10: CKC, Vay, order 3,
    filter, Godfrey NCI corrector, PEC z, moving window, boosted antenna, electrons + ions injected continuously from
    the lab-frame plasma bounds) on FOUR slabs along z: fields and both species (by id) against the single-box oracle."""
    from test_oracle import make_lwfa_oracle, _nci_lines
    from warpx_b200.engine import max_dt, nci_godfrey_stencils
    HS = hh.host_simulation_class()
    world, nsteps = 4, 24
    wl = workloads.laser_acceleration_boosted_3d(n_cell=(12, 12, 96), density=1.e22, use_fdtd_nci_corr=True)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    # six cells of vacuum above the antenna, as in tests/test_host_engine.py (the coarse grid's guard-cell tie at the wall)
    wl["prob_lo"] = wl["prob_lo"][:2] + (wl["prob_lo"][2] + 6 * dx[2],)
    wl["prob_hi"] = wl["prob_hi"][:2] + (wl["prob_hi"][2] + 6 * dx[2],)
    nci = nci_godfrey_stencils(hh.host_library(), _nci_lines(), workloads.C * wl["cfl"] * max_dt(wl["solver"], dx) / dx[2])

    def rank_fn(rank, dist):
        sim = HS(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"], dist=dist,
                 solver=wl["solver"], pusher=wl["pusher"], use_filter=True, sort_interval=4, nb=(1, 1, world),
                 boundaries=abi.make_boundaries(wl["field_lo"], wl["field_hi"]),
                 moving_window=(wl["moving_window_dir"], wl["moving_window_v"]),
                 gamma_boost=wl["gamma_boost"], nci_stencils=nci)
        for sp in wl["species"]:
            sim.add_plasma_species(sp["name"], sp["q"], sp["m"],
                                   abi.make_injector(sp["ppc"], sp["bound_lo"], sp["bound_hi"], sp["density"], True),
                                   capacity=12 * 12 * 200)
        la = wl["lasers"][0]
        sim.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"], la["e_max"],
                                     la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
        sim.Evolve(nsteps)
        return dict(fields={c: sim.field_numpy(c) for c in range(9)}, box=(sim.box_lo, sim.box_hi),
                    parts=[sim.species_numpy(i, sort_by_id=False) for i in (0, 1)], dz=sim.dx[2])

    res = hh.run_ranks(world, rank_fn)
    osim = make_lwfa_oracle(orc, wl)
    osim.evolve(nsteps)
    err, scale = _gather_fields(res, osim, world)
    for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):
        s = max(scale[c] for c in group)
        assert s > 0
        for c in group:
            assert err[c] <= 1e-9 * s, abi.COMP_NAMES[c]
    for isp in (0, 1):
        B = osim.particles(isp)
        ids = np.concatenate([res[r]["parts"][isp]["id"] for r in range(world)])
        order = np.argsort(ids)
        assert len(B["x"]) > 0 and np.array_equal(ids[order], np.arange(len(B["x"])))
        for k in ("x", "y", "z"):
            a = np.concatenate([res[r]["parts"][isp][k] for r in range(world)])[order]
            assert np.max(np.abs(a - B[k])) / res[0]["dz"] <= 1e-9, (isp, k)
        for k in ("ux", "uy", "uz"):
            a = np.concatenate([res[r]["parts"][isp][k] for r in range(world)])[order]
            assert np.max(np.abs(a - B[k])) / (10.0 * workloads.C) <= 1e-9, (isp, k)


def test_brick_decomposition_neighbours():
    assert parallel.brick_grid(1) == (1, 1, 1) and parallel.brick_grid(2) == (2, 1, 1)
    assert parallel.brick_grid(4) == (2, 2, 1) and parallel.brick_grid(8) == (2, 2, 2)
    dec = parallel.Decomposition((64, 64, 64), (2, 2, 2), 5)      # coord (1, 0, 1)
    assert dec.coord == (1, 0, 1) and dec.box_lo == (32, 0, 32) and dec.box_hi == (63, 31, 63)
    assert dec.neighbour(0, 1) == dec.neighbour(0, 0) == dec.rank_of((0, 0, 1))   # two bricks: same rank
    assert dec.neighbour(1, 1) == dec.rank_of((1, 1, 1))


@pytest.mark.parametrize("nb,periodic", [((2, 1, 1), (1, 1, 1)), ((2, 2, 2), (1, 1, 1)), ((1, 1, 2), (1, 1, 0))])
def test_halo_copy_and_add_match_oracle(orc, hh, nb, periodic):
    """pic_halo_copy / pic_halo_add -- the one-call replacements of ablastr's FillBoundary / SumBoundary -- on random
    data over bricks (thread ranks, NCCL stand-in) against the oracle's multi-box FillBoundary / SumBoundary: every
    staggering, ng below and at the allocated width, a non-periodic axis split into slabs."""
    import ctypes as C
    L = hh.host_library()
    world = nb[0] * nb[1] * nb[2]
    n = tuple(8 * v for v in nb)
    ngalloc = (3, 3, 3)
    geom = abi.make_geom(n, (0.0, 0.0, 0.0), tuple(float(v) for v in n), periodic=periodic)
    comps = (0, 4, 8, 6)                      # Ex, By, jz, jx staggerings
    decs = [parallel.Decomposition(n, nb, r) for r in range(world)]
    rng = np.random.default_rng(3)
    # valid points from one global array per component, so that the points shared by neighbouring boxes and the periodic
    # duplicates hold equal values (what every FillBoundary / SumBoundary of a run sees); guard cells start random
    start = [[None] * len(comps) for _ in decs]
    for k, c in enumerate(comps):
        stag = abi.YEE_STAG[c]
        G = rng.standard_normal(tuple(n[2 - ax] + stag[2 - ax] for ax in range(3)))
        for d in range(3):
            if periodic[d] and stag[d]:
                ax = 2 - d
                hi, lo = [slice(None)] * 3, [slice(None)] * 3
                hi[ax], lo[ax] = n[d], 0
                G[tuple(hi)] = G[tuple(lo)]
        for r, dec in enumerate(decs):
            f = abi.make_fab(None, dec.box_lo, dec.box_hi, ngalloc, stag)
            a = rng.standard_normal(f.shape)
            sl = tuple(slice(dec.box_lo[2 - ax], dec.box_hi[2 - ax] + 1 + stag[2 - ax]) for ax in range(3))
            a[f.valid_slices()] = G[sl]
            start[r][k] = a

    def run(op, ng, src_ng=None):
        def rank_fn(rank, dist):
            ident = __import__("torch").zeros(128, dtype=__import__("torch").uint8)
            if rank == 0:
                raw = (C.c_ubyte * 128)()
                assert L.pic_comm_unique_id(raw) == 0
                ident.copy_(__import__("torch").tensor(list(raw), dtype=__import__("torch").uint8))
            dist.broadcast(ident, 0)
            comm = L.pic_comm_create((C.c_ubyte * 128)(*ident.tolist()), world, rank)
            assert comm
            d = decs[rank]
            eng = L.pic_engine_create(C.byref(geom), abi.int3(d.box_lo), abi.int3(d.box_hi), 1, 1, 0, 0, 1.0, 0.0, 4, 0, abi.int3((1, 1, 1)))
            if not all(periodic):
                names = ["periodic" if p else "pec" for p in periodic]
                assert L.pic_engine_set_boundaries(eng, C.byref(abi.make_boundaries(names, names))) == 0
            assert L.pic_engine_set_comm(eng, comm, abi.int3(nb)) == 0, L.pic_last_error()
            fabs = [orc.HostFab(d.box_lo, d.box_hi, ngalloc, abi.YEE_STAG[c], data=start[rank][k].copy()) for k, c in enumerate(comps)]
            arr = orc.fab_array(fabs)
            if op == "copy":
                rc = L.pic_halo_copy(eng, arr, len(fabs), abi.int3(ng), None)
            else:
                rc = L.pic_halo_add(eng, arr, len(fabs), abi.int3(src_ng), abi.int3(ng), None)
            assert rc == 0, L.pic_last_error()
            dist.barrier()
            L.pic_engine_destroy(eng)
            L.pic_comm_destroy(comm)
            return [f.a.copy() for f in fabs]
        return hh.run_ranks(world, rank_fn)

    for op, ng, src_ng in (("copy", (2, 1, 3), None), ("copy", (3, 3, 3), None), ("add", (3, 3, 3), (2, 2, 2) if all(periodic) else (2, 2, 3)),
                           ("add", (3, 3, 3), (3, 3, 3))):
        got = run(op, ng, src_ng)
        for k, c in enumerate(comps):
            boxes = [orc.HostFab(d.box_lo, d.box_hi, ngalloc, abi.YEE_STAG[c], data=start[r][k].copy()) for r, d in enumerate(decs)]
            arr = orc.fab_array(boxes)
            if op == "copy":
                orc.lib().orc_fill_boundary(arr, world, abi.int3(ng), C.byref(geom))
            else:
                orc.lib().orc_sum_boundary(arr, world, abi.int3(src_ng), abi.int3(ng), C.byref(geom))
            for r in range(world):
                # AMReX touches the box grown by ng only; the axis sweeps here also rewrite (never-read) cells beyond it
                sl = tuple(slice(ngalloc[2 - ax] - ng[2 - ax], boxes[r].a.shape[ax] - (ngalloc[2 - ax] - ng[2 - ax])) for ax in range(3))
                scale = np.max(np.abs(boxes[r].a[sl]))
                assert np.max(np.abs(got[r][k][sl] - boxes[r].a[sl])) <= 1e-14 * scale, (op, ng, src_ng, abi.COMP_NAMES[c], r)


@pytest.mark.parametrize("world", [2, 8])
def test_redistribute_moves_every_particle_to_its_owner(orc, hh, world):
    """pic_engine_redistribute (HandleParticlesAtBoundaries as one call): particles displaced by up to 0.9 cell in every
    direction -- across brick faces, edges, corners and the periodic domain boundary -- end up on the rank that owns
    their cell, wrapped exactly like amrex's enforcePeriodic (the oracle's restatement), none lost, none duplicated."""
    import ctypes as C
    HS = hh.host_simulation_class()
    n = 16
    full = workloads.uniform_plasma_3d(n=n, ppc=(1, 1, 2), u_th=0.0)
    s = full["species"][0]
    dx = [(full["prob_hi"][d] - full["prob_lo"][d]) / n for d in range(3)]
    rng = np.random.default_rng(8)
    shift = [rng.uniform(-0.9, 0.9, len(s["x"])) * dx[d] for d in range(3)]
    gid = np.arange(len(s["x"]), dtype=np.float64)          # carried in uz: identifies a particle after the move

    def rank_fn(rank, dist):
        dec = parallel.Decomposition((n, n, n), parallel.brick_grid(world), rank)
        sim = HS(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=1, dist=dist, sort_interval=4)
        cell = [np.floor((s[k] - full["prob_lo"][d]) / dx[d]).astype(int) for d, k in enumerate("xyz")]
        m = np.ones(len(s["x"]), dtype=bool)
        for d in range(3):
            m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
        sim.add_species(s["name"], s["q"], s["m"], s["x"][m], s["y"][m], s["z"][m], s["w"][m], s["ux"][m], s["uy"][m], gid[m])
        sp = sim.species[0]
        torch = __import__("torch")
        who = sp.array("uz").to(torch.int64)               # the engine sorted the particles when they were registered
        for d, k in enumerate("xyz"):                       # the "push": host arrays are the device arrays here
            sp.array(k).add_(torch.from_numpy(shift[d])[who])
        assert sim.L.pic_engine_redistribute(sim.native, None) == 0, sim.L.pic_last_error()
        sim._sync_from_native()
        P = sim.species_numpy(0)
        return dict(P=P, box=(dec.box_lo, dec.box_hi))

    res = hh.run_ranks(world, rank_fn)
    got_id = np.concatenate([r["P"]["uz"] for r in res])
    assert len(got_id) == len(gid) and np.array_equal(np.sort(got_id), gid)          # none lost, none duplicated
    # expected positions: the displaced particles after the oracle's periodic wrap
    Q = orc.HostParticles(x=s["x"] + shift[0], y=s["y"] + shift[1], z=s["z"] + shift[2], w=s["w"], ux=s["ux"], uy=s["uy"], uz=gid)
    geom = abi.make_geom(full["n_cell"], full["prob_lo"], full["prob_hi"])
    orc.lib().orc_wrap_periodic(C.byref(Q.soa), C.byref(geom))
    moved_rank = 0
    for r in res:
        P, (blo, bhi) = r["P"], r["box"]
        idx = P["uz"].astype(np.int64)
        for d, k in enumerate("xyz"):
            assert np.array_equal(P[k], getattr(Q, k)[idx]), (k, float(np.max(np.abs(P[k] - getattr(Q, k)[idx]))),
                                                                  int(np.sum(P[k] != getattr(Q, k)[idx])))
            c = np.floor((P[k] - full["prob_lo"][d]) / dx[d]).astype(int)
            c = np.clip(c, 0, n - 1)                        # a particle wrapped onto prob_hi belongs to the last cell
            assert np.all((c >= blo[d]) & (c <= bhi[d])), (k, "a particle is on a rank that does not own its cell")
        cell0 = [np.floor((s[k][idx] - full["prob_lo"][d]) / dx[d]).astype(int) for d, k in enumerate("xyz")]
        moved_rank += int(np.sum(~np.all([(cell0[d] >= blo[d]) & (cell0[d] <= bhi[d]) for d in range(3)], axis=0)))
    assert moved_rank > 100                                  # the test did move particles between ranks


def test_classify_from_candidate_list_matches_full_sweep(orc, hh):
    """pic_particles_classify_listed (the migration's axis sweep over the push's list of brick leavers) against
    pic_particles_classify (every particle): same leavers when the list holds them, dead entries dropped, the full
    sweep when the list overflowed; pic_migrate_note_appended adds [np_old, np_new) of the last unpack."""
    import ctypes as C
    L = hh.host_library()
    rng = np.random.default_rng(3)
    n, npart = 16, 4000
    geom = abi.make_geom((n, n, n), (0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
    P = orc.HostParticles(**{k: rng.uniform(0.0, 1.0, npart) for k in orc.HostParticles.NAMES})
    lo, hi, cap = 4, 11, 4096

    def run(listed, cand=None):
        counts = np.zeros(2, dtype=np.int32)
        idx = [np.full(cap, -7, dtype=np.int32) for _ in range(2)]
        args = [C.byref(P.soa), C.byref(geom), 1, lo, hi, 0, counts.ctypes.data, idx[0].ctypes.data, idx[1].ctypes.data, cap, None]
        if listed:
            assert L.pic_particles_classify_listed(*args, C.byref(cand), None) == 0, L.pic_last_error()
        else:
            assert L.pic_particles_classify(*args, None) == 0, L.pic_last_error()
        return [set(idx[s][:counts[s]].tolist()) for s in range(2)], counts

    want, wc = run(False)
    assert wc[0] > 100 and wc[1] > 100 and wc[0] + wc[1] < npart
    cell = np.floor(P.y * n).astype(int)
    leavers = np.nonzero((cell < lo) | (cell > hi))[0]
    stay = np.nonzero((cell >= lo) & (cell <= hi))[0][:50]
    # the list: every leaver, some particles that stay, two entries behind the particle count, one dropped earlier
    entries = np.concatenate([leavers, stay, [npart + 5, npart], [-1]]).astype(np.int32)
    rng.shuffle(entries)
    store = np.concatenate([entries, np.full(64, -9, dtype=np.int32)])
    count = np.array([len(entries)], dtype=np.int32)
    cand = abi.pic_escape_list()
    cand.idx, cand.count, cand.capacity = store.ctypes.data, count.ctypes.data, len(store)
    got, gc = run(True, cand)
    assert got == want and list(gc) == list(wc)
    assert set(store[:len(entries)][entries >= npart].tolist()) == {-1}        # dead entries are dropped for good
    # appended arrivals of an unpack (work[4] = count before, work[5] = after) become candidates
    work = np.zeros(8, dtype=np.int32)
    work[4], work[5] = npart - 10, npart
    assert L.pic_migrate_note_appended(work.ctypes.data, C.byref(cand), None) == 0, L.pic_last_error()
    assert count[0] == len(entries) + 10 and store[len(entries):len(entries) + 10].tolist() == list(range(npart - 10, npart))
    work[4], work[5] = npart, npart - 3                                       # a net loss appends nothing
    assert L.pic_migrate_note_appended(work.ctypes.data, C.byref(cand), None) == 0
    assert count[0] == len(entries) + 10
    work[4], work[5] = 0, 1000                                                # more than the list holds: overflow mark
    assert L.pic_migrate_note_appended(work.ctypes.data, C.byref(cand), None) == 0
    assert count[0] == len(store) + 1
    got, gc = run(True, cand)                                                 # overflowed list: every particle is visited
    assert got == want and list(gc) == list(wc)


# ---------------------------------------------------------------------------------------------------------------------
# Gauss's law over the union of the bricks (tests/helpers.py: gauss_residual): a particle that migration loses or
# duplicates breaks G = div E - rho/ep0 by about 4e-2 of max|rho^0/ep0|.
# ---------------------------------------------------------------------------------------------------------------------
def union_state(sim):
    """What union_gauss needs of one rank: its box, the unique part of its valid E, and its particles."""
    E = []
    for c in range(3):
        d, a = sim.field_numpy(c)
        nb = [sim.box_hi[ax] - sim.box_lo[ax] + 1 for ax in range(3)]
        E.append(a[d.valid_slices()][:nb[2], :nb[1], :nb[0]].copy())
    parts = [{k: v.copy() for k, v in sim.species_numpy(i).items()} for i in range(len(sim.species))]   # host "device" memory
    return dict(box=(sim.box_lo, sim.box_hi), E=E, parts=parts)


def union_gauss(orc, states, full, nox, use_filter=False):
    """G of the whole box from every rank's state, rho from the oracle's charge deposit of every rank's particles;
    the first species' rho (the scale of G: a neutral plasma has almost none in total); the union's particle ids."""
    from helpers import gauss_residual, oracle_rho
    n = full["n_cell"]
    E = [np.full((n[2], n[1], n[0]), np.nan) for _ in range(3)]
    for st in states:
        lo, hi = st["box"]
        for c in range(3):
            E[c][lo[2]:hi[2] + 1, lo[1]:hi[1] + 1, lo[0]:hi[0] + 1] = st["E"][c]
    assert not any(np.isnan(e).any() for e in E)
    rho, first, ids = 0.0, None, []
    for isp, s in enumerate(full["species"]):
        parts = {k: np.concatenate([st["parts"][isp][k] for st in states]) for k in ("x", "y", "z", "w", "ux", "uy", "uz", "id")}
        one = oracle_rho(orc, n, full["prob_lo"], full["prob_hi"], nox, parts, s["q"], use_filter)
        first = one if first is None else first
        rho = rho + one
        ids.append(parts["id"])
    dx = [(full["prob_hi"][d] - full["prob_lo"][d]) / n[d] for d in range(3)]
    return gauss_residual(E, rho, dx, n), first, ids


def gauss_bricks(orc, hh, full, world, nox, checkpoints, **kw):
    """Run the bricks through the checkpoints and check G of their union at each: max|G^n - G^0| / max|rho^0/ep0|
    <= 1e-12 (rho^0 of the first species), every particle id exactly once, the particle count kept.  Returns whether particles changed brick."""
    from helpers import gauss_drift
    HS = hh.host_simulation_class()
    n = full["n_cell"]

    def rank_fn(rank, dist):
        dec = parallel.Decomposition(n, parallel.brick_grid(world), rank)
        sim = HS(n, full["prob_lo"], full["prob_hi"], nox=nox, dist=dist, sort_interval=4, **kw)
        for s in full["species"]:
            cell = [np.floor((s[k] - full["prob_lo"][d]) / sim.dx[d]).astype(int) for d, k in enumerate("xyz")]
            m = np.ones(len(s["x"]), dtype=bool)
            for d in range(3):
                m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
            sim.add_species(s["name"], s["q"], s["m"], *[s[k][m] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
        out, done, mine, moved = [union_state(sim)], 0, sim.species[0].np, False
        for step in checkpoints:
            sim.Evolve(step - done, synchronize_last=False)
            done = step
            out.append(union_state(sim))
            moved = moved or sim.species[0].np != mine
        return dict(states=out, moved=moved)

    res = hh.run_ranks(world, rank_fn)
    G0, rho0, ids0 = union_gauss(orc, [r["states"][0] for r in res], full, nox, kw.get("use_filter", False))
    for k, step in enumerate(checkpoints):
        G, _, ids = union_gauss(orc, [r["states"][k + 1] for r in res], full, nox, kw.get("use_filter", False))
        for a, b in zip(ids, ids0):
            assert len(a) == len(b) and np.array_equal(np.sort(a), np.sort(b)), step
        r = gauss_drift(G, G0, rho0)
        assert r <= 1e-12, (step, r)
    return any(r["moved"] for r in res)


def test_two_bricks_keep_gauss_law(orc, hh):
    """Two bricks as in test_two_bricks_periodic_loop_matches_oracle (16^3, order 1), with thermal electrons at
    u_th = 0.3 c so that particles cross between the bricks every step, 12 steps."""
    full = workloads.uniform_plasma_3d(n=16, ppc=(2, 1, 1), u_th=0.3, perturbation=0.01)
    assert gauss_bricks(orc, hh, full, 2, 1, (1, 4, 5, 12))


def test_eight_bricks_keep_gauss_law(orc, hh):
    """The eight-brick loop of test_eight_bricks_order3_thermal_loop_matches_oracle (order 3, bilinear filter, u_th =
    0.3 c: particles cross to face, edge and corner neighbours), 8 steps."""
    full = workloads.uniform_plasma_3d(n=16, ppc=(2, 1, 1), u_th=0.3, perturbation=0.01)
    assert gauss_bricks(orc, hh, full, 8, 3, (1, 4, 5, 8), use_filter=True)


def test_nccl_standins_export_the_nccl_entry_points(hh):
    """Both builds of fake_nccl.cpp -- host buffers (the ranks above) and device buffers (tests/test_gpu_multirank.py,
    -DPIC_STANDIN_DEVICE) -- export the nine symbols csrc/comm.cu binds, and the call counters a test reads to prove the
    stand-in was the library bound."""
    import subprocess
    want = {"ncclGetUniqueId", "ncclCommInitRank", "ncclCommDestroy", "ncclSend", "ncclRecv", "ncclGroupStart",
            "ncclGroupEnd", "ncclAllReduce", "ncclGetErrorString"}
    counters = {"standin_sends", "standin_recvs", "standin_allreduces"}
    for path in (hh.build_fake_nccl(), hh.build_device_nccl()):
        out = subprocess.run(["nm", "-D", "--defined-only", path], check=True, capture_output=True, text=True).stdout
        names = {line.split()[-1] for line in out.splitlines() if line.split()[1:2] == ["T"]}
        assert {n for n in names if n.startswith("nccl")} == want, path
        assert counters <= names, path
    # the device build binds the driver API at run time only: no CUDA library at link time
    out = subprocess.run(["readelf", "-d", hh.build_device_nccl()], check=True, capture_output=True, text=True).stdout
    assert "libcuda" not in out and "libcudart" not in out
