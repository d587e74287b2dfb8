"""CPU tests (-m "not gpu"): the WHOLE product library on the host.  tests/host_harness compiles every file of
warpx_b200/csrc -- kernels, argument builders and the C++ step driver engine.cu -- with g++ against its SIMT
emulator (kernel<<<...>>> rewritten to emulator launches by cuda2host.py, nothing else changed) and
warpx_b200.engine.Simulation drives that library through the same C ABI, with CPU tensors as "device" memory.
What this checks where no GPU exists: the step sequence of the C++ driver with every feature switched on, the
host-side argument builders and the kernel arithmetic -- against the oracle.  What it cannot check: races, launch
bounds, speed.  TEST INFRASTRUCTURE; the product has no CPU path."""
import numpy as np
import pytest

from helpers import rel_linf
from warpx_b200 import abi, workloads


@pytest.fixture(scope="module")
def HostSimulation():
    from host_harness import harness
    return harness.host_simulation_class()


def _compare(sim, osim, nspecies, ftol=1e-9, scale_u=workloads.C):
    for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):        # E, B, J: each against the scale of its vector
        got, want = [], []
        for c in group:
            d, a = sim.field_numpy(c)
            _, oa = osim.fab(c)
            got.append(a[d.valid_slices()])
            want.append(oa[d.valid_slices()])
        scale = max(np.max(np.abs(w)) for w in want)
        assert scale > 0
        for c, g, w in zip(group, got, want):
            assert np.max(np.abs(g - w)) <= ftol * scale, abi.COMP_NAMES[c]
    for isp in range(nspecies):
        A = sim.species_numpy(isp, sort_by_id=True)
        B = osim.particles(isp)
        assert len(A["x"]) == len(B["x"]) and np.array_equal(A["id"], np.arange(len(B["x"])))
        assert np.array_equal(A["w"], B["w"])
        for k in ("x", "y", "z"):
            assert np.max(np.abs(A[k] - B[k])) / sim.dx[2] <= 1e-9, k
        for k in ("ux", "uy", "uz"):
            assert np.max(np.abs(A[k] - B[k])) / scale_u <= 1e-9, k


def test_periodic_loop_on_the_host_matches_oracle(orc, HostSimulation):
    """Config 1 in the small (8^3 Langmuir wave, two species, order 1): six steps of the C++ driver with the cell
    sort, the supercell gather and the register-run deposition, all under emulation."""
    wl = workloads.langmuir_3d(n=8)
    sim = HostSimulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, sort_interval=4)
    osim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1)
    for s in wl["species"]:
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.Evolve(6)
    osim.evolve(6)
    for c in (0, 1, 2, 6, 7, 8):          # B is round-off in this electrostatic mode
        d, a = sim.field_numpy(c)
        _, oa = osim.fab(c)
        assert rel_linf(a[d.valid_slices()], oa[d.valid_slices()]) <= 1e-10, abi.COMP_NAMES[c]
    e, b = sim.field_energy()
    eo, bo = osim.field_energy()
    assert e == pytest.approx(eo, rel=1e-10)


@pytest.mark.parametrize("mode", [abi.PIC_DEPOSIT_CELLS, abi.PIC_DEPOSIT_CELLS2, abi.PIC_DEPOSIT_CELLS3])
def test_order3_loop_with_lane_per_cell_deposition_on_the_host_matches_oracle(orc, HostSimulation, mode):
    """Config 2 in the small (16^3, 8 ppc, order 3, hot enough that particles cross cell faces every step): nine steps of
    the C++ driver with pic_set_deposit_mode(PIC_DEPOSIT_CELLS) -- slices, extra rounds for the particles that left the
    cell of their bin (the sort runs every 4 steps), the list for those that left the supercell -- under emulation."""
    from host_harness import harness
    wl = workloads.uniform_plasma_3d(n=16, ppc=(2, 2, 2), u_th=0.1, lx=2.5e-6, perturbation=0.01)
    hl = harness.host_library()
    hl.pic_set_deposit_mode(mode)
    try:
        sim = HostSimulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
        osim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3)
        for s in wl["species"]:
            sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
            osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        sim.Evolve(9)
        osim.evolve(9)
    finally:
        hl.pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS)
    _compare(sim, osim, 1)
    e, b = sim.field_energy()
    eo, bo = osim.field_energy()
    assert e == pytest.approx(eo, rel=1e-10)


def test_boosted_deck_with_every_feature_on_the_host_matches_oracle(orc, HostSimulation):
    """BASELINE.json config 4 in the very small: gamma_boost = 10, CKC, Vay, order 3, bilinear filter, Godfrey NCI
    corrector, PEC walls in z, moving window, boosted Gaussian antenna, electrons + ions injected continuously from
    lab-frame bounds -- 14 steps through the C++ driver on the host against the oracle."""
    from test_oracle import make_lwfa_oracle, _nci_lines
    from warpx_b200.engine import max_dt, nci_godfrey_stencils
    from host_harness import harness
    wl = workloads.laser_acceleration_boosted_3d(n_cell=(12, 12, 48), density=1.e22, use_fdtd_nci_corr=True)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    # The deck puts the antenna in the cell next to the upper wall.  On a grid this coarse the huge, cancelling drift
    # currents of the +-w antenna pairs leave the periodic duplicate nodes of the tiny field components different at
    # the 1e-5 level there, and which duplicate a guard cell copies is a tie the oracle (canonical owner) and the
    # kernels (same-index image, AMReX's last-copy-wins order) break differently.  Six cells of vacuum above the
    # antenna remove the tie from the comparison; the full-size deck (tests/test_gpu_zz_lwfa.py) keeps the wall.
    wl["prob_lo"] = wl["prob_lo"][:2] + (wl["prob_lo"][2] + 6 * dx[2],)
    wl["prob_hi"] = wl["prob_hi"][:2] + (wl["prob_hi"][2] + 6 * dx[2],)
    nci = nci_godfrey_stencils(harness.host_library(), _nci_lines(), workloads.C * max_dt(wl["solver"], dx) / dx[2])
    sim = HostSimulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, cfl=1.0, solver=wl["solver"], pusher=wl["pusher"],
                         use_filter=True, sort_interval=4, boundaries=abi.make_boundaries(wl["field_lo"], wl["field_hi"]),
                         moving_window=(2, 1.0), gamma_boost=wl["gamma_boost"], nci_stencils=nci)
    for s in wl["species"]:
        sim.add_plasma_species(s["name"], s["q"], s["m"],
                               abi.make_injector(s["ppc"], s["bound_lo"], s["bound_hi"], s["density"], True), 12 * 12 * 100)
    la = wl["lasers"][0]
    sim.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"], la["e_max"],
                                 la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
    osim = make_lwfa_oracle(orc, wl)
    assert sim.ng_EB == osim.guards()["ng_EB"] == [4, 4, 8] and sim.ng_FG == osim.guards()["ng_FG"] == [2, 2, 6]
    for chunk, sync in ((9, False), (5, True)):
        sim.Evolve(chunk, synchronize_last=sync)
        osim.evolve(chunk, synchronize_last=sync)
    assert sim.time == pytest.approx(osim.time(), rel=1e-15)
    plo, phi = osim.prob_domain()
    assert sim.prob_lo == pytest.approx(plo, rel=0, abs=1e-18) and sim.prob_hi == pytest.approx(phi, rel=0, abs=1e-18)
    assert sim.species[0].np == osim.L.orc_sim_np(osim.h, 0) > 0
    _compare(sim, osim, 2, ftol=1e-9, scale_u=10.0 * workloads.C)
    LA, LB = sim.laser_numpy(0), osim.laser_particles(0)
    assert len(LA["x"]) == len(LB["x"]) > 0
    for k in ("x", "y", "z"):
        assert np.max(np.abs(LA[k] - LB[k])) / dx[2] <= 1e-10, k


def test_plotfile_of_a_host_run_reproduces_the_oracle_checksums(orc, HostSimulation, tmp_path):
    """warpx_b200.diagnostics.write_plotfile (the reference's `diag.format = plotfile` layout) read back with
    tests/plotfile_reader.py: the per-field / per-species sums the reference's checksum.py forms from a plotfile equal
    the oracle's own (cell-centred averages of ablastr/coarsen/sample.H, momenta in SI units)."""
    from warpx_b200 import diagnostics
    import plotfile_reader
    wl = workloads.langmuir_3d(n=8)
    sim = HostSimulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, sort_interval=4)
    osim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1)
    for s in wl["species"]:
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.Evolve(5)
    osim.evolve(5)
    root = diagnostics.write_plotfile(sim, str(tmp_path / "plt"))
    assert root.endswith("plt00005")
    got = plotfile_reader.checksums(root, species=("electrons", "positrons"))
    for c, name in enumerate(abi.COMP_NAMES):
        want = osim.checksum_field(c)
        tol = 1e-9 if c not in (3, 4, 5) else 1e-2         # B is round-off noise in this electrostatic mode
        assert abs(got["lev=0"][name] - want) <= tol * abs(want) + 1e-30, name
    for isp, sname in enumerate(("electrons", "positrons")):
        P = osim.particles(isp)
        assert got[sname]["particle_position_x"] == pytest.approx(float(np.sum(np.abs(P["x"]))), rel=1e-12)
        assert got[sname]["particle_momentum_z"] == pytest.approx(float(np.sum(np.abs(P["uz"]))) * workloads.M_E, rel=1e-9)
        assert got[sname]["particle_weight"] == pytest.approx(float(np.sum(P["w"])), rel=1e-12)
    _, hdr = plotfile_reader.read_fields(root)
    assert hdr["step"] == 5 and hdr["n_cell"] == [8, 8, 8] and hdr["names"] == list(abi.COMP_NAMES)


def test_checkpoint_restart_on_the_host_continues_the_run(orc, HostSimulation, tmp_path):
    """FlushFormatCheckpoint / InitFromCheckpoint in the small: 6 steps, checkpoint, restart in a new Simulation, 4 more
    steps == 10 steps in one go (the summation order of the deposition differs after the restart's sort: 1e-12)."""
    from warpx_b200 import diagnostics
    wl = workloads.uniform_plasma_3d(n=16, ppc=(1, 1, 2), u_th=0.05, lx=2.5e-6, perturbation=0.01)

    def fresh():
        return HostSimulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
    s = wl["species"][0]
    ref = fresh()
    ref.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    ref.Evolve(6)
    ref.Evolve(4)
    a = fresh()
    a.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    a.Evolve(6)
    root = diagnostics.write_checkpoint(a, str(tmp_path / "chk"))
    b = fresh()
    assert diagnostics.read_checkpoint(b, root) == 6
    b.Evolve(4)
    assert b.istep == ref.istep == 10 and b.time == pytest.approx(ref.time, rel=1e-14)
    for c in range(9):
        _, x = ref.field_numpy(c)
        _, y = b.field_numpy(c)
        assert np.max(np.abs(x - y)) <= 1e-11 * max(np.max(np.abs(x)), 1e-300), abi.COMP_NAMES[c]
    A, B = ref.species_numpy(0, sort_by_id=True), b.species_numpy(0, sort_by_id=True)
    assert np.array_equal(A["id"], B["id"])
    for k in ("x", "y", "z", "ux", "uy", "uz"):
        scale = ref.dx[0] if k in "xyz" else workloads.C
        assert np.max(np.abs(A[k] - B[k])) / scale <= 1e-11, k


@pytest.mark.parametrize("mode", [abi.PIC_DEPOSIT_RUNS, abi.PIC_DEPOSIT_CELLS])
def test_host_engine_keeps_gauss_law(HostSimulation, mode):
    """Gauss's law through the C++ driver's whole step (tests/helpers.py: gauss_residual): 16^3 x 8 ppc, order 3, hot
    enough to cross cell faces every step, 12 steps with a cell sort every 4, in the default deposition and with
    PIC_DEPOSIT_CELLS.  max|G^n - G^0| / max|rho^0/ep0| <= 1e-12 after steps 1, 4, 5 and 12; the particle count holds."""
    from helpers import gauss_drift, simulation_gauss
    from host_harness import harness
    wl = workloads.uniform_plasma_3d(n=16, ppc=(2, 2, 2), u_th=0.1, lx=2.5e-6)
    s = wl["species"][0]
    hl = harness.host_library()
    hl.pic_set_deposit_mode(mode)
    try:
        sim = HostSimulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        assert sim.native
        G0, rho0 = simulation_gauss(sim)
        done = 0
        for step in (1, 4, 5, 12):
            sim.Evolve(step - done, synchronize_last=False)
            done = step
            G, _ = simulation_gauss(sim)
            assert gauss_drift(G, G0, rho0) <= 1e-12, step
            assert sim.species[0].np == len(s["x"])
    finally:
        hl.pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS)
