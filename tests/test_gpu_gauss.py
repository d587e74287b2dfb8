"""GPU tests (-m gpu): Gauss's law through the whole step, at the benchmark's size and steady state, in every kernel mode.

Esirkepov deposition makes rho(x^{n+1}) - rho(x^n) = -dt div J hold to round-off, and EvolveE's downward differences
make div E^{n+1} - div E^n = -(dt/ep0) div J, for Yee and CKC alike.  So G = div E - rho/ep0 (tests/helpers.py:
gauss_residual) is the same at every step on every node of a periodic box.  Every check reports
max|G^n - G^0| / max|rho^0/ep0| and must stay <= 1e-11.  One particle missing from one deposition moves it by about
4e-2, so G breaks on a particle that the sort, the periodic wrap or the deposit drops or duplicates, on a J reduction
lost or applied twice, on a wrong or doubled J guard-cell sum, and on an EvolveE that reads a stale B plane.

What G cannot see: the gather, the momentum and position push, and EvolveB (continuity holds whatever velocity a
particle gets, and div curl B = 0 for any B).  div B = 0 is checked beside G for Yee; the gather and the push stay
covered by the oracle comparisons of test_gpu_parity.py and test_gpu_particle_sets.py.  rho comes from
Simulation.rho_numpy (charge.cu), and test_device_rho_matches_oracle holds that to the oracle's charge deposit.

Each run also keeps, at every checkpoint, its particle count, the weights by id bit for bit (so sum w too), and ids
that are a permutation of 0..np-1.  Checkpoints: steps 1, 4 (the step that sorts), 5 (the first step on fresh bins),
60, 61, 64 and 80 (the benchmark times from step 60 on)."""
import functools
import time

import pytest

from helpers import div_b_ratio, gauss_drift, oracle_rho, simulation_gauss
from test_gpu_particle_sets import DEPOSIT_MODES, GLOBAL
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu

TOL = 1e-11
CHECKPOINTS = (1, 4, 5, 60, 61, 64, 80)
ORDER_CHECKPOINTS = (1, 4, 5, 40)
BENCH_N, MODE_N, ORDER_N = 256, 128, 64
FULL_SIZE_FREE_BYTES = 40e9        # 256^3 x 8 ppc needs about 25 GB of device memory with rho and the checks


def bench_n(t):
    """The benchmark's 256^3 where the device has room, else 128^3 (as test_full_size_properties)."""
    free, _ = t.cuda.mem_get_info()
    return BENCH_N if free > FULL_SIZE_FREE_BYTES else MODE_N


@functools.lru_cache(maxsize=2)
def bench_workload(n):
    """The species bench.py builds (8 ppc on the lattice, u_th = 0.01, the benchmark's cell size) at n^3."""
    return workloads.uniform_plasma_3d(n=n, ppc=(2, 2, 2), u_th=0.01, lx=40.0e-6 * n / 256.0)


def make_sim(wl, nox=3, **kw):
    from warpx_b200.engine import Simulation
    kw.setdefault("sort_interval", 4)
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox, **kw)
    s = wl["species"][0]
    sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    return sim


def run_gauss(sim, checkpoints, label, check_div_b=True):
    """Evolve to every checkpoint (synchronize_last=False) and check G, div B and the particles there.  Prints and
    returns the largest max|G^n - G^0| / max|rho^0/ep0| of the run."""
    t = sim.torch
    sp = sim.species[0]
    np0 = sp.np
    ids0, order = t.sort(sp.id_array())
    assert t.equal(ids0, t.arange(np0, dtype=ids0.dtype, device=ids0.device))
    w0 = sp.array("w")[order].clone()
    sw0 = float(w0.sum())
    G0, rho0 = simulation_gauss(sim)
    worst, done, t_run = 0.0, 0, time.perf_counter()
    for step in checkpoints:
        sim.Evolve(step - done, synchronize_last=False)
        done = step
        G, _ = simulation_gauss(sim)
        r = gauss_drift(G, G0, rho0)
        worst = max(worst, r)
        assert r <= TOL, "%s: Gauss's law broken after step %d: %.3e" % (label, step, r)
        if check_div_b:
            B = [sim.data[c][sim.fab[c].valid_slices()] for c in range(3, 6)]
            assert div_b_ratio(B, sim.dx, sim.n_cell) <= 1e-9, (label, step)
        assert sp.np == np0, (label, step)
        ids, order = t.sort(sp.id_array())
        assert t.equal(ids, ids0), "%s: ids after step %d are not a permutation of 0..np-1" % (label, step)
        w = sp.array("w")[order]
        assert t.equal(w, w0) and float(w.sum()) == sw0, (label, step)
    print("GAUSS %s: %d^3, %d steps, max|G^n - G^0| / max|rho^0/ep0| = %.2e (%.1f s with the checks)"
          % (label, sim.n_cell[0], done, worst, time.perf_counter() - t_run))
    return worst


# ---------------------------------------------------------------------------------------------------------------------
def test_gauss_at_benchmark_state(cuda):
    """The benchmark's workload (256^3 x 8 ppc, order 3, Yee, Boris, a cell sort every 4 steps) in the default modes,
    through the spin-up the benchmark runs untimed and into its timed window."""
    n = bench_n(cuda)
    sim = make_sim(bench_workload(n))
    try:
        run_gauss(sim, CHECKPOINTS, "benchmark")
    finally:
        sim.close()
    if n == BENCH_N:
        bench_workload.cache_clear()


DEFAULT = ("default", None)
MODE_CASES = ([DEFAULT] + [("deposit", m) for m in DEPOSIT_MODES if m != abi.PIC_DEPOSIT_RUNS]
              + [("fdtd", 0), ("fdtd", 3), ("gather", abi.PIC_GATHER_PAIRS)])


@pytest.mark.parametrize("kind,mode", MODE_CASES)
def test_gauss_in_every_mode(cuda, kind, mode):
    """128^3 at the benchmark's cell size, the benchmark's checkpoints, one mode switched at a time.  default:
    PIC_DEPOSIT_RUNS, pic_set_fdtd_mode(1) (EvolveB staged) and the tile gather.  deposit: every entry of
    DEPOSIT_MODES (global = use_bins=False: the C++ driver without bins).  fdtd 0: plain loads; fdtd 3: EvolveE staged as well.
    gather: pair mode 1."""
    from warpx_b200.lib import lib as piclib
    L = piclib()
    kw = {}
    if kind == "deposit" and mode == GLOBAL:
        kw["use_bins"] = False
    elif kind == "deposit":
        L.pic_set_deposit_mode(mode)
    elif kind == "fdtd":
        L.pic_set_fdtd_mode(mode)
    elif kind == "gather":
        L.pic_set_gather_mode(mode)
    try:
        sim = make_sim(bench_workload(MODE_N), **kw)
        run_gauss(sim, CHECKPOINTS, "%s %s" % (kind, mode))
        sim.close()
    finally:
        L.pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS)
        L.pic_set_fdtd_mode(1)
        L.pic_set_gather_mode(abi.PIC_GATHER_TILE)


ORDER_CASES = [(1, abi.SOLVER_YEE, abi.PUSHER_BORIS, False), (2, abi.SOLVER_YEE, abi.PUSHER_BORIS, False),
               (4, abi.SOLVER_YEE, abi.PUSHER_BORIS, False), (3, abi.SOLVER_CKC, abi.PUSHER_VAY, False),
               (3, abi.SOLVER_YEE, abi.PUSHER_BORIS, True)]


@pytest.mark.parametrize("nox,solver,pusher,use_filter", ORDER_CASES)
def test_gauss_orders_solvers_filter(orc, cuda, nox, solver, pusher, use_filter):
    """64^3 for 40 steps: orders 1, 2 and 4, CKC with Vay, and the bilinear filter (rho filtered like J).  At the end
    the device rho also matches the oracle's charge deposit of the same particles."""
    wl = bench_workload(ORDER_N)
    sim = make_sim(wl, nox=nox, solver=solver, pusher=pusher, use_filter=use_filter)
    run_gauss(sim, ORDER_CHECKPOINTS, "order %d solver %d filter %d" % (nox, solver, use_filter),
              check_div_b=solver == abi.SOLVER_YEE)        # CKC's EvolveB smooths transversely
    check_rho_against_oracle(orc, sim, wl, nox, use_filter)
    sim.close()


def check_rho_against_oracle(orc, sim, wl, nox, use_filter):
    _, rho = simulation_gauss(sim)
    want = oracle_rho(orc, wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox, sim.species_numpy(0),
                      wl["species"][0]["q"], use_filter, sim.filter_npass)
    err = abs(rho.cpu().numpy() - want).max() / abs(want).max()
    print("GAUSS rho vs oracle, order %d filter %d: %.2e" % (nox, use_filter, err))
    assert err <= 1e-13, err


def test_device_rho_matches_oracle(orc, cuda):
    """The rho every check here rests on (pic_deposit_charge + SumBoundary on the device) against orc_deposit_charge of
    the same particles, at 128^3 after 5 steps (one sort, movers on fresh bins): 1e-13 of max|rho|."""
    wl = bench_workload(MODE_N)
    sim = make_sim(wl)
    sim.Evolve(5, synchronize_last=False)
    check_rho_against_oracle(orc, sim, wl, 3, False)
    sim.close()


def test_gauss_check_sees_one_edited_weight(cuda):
    """Negative control on the device: between two Evolve chunks one particle's weight grows by half in the species
    array the step driver works on.  Three steps later G is off by more than 1e-4 of max|rho^0/ep0| within the
    particle's stencil, and within the bar everywhere else."""
    t = cuda
    wl = bench_workload(ORDER_N)
    sim = make_sim(wl)
    sp = sim.species[0]
    G0, rho0 = simulation_gauss(sim)
    sim.Evolve(5, synchronize_last=False)
    target = 12345
    hit = (sp.id_array() == target).nonzero().flatten()
    assert hit.numel() == 1
    sp.array("w")[hit] *= 1.5
    sim.Evolve(3, synchronize_last=False)
    G, _ = simulation_gauss(sim)
    err = (G - G0).abs() / (float(rho0.abs().max()) / workloads.EP0)
    i = int((sp.id_array() == target).nonzero().flatten()[0])
    near = None
    for ax, k in enumerate("xyz"):
        n = sim.n_cell[ax]
        at = (float(sp.array(k)[i]) - sim.prob_lo[ax]) / sim.dx[ax]
        d = (t.arange(n, dtype=t.float64, device=G.device) - at).abs() % n
        d = t.minimum(d, n - d) <= 3
        shape = [1, 1, 1]
        shape[2 - ax] = n
        d = d.reshape(shape)
        near = d if near is None else near & d
    near = near.expand_as(err)
    assert float(err[near].max()) > 1e-4
    assert float(err[~near].max()) <= TOL
    sim.close()
