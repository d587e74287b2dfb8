"""GPU tests (-m gpu): a cell sort inside pic_engine_evolve stops at the permutation and the next gather + push moves
the particles.  Stage level through the C ABI on the seeded sets of tests/particle_sets.py (bit for bit by particle
id), then through Simulation: a run that defers against one that never does (Evolve(1) applies every sort at once),
and the gathers that must see the particles moved first (the pair kernels, order 4)."""
import numpy as np
import pytest

import deferred_sort_cases as cases
import particle_sets as ps
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu


@pytest.fixture()
def be(cuda):
    from warpx_b200.lib import lib
    return cases.Backend(cuda, lib(), "cuda")


@pytest.mark.parametrize("name", ps.SETS)
def test_index_then_apply_is_the_sort(be, name):
    cases.check_index_apply_is_the_sort(be, name)


@pytest.mark.parametrize("stale", [False, True], ids=["fresh_sort", "stale_bins"])
@pytest.mark.parametrize("pusher", [abi.PUSHER_BORIS, abi.PUSHER_VAY])
@pytest.mark.parametrize("nox", [1, 2, 3])
@pytest.mark.parametrize("stag", ["yee", "nodal"])
@pytest.mark.parametrize("name", ["steady", "poisson", "faces", "crowded_movers", "scrambled_rows"])
def test_permuting_gather_push_is_apply_then_push(be, orc, name, stag, nox, pusher, stale):
    cases.check_permuting_push_is_apply_then_push(be, orc, name, nox, 1, pusher, stag, stale_bins=stale)


def test_permuting_gather_push_refuses_what_it_does_not_serve(be, orc):
    be.L.pic_set_gather_mode(abi.PIC_GATHER_PAIRS)
    try:
        with pytest.raises(AssertionError, match="default gather kernel"):
            cases.check_permuting_push_is_apply_then_push(be, orc, "steady", 3, 1, abi.PUSHER_BORIS, "yee")
    finally:
        be.L.pic_set_gather_mode(abi.PIC_GATHER_TILE)


def _plasma(**kw):
    from warpx_b200.engine import Simulation
    wl = workloads.uniform_plasma_3d(n=16, ppc=(2, 2, 2), u_th=0.05, lx=2.5e-6, perturbation=0.01)
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=kw.pop("nox", 3), sort_interval=4, **kw)
    s = wl["species"][0]
    sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    return sim


def _state(sim):
    out = sim.species_numpy(0, sort_by_id=True)
    for c in range(9):
        d, a = sim.field_numpy(c)
        out[abi.COMP_NAMES[c]] = a[d.valid_slices()].copy()
    return out


def _cells_sorted(sim):
    p = sim.species_numpy(0)
    dx = sim.dx
    b = ps.bin_of(p["x"], p["y"], p["z"], sim.prob_lo, dx, sim.n_cell)
    return bool(np.all(np.diff(b) >= 0))


def _distance(a, b):
    return {k: float(np.max(np.abs(a[k] - b[k])) / max(np.max(np.abs(a[k])), 1e-300)) for k in a if k != "id"}


def test_evolve_that_defers_matches_evolve_that_never_does():
    """Evolve(8) carries the sort of step 4 into the push of step 5; eight Evolve(1) calls apply every sort at once.
    Each particle's arithmetic is the same; J is summed in another order, so the two runs agree as closely as two
    runs of one kind do (with a floor for the reordered sums)."""
    def run(chunks):
        sim = _plasma()
        sorted_after = []
        for n in chunks:
            sim.Evolve(n, synchronize_last=False)
            if sim.istep % 4 == 0:
                sorted_after.append(_cells_sorted(sim))          # the buffer the engine names holds the moved particles
        st = _state(sim)
        sim.close()
        return st, sorted_after
    deferred, seen_a = run([8])
    again, _ = run([8])
    stepwise, seen_b = run([1] * 8)
    assert seen_a == [True] and seen_b == [True, True]
    assert np.array_equal(deferred["id"], stepwise["id"]) and np.array_equal(deferred["w"], stepwise["w"])
    noise, diff = _distance(deferred, again), _distance(deferred, stepwise)
    for k in diff:
        assert diff[k] <= 10 * noise[k] + 1e-9, (k, diff[k], noise[k])


@pytest.mark.parametrize("case", ["pair_gather", "order4"])
def test_paths_that_need_the_particles_moved_first(case):
    """The pair kernels and order 4 do not permute: the pending sort is applied before them, and the run equals the
    one that never defers."""
    from warpx_b200.lib import lib
    def run(chunks):
        sim = _plasma(nox=4 if case == "order4" else 3)
        if case == "pair_gather":
            lib().pic_set_gather_mode(abi.PIC_GATHER_PAIRS)
        try:
            for n in chunks:
                sim.Evolve(n, synchronize_last=False)
        finally:
            lib().pic_set_gather_mode(abi.PIC_GATHER_TILE)
        st = _state(sim)
        sim.close()
        return st
    a, b = run([6]), run([1] * 6)
    assert np.array_equal(a["id"], b["id"])
    for k, v in _distance(a, b).items():
        assert v <= 1e-9, (k, v)
