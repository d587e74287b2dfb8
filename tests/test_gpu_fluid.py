"""GPU tests of the cold relativistic fluid species: each kernel against the numpy restatement (tests/fluid_oracle.py),
and the Langmuir fluid deck through the Python sequencer against WarpX's regression checksums and the oracle loop."""
import json
import os

import numpy as np
import pytest

import fluid_cases
import fluid_oracle as fo
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind,box_lo,box_hi", [("langmuir", (0, 0, 0), (31, 31, 31)),
                                                ("vacuum", (0, 0, 0), (31, 31, 31)),
                                                ("drift", (0, 0, 0), (31, 31, 31)),
                                                ("vacuum", (32, 16, 8), (63, 39, 35))])
def test_fluid_stages_match_oracle(cuda, kind, box_lo, box_hi):
    from warpx_b200.lib import lib
    err, counters = fluid_cases.check_stages(lib(), cuda, cuda.device("cuda", 0), kind, (64, 64, 64), box_lo, box_hi,
                                             1e-13)
    print(kind, box_lo, err, counters)
    if kind == "vacuum":
        assert counters["zero_edges"] > 0


def test_fluid_advection_matches_the_reference_headers(cuda):
    from warpx_b200.lib import lib
    print(fluid_cases.check_reference_fixture(lib(), cuda, cuda.device("cuda", 0)))


def _cell_centre_checksum(d, a):
    v = a[d.valid_slices()]
    for ax, dd in ((2, 0), (1, 1), (0, 2)):
        if d.stag[dd]:
            v = 0.5 * (np.take(v, range(v.shape[ax] - 1), axis=ax) + np.take(v, range(1, v.shape[ax]), axis=ax))
    return float(np.sum(np.abs(v)))


@pytest.fixture(scope="module")
def deck_oracle(orc):
    wl = workloads.langmuir_fluid_3d()
    run = fo.FluidRun(orc, wl["n_cell"], wl["prob_lo"], wl["prob_hi"])
    for f in wl["fluids"]:
        run.add_fluid(f["q"], f["m"], f["density"], f["momentum"])
    run.evolve(wl["max_step"])
    return run


def _deck(native):
    from warpx_b200.engine import Simulation
    wl = workloads.langmuir_fluid_3d()
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, native_driver=native)
    for f in wl["fluids"]:
        sim.add_fluid_species(f["name"], f["q"], f["m"], f["density"], f["momentum"])
    sim.Evolve(wl["max_step"])
    return sim


@pytest.mark.parametrize("native", [True, False])
def test_langmuir_fluid_deck_golden_checksums_and_oracle(cuda, deck_oracle, native):
    """inputs_test_3d_langmuir_fluid, 40 steps, on the device through the C++ driver (native) or the Python sequencer:
    WarpX's checksums at rtol 1e-9, and the oracle loop's fields (1e-9 of each vector's scale), field energy (1e-10)
    and fluid state (1e-9 of each component's scale)."""
    with open(os.path.join(ROOT, "tests", "golden", "warpx_fluid_checksums.json")) as f:
        g = json.load(f)["test_3d_langmuir_fluid"]["lev=0"]
    sim, run = _deck(native), deck_oracle
    for c, name in enumerate(abi.COMP_NAMES):
        d, a = sim.field_numpy(c)
        v = _cell_centre_checksum(d, a)
        assert abs(v - g[name]) <= 1e-9 * abs(g[name]), (name, v, g[name])
    rd, rho = sim.rho_numpy()
    v = _cell_centre_checksum(rd, rho)
    assert abs(v - g["rho"]) <= 1e-9 * g["rho"], (v, g["rho"])
    for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):
        scale = max(np.max(np.abs(run.fabs[c].a)) for c in group)
        for c in group:
            d, a = sim.field_numpy(c)
            V = d.valid_slices()
            assert np.max(np.abs(a[V] - run.fabs[c].a[V])) <= 1e-9 * scale, c
    e, eo = sim.field_energy(), run.field_energy()
    assert abs(e[0] - eo[0]) <= 1e-10 * eo[0] and abs(e[1] - eo[1]) <= 1e-10 * eo[1], (e, eo)
    for i in range(2):
        d, st = sim.fluid_numpy(i)
        V = d.valid_slices()
        for c, name in enumerate(("N", "NUx", "NUy", "NUz")):
            ref = run.fluids[i]["state"][c][V]
            assert np.max(np.abs(st[name][V] - ref)) <= 1e-9 * np.max(np.abs(ref)), (i, name)


def test_langmuir_fluid_deck_driver_matches_sequencer(cuda):
    """The C++ driver and the Python sequencer launch the same kernels in the same order: identical bits."""
    a, b = _deck(True), _deck(False)
    for c in range(9):
        assert np.array_equal(a.field_numpy(c)[1], b.field_numpy(c)[1]), c
    for i in range(2):
        V = a.fluid_numpy(i)[0].valid_slices()
        for name in ("N", "NUx", "NUy", "NUz"):
            assert np.array_equal(a.fluid_numpy(i)[1][name][V], b.fluid_numpy(i)[1][name][V]), (i, name)


def test_fluid_refusals_on_the_device(cuda):
    from warpx_b200.engine import Simulation
    wl = workloads.langmuir_fluid_3d(n=16)
    f = wl["fluids"][0]
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, gamma_boost=2.0)
    with pytest.raises(NotImplementedError, match="boost"):
        sim.add_fluid_species(f["name"], f["q"], f["m"], f["density"], f["momentum"])
    assert sim.fluids == []
