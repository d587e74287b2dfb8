"""CPU tests (-m "not gpu"): every particle set of tests/particle_sets.py contains what its parity cases are meant to
reach.  The product library has no event counters, so the kernels' classifications are restated in numpy
(particle_sets.quiet_kernel_events, cells_kernel_queue, gather_tile_events) and applied to the sets; a seed or size
change that removes a feature fails here instead of silently weakening the GPU cases."""
import numpy as np
import pytest

import particle_sets as ps

NG_J = (5, 5, 5)        # order 3 + 2
NG_EB = (4, 4, 4)


def cell_counts(s):
    return np.diff(s.cell_start)


@pytest.mark.parametrize("name", ps.SETS)
def test_set_stays_inside_the_preconditions(name):
    s = ps.get(name)
    assert set(s.p) == set(ps.NAMES) and all(len(v) == s.np for v in s.p.values())
    assert s.cell_start[0] == 0 and s.cell_start[-1] == s.np and np.all(np.diff(s.cell_start) >= 0)
    for d, k in enumerate(("x", "y", "z")):
        # inside the box, on its upper face, or one ulp below its lower face
        assert np.all(s.p[k] >= np.nextafter(s.origin[d], -np.inf)) and np.all(s.p[k] <= s.prob_hi[d]), k
    new, old = ps.grid_positions(s, NG_J)
    for d in range(3):
        assert np.max(np.abs(new[d] - old[d])) < 1.0
    # weights: log-uniform over 1e-3 .. 1e3 of the lattice weight
    w_lat = ps.DENSITY * np.prod(s.dx) / 8
    assert np.all(s.p["w"] >= 1e-3 * w_lat) and np.all(s.p["w"] <= 1e3 * w_lat)
    if s.np > 1000:
        assert np.min(s.p["w"]) < 1e-2 * w_lat and np.max(s.p["w"]) > 1e2 * w_lat


def test_steady_has_movers_lone_strays_and_jumps():
    s = ps.get("steady")
    for nox in (1, 2, 3):
        ev = ps.quiet_kernel_events(s, nox, NG_J)
        assert ev["movers"] > 0 and ev["lones"] > 0 and ev["jumps"] > 0, (nox, ev)
    # the gather's stray lists are used, without overflowing
    g = ps.gather_tile_events(s, NG_EB)
    assert g["leavers"] > 0 and 0 < g["isolated"].max() <= 1022 and g["leavers"] <= s.np // 8 + 1024


def test_poisson_has_the_chosen_cell_counts():
    s = ps.get("poisson")
    c = cell_counts(s)
    for n in (0, 1, 31, 32, 33, 600):
        assert np.sum(c == n) >= 1, n
    assert c.max() > 512                    # longer than one warp's span of 16 chunks
    assert ps.quiet_kernel_events(s, 3, NG_J)["movers"] > 0


def test_faces_has_particles_on_and_below_every_kind_of_face():
    s = ps.get("faces")
    f = ps.on_faces(s)
    for k in ("x", "y", "z"):
        assert f[k]["on"] > 100 and f[k]["below"] > 100 and f[k]["prob_hi"] > 10 and f[k]["supercell"] > 10, (k, f[k])
    assert np.sum(s.p["ux"] == 0.0) > 100       # at rest on a face: old position == new position


def test_crowded_movers_overflow_the_cells_queue():
    s = ps.get("crowded_movers")
    for nox in (1, 3):
        q = ps.cells_kernel_queue(s, nox, NG_J)
        t = ps.CROWDED_SUPERCELL
        nt = [(s.n[d] + ps.TILE - 1) // ps.TILE for d in range(3)]
        crowded = q["queued"][t[0] + nt[0] * (t[1] + nt[1] * t[2])]
        assert crowded > 768, (nox, crowded)     # QCAP of CELLS / CELLS2 (512 for CELLS3): the rest goes to the list
        assert q["listed"] > 0                   # sub-particles outside the supercell: deposit_general_kernel
    assert ps.quiet_kernel_events(s, 3, NG_J)["movers"] >= 240


def test_scrambled_rows_overflow_both_gather_lists():
    s = ps.get("scrambled_rows")
    g = ps.gather_tile_events(s, NG_EB)
    assert g["isolated"].max() > 1022            # GT_LOCAL_STRAYS: the rest is gathered inline from shared memory
    assert g["leavers"] > s.np // 8 + 1024       # the global stray list's capacity: the rest is gathered inline


@pytest.mark.parametrize("count", [1, 31, 33])
def test_sparse_sets_occupy_one_cell(count):
    s = ps.get("sparse%d" % count)
    c = cell_counts(s)
    assert s.np == count and np.sum(c > 0) == 1
    occupied = np.flatnonzero(c.reshape(-1, ps.TILE ** 3).sum(axis=1))
    assert len(occupied) == 1


def test_offset_box_keeps_the_bins_and_the_grid_positions():
    s, t = ps.get("poisson"), ps.get("poisson+offset")
    assert t.box_lo == ps.OFFSET_BOX_LO and all(v < 0 for v in t.prob_lo)
    assert np.array_equal(s.cell_start, t.cell_start)
    b = ps.bin_of(t.p["x"], t.p["y"], t.p["z"], t.origin, t.dx, t.n)
    assert np.all(np.diff(b) >= 0)
    a, c = ps.grid_positions(s, NG_J)[0], ps.grid_positions(t, NG_J)[0]
    for d in range(3):
        assert np.max(np.abs(a[d] - c[d])) < 1e-9


def test_reach_covers_the_oracle_deposition(orc):
    """The nodes a deposition changes lie inside particle_sets.reach (what the GPU cases require to stay bit-exact)."""
    import ctypes as C
    from warpx_b200 import abi
    s = ps.get("sparse33")
    for nox in (1, 4):
        ng = (nox + 2,) * 3
        xyzmin, lo = s.corner(ng)
        P = orc.HostParticles(**s.arrays())
        J = [orc.HostFab(s.box_lo, s.box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
        for f in J:
            f.a[...] = 1.0
        assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(s.dinv),
                                               abi.dbl3(xyzmin), abi.int3(lo), s.q, s.dt, -0.5 * s.dt, nox) == 0
        for f in J:
            r = ps.reach(s, f.a.shape, ng, nox)
            assert np.all(f.a[~r] == 1.0) and np.any(~r)
