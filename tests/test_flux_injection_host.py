"""CPU tests of the flux injection: the product's kernel source (csrc/flux_injection.cu and the step driver csrc/engine.cu,
through the SIMT host build of tests/host_harness) against the numpy restatement of tests/flux_oracle.py, bit for bit:
planes on each axis in both directions, fractional particles per cell, both Gaussian-flux branches, bounds that cut the
plane, boxes that do and do not own it, the injection window, and one step of the driver with a plane on a domain face
under periodic and absorbing particle boundaries; plus the refusals."""
import ctypes as C

import numpy as np
import pytest

import flux_oracle as fo
from warpx_b200 import abi

GEOM = ((6, 5, 4), (-1.0, 0.0, 2.0), (2.0, 2.5, 4.0))
FULL = ((0, 0, 0), (5, 4, 3))
NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")


@pytest.fixture(scope="module")
def host():
    import torch
    from host_harness import harness
    return harness.host_library(), torch


def call(L, torch, inj, geom, box, step, t, dt, first_id, index, np0=3, capacity=4000):
    """pic_add_flux_particles on the host build, behind np0 particles: (appended particles sorted by id, count, ids)"""
    g = abi.make_geom(*geom)
    buf = torch.zeros((7, capacity), dtype=torch.float64)
    ids = torch.full((capacity,), 7, dtype=torch.int64)
    soa = abi.pic_soa()
    for k, name in enumerate(NAMES):
        setattr(soa, name, buf[k].data_ptr())
    soa.idcpu, soa.np = ids.data_ptr(), np0
    nbytes = L.pic_flux_workspace_bytes(C.byref(inj), C.byref(g))
    assert nbytes > 0
    work = torch.zeros(nbytes, dtype=torch.uint8)
    used = C.c_uint64(0)
    n = L.pic_add_flux_particles(C.byref(inj), index, C.byref(g), abi.int3(box[0]), abi.int3(box[1]), step, t, dt,
                                 C.byref(soa), capacity, first_id, C.byref(used), work.data_ptr(), nbytes, None)
    assert n >= 0, L.pic_last_error().decode()
    assert np.all(ids[:np0].numpy() == 7) and np.all(buf[:, :np0].numpy() == 0)
    got = {name: buf[k, np0:np0 + n].numpy().copy() for k, name in enumerate(NAMES)}
    got["id"] = ids[np0:np0 + n].numpy().copy()
    return fo.sort_by_id(got), n, used.value


def assert_same(got, want):
    assert len(got["id"]) == len(want["id"])
    for k in want:
        assert np.array_equal(got[k], want[k]), k


CASES = {
    # name: (injector keywords, box)
    "x_plus_interior": (dict(num_particles_per_cell=3.0, surface_flux_pos=0.3, flux_normal_axis="x", flux_direction=1,
                             u_m=(0.05, 0.0, 0.0), u_th=(0.1, 0.1, 0.1)), FULL),
    "y_minus_face_of_a_cell": (dict(num_particles_per_cell=2.5, surface_flux_pos=1.5, flux_normal_axis="y",
                                    flux_direction=-1, u_m=(0.0, 0.2, 0.0), u_th=(0.1, 0.05, 0.1), flux=3.0), FULL),
    "z_plus_um_zero_bounds": (dict(num_particles_per_cell=4.0, surface_flux_pos=2.0, flux_normal_axis="z",
                                   flux_direction=1, u_th=(0.1, 0.2, 0.1), bound_lo=(-0.3, 0.7, -np.inf),
                                   bound_hi=(1.2, np.inf, np.inf)), FULL),
    "z_minus_negative_um": (dict(num_particles_per_cell=1.5, surface_flux_pos=3.2, flux_normal_axis="z",
                                 flux_direction=-1, u_m=(0.01, 0.0, -0.07), u_th=(0.0, 0.3, 0.1)), FULL),
    "x_minus_u_th_zero": (dict(num_particles_per_cell=2.0, surface_flux_pos=2.0, flux_normal_axis="x", flux_direction=-1,
                               u_m=(0.3, 0.0, 0.0), u_th=(0.0, 0.1, 0.1)), FULL),
    "bounds_behind_the_plane": (dict(num_particles_per_cell=3.0, surface_flux_pos=0.0, flux_normal_axis="x",
                                     flux_direction=1, u_th=(0.1, 0.1, 0.1), bound_lo=(0.2, -np.inf, -np.inf)), FULL),
    "sub_box_owns": (dict(num_particles_per_cell=2.0, surface_flux_pos=1.0, flux_normal_axis="y", flux_direction=1,
                          u_m=(0.0, 0.1, 0.0), u_th=(0.1, 0.1, 0.1)), ((3, 2, 2), (5, 3, 3))),
    "sub_box_lower_face_minus": (dict(num_particles_per_cell=2.0, surface_flux_pos=1.0, flux_normal_axis="y",
                                      flux_direction=-1, u_th=(0.1, 0.1, 0.1)), ((0, 0, 0), (2, 1, 1))),
    "sub_box_does_not_own": (dict(num_particles_per_cell=2.0, surface_flux_pos=1.0, flux_normal_axis="y",
                                  flux_direction=1, u_th=(0.1, 0.1, 0.1)), ((0, 0, 0), (5, 1, 3))),
    "no_flux": (dict(num_particles_per_cell=2.0, surface_flux_pos=1.0, flux_normal_axis="y", flux_direction=1,
                     u_th=(0.1, 0.1, 0.1), flux=0.0), FULL),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_call_matches_oracle(host, name):
    L, torch = host
    kw, box = CASES[name]
    inj = abi.make_flux_injector(seed=11, **kw)
    step, dt, first_id, index = 5, 2e-9, 1000, 2
    got, n, used = call(L, torch, inj, GEOM, box, step, 6 * dt, dt, first_id, index)
    want, want_used = fo.inject(fo.as_dict(inj), GEOM, box[0], box[1], step, 6 * dt, dt, first_id, index)
    assert used == want_used
    assert_same(got, fo.sort_by_id(want))
    if name in ("sub_box_does_not_own", "no_flux", "bounds_behind_the_plane"):
        assert n == 0
    else:
        assert n > 10
    if name == "bounds_behind_the_plane":
        assert n == 0 and used > 0          # cells overlap the bounds, every particle lies outside them


def test_host_streams_depend_on_step_and_index(host):
    L, torch = host
    inj = abi.make_flux_injector(2.0, 0.3, "x", 1, u_th=(0.1, 0.1, 0.1), seed=3)
    a, _, _ = call(L, torch, inj, GEOM, FULL, 1, 1.0, 1e-9, 0, 0)
    b, _, _ = call(L, torch, inj, GEOM, FULL, 2, 1.0, 1e-9, 0, 0)
    c, _, _ = call(L, torch, inj, GEOM, FULL, 1, 1.0, 1e-9, 0, 1)
    assert not np.array_equal(a["uy"][:5], b["uy"][:5]) and not np.array_equal(a["uy"][:5], c["uy"][:5])


@pytest.mark.parametrize("t,tmin,tmax,injects", [(1.0, -1.0, -1.0, True), (1.0, 1.0, -1.0, True), (1.0, 1.5, -1.0, False),
                                                 (1.0, -1.0, 1.0, False), (1.0, 0.5, 1.5, True)])
def test_host_injection_window(host, t, tmin, tmax, injects):
    L, torch = host
    inj = abi.make_flux_injector(2.0, 0.3, "x", 1, u_th=(0.1, 0.1, 0.1), flux_tmin=tmin, flux_tmax=tmax)
    got, n, used = call(L, torch, inj, GEOM, FULL, 0, t, 1e-9, 0, 0)
    assert (n > 0) == injects and (used == 5 * 4 * 3 if injects else used == 0)


def test_host_capacity_and_refusals(host):
    L, torch = host
    g = abi.make_geom(*GEOM)
    inj = abi.make_flux_injector(2.0, 0.3, "x", 1, u_th=(0.1, 0.1, 0.1))
    with pytest.raises(AssertionError):
        call(L, torch, inj, GEOM, FULL, 0, 1.0, 1e-9, 0, 0, np0=3, capacity=20)
    assert "capacity" in L.pic_last_error().decode()
    for bad in (dict(normal_axis=3), dict(direction=0), dict(num_ppc=0.0), dict(num_ppc=-1.0)):
        b = abi.make_flux_injector(2.0, 0.3, "x", 1, u_th=(0.1, 0.1, 0.1))
        for k, v in bad.items():
            setattr(b, k, v)
        assert L.pic_flux_workspace_bytes(C.byref(b), C.byref(g)) == -1
    b = abi.make_flux_injector(2.0, 0.3, "x", 1, u_th=(-0.1, 0.1, 0.1))
    assert L.pic_flux_workspace_bytes(C.byref(b), C.byref(g)) == -1


def wrap1(v, lo, hi):
    """amrex enforcePeriodic as particles_misc.cu's wrap1"""
    v = v.copy()
    L = hi - lo
    up, dn = v > hi, v < lo
    while np.any(v > hi):
        v[v > hi] -= L
    while np.any(v < lo):
        v[v < lo] += L
    v[up & (v < lo)] = lo
    v[dn & (v > hi)] = hi
    return v


@pytest.mark.parametrize("particles", ["periodic", "absorbing"])
def test_host_driver_step_on_a_domain_face(host, particles):
    """a z plane on the domain's lower face; transverse momenta carry particles across the x and y faces within t_fract:
    the step wraps them (periodic) or removes them (absorbing along x), as it treats pushed particles"""
    from host_harness import harness
    Sim = harness.host_simulation_class()
    n_cell, plo, phi = (8, 6, 4), (0.0, 0.0, 0.0), (4.0, 3.0, 2.0)
    bnd = None
    if particles == "absorbing":
        bnd = abi.make_boundaries(("pec", "periodic", "periodic"), ("pec", "periodic", "periodic"))
    dt = 6e-9
    sim = Sim(n_cell, plo, phi, nox=1, solver=abi.SOLVER_NONE, dt=dt, boundaries=bnd)
    sim.add_empty_species("e", 4000, q=-1.602176634e-19, m=9.1093837015e-31)
    inj = abi.make_flux_injector(6.0, 0.0, "z", 1, u_m=(0.0, 0.0, 0.1), u_th=(0.5, 0.5, 0.1), seed=9)
    assert sim.add_flux_injection("e", inj) == 0
    sim.Evolve(1)
    got = sim.species_numpy(0, sort_by_id=True)
    want, used = fo.inject(fo.as_dict(inj), (n_cell, plo, phi), (0, 0, 0), (7, 5, 3), 0, dt, dt, 0, 0)
    assert sim.species_next_id(0) == used == 8 * 6 * 7
    crossed = (want["x"] < plo[0]) | (want["x"] > phi[0])
    assert crossed.sum() > 10
    if particles == "periodic":
        want["x"] = wrap1(want["x"], plo[0], phi[0])
    else:
        want = {k: v[~crossed] for k, v in want.items()}
    want["y"] = wrap1(want["y"], plo[1], phi[1])
    assert_same(got, fo.sort_by_id(want))


def test_host_driver_refusals(host):
    from host_harness import harness
    Sim = harness.host_simulation_class()
    sim = Sim((4, 4, 4), (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), nox=1, solver=abi.SOLVER_NONE, dt=1e-9)
    sim.add_empty_species("e", 100, q=-1.0, m=1.0)
    with pytest.raises(RuntimeError, match="no species"):
        sim.add_flux_injection(3, abi.make_flux_injector(1.0, 0.5, "x", 1))
    with pytest.raises(RuntimeError, match="flux_direction"):
        sim.add_flux_injection(0, abi.make_flux_injector(1.0, 0.5, "x", 2))
    sim.add_flux_injection(0, abi.make_flux_injector(10.0, 0.5, "x", 1, u_th=(0.1, 0.1, 0.1)))
    assert sim.L.pic_engine_set_boost(sim.native, 2.0, 0.75 ** 0.5) != 0          # boosted frames take no injector
    assert "flux injection" in sim.L.pic_last_error().decode()
    with pytest.raises(RuntimeError, match="capacity"):
        sim.Evolve(1)
