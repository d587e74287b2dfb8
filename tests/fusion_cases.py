"""TEST INFRASTRUCTURE -- seeded reactant sets for the fusion stage and a runner of pic_collide_nuclear_fusion +
pic_fusion_create_products that works with the device library (CUDA tensors) and with the host build of
tests/host_harness (CPU tensors)."""
import ctypes as C

import numpy as np

import collision_cases as cc
from warpx_b200 import abi
from warpx_b200.engine import species_charge_mass

GEOM = cc.GEOM
KEV = 1.0e3 * 1.602176634e-19


def spec(ftype=abi.FUSION_DT_NHE4, mult=1.0, thr=0.02, target=0.002, seed=11, cidx=0):
    """reactants and products of a reaction: D + T -> He4 + n, D + D -> T + p, D + D -> He3 + n (products in that
    order, as a deck may list them)"""
    r1, r2, pa, pb = {abi.FUSION_DT_NHE4: ("deuterium", "tritium", "helium4", "neutron"),
                      abi.FUSION_DD_PT: ("deuterium", "deuterium", "tritium", "hydrogen1"),
                      abi.FUSION_DD_NHE3: ("deuterium", "deuterium", "helium3", "neutron")}[ftype]
    q1, m1 = species_charge_mass(r1)
    q2, m2 = species_charge_mass(r2)
    return dict(q1=q1, m1=m1, q2=q2, m2=m2, mA=species_charge_mass(pa)[1], mB=species_charge_mass(pb)[1], type=ftype,
                fusion_multiplier=mult, fusion_probability_threshold=thr, fusion_probability_target_value=target,
                seed=seed, collision_index=cidx, same_species=int(r1 == r2))


def reactants(seed, counts, m, E_keV, weights="equal", id_offset=0, w0=1.0e9, drift_keV=0.0):
    """particle_set with momenta of a Maxwellian of temperature E_keV (and a drift along z) for mass m"""
    u_th = np.sqrt(E_keV * KEV / m) / cc.workloads.C
    u_m = np.sqrt(2.0 * drift_keV * KEV / m) / cc.workloads.C
    return cc.particle_set(seed, GEOM, counts, (u_th, u_th, u_th), u_m=(0.0, 0.0, u_m), weights=weights,
                           id_offset=id_offset, w0=w0)


def fusion_spec(f):
    c = abi.pic_fusion_collision()
    for k in ("q1", "m1", "q2", "m2", "mA", "mB", "type", "fusion_multiplier", "fusion_probability_threshold",
              "fusion_probability_target_value", "seed", "collision_index", "same_species"):
        setattr(c, k, f[k])
    return c


class Products:
    def __init__(self, t, dev, cap):
        self.cap = cap
        self.buf = t.zeros((7, cap), dtype=t.float64, device=dev)
        self.ids = t.zeros(cap, dtype=t.int64, device=dev)

    def soa(self, n=0):
        s = abi.pic_soa()
        for k, name in enumerate(cc.DeviceSpecies.NAMES):
            setattr(s, name, self.buf[k].data_ptr())
        s.idcpu, s.np = self.ids.data_ptr(), n
        return s

    def numpy(self, n):
        out = {name: self.buf[k, :n].cpu().numpy().copy() for k, name in enumerate(cc.DeviceSpecies.NAMES)}
        out["id"] = self.ids[:n].cpu().numpy().copy()
        return out


def run_stage(L, t, dev, sp1, sp2, f, dt, step, pending=True, stream=None, sync=lambda: None, cap=None, scratch=True):
    """both passes on fresh copies: returns (species 1, species 2 or None, product A, product B, status), each species
    as arrays in storage order of the buffer the stage worked on"""
    d1 = cc.DeviceSpecies(L, t, dev, sp1, GEOM, stream=stream)
    d1.sort(pending)
    d2 = None
    if not f["same_species"]:
        d2 = cc.DeviceSpecies(L, t, dev, sp2, GEOM, stream=stream)
        d2.sort(pending)
    o = d2 if d2 is not None else d1
    pc = d1.n + (0 if d2 is None else d2.n)
    nb = L.pic_bins_count(abi.int3(GEOM["box_lo"]), abi.int3(GEOM["box_hi"]), abi.int3((8, 8, 8)))
    work = t.zeros(L.pic_fusion_workspace_bytes(pc, nb), dtype=t.uint8, device=dev)
    status = t.zeros(1, dtype=t.int32, device=dev)
    c = fusion_spec(f)
    rc = L.pic_collide_nuclear_fusion(C.byref(c), C.byref(d1.soa(d1.cur)), C.byref(d1.bins), d1.src,
                                      C.byref(o.soa(o.cur)), C.byref(o.bins), o.src, C.byref(d1.g), dt, step,
                                      L.pic_sort_scratch(d1.work.data_ptr(), d1.n) if scratch else None,
                                      L.pic_sort_scratch(o.work.data_ptr(), o.n) if scratch else None,
                                      work.data_ptr(), pc, status.data_ptr(), stream)
    assert rc == 0, L.pic_last_error()
    cap = 2 * pc if cap is None else cap
    pa, pb = Products(t, dev, max(cap, 1)), Products(t, dev, max(cap, 1))
    nev = C.c_long()
    rc = L.pic_fusion_create_products(C.byref(c), C.byref(d1.soa(d1.cur)), C.byref(d1.bins), C.byref(o.soa(o.cur)),
                                      C.byref(o.bins), C.byref(d1.g), step, work.data_ptr(), pc, C.byref(pa.soa()), cap, 0,
                                      C.byref(pb.soa()), cap, 0, C.byref(nev), stream)
    if rc != 0:
        raise RuntimeError(L.pic_last_error().decode())
    sync()
    n = 2 * nev.value
    return (d1.numpy(), d2.numpy() if d2 is not None else None, pa.numpy(n), pb.numpy(n), int(status.cpu()[0]))


def by_id(sp):
    return cc.by_id(sp)


def assert_matches(got, want, rtol, what):
    """reactants: same ids (spent ones included) and weights by id; products: same order, positions exact, momenta
    and weights to rtol of their scale"""
    if what == "reactant":
        g, w = by_id(got), by_id(want)
        assert np.array_equal(np.sort(got["id"]), np.sort(want["id"]))
        live = w["id"] != -1
        for k in ("x", "y", "z", "ux", "uy", "uz"):
            assert np.array_equal(g[k][live], w[k][live]), k
        scale = max(np.abs(w["w"]).max(), 1e-300)
        assert np.abs(g["w"][live] - w["w"][live]).max() <= rtol * scale
        return
    assert len(got["x"]) == len(want["x"])
    if len(want["x"]) == 0:
        return
    assert np.array_equal(got["id"], want["id"])
    for k in ("x", "y", "z"):
        assert np.array_equal(got[k], want[k]), k
    um = np.sqrt(want["ux"] ** 2 + want["uy"] ** 2 + want["uz"] ** 2).max()
    for k in ("ux", "uy", "uz"):
        err = np.abs(got[k] - want[k]).max() / um
        assert err <= rtol, (k, err)
    assert np.abs(got["w"] - want["w"]).max() <= rtol * np.abs(want["w"]).max()
