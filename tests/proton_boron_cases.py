"""TEST INFRASTRUCTURE -- seeded proton and boron sets for the proton-boron fusion stage and a runner of
pic_collide_nuclear_fusion + pic_fusion_create_products (type PIC_FUSION_PB_3HE4, one product species) that works with
the device library (CUDA tensors) and with the host build of tests/host_harness (CPU tensors)."""
import ctypes as C

import collision_cases as cc
import fusion_cases as fc
from warpx_b200 import abi
from warpx_b200.engine import species_charge_mass

GEOM = fc.GEOM


def spec(boron_first=False, mult=1.0, thr=0.02, target=0.002, seed=13, cidx=0):
    """p + B11 -> 3 He4 with the proton as species 1 (or the boron, boron_first)"""
    r = ("boron11", "hydrogen1") if boron_first else ("hydrogen1", "boron11")
    q1, m1 = species_charge_mass(r[0])
    q2, m2 = species_charge_mass(r[1])
    return dict(q1=q1, m1=m1, q2=q2, m2=m2, mA=species_charge_mass("helium4")[1], mB=0.0, type=abi.FUSION_PB_3HE4,
                fusion_multiplier=mult, fusion_probability_threshold=thr, fusion_probability_target_value=target,
                seed=seed, collision_index=cidx, same_species=0)


def run_stage(L, t, dev, sp1, sp2, f, dt, step, pending=True, stream=None, sync=lambda: None, cap=None):
    """both passes on fresh copies: (species 1, species 2, alphas, status), the species as arrays in storage order of the
    buffer the stage worked on"""
    d1 = cc.DeviceSpecies(L, t, dev, sp1, GEOM, stream=stream)
    d1.sort(pending)
    d2 = cc.DeviceSpecies(L, t, dev, sp2, GEOM, stream=stream)
    d2.sort(pending)
    pc = d1.n + d2.n
    nb = L.pic_bins_count(abi.int3(GEOM["box_lo"]), abi.int3(GEOM["box_hi"]), abi.int3((8, 8, 8)))
    work = t.zeros(L.pic_fusion_workspace_bytes(pc, nb), dtype=t.uint8, device=dev)
    status = t.zeros(1, dtype=t.int32, device=dev)
    c = fc.fusion_spec(f)
    rc = L.pic_collide_nuclear_fusion(C.byref(c), C.byref(d1.soa(d1.cur)), C.byref(d1.bins), d1.src,
                                      C.byref(d2.soa(d2.cur)), C.byref(d2.bins), d2.src, C.byref(d1.g), dt, step,
                                      L.pic_sort_scratch(d1.work.data_ptr(), d1.n),
                                      L.pic_sort_scratch(d2.work.data_ptr(), d2.n), work.data_ptr(), pc,
                                      status.data_ptr(), stream)
    assert rc == 0, L.pic_last_error()
    cap = 6 * pc if cap is None else cap
    pa = fc.Products(t, dev, max(cap, 1))
    nev = C.c_long()
    rc = L.pic_fusion_create_products(C.byref(c), C.byref(d1.soa(d1.cur)), C.byref(d1.bins), C.byref(d2.soa(d2.cur)),
                                      C.byref(d2.bins), C.byref(d1.g), step, work.data_ptr(), pc, C.byref(pa.soa()), cap,
                                      0, None, 0, 0, C.byref(nev), stream)
    if rc != 0:
        raise RuntimeError(L.pic_last_error().decode())
    sync()
    return d1.numpy(), d2.numpy(), pa.numpy(6 * nev.value), int(status.cpu()[0])
