#!/usr/bin/env python3
"""Multi-GPU parity check, launched by torchrun (one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29511 tests/multi_gpu_check.py

Config 1 (64^3 Langmuir, 40 steps) on a brick decomposition: WarpX's golden checksums at rtol 1e-9
(what the reference's own 2-rank CI runs compare, Examples/CMakeLists.txt:98-104), particle-count
conservation through migration, an order-3 thermal run compared with the single-box oracle, and Gauss's law over the
union of the bricks."""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle  # noqa: E402  (test infrastructure: the checker)
from warpx_b200 import abi, engine, parallel, workloads  # noqa: E402
from warpx_b200.engine import Simulation  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    import faulthandler
    faulthandler.dump_traceback_later(600, exit=True)      # a hang names its line instead of running into the job limit
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    ok = True
    sections = os.environ.get("PIC_CHECK_SECTIONS", "order3,gauss,lwfa,boosted").split(",")     # debugging: skip the slower sections
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "warpx_checksums.json")))["test_3d_langmuir_multi"]
    L = oracle.lib()

    # ---------------- config 1 on `world` GPUs ----------------
    n = 64
    nb = parallel.brick_grid(world)
    dec = parallel.Decomposition((n, n, n), nb, rank)
    full = workloads.langmuir_3d(n=n)
    sim = Simulation(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=1, dist=dist, sort_interval=4)
    dx = sim.dx[0]
    for s in full["species"]:
        cell = [np.floor((s[k] - full["prob_lo"][d]) / dx).astype(int) for d, k in enumerate("xyz")]
        m = np.ones(len(s["x"]), dtype=bool)
        for d in range(3):
            m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
        sim.add_species(s["name"], s["q"], s["m"], *[s[k][m] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
    ntot0 = sim.total_particles()
    sim.Evolve(40)
    torch.cuda.synchronize()
    assert sim.total_particles() == ntot0 == 2 * n ** 3
    sums = []
    for c in range(9):
        d, a = sim.field_numpy(c)
        hf = oracle.HostFab(sim.box_lo, sim.box_hi, d.ng, abi.YEE_STAG[c], data=a)
        sums.append(L.orc_checksum_cell_centered(C.byref(hf.desc), abi.int3(sim.box_lo), abi.int3(sim.box_hi)))
    psum = []
    for isp in range(2):
        P = sim.species_numpy(isp)
        psum += [np.sum(np.abs(P["x"])), np.sum(np.abs(P["y"])), np.sum(np.abs(P["z"])),
                 np.sum(np.abs(P["ux"])) * workloads.M_E, np.sum(np.abs(P["uz"])) * workloads.M_E, np.sum(P["w"])]
    t = torch.tensor(sums + psum, dtype=torch.float64, device="cuda")
    dist.all_reduce(t)
    v = t.cpu().numpy()
    if rank == 0:
        for c, name in enumerate(abi.COMP_NAMES):
            g = golden["lev=0"][name]
            good = abs(v[c] - g) <= 1e-9 * abs(g)
            ok &= good
            print(f"[langmuir x{world}] {name}: {v[c]:.15e} golden {g:.15e} {'ok' if good else 'FAIL'}")
        keys = ["particle_position_x", "particle_position_y", "particle_position_z", "particle_momentum_x",
                "particle_momentum_z", "particle_weight"]
        for isp, sname in enumerate(("electrons", "positrons")):
            for j, key in enumerate(keys):
                if key in golden[sname]:
                    g = golden[sname][key]
                    good = abs(v[9 + 6 * isp + j] - g) <= 1e-9 * abs(g)
                    ok &= good
                    print(f"[langmuir x{world}] {sname}.{key}: {'ok' if good else 'FAIL'} ({v[9 + 6 * isp + j]:.15e} vs {g:.15e})")

    # ---------------- order-3 thermal plasma with migration vs the single-box oracle ----------------
    n3 = 32
    wl = workloads.uniform_plasma_3d(n=n3, ppc=(2, 2, 2), u_th=0.05, lx=5e-6, perturbation=0.01)
    dec3 = parallel.Decomposition((n3,) * 3, nb, rank)
    mine = workloads.uniform_plasma_3d(n=n3, ppc=(2, 2, 2), u_th=0.05, lx=5e-6, perturbation=0.01,
                                       box_lo=dec3.box_lo, box_hi=dec3.box_hi)
    s = mine["species"][0]
    so = wl["species"][0]
    # warpx.use_filter = 0 / 1 (bilinear, 1 pass); C++ driver over its own NCCL communicator
    for filt in (False, True) if "order3" in sections else ():
        sim3 = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, dist=dist, sort_interval=4,
                          use_filter=filt)
        sim3.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        sim3.Evolve(12)
        e, b = sim3.field_energy()
        npart = sim3.total_particles()
        if rank == 0:
            osim = oracle.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, use_filter=filt)
            osim.add_species(so["q"], so["m"], so["x"], so["y"], so["z"], so["w"], so["ux"], so["uy"], so["uz"])
            osim.evolve(12)
            eo, bo = osim.field_energy()
            good = abs(e - eo) <= 1e-10 * eo and abs(b - bo) <= 1e-8 * bo and npart == len(so["x"])
            ok &= good
            print(f"[order3 x{world} filter={int(filt)}] field energy E {e:.12e} vs oracle {eo:.12e}; "
                  f"B {b:.12e} vs {bo:.12e}; particles {npart}: {'ok' if good else 'FAIL'}")
        sim3.close()
        del sim3
    # ---------------- Gauss's law over the union of the bricks (tests/test_host_multirank.py: union_gauss) ----------------
    # (order 3, thermal electrons at u_th = 0.3 c crossing between bricks every step: a particle that migration loses or
    #  duplicates breaks G = div E - rho/ep0 by about 4e-2 of max|rho^0/ep0|)
    if "gauss" in sections:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from helpers import gauss_drift
        from test_host_multirank import union_gauss, union_state
        wl = workloads.uniform_plasma_3d(n=n3, ppc=(2, 1, 1), u_th=0.3, lx=5e-6, perturbation=0.01)
        mine = workloads.uniform_plasma_3d(n=n3, ppc=(2, 1, 1), u_th=0.3, lx=5e-6, perturbation=0.01,
                                           box_lo=dec3.box_lo, box_hi=dec3.box_hi)
        s = mine["species"][0]
        simg = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, dist=dist, sort_interval=4)
        simg.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        done, states = 0, []
        for step in (0, 1, 4, 5, 12):
            if step > done:
                simg.Evolve(step - done, synchronize_last=False)
                done = step
            torch.cuda.synchronize()
            got = [None] * world
            dist.all_gather_object(got, union_state(simg))
            states.append(got)
        if rank == 0:
            G0, rho0, ids0 = union_gauss(oracle, states[0], wl, 3)
            for step, st in zip((1, 4, 5, 12), states[1:]):
                G, _, ids = union_gauss(oracle, st, wl, 3)
                r = gauss_drift(G, G0, rho0)
                good = r <= 1e-11 and len(ids[0]) == len(ids0[0]) and np.array_equal(np.sort(ids[0]), np.sort(ids0[0]))
                ok &= good
                print(f"[gauss x{world}] step {step}: max|G^n - G^0| / max|rho^0/ep0| {r:.3e}, "
                      f"{len(ids[0])} particles, ids kept: {'ok' if good else 'FAIL'}")
        simg.close()
        del simg
    # ---------------- laser-acceleration deck on z slabs: moving window over several ranks ----------------
    # (PEC walls on the end slabs, neighbour planes pulled in by the window shift, one cell layer of
    #  particles migrating down per shift, injection on the top slab, replicated antenna) against WarpX's
    #  golden checksums of test_3d_laser_acceleration -- the decomposition must not change them.
    if 256 % world == 0 and 256 // world >= 16 and "lwfa" in sections:
        gl = json.load(open(os.path.join(ROOT, "tests", "golden", "warpx_checksums.json")))["test_3d_laser_acceleration"]
        wl = workloads.laser_acceleration_3d()
        simw = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"], dist=dist,
                          use_filter=wl["use_filter"], sort_interval=4, nb=(1, 1, world),
                          boundaries=abi.make_boundaries(wl["field_lo"], wl["field_hi"]),
                          moving_window=(wl["moving_window_dir"], wl["moving_window_v"]))
        sp = wl["species"][0]
        simw.add_plasma_species(sp["name"], sp["q"], sp["m"],
                                abi.make_injector(sp["ppc"], sp["bound_lo"], sp["bound_hi"], sp["density"], True),
                                capacity=22 * 22 * 256)
        la = wl["lasers"][0]
        simw.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"], la["e_max"],
                                      la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
        simw.Evolve(wl["max_step"])
        torch.cuda.synchronize()
        sums = []
        for c in range(9):
            d, a = simw.field_numpy(c)
            hf = oracle.HostFab(simw.box_lo, simw.box_hi, d.ng, abi.YEE_STAG[c], data=a)
            sums.append(L.orc_checksum_cell_centered(C.byref(hf.desc), abi.int3(simw.box_lo), abi.int3(simw.box_hi)))
        P = simw.species_numpy(0)
        psum = [np.sum(np.abs(P["x"])), np.sum(np.abs(P["y"])), np.sum(np.abs(P["z"])),
                np.sum(np.abs(P["ux"])) * workloads.M_E, np.sum(np.abs(P["uy"])) * workloads.M_E,
                np.sum(np.abs(P["uz"])) * workloads.M_E, np.sum(P["w"]), float(len(P["x"]))]
        t = torch.tensor(sums + psum, dtype=torch.float64, device="cuda")
        dist.all_reduce(t)
        v = t.cpu().numpy()
        if rank == 0:
            keys = ["particle_position_x", "particle_position_y", "particle_position_z", "particle_momentum_x",
                    "particle_momentum_y", "particle_momentum_z", "particle_weight"]
            pairs = [(name, v[c], gl["lev=0"][name]) for c, name in enumerate(abi.COMP_NAMES)] + \
                    [("electrons." + k, v[9 + j], gl["electrons"][k]) for j, k in enumerate(keys)]
            for name, got, g in pairs:
                good = abs(got - g) <= 1e-9 * abs(g)
                ok &= good
                print(f"[lwfa z-slabs x{world}] {name}: {got:.15e} golden {g:.15e} {'ok' if good else 'FAIL'}")
            good = int(v[9 + 7]) == 22 * 22 * (45 + 98)
            ok &= good
            print(f"[lwfa z-slabs x{world}] particles {int(v[9 + 7])}: {'ok' if good else 'FAIL'}")
        simw.close()
        del simw
    # ---------------- BASELINE.json configs[3] in the small: boosted-frame laser acceleration on z slabs ----------------
    # (gamma_boost = 10, CKC, Vay, order 3, filter, Godfrey NCI corrector, PEC z, moving window, boosted antenna, electrons
    #  + ions injected continuously) -- every rank runs the small single-box oracle and compares its own slab and its own
    #  particles (by global id) with it.
    if "boosted" in sections and 128 % world == 0 and 128 // world >= 17:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_oracle import make_lwfa_oracle, _nci_lines
        from warpx_b200.engine import max_dt, nci_godfrey_stencils
        from warpx_b200.lib import lib as piclib
        wl = workloads.laser_acceleration_boosted_3d(use_fdtd_nci_corr=True)
        dxb = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
        nci = nci_godfrey_stencils(piclib(), _nci_lines(), workloads.C * wl["cfl"] * max_dt(wl["solver"], dxb) / dxb[2])
        simb = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"], dist=dist,
                          solver=wl["solver"], pusher=wl["pusher"], use_filter=True, sort_interval=4, nb=(1, 1, world),
                          boundaries=abi.make_boundaries(wl["field_lo"], wl["field_hi"]),
                          moving_window=(wl["moving_window_dir"], wl["moving_window_v"]),
                          gamma_boost=wl["gamma_boost"], nci_stencils=nci)
        for sp in wl["species"]:
            simb.add_plasma_species(sp["name"], sp["q"], sp["m"],
                                    abi.make_injector(sp["ppc"], sp["bound_lo"], sp["bound_hi"], sp["density"], True),
                                    capacity=16 * 16 * 200)
        la = wl["lasers"][0]
        simb.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"], la["e_max"],
                                      la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
        osim = make_lwfa_oracle(oracle, wl)
        simb.Evolve(40)
        osim.evolve(40)
        torch.cuda.synchronize()
        err, scale = [], []
        for c in range(9):
            d, a = simb.field_numpy(c)
            od, oa = osim.fab(c)
            sl = tuple(slice(od.ng[2 - ax] + simb.box_lo[2 - ax], od.ng[2 - ax] + simb.box_hi[2 - ax] + 1 + abi.YEE_STAG[c][2 - ax])
                       for ax in range(3))
            err.append(float(np.max(np.abs(a[d.valid_slices()] - oa[sl]))))
            scale.append(float(np.max(np.abs(oa))))
        perr, nmine = 0.0, 0
        for isp in (0, 1):
            A = simb.species_numpy(isp, sort_by_id=False)
            B = osim.particles(isp)
            ids = A["id"].astype(np.int64)
            nmine += len(ids)
            if len(ids):
                assert ids.min() >= 0 and ids.max() < len(B["x"])
                for k in ("x", "y", "z"):
                    perr = max(perr, float(np.max(np.abs(A[k] - B[k][ids]))) / simb.dx[2])
                for k in ("ux", "uy", "uz"):
                    perr = max(perr, float(np.max(np.abs(A[k] - B[k][ids]))) / (10.0 * workloads.C))
        ntotal = len(osim.particles(0)["x"]) + len(osim.particles(1)["x"])
        t = torch.tensor(err + [perr], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        cnt = torch.tensor([nmine], dtype=torch.int64, device="cuda")
        dist.all_reduce(cnt)
        v = t.cpu().numpy()
        if rank == 0:
            for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):
                sg = max(scale[c] for c in group)
                for c in group:
                    good = sg > 0 and v[c] <= 1e-8 * sg
                    ok &= good
                    print(f"[boosted z-slabs x{world}] {abi.COMP_NAMES[c]}: max |difference to the single-box oracle| {v[c]:.3e} "
                          f"of scale {sg:.3e}: {'ok' if good else 'FAIL'}")
            good = v[9] <= 1e-9 and int(cnt.item()) == ntotal > 0
            ok &= good
            print(f"[boosted z-slabs x{world}] electrons + ions by id: {int(cnt.item())} of {ntotal} particles, "
                  f"max difference {v[9]:.3e} (cells, 10 c): {'ok' if good else 'FAIL'}")
        simb.close()
        del simb
    if rank == 0:
        print("MULTI_GPU_CHECK", "PASS" if ok else "FAIL", flush=True)
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.broadcast(flag, 0)
    code = 0 if int(flag.item()) else 1
    # collective, explicit teardown: engines closed above, every rank releases the private communicator at the
    # same point, then torch's process group; no NCCL object is left for the interpreter's shutdown
    sim.close()
    torch.cuda.synchronize()
    dist.barrier()
    engine.release_comm(dist)
    dist.barrier()
    dist.destroy_process_group()
    sys.stdout.flush()
    os._exit(code)


if __name__ == "__main__":
    main()
