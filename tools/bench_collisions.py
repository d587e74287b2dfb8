#!/usr/bin/env python3
"""Cost of the pairwise Coulomb collisions, from the C++ driver's CUDA events, on two workloads:

  bench   the benchmark's plasma (256^3 cells, 8 ppc, order 3, Yee) with electron-electron collisions every step
          (ndt = 1: the species is sorted before every collision), against the same run without collisions;
  xyz     64^3 cells of the xyz collision deck's size, 200 ppc of electrons and of ions, algo.maxwell_solver = none,
          electron-ion collisions every step.

Per workload: the `collisions` stage in ms per call, the `sort` stage per step with and without collisions (the extra
sorts ndt = 1 forces), the whole step with and without collisions, and the achieved bandwidth against the collision
stage's algorithmic bytes -- per particle: read id, w, ux, uy, uz and src, write ux, uy, uz (68 B); per bin and species:
one cell_start entry (4 B).  The card's name, power limit and maximum SM clock are read in the same run.
The fp64 instruction count is the static count of double-precision instructions in the SASS of the collision kernels
(cuobjdump of the library): the cell walk's kernels instantiated with PairwiseCoulomb.

    python tools/bench_collisions.py --steps 10 --warmup 3 > bench_collisions.json"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def sass_fp64_counts():
    from warpx_b200 import build
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", build.LIB], capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "kernel" in m.group(1) and "PairwiseCoulomb" in m.group(1) else None
            if cur:
                out[cur] = {"fp64": 0, "all": 0}
            continue
        if cur and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            out[cur]["all"] += 1
            if re.search(r"\b(DADD|DMUL|DFMA|DSETP|DMNMX|MUFU\.RSQ64H|MUFU\.RCP64H|F2F\.F64|I2F\.F64|F2I\.F64)", line):
                out[cur]["fp64"] += 1
    return out


def run(sim, steps, warmup):
    import torch
    sim.Evolve(warmup, synchronize_last=False)
    sim.enable_stage_timing(True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sim.Evolve(steps, synchronize_last=False)
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / steps * 1e3
    st = sim.stage_ms()
    sim.enable_stage_timing(False)
    return wall, st


def summarise(name, with_c, without, nparticles, nbins_species):
    wall_c, st_c = with_c
    wall_0, st_0 = without
    coll_ms, coll_calls = st_c["collisions"]
    bytes_call = 68 * nparticles + 4 * nbins_species
    sort_c = st_c.get("sort", (0.0, 0))
    sort_0 = st_0.get("sort", (0.0, 0))
    return {
        "workload": name, "particles": nparticles,
        "collisions_ms_per_call": coll_ms, "collision_calls": coll_calls,
        "algorithmic_bytes_per_call": bytes_call,
        "achieved_GB_per_s": bytes_call / (coll_ms * 1e-3) / 1e9,
        "hbm_floor_ms": bytes_call / HBM_BYTES_PER_S * 1e3,
        "sort_ms_per_step_with_collisions": sort_c[0] * sort_c[1] / coll_calls,
        "sort_ms_per_step_without": (sort_0[0] * sort_0[1] / coll_calls) if sort_0[1] else 0.0,
        "step_ms_with_collisions": wall_c, "step_ms_without": wall_0,
        "stages_with": {k: v[0] for k, v in st_c.items()}, "stages_without": {k: v[0] for k, v in st_0.items()},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cells", type=int, default=256)
    ap.add_argument("--xyz-cells", type=int, default=64)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_collisions.py needs a CUDA device")
    from warpx_b200 import abi, workloads
    from warpx_b200.engine import Simulation
    result = {"card": card(), "sass": sass_fp64_counts(), "runs": []}

    n = args.cells
    wl = workloads.uniform_plasma_3d(n=n, ppc=(2, 2, 2), u_th=0.01, lx=40.0e-6 * n / 256.0)
    s = wl["species"][0]
    arrays = [torch.from_numpy(s[k]) for k in ("x", "y", "z", "w", "ux", "uy", "uz")]
    nb = None
    runs = {}
    for with_coll in (True, False):
        sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
        sim.add_species("electrons", s["q"], s["m"], *arrays)
        nb = sim.L.pic_bins_count(abi.int3(sim.box_lo), abi.int3(sim.box_hi), abi.int3(sim.tile))
        if with_coll:
            sim.add_collision(0, 0, coulomb_log=-1.0, ndt=1, seed=1)
        runs[with_coll] = run(sim, args.steps, args.warmup)
        sim.close()
        del sim
        torch.cuda.empty_cache()
    result["runs"].append(summarise("bench %d^3 x 8 ppc, e-e" % n, runs[True], runs[False], len(s["x"]), nb + 1))
    del arrays, wl, s

    m = args.xyz_cells
    wl = workloads.collision_xyz_3d(n=m, ppc=200)
    runs = {}
    for with_coll in (True, False):
        sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=wl["dt"],
                         sort_interval=4)
        for sp in wl["species"]:
            sim.add_species(sp["name"], sp["q"], sp["m"], *[torch.from_numpy(sp[k]) for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
        nb = sim.L.pic_bins_count(abi.int3(sim.box_lo), abi.int3(sim.box_hi), abi.int3(sim.tile))
        if with_coll:
            sim.add_collision(0, 1, coulomb_log=15.9, ndt=1, seed=1)
        runs[with_coll] = run(sim, args.steps, args.warmup)
        sim.close()
        del sim
        torch.cuda.empty_cache()
    npart = sum(len(sp["x"]) for sp in wl["species"])
    result["runs"].append(summarise("xyz %d^3 x 200 ppc x 2 species, e-i" % m, runs[True], runs[False], npart, 2 * (nb + 1)))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
