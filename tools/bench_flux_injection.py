#!/usr/bin/env python3
"""Cost of the flux injection, from the C++ driver's CUDA events: the benchmark's plasma (256^3 cells, 8 ppc, order 3,
Yee) plus one injector of 64 particles per cell on the z plane through the middle of the domain (65536 plane cells:
about 4.2 M particles per call), against the same run without the injector.  The two runs alternate in this process
(with, without, with, without), each on a fresh Simulation with the same capacity; the particle count grows by a call's
particles every step of the run with the injector, so its step time includes pushing and depositing them.

Reported: the `flux_injection` stage in ms per call, the particles per call, the stage's algorithmic bytes -- per
particle the written SoA and id (64 B), per particle slot (plane cell x (floor(ppc) + 1)) the keep flag written,
scanned in place and read twice (20 B) -- the achieved bandwidth and its share of the H100 SXM's 3.35 TB/s, and the
step time of both runs.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_flux_injection.py --steps 20 --warmup 2 > bench_flux_injection.json"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cells", type=int, default=256)
    ap.add_argument("--ppc", type=float, default=64.0, help="particles per plane cell of the injector")
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_flux_injection.py needs a CUDA device")
    from warpx_b200 import abi, workloads
    from warpx_b200.engine import Simulation
    n = args.cells
    wl = workloads.uniform_plasma_3d(n=n, ppc=(2, 2, 2), u_th=0.01, lx=40.0e-6 * n / 256.0)
    s = wl["species"][0]
    arrays = [torch.from_numpy(s[k]).pin_memory() for k in ("x", "y", "z", "w", "ux", "uy", "uz")]
    per_call_max = n * n * (int(args.ppc) + 1)
    capacity = len(s["x"]) + (args.warmup + args.steps) * per_call_max
    z_mid = 0.5 * (wl["prob_lo"][2] + wl["prob_hi"][2]) + 0.25 * (wl["prob_hi"][2] - wl["prob_lo"][2]) / n
    injector = dict(num_particles_per_cell=args.ppc, surface_flux_pos=z_mid, flux_normal_axis="z", flux_direction=1,
                    flux=1.0e30, u_m=(0.0, 0.0, 0.01), u_th=(0.01, 0.01, 0.01), seed=1)
    result = {"card": card(), "cells": n, "injector_ppc": args.ppc, "steps": args.steps, "rounds": []}
    for rnd in range(args.rounds):
        entry = {}
        for with_inj in (True, False):
            sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
            sim.add_species("electrons", s["q"], s["m"], *arrays, capacity=capacity)
            if with_inj:
                sim.add_flux_injection("electrons", abi.make_flux_injector(**injector))
            np0 = sim.species[0].np
            sim.Evolve(args.warmup, synchronize_last=False)
            np1 = sim.species[0].np
            sim.enable_stage_timing(True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sim.Evolve(args.steps, synchronize_last=False)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) / args.steps * 1e3
            st = sim.stage_ms()
            np2 = sim.species[0].np
            sim.close()
            del sim
            torch.cuda.empty_cache()
            key = "with" if with_inj else "without"
            entry["step_ms_" + key] = wall
            entry["stages_" + key] = {k: v[0] for k, v in st.items()}
            if with_inj:
                ms, calls = st["flux_injection"]
                per_call = (np2 - np1) / args.steps
                bytes_call = 64 * per_call + 20 * n * n * (int(args.ppc) + 1)
                entry.update(flux_injection_ms_per_call=ms, calls=calls, particles_per_call=per_call,
                             particles_at_start=np0, particles_at_end=np2, algorithmic_bytes_per_call=bytes_call,
                             achieved_GB_per_s=bytes_call / (ms * 1e-3) / 1e9,
                             share_of_hbm_peak=bytes_call / (ms * 1e-3) / HBM_BYTES_PER_S)
        result["rounds"].append(entry)
        print(json.dumps(dict(round=rnd, **{k: v for k, v in entry.items() if not k.startswith("stages")})),
              file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
