#!/usr/bin/env python3
"""Per-kernel GPU time of the benchmark workload (256^3 x 8 ppc, order 3, sort every 4 steps), from torch.profiler
with CUDA activities over the timed steps -- the same state bench.py measures:

    python tools/profile_kernels.py --spinup 60 --steps 8 > steady.json     # steady state
    python tools/profile_kernels.py --spinup 0 --steps 8 > fresh.json       # fresh lattice

Prints one JSON document: the card (name, power limit, max SM clock), the deposition mode, whole-step time from CUDA
events in an unprofiled pass over the same steps, and for every kernel its total time per step and launches."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=256)
    ap.add_argument("--ppc", type=int, default=2)
    ap.add_argument("--spinup", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--steps", type=int, default=8, help="profiled steps (a multiple of the sort interval)")
    ap.add_argument("--deposit-mode", type=int, default=None, help="pic_set_deposit_mode (default: the library's)")
    args = ap.parse_args()
    import torch
    from bench import device_info
    from warpx_b200 import workloads
    from warpx_b200.engine import Simulation
    from warpx_b200.lib import lib
    if not torch.cuda.is_available():
        raise SystemExit("tools/profile_kernels.py needs a CUDA device")
    L = lib()
    if args.deposit_mode is not None:
        L.pic_set_deposit_mode(args.deposit_mode)
    n = args.cells
    lx = 40.0e-6 * n / 256.0
    wl = workloads.uniform_plasma_3d(n_cell=(n, n, n), ppc=(args.ppc,) * 3, lx=(lx,) * 3, u_th=0.01)
    s = wl["species"][0]
    sim = Simulation((n, n, n), wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
    sim.add_species("electrons", s["q"], s["m"], *[torch.from_numpy(s[k]) for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
    sim.Evolve(args.spinup + args.warmup, synchronize_last=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sim.Evolve(args.steps, synchronize_last=False)
    e1.record()
    torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / args.steps
    # the profiled steps start at the same phase of the sort cycle as the timed ones
    sim.Evolve((-args.steps) % 4, synchronize_last=False)
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sim.Evolve(args.steps, synchronize_last=True)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.split("(")[0].split("<")[0].strip()
        k = kernels.setdefault(name, {"ms_per_step": 0.0, "launches": 0})
        k["ms_per_step"] += ev.time_range.elapsed_us() / 1e3 / args.steps
        k["launches"] += 1
    total = sum(k["ms_per_step"] for k in kernels.values())
    ranked = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms_per_step"]))
    sim.close()
    print(json.dumps({"device": device_info(torch.cuda.current_device()), "cells": n, "ppc": args.ppc ** 3,
                      "spinup": args.spinup, "steps": args.steps, "deposit_mode": args.deposit_mode,
                      "ms_per_step_unprofiled": ms_step, "kernel_ms_per_step_sum": total, "kernels": ranked}, indent=1))
    for name, k in list(ranked.items())[:12]:
        print("%-40s %8.3f ms/step  %4d launches" % (name[:40], k["ms_per_step"], k["launches"]), file=sys.stderr)


if __name__ == "__main__":
    main()
