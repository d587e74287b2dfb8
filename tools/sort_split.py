#!/usr/bin/env python3
"""What deferring the cell sort's move trades, on the benchmark workload: per-call times (the C++ driver's CUDA events)
of `sort` when it stops at the permutation and when it also moves the particles, and of `gather_push` on the step after
a deferred sort (it carries the move) and on other steps.

A sort is deferred when another step of the same Evolve call follows it.  With a sort every 4 steps the script runs,
from a spun-up state, cycles of Evolve(3), Evolve(2), Evolve(3): the first call ends before the sort of step 4, the
second holds that sort (deferred) and the push that carries it, the third ends with the sort of step 8 (moved at once).

    python tools/sort_split.py --cells 256 > sort_split.json"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=256)
    ap.add_argument("--ppc", type=int, default=2)
    ap.add_argument("--spinup", type=int, default=64, help="a multiple of 8")
    ap.add_argument("--cycles", type=int, default=4)
    args = ap.parse_args()
    import torch
    from warpx_b200 import workloads
    from warpx_b200.engine import Simulation
    if not torch.cuda.is_available():
        raise SystemExit("tools/sort_split.py needs a CUDA device")
    n = args.cells
    wl = workloads.uniform_plasma_3d(n_cell=(n, n, n), ppc=(args.ppc,) * 3, lx=(40.0e-6,) * 3, u_th=0.01)
    s = wl["species"][0]
    sim = Simulation((n, n, n), wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
    sim.add_species("electrons", s["q"], s["m"], *[torch.from_numpy(s[k]) for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
    sim.Evolve(args.spinup, synchronize_last=False)

    def call(steps):
        sim.enable_stage_timing(True)
        sim.Evolve(steps, synchronize_last=False)
        st = sim.stage_ms()                    # {stage: (ms per call, calls)}
        sim.enable_stage_timing(False)
        return {k: st[k][0] * st[k][1] for k in ("sort", "gather_push") if k in st}

    rows = {"sort_deferred": [], "sort_with_move": [], "gather_push_other_steps": [], "gather_push_after_deferred_sort": []}
    for _ in range(args.cycles):
        a, b, c = call(3), call(2), call(3)
        plain = (a["gather_push"] + c["gather_push"]) / 6
        rows["gather_push_other_steps"].append(plain)
        rows["gather_push_after_deferred_sort"].append(b["gather_push"] - plain)
        rows["sort_deferred"].append(b["sort"])
        rows["sort_with_move"].append(c["sort"])
    dev = torch.cuda.get_device_properties(0)
    print(json.dumps({"device": dev.name, "cells": n, "ppc": args.ppc ** 3, "unit": "ms per call",
                      **{k: {"mean": sum(v) / len(v), "min": min(v), "max": max(v)} for k, v in rows.items()}}))
    sim.close()


if __name__ == "__main__":
    main()
