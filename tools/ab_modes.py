#!/usr/bin/env python3
"""A/B of the experimental kernel variants on the benchmark workload, in ONE process (the 256^3 x 8 ppc state is
generated and uploaded once): for every deposition variant (pic_set_deposit_mode 0..7, 12) and gather variant
(pic_set_gather_mode 0..2) the per-stage times of the step (CUDA events around every stage, Python sequencer)
and the whole-step time of the C++ driver.  Not a bench value -- a ranking tool for a scarce GPU slot:

    python tools/ab_modes.py --cells 256 > ab_modes.json

Every variant passes the same parity tests (tests/test_gpu_zz_lwfa.py::test_deposit_variants_match_oracle,
::test_gather_variants_match_oracle); this script only times them."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=256)
    ap.add_argument("--ppc", type=int, default=2)
    ap.add_argument("--steps", type=int, default=8, help="timed steps per variant (a multiple of the sort interval)")
    ap.add_argument("--u-th", type=float, default=0.01)
    ap.add_argument("--jitter", action="store_true", help="random in-cell positions (the steady state of the lattice)")
    ap.add_argument("--sort-intervals", default="", help="comma list: steady-state ms/step for each cell-sort interval "
                    "(64 spin-up steps, then 16 timed), default kernels")
    ap.add_argument("--fresh", action="store_true", help="a new Simulation per variant: stage times on the FRESH state "
                    "(steps 4..12 after the upload) instead of one long-running state")
    ap.add_argument("--deposit-modes", default="0,12,7,2,5,6")
    ap.add_argument("--gather-modes", default="0,1,2,3")
    args = ap.parse_args()
    import torch
    from warpx_b200 import workloads
    from warpx_b200.engine import Simulation
    from warpx_b200.lib import lib
    if not torch.cuda.is_available():
        raise SystemExit("tools/ab_modes.py needs a CUDA device")
    L = lib()
    n = args.cells
    wl = workloads.uniform_plasma_3d(n_cell=(n, n, n), ppc=(args.ppc,) * 3, lx=(40.0e-6,) * 3, u_th=args.u_th)
    s = wl["species"][0]
    if args.jitter:
        import numpy as np
        rng = np.random.default_rng(1234)
        for d, k in enumerate(("x", "y", "z")):
            dxd = 40.0e-6 / n
            cell = np.floor((s[k] - wl["prob_lo"][d]) / dxd)
            s[k] = wl["prob_lo"][d] + (cell + rng.uniform(0.0, 1.0, len(cell))) * dxd
    names = ("x", "y", "z", "w", "ux", "uy", "uz")

    def make(native):
        sim = Simulation((n, n, n), wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4, native_driver=native)
        sim.add_species("electrons", s["q"], s["m"], *[torch.from_numpy(s[k]) for k in names])
        return sim

    def timed(sim, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        sim.Evolve(steps, synchronize_last=False)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    if args.sort_intervals:
        out = {"cells": n, "ppc": args.ppc ** 3, "sort_intervals": []}
        for si in (int(v) for v in args.sort_intervals.split(",")):
            sim = Simulation((n, n, n), wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=si)
            sim.add_species("electrons", s["q"], s["m"], *[torch.from_numpy(s[k]) for k in names])
            sim.Evolve(64, synchronize_last=False)
            sim.enable_stage_timing(True)
            ms = timed(sim, 16)
            st = {k: (t[0], t[1]) for k, t in sim.stage_ms().items()}
            sim.close()
            del sim
            torch.cuda.empty_cache()
            out["sort_intervals"].append({"sort_interval": si, "ms_per_step": ms, "stage_ms": st})
            print("sort every %2d steps : %7.2f ms/step   gather %6.2f  deposit %6.2f  sort %5.2f x %d" %
                  (si, ms, st["gather_push"][0], st["deposit"][0], st.get("sort", (0, 0))[0], st.get("sort", (0, 0))[1]), file=sys.stderr)
        print(json.dumps(out, indent=1))
        return
    if args.fresh:
        out = {"cells": n, "ppc": args.ppc ** 3, "steps": args.steps, "fresh": True, "variants": []}
        for d in (int(v) for v in args.deposit_modes.split(",")):
            for g in (int(v) for v in args.gather_modes.split(",")):
                L.pic_set_deposit_mode(d)
                L.pic_set_gather_mode(g)
                sim = make(True)
                sim.Evolve(4, synchronize_last=False)
                sim.enable_stage_timing(True)
                ms = timed(sim, args.steps)
                st = {k: t[0] for k, t in sim.stage_ms().items()}
                sim.close()
                del sim
                torch.cuda.empty_cache()
                out["variants"].append({"deposit_mode": d, "gather_mode": g, "ms_per_step": ms, "stage_ms": st})
                print("fresh: deposit_mode %d gather_mode %d : %7.2f ms/step   gather %6.2f  deposit %6.2f" %
                      (d, g, ms, st.get("gather_push", float("nan")), st.get("deposit", float("nan"))), file=sys.stderr)
        L.pic_set_deposit_mode(0)
        L.pic_set_gather_mode(0)
        print(json.dumps(out, indent=1))
        return
    combos = [(d, 0) for d in (int(v) for v in args.deposit_modes.split(","))] + \
             [(0, g) for g in (int(v) for v in args.gather_modes.split(",")) if g]
    out = {"cells": n, "ppc": args.ppc ** 3, "steps": args.steps, "variants": []}
    # whole step, C++ driver
    sim = make(True)
    sim.Evolve(4, synchronize_last=False)
    for d, g in combos + [combos[0]]:                    # the default again at the end: drift of the state
        L.pic_set_deposit_mode(d)
        L.pic_set_gather_mode(g)
        sim.Evolve(4, synchronize_last=False)            # warm-up of this variant (one sort period)
        out["variants"].append({"deposit_mode": d, "gather_mode": g, "ms_per_step": timed(sim, args.steps)})
    # per stage: CUDA events of the C++ driver
    for v in out["variants"][:-1]:
        L.pic_set_deposit_mode(v["deposit_mode"])
        L.pic_set_gather_mode(v["gather_mode"])
        sim.enable_stage_timing(False)
        sim.Evolve(4, synchronize_last=False)            # warm-up of this variant
        sim.enable_stage_timing(True)                    # fresh sums
        sim.Evolve(4, synchronize_last=False)
        v["stage_ms"] = {k: t[0] for k, t in sim.stage_ms().items()}
    L.pic_set_deposit_mode(0)
    L.pic_set_gather_mode(0)
    # the two FDTD data paths (stage times only)
    out["fdtd"] = {}
    for fm in (0, 3):
        L.pic_set_fdtd_mode(fm)
        sim.enable_stage_timing(False)
        sim.Evolve(2, synchronize_last=False)
        sim.enable_stage_timing(True)
        sim.Evolve(4, synchronize_last=False)
        st = sim.stage_ms()
        out["fdtd"]["bulk" if fm else "plain"] = {k: st[k][0] for k in ("evolve_b", "evolve_e")}
        print("fdtd mode %d : evolve_b %.3f ms  evolve_e %.3f ms" % (fm, st["evolve_b"][0], st["evolve_e"][0]), file=sys.stderr)
    L.pic_set_fdtd_mode(1)
    # best of each family together
    best_d = min((v for v in out["variants"][:-1] if v["gather_mode"] == 0), key=lambda v: v["ms_per_step"])
    best_g = min((v for v in out["variants"][:-1] if v["deposit_mode"] == 0), key=lambda v: v["ms_per_step"])
    out["best"] = {"deposit_mode": best_d["deposit_mode"], "gather_mode": best_g["gather_mode"]}
    print(json.dumps(out, indent=1))
    # the same, compact, for the tail of a log (stderr, so that stdout stays one JSON document)
    for v in out["variants"]:
        st = v.get("stage_ms", {})
        print("deposit_mode %d gather_mode %d : %7.2f ms/step   gather %6.2f  deposit %6.2f" %
              (v["deposit_mode"], v["gather_mode"], v["ms_per_step"], st.get("gather_push", float("nan")),
               st.get("deposit", float("nan"))), file=sys.stderr)


if __name__ == "__main__":
    main()
