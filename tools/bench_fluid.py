"""Stage times of the cold fluid Langmuir plasma (two fluid species, Yee, periodic) at 256^3 on one GPU.

    python tools/bench_fluid.py [--n 256] [--steps 40] [--warmup 5]

Per fluid stage: milliseconds per call from CUDA events over the timed steps (Simulation.enable_stage_timing), the
algorithmic bytes per node the stage must move (computed here from the array shapes, fp64), the achieved rate and its
fraction of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card's name and power limit are read in the same
run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BW = 3.35e12

# Algorithmic HBM bytes per valid node and call (8 B per double read or written once):
#   gather_push:  N, NU read (32), 6 field components read (48), NU written (24)
#   advect:       N, NU read (32), N, NU written (32)        (edge states stay on chip)
#   deposit:      one launch per J component, each reads N, NU (3 x 32) and reads and writes its J component (3 x 16)
BYTES_PER_NODE = {"fluid_gather_push": 104, "fluid_advect": 64, "fluid_deposit": 144}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [v.strip() for v in out.split(",")]
        return name, limit
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    from warpx_b200 import workloads
    from warpx_b200.engine import Simulation
    if not torch.cuda.is_available():
        raise SystemExit("bench_fluid: needs a CUDA device")
    wl = workloads.langmuir_fluid_3d(n=a.n)
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, native_driver=False)
    for f in wl["fluids"]:
        sim.add_fluid_species(f["name"], f["q"], f["m"], f["density"], f["momentum"])
    sim.Evolve(a.warmup, synchronize_last=False)
    torch.cuda.synchronize()
    sim.enable_stage_timing(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sim.Evolve(a.steps, synchronize_last=False)
    e1.record()
    torch.cuda.synchronize()
    nodes = (a.n + 1) ** 3
    stages = {}
    for name, (ms, calls) in sorted(sim.stage_ms().items()):
        row = {"ms": ms, "calls": calls}
        if name in BYTES_PER_NODE:
            b = BYTES_PER_NODE[name] * nodes
            row.update(bytes_per_node=BYTES_PER_NODE[name], gb_s=b / (ms * 1e-3) / 1e9,
                       fraction_of_3_35_TB_s=b / (ms * 1e-3) / PEAK_BW)
        stages[name] = row
    name, limit = card()
    print(json.dumps({"workload": "langmuir_fluid_3d", "n": a.n, "fluids": len(sim.fluids), "steps": a.steps,
                      "step_ms": e0.elapsed_time(e1) / a.steps, "stages": stages, "gpu": name or torch.cuda.get_device_name(),
                      "power_limit": limit}))


if __name__ == "__main__":
    main()
