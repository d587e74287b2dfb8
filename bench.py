#!/usr/bin/env python3
"""Benchmark of the hot path: particle-steps/s of the explicit EM-PIC step on the 3D
uniform-plasma workload of BASELINE.json (configs[1]: 256^3 cells per GPU, 8 particles per cell,
Yee FDTD, Boris pusher, order-3 Esirkepov deposition, fp64).

    python bench.py --gpus N --steps K --warmup W                    # this repo's CUDA engine
    python bench.py --impl reference --gpus N --steps K --warmup W   # reference CPU algorithm (oracle)

Prints ONE JSON line (rank 0).  See DESIGN.md "Measurement" for the definition of every field.
"""
import argparse
import atexit
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "particle-steps/sec (3D uniform plasma, 256^3, 8 ppc)"
_LINE_FD = None        # the process's original stdout; everything else written to fd 1 is sent to stderr (see main)


def emit_line(line):
    """The ONE JSON line, on the original stdout."""
    data = (json.dumps(line) + "\n").encode()
    if _LINE_FD is None:
        sys.stdout.write(data.decode()); sys.stdout.flush()
    else:
        os.write(_LINE_FD, data)
HBM_PEAK_GBS = 3350.0          # H100 SXM data sheet (HBM3, 3.35 TB/s)
HBM_PEAK_SOURCE = "NVIDIA H100 SXM data sheet (3.35 TB/s)"


def device_info(gpu_index):
    """Name, power limit and maximum SM clock of the card the numbers are measured on (read-only queries)."""
    info = {"name": None, "power_limit_w": None, "sm_max_mhz": None}
    try:
        import torch
        info["name"] = torch.cuda.get_device_name(gpu_index)
    except Exception:
        pass
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        f = [v.strip() for v in out.strip().split(",")]
        info["power_limit_w"], info["sm_max_mhz"] = float(f[0]), float(f[1])
    except Exception:
        pass
    return info


class ClockSampler:
    """SM clocks / throttle reasons during the timed region (NVML, else an nvidia-smi query loop)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.rows, self.proc, self.idx = [], None, gpu_index

    def start(self):
        # NVML (pynvml) when it loads: a sample every 5 ms, so that even a 100 ms timed region is covered;
        # otherwise an nvidia-smi query loop (one sample per 100 ms)
        self.nvml_rows, self._stop, self._thread = [], threading.Event(), None
        try:
            import pynvml
            pynvml.nvmlInit()
            h = pynvml.nvmlDeviceGetHandleByIndex(self.idx)
            smax = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            reasons_fn = getattr(pynvml, "nvmlDeviceGetCurrentClocksEventReasons", None) or \
                pynvml.nvmlDeviceGetCurrentClocksThrottleReasons
            reasons_fn(h)                                   # raises here if unsupported, before the thread starts

            def poll():
                while not self._stop.is_set():
                    try:
                        self.nvml_rows.append((float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)), smax,
                                               int(reasons_fn(h))))
                    except Exception:
                        pass
                    time.sleep(0.005)
            self._thread = threading.Thread(target=poll, daemon=True)
            self._thread.start()
            return
        except Exception:
            self._thread = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    # NVML clocks-event-reason bits (nvml.h): SwPowerCap 0x4, HwSlowdown 0x8, SwThermalSlowdown 0x20, HwThermalSlowdown 0x40
    NVML_REASONS = ((0x8, "hw_slowdown"), (0x40, "hw_thermal_slowdown"), (0x20, "sw_thermal_slowdown"), (0x4, "sw_power_cap"))

    def stop(self):
        if getattr(self, "_thread", None) is not None:
            self._stop.set()
            self._thread.join(timeout=1.0)
            sm = sorted(r[0] for r in self.nvml_rows)
            reasons = set()
            for r in self.nvml_rows:
                for bit, name in self.NVML_REASONS:
                    if r[2] & bit:
                        reasons.add(name)
            return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": self.nvml_rows[0][1] if sm else None,
                    "reasons": sorted(reasons), "samples": len(sm), "source": "nvml"}
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, smax, reasons = [], None, set()
        for r in self.rows:
            f = [v.strip() for v in r.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); smax = float(f[2])
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": smax, "reasons": sorted(reasons),
                "samples": len(sm), "source": "nvidia-smi"}


# ---------------------------------------------------------------------------------------------
def cpu_reference_run(n, ppc, steps, warmup, nox=3, use_filter=False, solver="yee"):
    """The reference algorithm on the host cores: the oracle's whole-loop driver (OpenMP, all
    cores) on a bounded sample of the workload (n^3 cells of the same plasma).  Test infrastructure
    used as the measured CPU baseline -- the only place bench.py executes oracle/."""
    # threads pinned to cores (set before libgomp starts): the same box gave 4x different numbers unpinned
    os.environ.setdefault("OMP_PROC_BIND", "close")
    os.environ.setdefault("OMP_PLACES", "cores")
    os.environ.setdefault("OMP_WAIT_POLICY", "active")
    from oracle import oracle
    from warpx_b200 import abi, workloads
    oracle.lib()                 # as build() left it; compiled here only when it is missing
    # same cell size and plasma as the GPU run (dx = 40um/256), smaller box
    lx = 40.0e-6 * n / 256.0
    wl = workloads.uniform_plasma_3d(n=n, ppc=ppc, lx=lx)
    kind = "reference" if oracle.have_ref() else "restated"
    # host cores this process may use (torchrun exports OMP_NUM_THREADS=1; cgroup-limited boxes
    # report more logical CPUs than they grant).  SMT siblings rarely help this fp64 loop, so both
    # "all logical CPUs" and half of them are timed and the better one is reported.
    try:
        ncores = len(os.sched_getaffinity(0))
    except AttributeError:
        ncores = os.cpu_count() or 1
    env = os.environ.get("PIC_CPU_THREADS")
    candidates = [int(env)] if env else sorted({ncores, max(1, ncores // 2)}, reverse=True)
    s = wl["species"][0]
    npart = len(s["x"])
    best = None
    for threads in candidates:
        sim = oracle.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox, kind=kind, use_filter=use_filter,
                               solver=abi.SOLVER_CKC if solver == "ckc" else abi.SOLVER_YEE)
        sim.L.orc_set_num_threads(threads)
        sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        sim.evolve(max(warmup, 1), synchronize_last=False)
        t0 = time.perf_counter()
        sim.evolve(steps, synchronize_last=False)
        dt = time.perf_counter() - t0
        if best is None or dt < best[0]:
            best = (dt, threads, sim.timers())
        del sim
    dt, cores, timers = best
    return dict(value=npart * steps / dt, unit="particle-steps/s", cores=cores,
                kind="reference-leaves+port" if kind == "reference" else "port",
                sample="%d^3 cells x %d ppc (%d particles), order %d, %s, bilinear filter %s, %d steps, OpenMP %d threads "
                       "pinned to cores (best of %s); oracle = loop-for-loop restatement of the reference CPU path"
                       % (n, ppc[0] * ppc[1] * ppc[2], npart, nox, solver.upper(), "on" if use_filter else "off", steps,
                          cores, candidates),
                seconds=dt, ms_per_step=1e3 * dt / steps, timers=timers)


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    ppc = (args.ppc,) * 3
    steps = max(2, min(args.steps, 10))          # a bounded sample: the whole arm ends within a few minutes
    r = cpu_reference_run(args.cpu_n, ppc, steps, min(args.warmup, 2), nox=args.order, use_filter=bool(args.filter),
                          solver=args.solver)
    line = {"impl": "reference", "metric": METRIC, "value": r["value"], "unit": "particle-steps/s",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": r["ms_per_step"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": "3D uniform plasma, %s FDTD, Boris, order-%d Esirkepov, %d ppc; CPU sample "
                                   % (args.solver.upper(), args.order, args.ppc ** 3) + r["sample"],
                       "use_filter": int(args.filter), "timed_steps_of_the_sample": steps},
            "cpu_baseline": {k: r[k] for k in ("value", "unit", "cores", "kind", "sample")},
            "e2e": {"value": r["value"], "unit": "particle-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    emit_line(line)


DUMP_FIELD_POINTS = 1 << 18        # per component: 9 x 2 MB
DUMP_PARTICLES = 1 << 18           # 8 arrays x 2 MB


def dump_outputs(sim, out_dir, npart_local):
    """What the timed steps computed, as a caller of Simulation.Evolve receives it: the FieldEnergy diagnostic, the
    field components Ex..jz at a fixed, seeded sample of their valid points ([k, j, i] order), and the particle
    arrays (x y z w ux uy uz) of a fixed, seeded sample of particle ids, ordered by id.  The sample depends on the
    grid and particle count only, so two builds run with the same arguments can be compared array by array."""
    import numpy as np
    import torch
    from warpx_b200 import abi
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "field_energy.npy"), np.array(sim.field_energy(), dtype=np.float64))
    rng = np.random.default_rng(20240917)
    for c, name in enumerate(abi.COMP_NAMES):
        valid = sim.data[c][sim.fab[c].valid_slices()]
        n = valid.numel()
        idx = np.sort(rng.choice(n, size=min(n, DUMP_FIELD_POINTS), replace=False))
        sample = valid.reshape(-1)[torch.from_numpy(idx).to(valid.device)]
        np.save(os.path.join(out_dir, name + ".npy"), sample.cpu().numpy().astype(np.float64))
    sp = sim.species[0]
    want = torch.from_numpy(np.sort(rng.choice(npart_local, size=min(npart_local, DUMP_PARTICLES), replace=False)))
    ids = sp.id_array()
    keep = torch.isin(ids, want.to(ids.device))
    order = torch.argsort(ids[keep])
    np.save(os.path.join(out_dir, "particle_id.npy"), ids[keep][order].cpu().numpy().astype(np.float64))
    for name in sp.NAMES:
        np.save(os.path.join(out_dir, "particle_" + name + ".npy"),
                sp.array(name)[keep][order].cpu().numpy().astype(np.float64))


def start_watchdog(rank):
    """A hang must name its line: dump every thread's Python stack to stderr after 4 minutes and leave (status 3)
    after 11 -- before an outer limit kills the job without a trace."""
    import faulthandler

    def watch():
        time.sleep(240)
        sys.stderr.write("[bench watchdog] rank %d still running after 240 s\n" % rank)
        faulthandler.dump_traceback(file=sys.stderr, all_threads=True)
        sys.stderr.flush()
        time.sleep(420)
        sys.stderr.write("[bench watchdog] rank %d still running after 660 s: giving up\n" % rank)
        faulthandler.dump_traceback(file=sys.stderr, all_threads=True)
        sys.stderr.flush()
        os._exit(3)
    threading.Thread(target=watch, daemon=True).start()


# ---------------------------------------------------------------------------------------------
def run_engine(args):
    import numpy as np
    import torch
    from warpx_b200 import abi, engine, workloads
    from warpx_b200.engine import Simulation
    from warpx_b200.lib import lib
    from warpx_b200 import parallel

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    start_watchdog(rank)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the CUDA engine has no CPU fallback")
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    L = lib()
    L.pic_set_deposit_mode(args.deposit_mode)
    L.pic_set_gather_mode(args.gather_mode)

    n, ppc = args.n, (args.ppc,) * 3
    nb = parallel.brick_grid(world)
    n_cell = tuple(n * nb[d] for d in range(3))               # weak scaling: n^3 cells per GPU
    lx = 40.0e-6 * np.array(nb) * (n / 256.0)                  # same dx as configs[1]
    dec = parallel.Decomposition(n_cell, nb, rank)
    prob_lo = tuple(-0.5 * lx); prob_hi = tuple(0.5 * lx)
    solver = abi.SOLVER_CKC if args.solver == "ckc" else abi.SOLVER_YEE

    # ---- synthetic input, generated on the host into pinned memory (seeded, counter based) ----
    t_gen = time.perf_counter()
    wl = workloads.uniform_plasma_3d(n_cell=n_cell, ppc=ppc, lx=tuple(lx), box_lo=dec.box_lo if world > 1 else None,
                                     box_hi=dec.box_hi if world > 1 else None, u_th=args.u_th)
    if args.jitter:
        rng = np.random.default_rng(1234 + rank)
        s0 = wl["species"][0]
        for d, k in enumerate(("x", "y", "z")):
            dxd = lx[d] / n_cell[d]
            cell = np.floor((s0[k] - prob_lo[d]) / dxd)
            s0[k] = prob_lo[d] + (cell + rng.uniform(0.0, 1.0, len(cell))) * dxd
    s = wl["species"][0]
    names = ("x", "y", "z", "w", "ux", "uy", "uz")
    pinned = {k: torch.from_numpy(s[k]).pin_memory() for k in names}
    npart_local = len(s["x"])
    t_gen = time.perf_counter() - t_gen

    def make_sim():
        sim = Simulation(n_cell, prob_lo, prob_hi, nox=args.order, dist=dist, sort_interval=args.sort_interval,
                         solver=solver, use_filter=bool(args.filter))
        sim.add_species("electrons", s["q"], s["m"], *[pinned[k] for k in names])
        return sim

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(v):
        t = torch.tensor([v], dtype=torch.float64, device="cuda")
        if dist is not None:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # =================== device-resident measurement (`value`) ===================
    sim = make_sim()
    ntot = sim.total_particles()
    # spin-up: the NUniformPerCell lattice decays into random in-cell positions within ~50 steps (u_th dt = 0.006 dx
    # per step); particles then change cell all the time and the kernels see their steady-state load
    sim.Evolve(args.spinup, synchronize_last=False)
    sim.Evolve(args.warmup, synchronize_last=False)
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()       # before the barrier: spawning the sampler must not delay rank 0 inside the timed region
    sim.enable_stage_timing(True)       # CUDA events around every stage, inside the same timed steps
    barrier()
    launches0 = L.pic_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t_host0 = time.perf_counter()
    sim.Evolve(args.steps, synchronize_last=False)
    t_host_enqueue = time.perf_counter() - t_host0      # host time to issue the K steps
    e1.record()
    barrier()
    ms = max_over_ranks(e0.elapsed_time(e1))
    launches = L.pic_launch_count() - launches0
    clk = clocks.stop() if rank == 0 else None
    stage = sim.stage_ms()                               # {stage: (ms per call, calls)} of the timed steps
    sim.enable_stage_timing(False)
    fe = sim.field_energy()
    if args.dump_outputs and rank == 0:
        dump_outputs(sim, args.dump_outputs, npart_local)
    value = ntot * args.steps / (ms * 1e-3)
    sim.close()
    del sim
    torch.cuda.empty_cache()

    e2e = None
    if not args.profile_only:
        # =================== end-to-end through the public API (`e2e`) ===================
        # Job-level: every rank uploads its initial particle state from pinned host memory, runs K
        # steps through Simulation.Evolve, and reads the FieldEnergy reduced diagnostic back to the
        # host after EVERY step (what a WarpX run with reduced diagnostics does).  A PIC run has no
        # per-step host input: the upload happens once and is reported separately as well.
        barrier()
        t0 = time.perf_counter()
        sim2 = make_sim()
        torch.cuda.synchronize()
        t_up = time.perf_counter() - t0
        d2h = 0
        for _ in range(args.steps):
            sim2.Evolve(1, synchronize_last=False)
            sim2.field_energy()
            d2h += 16
        barrier()
        t_all = max_over_ranks(time.perf_counter() - t0)
        t_up = max_over_ranks(t_up)
        h2d_total = npart_local * 7 * 8
        e2e = {"value": ntot * args.steps / t_all, "unit": "particle-steps/s",
               "h2d_bytes_per_step": h2d_total / args.steps, "d2h_bytes_per_step": d2h / args.steps,
               "upload_and_first_sort_s": t_up, "loop_s": t_all - t_up,
               "loop_value": ntot * args.steps / max(t_all - t_up, 1e-9),
               "definition": "job-level wall clock, max over ranks: H2D upload of the initial particle state from pinned "
                             "host memory + initial cell sort (upload_and_first_sort_s) + K steps via Simulation.Evolve "
                             "with a D2H read of the FieldEnergy diagnostic after every step (loop_s; these steps start "
                             "from the lattice, not from the spun-up state)"}
        sim2.close()
        del sim2

    # =================== teardown, collective and explicit, BEFORE the CPU leg ===================
    barrier()
    if dist is not None:
        engine.release_comm(dist)
        barrier()
        dist.destroy_process_group()
    if rank != 0:
        return

    # =================== roofline of the kernels (algorithmic bytes / CUDA-event time) ==========
    hbm = HBM_PEAK_GBS
    ncell = n ** 3
    alg = {  # bytes per launch, DESIGN.md "Kernels"
        "evolve_b": 72.0 * ncell,
        "evolve_e": 96.0 * ncell,
        "gather_push": 96.0 * npart_local + 48.0 * ncell,
        "deposit": 56.0 * npart_local + 72.0 * ncell,
        "filter_j": 48.0 * ncell,        # --filter 1: three components, one read + one write each (no copy back)
    }
    kernels = {}
    for k, b in alg.items():
        if k in stage:
            t_ms, calls = stage[k]
            kernels[k] = {"ms": t_ms, "calls": calls, "achieved_gbs": b / (t_ms * 1e-3) / 1e9,
                          "frac_of_hbm_peak": b / (t_ms * 1e-3) / 1e9 / hbm, "algorithmic_bytes": b}
    dom = max((k for k in kernels), key=lambda k: kernels[k]["ms"] * kernels[k]["calls"])
    roofline = {"kernel": dom, "bound": "hbm", "achieved": kernels[dom]["achieved_gbs"], "peak": hbm, "unit": "GB/s",
                "frac": kernels[dom]["frac_of_hbm_peak"], "peak_source": HBM_PEAK_SOURCE,
                "kernels": kernels,
                "note": "stage durations from CUDA events recorded by the C++ driver inside the timed steps (a stage = "
                        "its main kernel plus the small ones it needs: stray / listed particles); gather_push and "
                        "deposit are fp64-FMA / shared-memory bound at order 3 (DESIGN.md); the HBM fraction is "
                        "reported because BASELINE.json asks for it"}
    step_sum = sum(t * c for t, c in stage.values()) / args.steps
    line = {"metric": METRIC, "value": value, "unit": "particle-steps/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": "3D uniform plasma %dx%dx%d cells (%d^3 per GPU), %d ppc (%d particles), %s FDTD, "
                                   "Boris pusher, order-%d Esirkepov, Galerkin gather, cfl 1, u_th %gc%s, "
                                   "bilinear current filter %s, cell sort every %d steps"
                                   % (n_cell + (n, args.ppc ** 3, ntot, args.solver.upper(), args.order, args.u_th,
                                                ", random in-cell positions" if args.jitter else "",
                                                "on (1 pass)" if args.filter else "off (SURVEY 8d)",
                                                args.sort_interval)),
                       "state": "steady state: %d untimed spin-up steps + %d warm-up steps before the timed region "
                                "(the initial lattice has decayed into random in-cell positions)" % (args.spinup, args.warmup),
                       "use_filter": int(args.filter), "deposit_mode": int(args.deposit_mode), "gather_mode": int(args.gather_mode),
                       "brick_grid": list(nb), "l2": "inputs (%.1f GB of particles per GPU) exceed the 50 MB L2"
                                                     % (npart_local * 56 / 1e9)},
            "e2e": e2e, "gpu_launches": launches, "device": device_info(local), "clocks": clk, "roofline": roofline,
            "stage_ms": {k: v[0] for k, v in stage.items()}, "stage_calls": {k: v[1] for k, v in stage.items()},
            "stage_sum_ms_per_step": step_sum, "host_enqueue_ms_per_step": 1e3 * t_host_enqueue / args.steps,
            "field_energy_J": list(fe), "host_generation_s": t_gen}
    if args.profile_only:
        line["profile_only"] = True
    else:
        try:         # last: NCCL and the engines are gone, a slow or failing CPU leg cannot hang a collective
            cpu = cpu_reference_run(args.cpu_n, ppc, args.cpu_steps, 1, nox=args.order, use_filter=bool(args.filter),
                                    solver=args.solver)
            line["cpu_baseline"] = {k: cpu[k] for k in ("value", "unit", "cores", "kind", "sample")}
        except Exception as exc:     # noqa: BLE001 -- the GPU line must still be printed
            line["cpu_baseline"] = {"value": None, "unit": "particle-steps/s", "cores": 0, "kind": "port",
                                    "sample": "failed: %r" % (exc,)}
    emit_line(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="engine", choices=["engine", "reference"])
    ap.add_argument("--cells", dest="n", type=int, default=256, help="cells per GPU and direction")
    ap.add_argument("--cpu-cells", dest="cpu_n", type=int, default=128, help="cells per direction of the CPU sample")
    ap.add_argument("--cpu-steps", type=int, default=5, help="timed steps of the in-line cpu_baseline sample")
    ap.add_argument("--sort-interval", type=int, default=4)
    ap.add_argument("--spinup", type=int, default=60,
                    help="untimed steps before the warm-up that take the lattice to its steady state (0: measure the "
                         "fresh lattice)")
    ap.add_argument("--solver", default="yee", choices=["yee", "ckc"], help="algo.maxwell_solver (configs[2] uses ckc)")
    ap.add_argument("--profile-only", action="store_true", help="spin-up + warm-up + steps only (for runs under ncu)")
    ap.add_argument("--ppc", type=int, default=2, help="particles per cell and direction (2 -> 8 ppc, 4 -> 64 ppc)")
    ap.add_argument("--u-th", type=float, default=0.01, help="thermal momentum spread u/c")
    ap.add_argument("--jitter", action="store_true", help="stress variant: random positions inside the cells "
                    "instead of the NUniformPerCell lattice (particles cross cell faces from step 1)")
    ap.add_argument("--order", type=int, default=3)
    ap.add_argument("--filter", type=int, default=0, choices=[0, 1],
                    help="warpx.use_filter: bilinear current filter, 1 pass.  Off by default: SURVEY.md 8(d) "
                         "fixes use_filter = 0 for the benchmark configurations; --filter 1 measures the "
                         "reference's own default (WarpX.cpp:158)")
    ap.add_argument("--deposit-mode", type=int, default=0, choices=list(range(12)),
                    help="pic_set_deposit_mode: 0 register runs, 1 shared-memory tile block, 2 two lines per "
                         "lane, 3 per-slot reductions, 4 both, 5 four lines per lane, 6 four lines + per-slot reductions, "
                         "7 one lane per cell (every mode passes the parity tests)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what they computed as DIR/<name>.npy: the field energy, a "
                         "seeded sample of every field component and of the particles (by id), float64, < 64 MB")
    ap.add_argument("--gather-mode", type=int, default=0, choices=[0, 1, 2, 3],
                    help="pic_set_gather_mode: 0 one particle per lane (default), 1 two particles of a cell per lane, "
                         "2 the same without the 128-register cap (A/B measurement; same parity tests)")
    args = ap.parse_args()
    # Only the JSON line may reach stdout: libraries write there too (NCCL prints its version line when NCCL_DEBUG is
    # set).  Keep the original stdout for the line and point fd 1 at stderr for everybody else.
    global _LINE_FD
    sys.stdout.flush()
    _LINE_FD = os.dup(1)
    os.dup2(2, 1)
    if args.warmup < 3 and args.impl == "engine":
        args.warmup = 3
    if args.impl == "reference":
        run_reference(args)
    else:
        run_engine(args)
    # the line is out and flushed.  The handlers registered with atexit still run (a profiler or tracer may have output
    # to write); the interpreter's teardown of CUDA / NCCL state is skipped: nothing below may hang the job
    atexit._run_exitfuncs()
    sys.stdout.flush()
    sys.stderr.flush()
    os._exit(0)


if __name__ == "__main__":
    main()
