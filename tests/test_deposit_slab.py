"""CPU tests (-m "not gpu"): the register-run deposition kernel of warpx_b200/csrc/deposit_runs.cu with its per-warp
shared-memory J slab (PIC_DEPOSIT_RUNS_SLAB) and without it (the default, PIC_DEPOSIT_RUNS), under the SIMT emulator of
tests/host_harness, against the oracle on a steady-state particle set: a thermal plasma evolved by the oracle, cell
sorted as the engine sorts it, then evolved three more steps -- so the deposited step has particles that changed cell
(movers), particles that drifted out of their sorted place (lone strays) and warps whose span leaves one slab (rebases).
The kernel is built here with -DPIC_DEPOSIT_COUNTERS, which counts those events; the library never sets it.

    python tests/test_deposit_slab.py      # prints the counts per deposited step (steady state, 32 x 32 x 16 x 8 ppc)"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import particle_sets as ps  # noqa: E402
from helpers import lower_corner, rel_linf  # noqa: E402
from particle_sets import steady_state  # noqa: E402
from warpx_b200 import abi, workloads  # noqa: E402

COUNTERS = ("chunks", "particles", "movers", "runs", "slides", "jumps", "lones", "lones_outside", "rebases", "cells",
            "red_retire", "red_lone", "red_slab")
VARIANT_SLAB = 8        # g_runs_variant of PIC_DEPOSIT_RUNS_SLAB


def counting_simt():
    """The SIMT build of tests/host_harness with the event counters compiled in (its own library file)."""
    from host_harness import harness
    out = os.path.join(harness.HERE, "_build", "libpic_simt_counters.so")
    deps = [os.path.join(harness.HERE, f) for f in ("simt_host.h", "simt_deposit.cpp")] + \
           [os.path.join(harness.CSRC, f) for f in ("deposit_runs.cu", "deposit_common.cuh", "pic_common.cuh", "runtime.cu")] + \
           [os.path.join(harness.ROOT, "include", "pic_b200.h")]
    if not (os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cuda = os.path.dirname(os.path.dirname(harness.NVCC))
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-DPIC_SIMT_HOST", "-DPIC_DEPOSIT_COUNTERS",
                        "-include", os.path.join(harness.HERE, "simt_host.h"), "-x", "c++", "-I", os.path.join(cuda, "include"),
                        "-I", harness.CSRC, "-ffp-contract=off", "-Wno-attributes", "-Wno-unknown-pragmas",
                        os.path.join(harness.HERE, "simt_deposit.cpp"), os.path.join(harness.CSRC, "runtime.cu"), "-o", out,
                        "-L", os.path.join(cuda, "lib64"), "-lcudart"], check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    L = C.CDLL(out)
    L.simt_deposit_runs.restype = C.c_int
    L.simt_deposit_runs.argtypes = [C.POINTER(abi.pic_soa), C.c_long, C.c_long, C.POINTER(abi.pic_fab), abi.c_double_p,
                                    abi.c_double_p, abi.c_int_p, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int]
    L.pic_runs_counters.argtypes = [C.POINTER(C.c_long), C.c_int]
    return L


def deposit_both(L, wl, dt, p, variant, nox=3):
    from oracle import oracle as orc
    n = wl["n_cell"]
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    q = wl["species"][0]["q"]
    P = orc.HostParticles(**{k: p[k] for k in orc.HostParticles.NAMES})
    ngJ = (nox + 2,) * 3
    xyzmin, lo = lower_corner(prob_lo, dx, (0, 0, 0), ngJ)
    box_hi = tuple(v - 1 for v in n)
    J = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    K = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                           abi.int3(lo), q, dt, -0.5 * dt, nox) == 0
    cnt = (C.c_long * len(COUNTERS))()
    L.pic_runs_counters(cnt, 1)
    assert L.simt_deposit_runs(C.byref(P.soa), 0, P.np, orc.fab_array(K), abi.dbl3(dinv), abi.dbl3(xyzmin),
                               abi.int3(lo), q, dt, -0.5 * dt, nox, variant) == 0
    L.pic_runs_counters(cnt, 1)
    return J, K, dict(zip(COUNTERS, cnt))


@pytest.fixture(scope="module")
def state():
    wl, dt, p, _ = steady_state()
    return counting_simt(), (wl, dt, p)


@pytest.mark.parametrize("variant", [0, VARIANT_SLAB])
def test_run_kernel_matches_oracle_in_steady_state(orc, state, variant):
    L, (wl, dt, p) = state
    J, K, cnt = deposit_both(L, wl, dt, p, variant)
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]
    # the paths this state is meant to exercise did run
    assert cnt["movers"] > 0 and cnt["lones"] > 0 and cnt["jumps"] > 0 and cnt["slides"] > 0
    if variant == VARIANT_SLAB:
        assert cnt["rebases"] > 0 and cnt["red_slab"] > 0 and cnt["red_retire"] == 0
        assert cnt["lones"] > cnt["lones_outside"]           # strays inside the slab stay in shared memory
    else:
        assert cnt["rebases"] == 0 and cnt["red_slab"] == 0 and cnt["red_retire"] > 0


@pytest.mark.parametrize("variant", [0, VARIANT_SLAB])
@pytest.mark.parametrize("name", ["steady", "poisson", "crowded_movers"])
def test_run_kernel_matches_oracle_on_particle_sets(orc, state, name, variant):
    """The sets of tests/particle_sets.py (log-uniform weights; Poisson counts with runs longer than a warp's span;
    a supercell of diagonal movers) through both retire paths, order 3."""
    L = state[0]
    s = ps.get(name)
    wl = dict(n_cell=s.n, prob_lo=s.prob_lo, prob_hi=s.prob_hi, species=[dict(q=s.q)])
    J, K, cnt = deposit_both(L, wl, s.dt, s.p, variant)
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]
    # the kernel classifies the particles as the numpy restatement of tests/test_particle_sets.py does
    want = ps.quiet_kernel_events(s, 3, (5, 5, 5))
    assert cnt["movers"] == want["movers"] and cnt["lones"] == want["lones"], (cnt, want)
    assert cnt["runs"] > 0 and (name != "steady" or cnt["lones"] > 0)
    if variant == VARIANT_SLAB:
        assert cnt["red_slab"] > 0 and cnt["red_retire"] == 0


def main():
    """Counts per deposited step over one sort interval (1..4 steps after the sort), both retire paths."""
    L = counting_simt()
    tot = {v: dict.fromkeys(COUNTERS, 0) for v in (0, VARIANT_SLAB)}
    for k in range(4):
        wl, dt, p, _ = steady_state(n=(32, 32, 16), u_th=0.01, steps=60, after_sort=k + 1)
        for v in tot:
            _, _, cnt = deposit_both(L, wl, dt, p, v)
            for f in COUNTERS:
                tot[v][f] += cnt[f] / 4.0
    for v, c in tot.items():
        cells = max(c["cells"], 1)
        print("%s: %s" % ("slab" if v == VARIANT_SLAB else "L2  ", " ".join("%s %.0f" % kv for kv in c.items())))
        print("      per particle: movers %.4f lones %.4f jumps %.4f   per visited cell: reductions to J %.2f "
              "(retire %.2f, lone %.2f, slab flush %.2f)" %
              (c["movers"] / c["particles"], c["lones"] / c["particles"], c["jumps"] / c["particles"],
               (c["red_retire"] + c["red_lone"] + c["red_slab"]) / cells, c["red_retire"] / cells, c["red_lone"] / cells,
               c["red_slab"] / cells))


if __name__ == "__main__":
    main()
