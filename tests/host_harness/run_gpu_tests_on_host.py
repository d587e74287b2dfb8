#!/usr/bin/env python3
"""TEST INFRASTRUCTURE -- runs the `-m gpu` test functions (tests/test_gpu_parity.py, tests/test_gpu_particle_sets.py,
tests/test_gpu_gauss.py, tests/test_gpu_zz_lwfa.py)
against the HOST build of the library (harness.host_library: every csrc file compiled by g++ against the SIMT emulator),
for a container without a GPU:

    python tests/host_harness/run_gpu_tests_on_host.py                     # everything (about an hour of emulation)
    python tests/host_harness/run_gpu_tests_on_host.py boosted nci order4  # the tests whose names contain one of the words
    python tests/host_harness/run_gpu_tests_on_host.py -langmuir_loop      # ... all but those containing the word

The test functions run unchanged, with their own tolerances.  Substitutions: warpx_b200.engine.Simulation -> the host
subclass of harness.host_simulation_class(); the library loader -> harness.host_library; the `cuda` fixture -> an
object whose synchronize() does nothing; the `dev` fixture -> the same helper with CPU tensors ("upload" = a copy).
The Gauss's-law module runs its cases at 16^3 for 8 steps (checkpoints 1, 4, 5, 8) instead of the benchmark's sizes.
This checks the step sequence, argument builders and kernel arithmetic; it cannot check races, launch bounds or
speed -- it does not replace the device run, and nothing in the product uses it."""
import inspect
import itertools
import json
import os
import sys
import time
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))

import pytest  # noqa: E402
import torch  # noqa: E402

from host_harness import harness  # noqa: E402
import warpx_b200.engine as engine  # noqa: E402
import warpx_b200.lib as piclib  # noqa: E402

engine.Simulation = harness.host_simulation_class()
piclib.lib = harness.host_library
torch.Tensor.cuda = lambda self, *a, **k: self.clone()          # "upload": a separate copy, like a device buffer


class _TorchOnHost:
    """torch, with device="cuda" read as the host and torch.cuda.* as no-ops."""

    def __getattr__(self, name):
        obj = getattr(torch, name)
        if callable(obj) and not isinstance(obj, type):
            def wrapped(*a, **k):
                if k.get("device") == "cuda":
                    k["device"] = "cpu"
                return obj(*a, **k)
            return wrapped
        return obj

    class cuda:
        @staticmethod
        def synchronize():
            pass

        @staticmethod
        def current_stream():
            class S:
                cuda_stream = None
            return S


import test_gpu_parity as TP  # noqa: E402
import test_gpu_particle_sets as TS  # noqa: E402
import test_gpu_gauss as TG  # noqa: E402
import test_gpu_zz_lwfa as TL  # noqa: E402
from oracle import oracle as orc  # noqa: E402


TG.BENCH_N = TG.MODE_N = TG.ORDER_N = 16
TG.CHECKPOINTS = TG.ORDER_CHECKPOINTS = (1, 4, 5, 8)
TG.bench_n = lambda t: TG.BENCH_N


class HostDev(TP.Dev):
    def __init__(self):
        self.t, self.L, self.keep = _TorchOnHost(), harness.host_library(), []

    @property
    def stream(self):
        return None

    def sync(self):
        pass


def cases(fn):
    marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]
    names = [[s.strip() for s in m.args[0].split(",")] for m in marks]
    for combo in itertools.product(*[m.args[1] for m in marks]):
        kw = {}
        for n, v in zip(names, combo):
            kw.update({n[0]: v} if len(n) == 1 else dict(zip(n, v)))
        yield kw


SKIP = {"test_full_size_properties": "benchmark-size arrays", "test_two_gpu_halo_and_migration": "spawns torchrun on two GPUs"}


def main():
    words = [w for w in sys.argv[1:] if not w.startswith("-")]
    minus = [w[1:] for w in sys.argv[1:] if w.startswith("-")]
    golden = json.load(open(os.path.join(TESTS, "golden", "warpx_checksums.json")))
    npass = nfail = 0
    for mod in (TP, TS, TG, TL):
        for name, fn in sorted(vars(mod).items()):
            if not name.startswith("test_") or not inspect.isfunction(fn) or fn.__module__ != mod.__name__:
                continue
            if (words and not any(w in name for w in words)) or any(w in name for w in minus):
                continue
            if name in SKIP:
                print("SKIP", name, "--", SKIP[name], flush=True)
                continue
            sig = inspect.signature(fn).parameters
            for kw in cases(fn):
                full = dict(kw)
                if "orc" in sig:
                    full["orc"] = orc
                if "dev" in sig:
                    full["dev"] = HostDev()
                if "cuda" in sig:
                    full["cuda"] = _TorchOnHost()
                if "golden" in sig:
                    full["golden"] = golden
                t = time.time()
                try:
                    fn(**full)
                    npass += 1
                    print("PASS %s %s %.1fs" % (name, kw or "", time.time() - t), flush=True)
                except pytest.skip.Exception as e:
                    print("SKIP", name, kw, "--", e, flush=True)
                except Exception:                                    # noqa: BLE001 -- reported, the run goes on
                    nfail += 1
                    print("FAIL", name, kw, flush=True)
                    traceback.print_exc()
    print("passed %d, failed %d" % (npass, nfail))
    return 1 if nfail else 0


if __name__ == "__main__":
    sys.exit(main())
