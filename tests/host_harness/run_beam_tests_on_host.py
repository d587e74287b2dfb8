#!/usr/bin/env python3
"""TEST INFRASTRUCTURE -- runs the `-m gpu` test functions of tests/test_gpu_beam.py against the HOST build of the
library, for a container without a GPU, with the substitutions of run_gpu_tests_on_host.py (host Simulation, host
library, `cuda` fixture read as the host):

    python tests/host_harness/run_beam_tests_on_host.py            # all five (a few minutes of emulation)
    python tests/host_harness/run_beam_tests_on_host.py bricks     # the tests whose names contain one of the words

The functions run unchanged, with their own tolerances.  Like the other runner it checks argument builders, kernel
arithmetic and the step sequence, not races, launch bounds or speed; nothing in the product uses it."""
import inspect
import os
import sys
import time
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))

import pytest  # noqa: E402

from host_harness import run_gpu_tests_on_host as R  # noqa: E402  (installs the host substitutions)
import test_gpu_beam as TB  # noqa: E402


def main():
    words = [w for w in sys.argv[1:] if not w.startswith("-")]
    npass = nfail = 0
    for name, fn in sorted(vars(TB).items()):
        if not name.startswith("test_") or not inspect.isfunction(fn) or fn.__module__ != TB.__name__:
            continue
        if words and not any(w in name for w in words):
            continue
        sig = inspect.signature(fn).parameters
        for kw in R.cases(fn):
            full = dict(kw)
            if "orc" in sig:
                full["orc"] = R.orc
            if "cuda" in sig:
                full["cuda"] = R._TorchOnHost()
            t = time.time()
            try:
                fn(**full)
                npass += 1
                print("PASS %s %s %.1fs" % (name, kw or "", time.time() - t), flush=True)
            except pytest.skip.Exception as e:
                print("SKIP", name, kw, "--", e, flush=True)
            except Exception:                                        # noqa: BLE001 -- reported, the run goes on
                nfail += 1
                print("FAIL", name, kw, flush=True)
                traceback.print_exc()
    print("passed %d, failed %d" % (npass, nfail))
    return 1 if nfail else 0


if __name__ == "__main__":
    sys.exit(main())
