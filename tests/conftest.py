import json
import os
import sys

import pytest

# The oracle is OpenMP code on all host cores.  Let idle threads sleep instead of spinning, so that a box that is
# shared (or grants fewer cores than it reports) does not turn every barrier into a time slice: set before libgomp loads.
os.environ.setdefault("OMP_WAIT_POLICY", "passive")
try:
    os.environ.setdefault("OMP_NUM_THREADS", str(max(1, len(os.sched_getaffinity(0)))))
except AttributeError:            # not Linux
    pass
os.environ.setdefault("GOMP_SPINCOUNT", "0")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """Whole-deck golden runs go last: a failing deck (under the driver's -x) must not keep the stage-level parity
    cases -- kernel variants, charge deposition -- from running at all (stable order otherwise)."""
    # ... and behind them the stage cases of the kernel that was rewritten after the last single-GPU run of the round (the
    # streaming bilinear filter: on devices it has only run inside the 8-GPU check -- these cases must not be able to
    # stop anything else)
    unproven = ("test_bilinear_filter_three_components_in_one_launch", "test_bilinear_filter_matches_oracle")
    items.sort(key=lambda it: 2 if it.name.startswith(unproven) else (1 if "golden_checksum" in it.name else 0))


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "warpx_checksums.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def reference_leaves():
    """Digests of what the reference's own leaf headers compute on the seeded inputs of tests/helpers.py."""
    with open(os.path.join(ROOT, "tests", "golden", "reference_leaves.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle module (test infrastructure)."""
    from oracle import oracle
    oracle.build(ref=True)
    return oracle


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch
