"""CPU test: the Gaussian-flux sampler of the restatement (tests/flux_oracle.py, the kernel's gaussian_flux restated) against
what the reference's own SampleGaussianFluxDistribution.H computes on the project's random streams --
tests/golden/flux_reference.npz, made by tests/golden/make_flux_reference.py from the header, unchanged.  Every sample
and the number of random words it consumed agree bit for bit."""
import os

import numpy as np
import pytest

import flux_oracle as fo
from collision_oracle import Streams

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flux_reference.npz"))
NAMES = sorted({k.split("/")[0] for k in Z.files})


def test_fixture_covers_the_cases():
    assert len(NAMES) == 8
    p = {n: Z[n + "/params"] for n in NAMES}
    assert any(v[0] == 0.0 for v in p.values()) and any(v[1] == 0.0 for v in p.values())
    assert any(0 < abs(v[0]) < 0.6 * v[1] for v in p.values()) and any(abs(v[0]) >= 0.6 * v[1] > 0 for v in p.values())
    assert any(v[0] < 0 for v in p.values())
    assert Z["long_rejection_runs/words"].max() > 1000


@pytest.mark.parametrize("name", NAMES)
def test_restated_sampler_reproduces_the_reference_header(name):
    u_m, u_th = (float(v) for v in Z[name + "/params"])
    seed, step, index, tag, n = (int(v) for v in Z[name + "/ints"])
    rng = Streams(seed, step, np.arange(n), fo.FLUX_BIT | index, np.full(n, tag, dtype=np.uint64))
    u = fo.gaussian_flux(u_m, u_th, rng, np.arange(n))
    assert np.array_equal(u.view(np.int64), Z[name + "/u"].view(np.int64))
    assert np.array_equal(rng.drawn, Z[name + "/words"])
