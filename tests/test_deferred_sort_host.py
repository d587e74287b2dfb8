"""CPU tests: the two halves of the cell sort and the gather + push that carries out a pending sort
(pic_gather_push_permuted, the PERM instantiation of gather_push_tile_kernel), compiled from the product's sources for
the SIMT host emulator -- the host twin of tests/test_gpu_deferred_sort.py.  TEST INFRASTRUCTURE."""
import pytest

import deferred_sort_cases as cases
from warpx_b200 import abi


@pytest.fixture(scope="module")
def be():
    import torch
    from host_harness import harness
    return cases.Backend(torch, harness.host_library(), "cpu")


@pytest.mark.parametrize("name", ["steady", "poisson", "faces"])
def test_index_then_apply_is_the_sort_on_the_host(be, name):
    cases.check_index_apply_is_the_sort(be, name)


@pytest.mark.parametrize("name,nox,pusher,stag,stale", [
    ("steady", 3, abi.PUSHER_BORIS, "yee", False), ("steady", 3, abi.PUSHER_BORIS, "yee", True),
    ("scrambled_rows", 3, abi.PUSHER_VAY, "yee", True), ("faces", 1, abi.PUSHER_BORIS, "nodal", True)])
def test_permuting_gather_push_is_apply_then_push_on_the_host(be, orc, name, nox, pusher, stag, stale):
    cases.check_permuting_push_is_apply_then_push(be, orc, name, nox, 1, pusher, stag, stale_bins=stale)
