#!/usr/bin/env python3
"""Regenerates tests/golden/reference_leaves.json: SHA-256 digests of what the oracle computes with the reference's
own leaf headers compiled in (oracle/_ref/libpic_oracle_ref.so) on the seeded inputs of tests/helpers.py.

    make -C oracle ref REF=<WarpX source tree>
    python tests/golden/make_reference_leaves.py

The tests recompute the same outputs with the hand-restated leaves and compare the digests, so they pin the
restatement to the reference bit for bit without the reference tree."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import helpers  # noqa: E402
from oracle import oracle as orc  # noqa: E402

if not orc.have_ref():
    sys.exit("oracle/_ref/libpic_oracle_ref.so is missing: make -C oracle ref REF=<WarpX source tree>")
L = orc.lib("reference")
assert L.orc_leaf_name() == b"reference"


def digests(d):
    return {k: helpers.digest(v) for k, v in sorted(d.items())}


gold = {
    "_provenance": "oracle/pic_oracle.cpp with the leaf headers of ECP-WarpX/WarpX Source (ShapeFactors.H, "
                   "UpdateMomentum*.H, UpdatePosition.H, CartesianYeeAlgorithm.H, CartesianCKCAlgorithm.H) compiled "
                   "verbatim (oracle/leaf_reference.hpp); inputs and outputs: tests/helpers.py; digests: helpers.digest",
    "leaves": digests(helpers.leaf_outputs(orc, L)),
    "stages": digests(helpers.stage_outputs(orc, L)),
    "order4_loop": digests(helpers.order4_loop_fields(orc, "reference")),
    "shape_factors": {str(order): digests(helpers.shape_factor_outputs(order, L.orc_shape, L.orc_shifted_shape))
                      for order in (1, 2, 3, 4)},
}
out = os.path.join(HERE, "reference_leaves.json")
with open(out, "w") as f:
    json.dump(gold, f, indent=1, sort_keys=True)
    f.write("\n")
print("wrote", out)
