#!/usr/bin/env python3
"""Regenerates tests/golden/warpx_checksums.json and nci_godfrey_lines.json from a WarpX source tree:

    python tests/golden/make_golden.py <WarpX source tree>

The values are WarpX's own regression checksums for the tests that pin the hot path
(SURVEY.md section 8c): the 3D Langmuir wave (full loop, order 1), the force-free particle pusher and
the 3D laser-acceleration deck (full loop at order 3 with the bilinear filter, PEC walls, the moving
window, the laser antenna and continuous injection -- no RNG in that deck).
Nothing else is taken from the reference."""
import json
import os
import sys

WARPX = sys.argv[1]
REF = os.path.join(WARPX, "Regression", "Checksum", "benchmarks_json")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "warpx_checksums.json")

gold = {
    "_provenance": {
        "source": "ECP-WarpX/WarpX Regression/Checksum/benchmarks_json/{test_3d_langmuir_multi,test_3d_particle_pusher,test_3d_laser_acceleration,test_3d_pec_field,test_3d_pec_particle,test_3d_laser_injection,test_3d_particle_boundaries}.json",
        "tolerance": "rtol 1e-9, atol 1e-40 (Regression/Checksum/checksum.py:219-301)",
        "decks": ["Examples/Tests/langmuir/inputs_test_3d_langmuir_multi",
                  "Examples/Tests/particle_pusher/inputs_test_3d_particle_pusher",
                  "Examples/Physics_applications/laser_acceleration/inputs_test_3d_laser_acceleration",
                  "Examples/Tests/pec/inputs_test_3d_pec_field", "Examples/Tests/pec/inputs_test_3d_pec_particle",
                  "Examples/Tests/laser_injection/inputs_test_3d_laser_injection",
                  "Examples/Tests/boundaries/inputs_test_3d_particle_boundaries"],
        "pusher_expected_error": {"boris": 2321.3958529, "vay": 0.00010467, "higuera_cary": 0.00011403,
                                  "source": "Examples/Tests/particle_pusher/analysis.py:17-21"},
    }
}
for name in ("test_3d_langmuir_multi", "test_3d_particle_pusher", "test_3d_laser_acceleration", "test_3d_pec_field",
             "test_3d_pec_particle", "test_3d_laser_injection", "test_3d_particle_boundaries"):
    with open(os.path.join(REF, name + ".json")) as f:
        gold[name] = json.load(f)
with open(OUT, "w") as f:
    json.dump(gold, f, indent=1, sort_keys=True)
print("wrote", OUT)

# ---- a few lines of the Godfrey NCI-corrector coefficient tables (Source/Utils/NCIGodfreyTables.H): the lines
# the parity tests interpolate between for c dt / dz = 0, 0.5, 0.9 / sqrt(3), 0.98 and 1.  The tables are fitted
# data of the reference; a WarpX build passes the stencils it computed from them through the C ABI
# (pic_apply_nci_filter), the tests need a handful of lines to check the restated interpolation.
import re

TABLES = os.path.join(WARPX, "Source", "Utils", "NCIGodfreyTables.H")
OUT2 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "nci_godfrey_lines.json")
text = open(TABLES).read()
tab_length = int(re.search(r"const int tab_length = (\d+);", text).group(1))
tab_width = int(re.search(r"const int tab_width = (\d+);", text).group(1))
lines = {"_provenance": {"source": "ECP-WarpX/WarpX Source/Utils/NCIGodfreyTables.H (lines 0,1,50-53,98-100 of each table)",
                         "tab_length": tab_length, "tab_width": tab_width}}
WANT = (0, 1, 50, 51, 52, 53, 98, 99, 100)
for m in re.finditer(r"table_nci_godfrey_(\w+)\[tab_length\]\[tab_width\]\{(.*?)\};", text, re.S):
    rows = re.findall(r"\{([^{}]*)\}", m.group(2))
    assert len(rows) == tab_length
    parsed = [[float(v.replace("_rt", "")) for v in r.split(",")] for r in rows]
    lines[m.group(1)] = {str(i): parsed[i] for i in WANT}
with open(OUT2, "w") as f:
    json.dump(lines, f, indent=1, sort_keys=True)
print("wrote", OUT2)
