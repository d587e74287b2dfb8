"""CPU test: the restated analysis of Examples/Tests/flux_injection/analysis_flux_injection_3d.py (tests/
flux_deck_analysis.py) passes on the numpy restatement of the injection (tests/flux_oracle.py) run on the deck of
warpx_b200.workloads.flux_injection_3d, on a coarser grid with the same plane area and a larger number of particles per
cell (the same number of particles per step, so the histograms keep the deck's statistics)."""
import flux_deck_analysis as fda
import flux_oracle as fo
from warpx_b200 import workloads


def test_restated_deck_passes_the_analysis():
    wl = workloads.flux_injection_3d(n=8, ppc=400.0)
    data = fo.deck(wl)
    C = fo.C
    out = fda.check(wl, {k: dict(ux=v["ux"] / C, uy=v["uy"] / C, uz=v["uz"] / C, w=v["w"]) for k, v in data.items()},
                    wl["max_step"] * wl["dt"])
    assert len(out) == 12
    n = len(data["electron"]["w"])
    assert 2 * 8 * 8 * 400 <= n <= 2 * 8 * 8 * 401
