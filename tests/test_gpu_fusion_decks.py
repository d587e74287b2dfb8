"""GPU tests (-m gpu): the reference's four 3D nuclear fusion decks at full size through Simulation (warpx_b200.workloads
fusion_dt_3d, fusion_dd_3d, fusion_dd_intraspecies_3d, proton_boron_3d), checked by the restated analyses of
tests/fusion_deck_analysis.py with the reference's own tolerances on what plotfiles written at the first and the last
step hold (read back by tests/plotfile_reader.py); ids and rho come from the run itself.  Each test prints the measured
values beside their tolerances and the fusion stage times."""
import json

import numpy as np
import pytest

import fusion_deck_analysis as fda
import plotfile_reader as pr
from warpx_b200 import workloads

pytestmark = pytest.mark.gpu


def build(wl):
    from warpx_b200.engine import Simulation
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"])
    for s in wl["species"]:
        if "x" in s:
            sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"],
                            species_type=s["species_type"])
        else:
            sim.add_empty_species(s["name"], s["capacity"], species_type=s["species_type"])
        sim.set_species_flags(s["name"], do_not_push=s["do_not_push"], do_not_deposit=s["do_not_deposit"])
    names = [s["name"] for s in wl["species"]]
    for f in wl["fusions"]:
        sim.add_fusion(names[f["species"][0]], names[f["species"][1]], [names[p] for p in f["products"]],
                       multiplier=f["multiplier"], probability_threshold=f["threshold"],
                       probability_target_value=f["target"], seed=wl["seed"])
    return sim, names


def state(root, wl):
    out = {}
    for s in wl["species"]:
        d = pr.read_species(root, s["name"])
        m = fda.fo_mass(s)
        out[s["name"]] = dict(x=d["position_x"], y=d["position_y"], z=d["position_z"], w=d["weight"],
                              ux=d["momentum_x"] / m, uy=d["momentum_y"] / m, uz=d["momentum_z"] / m)
    return out


def report(name, out, stages):
    print("DECK", name, json.dumps({k: [float(v[0]), float(v[1])] for k, v in out.items()}))
    print("STAGES", name, json.dumps({k: stages[k] for k in ("fusion", "fusion_products") if k in stages}))


@pytest.mark.parametrize("deck", ["fusion_dt_3d", "fusion_dd_3d", "proton_boron_3d"])
def test_deck_passes_the_restated_analysis(cuda, tmp_path, deck):
    from warpx_b200 import diagnostics
    wl = getattr(workloads, deck)()
    sim, names = build(wl)
    rho0 = sim.rho_numpy()[1]
    p0 = diagnostics.write_plotfile(sim, str(tmp_path / "plt"), 0)
    sim.enable_stage_timing()
    sim.Evolve(wl["max_step"])
    stages = sim.stage_ms()
    p1 = diagnostics.write_plotfile(sim, str(tmp_path / "plt"), wl["max_step"])
    out = fda.check_deck(wl, state(p0, wl), state(p1, wl), sim.dt)
    rho1 = sim.rho_numpy()[1]
    assert np.all(np.abs(rho1 - rho0) <= wl["analysis"]["rho_tol"] * np.abs(rho0))
    for isp in range(len(names)):
        ids = sim.species_numpy(isp)["id"]
        assert np.unique(ids).size == ids.size, names[isp]
    report(deck, out, stages)


def test_intraspecies_deck_sigma_v(cuda):
    wl = workloads.fusion_dd_intraspecies_3d()
    sim, names = build(wl)
    sim.enable_stage_timing()
    times, neutrons = [sim.time], [sim.particle_number()[2][1]]
    for _ in range(wl["max_step"]):
        sim.Evolve(1)
        times.append(sim.time)
        neutrons.append(sim.particle_number()[2][1])
    stages = sim.stage_ms()
    sv = fda.sigma_v_intraspecies(wl, times, neutrons)
    err = abs(sv - wl["analysis"]["sigma_v"]) / wl["analysis"]["sigma_v"]
    report("fusion_dd_intraspecies_3d", {"sigma_v_error": (err, wl["analysis"]["tolerance"])}, stages)
    assert err < wl["analysis"]["tolerance"], sv
