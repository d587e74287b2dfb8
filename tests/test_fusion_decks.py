"""CPU tests: the reference's acceptance checks of its 3D nuclear fusion decks (restated in tests/fusion_deck_analysis.py)
on the numpy restatements of the fusion stage (tests/fusion_oracle.py, tests/proton_boron_oracle.py) run over the decks of
warpx_b200.workloads with fewer particles per cell.  The statistical checks take their 5 sigma bounds from the counts;
a failure on the device then points at the kernels, not at the workloads or the analysis."""
import numpy as np
import pytest

import fusion_deck_analysis as fda
import fusion_oracle as fo
import proton_boron_oracle as po
from warpx_b200 import abi, workloads
from warpx_b200.engine import max_dt, nuclear_fusion_type

NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")


def _geom(wl):
    return dict(n_cell=wl["n_cell"], prob_lo=wl["prob_lo"], prob_hi=wl["prob_hi"], box_lo=(0, 0, 0),
                box_hi=tuple(v - 1 for v in wl["n_cell"]))


def _dt(wl):
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    return wl["cfl"] * max_dt(abi.SOLVER_YEE, dx)


def run_oracle(wl, steps=1):
    """the deck's fusion entries, in order, for `steps` steps; returns (start, end, neutron weight history)"""
    geom, dt = _geom(wl), _dt(wl)
    sp = wl["species"]
    state = {}
    for s in sp:
        n = len(s.get("x", ()))
        state[s["name"]] = {k: (np.array(s[k]) if n else np.zeros(0)) for k in NAMES}
        state[s["name"]]["id"] = np.arange(n, dtype=np.int64)
    start = {k: {a: v.copy() for a, v in d.items()} for k, d in state.items()}
    history = []
    for step in range(steps):
        for k, f in enumerate(wl["fusions"]):
            i, j = f["species"]
            types = [sp[n]["species_type"] for n in f["species"] + f["products"]]
            ftype = nuclear_fusion_type(types[:2], types[2:])
            coll = dict(m1=fda.fo_mass(sp[i]), m2=fda.fo_mass(sp[j]), mA=fda.fo_mass(sp[f["products"][0]]),
                        mB=fda.fo_mass(sp[f["products"][-1]]), type=ftype, fusion_multiplier=f["multiplier"],
                        fusion_probability_threshold=f["threshold"], fusion_probability_target_value=f["target"],
                        seed=wl["seed"], collision_index=k, same_species=int(i == j))
            s1, s2 = state[sp[i]["name"]], state[sp[j]["name"]]
            if ftype == abi.FUSION_PB_3HE4:
                r1, r2, al = po.fuse(s1, s2, coll, geom, dt, step)
                made = [al]
            else:
                r1, r2, pa, pb = fo.fuse(s1, s2, coll, geom, dt, step)
                made = [pa, pb]
            for n, r in ((sp[i]["name"], r1), (sp[j]["name"], r2)):
                if r is not None:
                    live = r["id"] != -1
                    state[n] = {a: v[live] for a, v in r.items()}
            for p, new in zip(f["products"], made):
                old = state[sp[p]["name"]]
                nxt = len(old["id"])
                state[sp[p]["name"]] = {a: np.concatenate([old[a], new[a] + (nxt if a == "id" else 0)]) for a in old}
        history.append(float(state[sp[-1]["name"]]["w"].sum()))
    return start, state, history, dt


@pytest.mark.parametrize("deck", ["fusion_dt_3d", "fusion_dd_3d", "proton_boron_3d"])
def test_oracle_deck_passes_the_restated_analysis(deck):
    wl = getattr(workloads, deck)(scale=0.05)
    start, end, _, dt = run_oracle(wl)
    out = fda.check_deck(wl, start, end, dt, reduced=True)
    assert any(k.endswith("yield_per_slice_sigma") for k in out)
    for s in wl["species"]:                                  # unique ids of every product species
        ids = end[s["name"]]["id"]
        assert np.unique(ids).size == ids.size


def test_oracle_intraspecies_deck_sigma_v():
    """<sigma v> from the neutron history: 2 % at the deck's size, here the 5 sigma bound of the event count when wider"""
    wl = workloads.fusion_dd_intraspecies_3d(scale=0.1)
    start, end, history, dt = run_oracle(wl, steps=wl["max_step"] + 1)
    times = dt * np.arange(len(history) + 1)
    hist = [0.0] + history
    sv = fda.sigma_v_intraspecies(wl, times, hist)
    events = len(end["neutron"]["w"]) / 2
    tol = max(wl["analysis"]["tolerance"], 5.0 / np.sqrt(events))
    assert abs(sv - wl["analysis"]["sigma_v"]) / wl["analysis"]["sigma_v"] < tol, (sv, events)
