"""CPU tests: the reference's own acceptance tests of its 3D collision decks (Examples/Tests/collision/
analysis_collision_3d.py and analysis_collision_3d_isotropization.py), run through the numpy restatement of
tests/collision_oracle.py on the full decks of warpx_b200.workloads."""
import numpy as np

import collision_oracle as co
from warpx_b200 import workloads


def _deck(wl):
    geom = dict(n_cell=wl["n_cell"], prob_lo=wl["prob_lo"], prob_hi=wl["prob_hi"], box_lo=(0, 0, 0),
                box_hi=tuple(v - 1 for v in wl["n_cell"]))
    species = [dict(s, id=np.arange(len(s["x"]), dtype=np.int64)) for s in wl["species"]]
    return geom, species


def test_oracle_xyz_deck_passes_the_reference_analysis():
    """mean over steps 0, 10, ..., 150 of |a exp(b j) - (<ux>_e - <ux>_i)/c| < 0.001"""
    wl = workloads.collision_xyz_3d()
    geom, species = _deck(wl)
    an = wl["analysis"]
    err = []
    for j in range(0, wl["max_step"] + 1, 10):
        if j:
            co.deck_loop(species, wl["collisions"], geom, wl["dt"], 10, first_step=j - 10)
        vxd = species[0]["ux"].mean() / workloads.C - species[1]["ux"].mean() / workloads.C
        err.append(abs(an["a"] * np.exp(an["b"] * j) - vxd))
    assert np.mean(err) < an["tolerance"], np.mean(err)


def test_oracle_iso_deck_passes_the_reference_analysis():
    """Tx and Ty after 100 steps within 5 % of the analytic relaxation of the deck's anisotropic temperature"""
    wl = workloads.collision_iso_3d()
    geom, species = _deck(wl)
    co.deck_loop(species, wl["collisions"], geom, wl["dt"], wl["max_step"])
    an = wl["analysis"]
    e, me, dt = workloads.Q_E, workloads.M_E, wl["dt"]
    T_par, T_per = an["T_par"] * e, an["T_per"] * e
    A = 1.0 - T_per / T_par
    mu = (e ** 4 * an["ne"] * an["coulomb_log"] / (8.0 * np.pi ** 1.5 * workloads.EP0 ** 2 * me ** 0.5 * T_par ** 1.5)
          * A ** (-2) * (-3.0 + (3.0 - A) * np.arctanh(A ** 0.5) / A ** 0.5))
    Tx0, Ty0 = T_par, T_per
    for _ in range(wl["max_step"] - 1):
        Tx0 = Tx0 + dt * mu * (Ty0 - Tx0) * 2.0
        Ty0 = Ty0 + dt * mu * (Tx0 - Ty0)
    Tx = np.mean(species[0]["ux"] ** 2) * me / e
    Ty = np.mean(species[0]["uy"] ** 2) * me / e
    err = max(abs(Tx - Tx0 / e) / Tx, abs(Ty - Ty0 / e) / Ty)
    assert err < an["tolerance"], (Tx, Tx0 / e, Ty, Ty0 / e)
