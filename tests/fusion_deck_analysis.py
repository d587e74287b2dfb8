"""TEST INFRASTRUCTURE -- the acceptance checks of the reference's 3D nuclear fusion decks (Examples/Tests/nuclear_fusion/
analysis_two_product_fusion.py, analysis_proton_boron_fusion.py, analysis_deuterium_deuterium_3d_intraspecies.py),
restated in this project's terms for the decks of warpx_b200.workloads.

A state is {species name: dict(x, y, z, w, ux, uy, uz)} (u in m/s, as the engine stores it).  check_deck(wl, start, end,
dt) applies, per fusion set of the deck: conservation of weight, charge, momentum and energy (with the reaction's Q), the
number of product macroparticles (5 sigma), the yield per z slice against the cross section (5 sigma), isotropy, and for
proton-boron the thermal yield against the Tentori-Belloni reactivity fit and the boron of sets 4 and 5.  It returns the
measured values beside their tolerances."""
import numpy as np

import fusion_oracle as fo
import proton_boron_oracle as po

C = fo.C
C_SQ = fo.C_SQ
Q_E = fo.Q_E
REACTION = {"dt": fo.DT_NHE4, "dd": fo.DD_NHE3}


def kinetic(m, s):
    """sum of w (gamma - 1) m c^2"""
    usq = (s["ux"] ** 2 + s["uy"] ** 2 + s["uz"] ** 2) / C_SQ
    return float(np.sum(s["w"] * m * C_SQ * usq / (np.sqrt(1.0 + usq) + 1.0)))


def momentum(m, s):
    return np.array([np.sum(s["w"] * m * s[k]) for k in ("ux", "uy", "uz")])


def _rel(a, b, scale=None):
    return abs(a - b) / (abs(b) if scale is None else scale)


def _slices(s, nz):
    return np.histogram(s["z"], bins=nz, range=(0, nz), weights=s["w"])[0]


def _thermal_sigma_v(T, m_reduced):
    """Maxwellian <sigma v> [m^3/s] of p + B11 at T keV (< 70 keV): the non-resonant saddle-point estimate with the
    low-energy polynomial of the Tentori-Belloni S factor, plus the 148 keV resonance (Tentori & Belloni 2023, eqs. for the
    low-energy thermal reactivity)"""
    a = Q_E * Q_E * 5.0 / (2.0 * po.EP0 * po.HBAR)
    E_G = m_reduced / 2.0 * a * a / (1e3 * Q_E)     # Gamow energy [keV] (the factor of ProtonBoronFusionCrossSection)
    E0 = (E_G / 4.0) ** (1.0 / 3.0) * T ** (2.0 / 3.0)
    dE0 = 4.0 * np.sqrt(T * E0 / 3.0)
    tau = 3.0 * E0 / T
    S = (197.0e3 * (1.0 + 5.0 / (12.0 * tau)) + 0.269e3 * (E0 + 35.0 / 36.0 * T) +
         2.54e-4 * 1e3 * (E0 * E0 + 89.0 / 36.0 * E0 * T))
    nonres = np.sqrt(2.0 * T * 1e3 * Q_E / m_reduced) * dE0 * S / (T * T) * np.exp(-tau) * 1e-28
    return nonres + 5.41e-21 * np.exp(-148.0 / T) / T ** 1.5


def check_deck(wl, start, end, dt, reduced=False):
    """every check of the deck's analysis; returns {check: (measured, tolerance)} and raises on a failed check.
    reduced: a deck with fewer particles per cell than the reference's; the isotropy and thermal-yield tolerances widen
    to 5 sigma of what the events measure when that is larger (relative variance 4/5 of p_x^2 for isotropic directions;
    the compound-Poisson variance of the yield)."""
    an = wl["analysis"]
    sp = wl["species"]
    name = [s["name"] for s in sp]
    mass = {s["name"]: fo_mass(s) for s in sp}
    charge = {s["name"]: s_charge(s) for s in sp}
    nx, ny, nz = wl["n_cell"]
    dV_slice = nx * ny * (wl["prob_hi"][0] - wl["prob_lo"][0]) / nx * (wl["prob_hi"][1] - wl["prob_lo"][1]) / ny * \
        (wl["prob_hi"][2] - wl["prob_lo"][2]) / nz
    pb = an["reaction"] == "pb"
    out = {}
    for k, st in enumerate(an["sets"]):
        r1, r2 = (name[i] for i in st["reactants"])
        prods = [name[i] for i in st["products"]]
        tag = "set%d/" % (k + 1)
        W = {n: (float(start[n]["w"].sum()) if n in start else 0.0, float(end[n]["w"].sum())) for n in [r1, r2] + prods}
        c1, c2 = W[r1][0] - W[r1][1], W[r2][0] - W[r2][1]
        scale = max(W[r1][0], W[r2][0])
        assert c1 >= 0 and c2 >= 0
        out[tag + "weight_reactants"] = (_rel(c1, c2, scale), an["tol"])
        for p in prods:
            made = W[p][1] / (3.0 if pb else 1.0)
            out[tag + "weight_" + p] = (_rel(made, c1, scale), an["tol"])
        names = [r1, r2] + prods
        q0 = sum(charge[n] * W[n][0] for n in names)
        q1 = sum(charge[n] * W[n][1] for n in names)
        out[tag + "charge"] = (_rel(q1, q0, max(abs(charge[r1]) * W[r1][0], abs(charge[r2]) * W[r2][0])), an["tol"])
        p0 = sum(momentum(mass[n], start[n]) for n in names if n in start)
        p1 = sum(momentum(mass[n], end[n]) for n in names)
        pscale = sum(np.abs(momentum(mass[n], start[n])).sum() for n in (r1, r2)) + 1e-300
        out[tag + "momentum"] = (float(np.abs(p1 - p0).max() / pscale), an["tol"])
        Q = po.Q_TOTAL if pb else fo.E_FUSION[REACTION[an["reaction"]]]
        e0 = sum(kinetic(mass[n], start[n]) for n in names if n in start)
        e1 = sum(kinetic(mass[n], end[n]) for n in names)
        n_reactions = W[prods[0]][1] / (3.0 if pb else 1.0)
        out[tag + "energy"] = (_rel(e1, e0 + Q * n_reactions), an["energy_tol"])
        if "densities" not in st and not (pb and k == 2):
            continue
        # product macroparticles and isotropy
        per_event = 6 if pb else 2
        nprod = len(end[prods[0]]["w"])
        if "densities" in st:
            expected = nx * ny * (nz - 1) * st["pairs_per_cell"] * st["target"]
            out[tag + "macroparticles"] = (abs(nprod - per_event * expected) / (per_event * np.sqrt(expected)), 5.0)
        floor = 5.0 * np.sqrt(2.0 * 0.8 / max(nprod / per_event, 1.0)) if reduced else 0.0
        for p in prods:
            pp = [np.mean((end[p][c] * mass[p]) ** 2) for c in ("ux", "uy", "uz")]
            if st.get("beam_only"):
                out[tag + "xy_isotropy_" + p] = (_rel(pp[0], pp[1]), max(an["xy_isotropy"], floor))
                assert pp[2] > pp[0] and pp[2] > pp[1]
            else:
                iso = an["thermal_isotropy"] if (pb and k == 2) else an["isotropy"]
                out[tag + "isotropy_" + p] = (max(_rel(pp[0], pp[1]), _rel(pp[0], pp[2])), max(iso, floor))
        if pb and k == 2:
            th = an["thermal"]
            m1, m2 = mass[r1], mass[r2]
            V = dV_slice * nz
            want = 3.0 * th["n_p"] * th["n_b"] * _thermal_sigma_v(th["T_keV"], m1 * m2 / (m1 + m2)) * V * dt
            a = end[prods[0]]["w"]
            # a reduced deck: 5 sigma of the compound-Poisson yield (each event adds six alphas of equal weight)
            floor = 5.0 * np.sqrt(6.0 * np.sum(a * a)) / max(np.sum(a), 1e-300) if reduced else 0.0
            out[tag + "thermal_yield"] = (_rel(W[prods[0]][1], want), max(th["tolerance"], floor))
            continue
        # yield per z slice against the cross section at the slice's momenta
        m1, m2 = mass[r1], mass[r2]
        u1 = [np.zeros(nz), np.zeros(nz), _slice_u(start[r1], nz, st.get("beam_only"))]
        u2 = [np.zeros(nz), np.zeros(nz), _slice_u(start[r2], nz, st.get("beam_only"))]
        E, v, lab_to_com = fo.collision_parameters(u1, u2, m1, m2)
        sigma = po.cross_section(E) if pb else fo.bosch_hale(E, REACTION[an["reaction"]], m1, m2)
        theory = st["densities"][0] * st["densities"][1] * sigma * v * lab_to_com * dV_slice * dt * (3.0 if pb else 1.0)
        std = 1.0 / np.sqrt(expected / (nz - 1))
        worst = 0.0
        for p in prods:
            got = _slices(end[p], nz)
            worst = max(worst, float(np.max(np.abs(got[1:] - theory[1:]) / (theory[1:] * std))))
            assert got[0] == 0.0
        out[tag + "yield_per_slice_sigma"] = (worst, 5.0)
    if pb:
        out["set4/boron_left"] = (len(end[name[an["sets"][3]["reactants"][1]]]["w"]), 0)
        out["set5/boron_left"] = (len(end[name[an["sets"][4]["reactants"][1]]]["w"]), 1)
    bad = {k: v for k, v in out.items() if not _ok(k, v)}
    assert not bad, bad
    return out


def _ok(k, v):
    got, tol = v
    if k == "set4/boron_left":
        return got == 0
    if k == "set5/boron_left":
        return got >= tol
    return got <= tol


def _slice_u(s, nz, beam_only):
    """uz of the species in each z slice (constant per slice in the decks; the moving part for a beam on a background)"""
    out = np.zeros(nz)
    for j in range(nz):
        sel = (s["z"] >= j) & (s["z"] < j + 1)
        if beam_only:
            sel &= s["uz"] != 0.0
        if sel.any():
            out[j] = s["uz"][sel][0]
    return out


def fo_mass(s):
    from warpx_b200.engine import species_charge_mass
    return species_charge_mass(s["species_type"])[1]


def s_charge(s):
    from warpx_b200.engine import species_charge_mass
    return species_charge_mass(s["species_type"])[0]


def sigma_v_intraspecies(wl, times, neutron_weights):
    """<sigma v> [cm^3/s] from the neutrons' weight history: dY/dt (1 + delta_ij) / n^2 / V"""
    an = wl["analysis"]
    dY_dt = abs(neutron_weights[-1] - neutron_weights[0]) / (times[-1] - times[0])
    return dY_dt * 2.0 / an["density"] ** 2 / an["volume"] * 1e6
