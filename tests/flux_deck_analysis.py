"""TEST INFRASTRUCTURE -- Examples/Tests/flux_injection/analysis_flux_injection_3d.py restated for the flux deck of
warpx_b200.workloads.flux_injection_3d: each species' momenta (in units of c) histogrammed over [-0.5, 0.5] in 50 bins,
weighted by w / du, against N_tot = flux * 64 m^2 * t_max times the Gaussian of u_th (the transverse axes, within 0.07
of the expected peak) and the Gaussian-flux distribution of u_m, u_th (the normal axis, its sign flipped for
flux_direction = -1, within 0.05).  check() returns {name/axis: (measured max |hist - expected| / expected peak,
tolerance)}."""
import numpy as np
from scipy.special import erf


def gaussian_dist(u, u_th):
    return 1.0 / ((2 * np.pi) ** 0.5 * u_th) * np.exp(-(u ** 2) / (2 * u_th ** 2))


def gaussian_flux_dist(u, u_th, u_m):
    normalization_factor = u_th ** 2 * np.exp(-(u_m ** 2) / (2 * u_th ** 2)) + (np.pi / 2) ** 0.5 * u_m * u_th * (
        1 + erf(u_m / (2 ** 0.5 * u_th)))
    return 1.0 / normalization_factor * np.where(u > 0, u * np.exp(-((u - u_m) ** 2) / (2 * u_th ** 2)), 0)


def _compare(u, w, expected, Ntot, a, tol):
    du = (a["hist_range"][1] - a["hist_range"][0]) / a["hist_bins"]
    w_hist, edges = np.histogram(u, bins=a["hist_bins"], weights=w / du, range=a["hist_range"])
    centres = 0.5 * (edges[1:] + edges[:-1])
    w_th = Ntot * expected(centres)
    ok = bool(np.allclose(w_hist, w_th, atol=tol * w_th.max()))
    return float(np.abs(w_hist - w_th).max() / w_th.max()), ok


def check(wl, data, t_max):
    """data: {species name: dict with ux, uy, uz (units of c) and w}; raises AssertionError naming the first failure"""
    a = wl["analysis"]
    Ntot = a["flux"] * a["emission_surface"] * t_max
    out, failed = {}, []
    for s in wl["species"]:
        f = s["flux"]
        axis = "xyz".index(f["flux_normal_axis"]) if isinstance(f["flux_normal_axis"], str) else f["flux_normal_axis"]
        d = data[s["name"]]
        for k, comp in enumerate(("ux", "uy", "uz")):
            u_th = f["u_th"][k]
            if k == axis:
                u = d[comp] if f["flux_direction"] > 0 else -d[comp]
                u_m = f["u_m"][k]
                err, ok = _compare(u, d["w"], lambda c: gaussian_flux_dist(c, u_th, u_m), Ntot, a, a["flux_tol"])
                tol = a["flux_tol"]
            else:
                err, ok = _compare(d[comp], d["w"], lambda c: gaussian_dist(c, u_th), Ntot, a, a["gaussian_tol"])
                tol = a["gaussian_tol"]
            key = "%s/%s" % (s["name"], comp)
            out[key] = (err, tol)
            if not ok:
                failed.append(key)
    assert not failed, ("flux deck analysis failed", failed, out)
    return out
