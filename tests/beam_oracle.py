"""TEST INFRASTRUCTURE -- oracle of the Gaussian beam: WarpX's beam injection restated in numpy, operation by operation,
from given normals (warpx_b200.workloads.beam_normals, or the normals a library build reports with
pic_gaussian_beam_normals).  Every elementwise numpy operation is one IEEE rounding, as in the reference's CPU build,
so the result is bit-comparable with the library's (which keeps nvcc from contracting to FMA).

Restated (paths relative to Source/ of ECP-WarpX/WarpX):
  PhysicalParticleContainer::AddGaussianBeam            Particles/PhysicalParticleContainer.cpp:503-677
  PhysicalParticleContainer::CheckAndAddParticle        Particles/PhysicalParticleContainer.cpp:830-853
  PhysicalParticleContainer::MapParticletoBoostedFrame  Particles/PhysicalParticleContainer.cpp:456-500
  WarpXParticleContainer::AddNParticles (ids)           Particles/WarpXParticleContainer.cpp:163-240
  PhysicalParticleContainer::InitData -> Redistribute   Particles/PhysicalParticleContainer.cpp:450-454, with the
      oracle's semantics: amrex::enforcePeriodic (oracle/pic_oracle_core.hpp, wrap_periodic) along periodic axes,
      removal outside a non-periodic face (x < prob_lo or x > prob_hi, oracle/pic_oracle_lwfa.hpp).
The result goes into an oracle run with OracleSim.add_species (add_beam below)."""
import numpy as np

from warpx_b200 import workloads

C = workloads.C
NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")


def params(beam):
    """abi.pic_gaussian_beam -> plain Python values."""
    v = lambda a: np.array([float(a[d]) for d in range(3)])   # noqa: E731
    return dict(x_m=v(beam.x_m), rms=v(beam.rms), cut=v(beam.cut), blo=v(beam.bound_lo), bhi=v(beam.bound_hi),
                u_m=v(beam.u_m), u_th=v(beam.u_th), q_tot=float(beam.q_tot), npart=int(beam.npart),
                do_symmetrize=bool(beam.do_symmetrize), order=int(beam.symmetrization_order),
                do_focusing=bool(beam.do_focusing), focal_distance=float(beam.focal_distance), seed=int(beam.seed),
                gamma_boost=float(beam.gamma_boost), beta_boost=float(beam.beta_boost))


def ndraws(beam):
    p = params(beam)
    return p["npart"] // p["order"] if p["do_symmetrize"] else p["npart"]       # npart /= symmetrization_order (:530-532)


def creation_list(beam, charge, normals, t0=0.0):
    """AddGaussianBeam + CheckAndAddParticle for the draws whose normals are given (rows 0..ndraws-1, columns x y z ux
    uy uz first): the particles in the order the reference creates them; their index is their id."""
    p = params(beam)
    n = ndraws(beam)
    g = np.asarray(normals, dtype=np.float64)[:n]
    assert g.shape[0] == n and g.shape[1] >= 6
    weight = p["q_tot"] / (n * charge)                                           # :538
    x = [p["x_m"][d] + p["rms"][d] * g[:, d] for d in range(3)]                  # RandomNormal(x_m, x_rms) (:539-541)
    keep = np.ones(n, dtype=bool)
    for d in range(3):                                                           # insideBounds + cuts (:546-549)
        keep &= (x[d] < p["bhi"][d]) & (x[d] >= p["blo"][d])
        keep &= np.abs(x[d] - p["x_m"][d]) <= p["cut"][d] * p["rms"][d]
    x = [a[keep] for a in x]
    u = [p["u_m"][d] + p["u_th"][d] * g[keep, 3 + d] for d in range(3)]          # InjectorMomentumGaussian::getMomentum
    if p["do_focusing"]:                                                         # :559-593
        um = p["u_m"]
        norm = np.sqrt(um[0] * um[0] + um[1] * um[1] + um[2] * um[2])
        nv = [um[d] / norm for d in range(3)]
        xf = [p["x_m"][d] + p["focal_distance"] * nv[d] for d in range(3)]
        gamma = np.sqrt(1.0 + (u[0] * u[0] + u[1] * u[1] + u[2] * u[2]))
        v = [u[d] / gamma * C for d in range(3)]
        v_dot_n = v[0] * nv[0] + v[1] * nv[1] + v[2] * nv[2]
        t = ((xf[0] - x[0]) * nv[0] + (xf[1] - x[1]) * nv[1] + (xf[2] - x[2]) * nv[2]) / v_dot_n
        x = [x[d] - (v[d] - v_dot_n * nv[d]) * t for d in range(3)]
    u = [a * C for a in u]                                                       # :594-596
    m = len(x[0])
    if p["do_symmetrize"]:                                                       # :598-631, image by image
        imgs = [(x[0], x[1], u[0], u[1]), (x[0], -x[1], u[0], -u[1]), (-x[0], x[1], -u[0], u[1]),
                (-x[0], -x[1], -u[0], -u[1])]
        if p["order"] == 8:
            imgs += [(x[1], x[0], u[1], u[0]), (-x[1], x[0], -u[1], u[0]), (x[1], -x[0], u[1], -u[0]),
                     (-x[1], -x[0], -u[1], -u[0])]
        w = weight / 8.0 if p["order"] == 8 else weight / 4.0
    else:
        imgs = [(x[0], x[1], u[0], u[1])]
        w = weight
    k = len(imgs)
    out = dict(x=np.empty(m * k), y=np.empty(m * k), z=np.empty(m * k), w=np.full(m * k, w),
               ux=np.empty(m * k), uy=np.empty(m * k), uz=np.empty(m * k))
    for j, (a, b, ua, ub) in enumerate(imgs):                                    # draw-major, image-minor
        out["x"][j::k], out["y"][j::k], out["z"][j::k] = a, b, x[2]
        out["ux"][j::k], out["uy"][j::k], out["uz"][j::k] = ua, ub, u[2]
    if p["gamma_boost"] > 1.0:
        boost_map(out, p["gamma_boost"], p["beta_boost"], t0)
    out["id"] = np.arange(m * k, dtype=np.int64)                                 # AddNParticles: creation order
    return out


def boost_map(P, gamma_boost, beta_boost, t0):
    """MapParticletoBoostedFrame (:456-500) at t_lab = 0, forward propagation, transverse positions unchanged."""
    uz_boost = gamma_boost * beta_boost * C
    z, ux, uy, uz = P["z"], P["ux"], P["uy"], P["uz"]
    tpr = gamma_boost * 0.0 - uz_boost * z / (C * C)
    zpr = gamma_boost * z - uz_boost * 0.0
    gamma_lab = np.sqrt(1.0 + (ux * ux + uy * uy + uz * uz) / (C * C))
    uzp = gamma_boost * uz - uz_boost * gamma_lab
    gammapr = np.sqrt(1.0 + (ux * ux + uy * uy + uzp * uzp) / (C * C))
    vzpr = uzp / gammapr
    P["uz"] = uzp
    P["z"] = zpr - (tpr - t0) * vzpr


def redistribute(P, prob_lo, prob_hi, periodic):
    """InitData's Redistribute: wrap along periodic axes, drop beyond non-periodic faces (order kept)."""
    keep = np.ones(len(P["x"]), dtype=bool)
    for d, k in enumerate(("x", "y", "z")):
        lo, hi = float(prob_lo[d]), float(prob_hi[d])
        v = P[k].copy()
        if periodic[d]:
            ln = hi - lo
            up = v > hi
            while np.any(v[up] > hi):
                sel = up & (v > hi)
                v[sel] = v[sel] - ln
            v[up & (v < lo)] = lo
            dn = ~up & (v < lo)
            while np.any(v[dn] < lo):
                sel = dn & (v < lo)
                v[sel] = v[sel] + ln
            v[dn & (v > hi)] = hi
            P[k] = v
        else:
            keep &= ~((v < lo) | (v > hi))
    return {k: a[keep] for k, a in P.items()}


def gaussian_beam(beam, charge, normals, prob_lo, prob_hi, periodic, t0=0.0):
    """The beam of one box covering the domain, after InitData: dict of x y z w ux uy uz id."""
    return redistribute(creation_list(beam, charge, normals, t0), prob_lo, prob_hi, periodic)


def add_beam(osim, q, m, beam, normals=None, t0=0.0, periodic=(1, 1, 0)):
    """Put a beam species into an oracle run (single box): the restated beam, added like any species.  Returns the
    particles added (ids included), in the order the oracle keeps them."""
    if normals is None:
        normals = workloads.beam_normals(int(beam.seed), 0, ndraws(beam))
    plo, phi = osim.prob_domain()
    P = gaussian_beam(beam, q, normals, plo, phi, periodic, t0)
    osim.add_species(q, m, *[P[k] for k in NAMES])
    return P
