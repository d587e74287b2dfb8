#!/usr/bin/env python3
"""Regenerates tests/golden/fusion_reference.npz: what the reference's own fusion headers compute.

    python tests/golden/make_fusion_reference.py <WarpX source tree>

A small C++ program includes, from the given tree and unchanged, Source/Particles/Collision/BinaryCollision/
NuclearFusion/SingleNuclearFusionEvent.H (with BoschHaleFusionCrossSection.H and BinaryCollisionUtils.H's
get_collision_parameters and remove_weight_from_colliding_particle), NuclearFusion/TwoProductFusionUtil.H and
ShuffleFisherYates.H, against a stand-in written here: the AMReX macros, literals, max / min / powi, PhysConst /
MathConst with the values of Source/ablastr/constant.H, ParticleIdCpus::Invalid and the atomics as plain updates,
ParticleUtils::RandomizeVelocity (theta, then z, as Utils/ParticleUtils.H:137-175) and an amrex::RandomEngine that
replays this project's Philox4x64-10 streams (make_collision_reference.py's stand-in).  Its per-cell loop has the shape
of doCollisionsWithinTile (BinaryCollision.H:383-472 intra-species, :613-730 inter-species) with
NuclearFusionFunc::Executor's chain loop (NuclearFusionFunc.H:127-234): ShuffleFisherYates, then per independent pair
chain SingleNuclearFusionEvent with multiplier_ratio, the weight removal and the skip of spent particles; the products
of the events in pair order get TwoProductFusionComputeProductMomenta.  The particles of a cell are handed over in this
project's canonical order (ascending id), and the product streams are the contract's (tag 2^62 | event index).

Cases: each reaction; E* = 0 (identical momenta), keV and MeV energies; the threshold branch with and without the
multiplier floor of 1; tiny probabilities (where expm1 matters); unequal weights; reactants spent mid-chain; n1 != n2;
odd intra-species counts; mildly relativistic pairs.  The fixture stores inputs and outputs."""
import importlib.util
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

_spec = importlib.util.spec_from_file_location("make_collision_reference", os.path.join(HERE, "make_collision_reference.py"))
_mcr = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_mcr)

SHIM = {
    "AMReX_Random.H": _mcr.SHIM["AMReX_Random.H"],
    "AMReX_Math.H": r'''#pragma once
#include <cmath>
#include <algorithm>
#include "AMReX_REAL.H"
#define AMREX_GPU_HOST_DEVICE
#define AMREX_INLINE inline
#define AMREX_FORCE_INLINE inline
#define AMREX_RESTRICT __restrict__
#define AMREX_ASSERT(x) ((void)0)
namespace amrex {
template <class T> const T& max(const T& a, const T& b) { return std::max(a, b); }
template <class T> const T& min(const T& a, const T& b) { return std::min(a, b); }
namespace Math {
template <class T> T abs(T v) { return std::abs(v); }
template <int N, class T> T powi(T x) { T r = x; for (int i = 1; i < N; ++i) r *= x; return r; }
}
}
''',
    "AMReX_REAL.H": r'''#pragma once
namespace amrex {
using Real = double;
using ParticleReal = double;
namespace literals {
constexpr double operator""_prt(long double x) { return double(x); }
constexpr double operator""_prt(unsigned long long x) { return double(x); }
constexpr double operator""_rt(long double x) { return double(x); }
constexpr double operator""_rt(unsigned long long x) { return double(x); }
}
}
using namespace amrex::literals;
''',
    "AMReX_Algorithm.H": '#pragma once\n#include "AMReX_Math.H"\n',
    "Utils/WarpXConst.H": "#pragma once\nnamespace PhysConst { constexpr double c = 299792458.0; "
                          "constexpr double q_e = 1.602176634e-19; constexpr double m_u = 1.66053906660e-27; "
                          "constexpr double m_p = 1.67262192369e-27; constexpr double alpha = 0.007297352573748943; "
                          "constexpr double ep0 = 8.8541878128e-12; constexpr double hbar = 1.054571817e-34; }\n"
                          "namespace MathConst { constexpr double pi = 3.14159265358979323846; }\n",
    "Particles/MultiParticleContainer.H": r'''#pragma once
#include <cstdint>
#include <limits>
#include "AMReX_REAL.H"
#include "Utils/WarpXConst.H"
class MultiParticleContainer;
namespace amrex {
struct ParticleIdCpus { static constexpr uint64_t Invalid = 16777216; };
namespace Gpu { namespace Atomic {
inline void AddNoRet(double* p, double v) { *p += v; }
template <class T> T Exch(T* p, T v) { T o = *p; *p = v; return o; }
} }
}
''',
    "Utils/ParticleUtils.H": r'''#pragma once
#include <cmath>
#include "AMReX_Random.H"
#include "AMReX_REAL.H"
#include "Utils/WarpXConst.H"
namespace ParticleUtils {
inline void getRandomVector(double& x, double& y, double& z, amrex::RandomEngine const& engine) {
    auto const theta = amrex::Random(engine) * 2.0 * MathConst::pi;
    z = 2.0 * amrex::Random(engine) - 1.0;
    auto const xy = std::sqrt(1.0 - z * z);
    x = xy * std::cos(theta);
    y = xy * std::sin(theta);
}
inline void RandomizeVelocity(double& ux, double& uy, double& uz, const double vp, amrex::RandomEngine const& engine) {
    double x, y, z;
    getRandomVector(x, y, z, engine);
    ux = x * vp; uy = y * vp; uz = z * vp;
}
}
''',
}

PROGRAM = r'''
#include <cstdio>
#include <vector>
#include "Particles/Collision/BinaryCollision/NuclearFusion/SingleNuclearFusionEvent.H"
#include "Particles/Collision/BinaryCollision/NuclearFusion/TwoProductFusionUtil.H"
#include "Particles/Collision/BinaryCollision/ShuffleFisherYates.H"
static amrex::RandomEngine engine(uint64_t seed, uint64_t step, uint64_t cell, uint64_t cidx, uint64_t tag) {
    amrex::RandomEngine e; e.seed = seed; e.c1 = step; e.c2 = cell; e.c3 = (1ull << 63) | (cidx << 32) | tag; return e;
}
int main(int argc, char** argv) {
    FILE* in = fopen(argv[1], "r");
    int same, type; double m1, m2, mA, mB, mult, thr, target, dt, dV; unsigned long long seed, step, cidx; int ncell;
    fscanf(in, "%d %d %lf %lf %lf %lf %lf %lf %lf %lf %lf %llu %llu %llu %d", &same, &type, &m1, &m2, &mA, &mB, &mult,
           &thr, &target, &dt, &dV, &seed, &step, &cidx, &ncell);
    const NuclearFusionType ft = type == 0 ? NuclearFusionType::DeuteriumTritiumToNeutronHelium
        : (type == 1 ? NuclearFusionType::DeuteriumDeuteriumToProtonTritium : NuclearFusionType::DeuteriumDeuteriumToNeutronHelium);
    const double E_fusion = type == 0 ? 17.5893e6_prt * PhysConst::q_e
        : (type == 1 ? 4.032667e6_prt * PhysConst::q_e : 3.268911e6_prt * PhysConst::q_e);   // ParticleCreationFunc.H:205-217
    for (int c = 0; c < ncell; ++c) {
        unsigned long long cell; int n1, n2;
        fscanf(in, "%llu %d %d", &cell, &n1, &n2);
        std::vector<double> a[2][4];
        std::vector<uint64_t> id[2];
        for (int s = 0; s < 2; ++s)
            for (int i = 0; i < (s ? n2 : n1); ++i) {
                for (int k = 0; k < 4; ++k) { double v; fscanf(in, "%lf", &v); a[s][k].push_back(v); }
                id[s].push_back(0);
            }
        const int S2 = same ? 0 : 1;
        std::vector<int> I1(n1), I2(n2);
        for (int i = 0; i < n1; ++i) I1[i] = i;
        for (int i = 0; i < n2; ++i) I2[i] = i;
        int NI1, NI2; const int *J1, *J2;
        if (same) {                               // BinaryCollision.H:383-472: halves of the shuffled cell
            ShuffleFisherYates(I1.data(), 0, n1, engine(seed, step, cell, cidx, 0));
            NI1 = n1 / 2; NI2 = n1 - n1 / 2; J1 = I1.data(); J2 = I1.data() + n1 / 2;
        } else {                                  // :613-730
            ShuffleFisherYates(I1.data(), 0, n1, engine(seed, step, cell, cidx, 0));
            ShuffleFisherYates(I2.data(), 0, n2, engine(seed, step, cell, cidx, 1));
            NI1 = n1; NI2 = n2; J1 = I1.data(); J2 = I2.data();
        }
        const int max_N = std::max(NI1, NI2), min_N = std::min(NI1, NI2);
        const int multiplier_ratio = same ? min_N + max_N - 1 : min_N;
        std::vector<int> mask(max_N, 0), p1(max_N), p2(max_N);
        std::vector<double> wr(max_N, 0.0);
        for (int ci = 0; ci < min_N; ++ci) {      // NuclearFusionFunc::Executor, one independent chain
            const amrex::RandomEngine eng = engine(seed, step, cell, cidx, 2 + ci);
            int i1 = ci, i2 = ci;
            for (int k = ci; k < max_N; k += min_N) {
                const int e1 = J1[i1], e2 = J2[i2];
                p1[k] = e1; p2[k] = e2;
                if (id[0][e1] == amrex::ParticleIdCpus::Invalid || id[S2][e2] == amrex::ParticleIdCpus::Invalid) {
                    mask[k] = 0;
                } else {
                    SingleNuclearFusionEvent(a[0][1][e1], a[0][2][e1], a[0][3][e1], a[S2][1][e2], a[S2][2][e2],
                                             a[S2][3][e2], m1, m2, a[0][0][e1], a[S2][0][e2], dt, dV, k, mask.data(),
                                             wr.data(), mult, multiplier_ratio, thr, target, ft, eng);
                    if (mask[k]) {
                        BinaryCollisionUtils::remove_weight_from_colliding_particle(a[0][0][e1], id[0][e1], wr[k]);
                        BinaryCollisionUtils::remove_weight_from_colliding_particle(a[S2][0][e2], id[S2][e2], wr[k]);
                    }
                }
                if (max_N == NI1) { i1 += min_N; }
                if (max_N == NI2) { i2 += min_N; }
            }
        }
        for (int s = 0; s < (same ? 1 : 2); ++s)
            for (int i = 0; i < (s ? n2 : n1); ++i)
                printf("%.17g %d\n", a[s][0][i], id[s][i] == amrex::ParticleIdCpus::Invalid ? 1 : 0);
        int nev = 0;
        for (int k = 0; k < max_N; ++k) nev += mask[k] ? 1 : 0;
        printf("%d\n", nev);
        int j = 0;
        for (int k = 0; k < max_N; ++k) {
            if (!mask[k]) continue;
            double uA[3], uB[3];
            const int e1 = p1[k], e2 = p2[k];
            TwoProductFusionComputeProductMomenta(a[0][1][e1], a[0][2][e1], a[0][3][e1], m1, a[S2][1][e2], a[S2][2][e2],
                                                  a[S2][3][e2], m2, uA[0], uA[1], uA[2], mA, uB[0], uB[1], uB[2], mB,
                                                  E_fusion, engine(seed, step, cell, cidx, (1ull << 62) | (uint64_t)j));
            printf("%d %d %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", k, e1, e2, wr[k], uA[0], uA[1], uA[2], uB[0],
                   uB[1], uB[2]);
            ++j;
        }
    }
    return 0;
}
'''


def build(tree, d):
    for name, text in SHIM.items():
        p = os.path.join(d, "shim", name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            f.write(text)
    src = os.path.join(d, "ref.cpp")
    with open(src, "w") as f:
        f.write(PROGRAM)
    exe = os.path.join(d, "ref")
    # the stand-in's headers first, so that the tree's own Utils/WarpXConst.H, ParticleUtils.H, ... are not used
    subprocess.run(["g++", "-std=c++17", "-O0", "-ffp-contract=off", "-I", os.path.join(d, "shim"), "-I",
                    os.path.join(tree, "Source"), src, "-o", exe], check=True)
    return exe


def run_case(exe, d, sp1, sp2, f, geom, dt, step, tile=(8, 8, 8)):
    """the reference on one particle set: (w1, spent1, w2, spent2, products A, products B) in the project's layout"""
    import fusion_oracle as fo
    same = bool(f["same_species"])
    dxs = [(geom["prob_hi"][k] - geom["prob_lo"][k]) / geom["n_cell"][k] for k in range(3)]
    dV = dxs[0] * dxs[1] * dxs[2]
    idx1, c1, st1, n1 = fo._live_canonical(sp1, geom)
    if same:
        keep = n1 >= 2
        cells, st1, n1 = c1[keep], st1[keep], n1[keep]
        idx2, st2, n2 = idx1, st1, np.zeros_like(n1)
    else:
        idx2, c2, st2, n2 = fo._live_canonical(sp2, geom)
        cells, i1, i2 = np.intersect1d(c1, c2, assume_unique=True, return_indices=True)
        st1, n1, st2, n2 = st1[i1], n1[i1], st2[i2], n2[i2]
    order = np.argsort(fo.bins_of(cells, geom, tile), kind="stable")
    m2 = f["m1"] if same else f["m2"]
    lines = ["%d %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %d %d %d %d" % (
        int(same), f["type"], f["m1"], m2, f["mA"], f["mB"], f["fusion_multiplier"], f["fusion_probability_threshold"],
        f["fusion_probability_target_value"], dt, dV, f["seed"], step, f["collision_index"], len(cells))]
    for c in order:
        lines.append("%d %d %d" % (cells[c], n1[c], n2[c]))
        for idx, sp, st, n in ((idx1, sp1, st1, n1), (idx2, sp2, st2, n2)):
            for p in idx[st[c]:st[c] + n[c]]:
                lines.append("%.17g %.17g %.17g %.17g" % (sp["w"][p], sp["ux"][p], sp["uy"][p], sp["uz"][p]))
    inp = os.path.join(d, "in.txt")
    with open(inp, "w") as fh:
        fh.write("\n".join(lines) + "\n")
    out = subprocess.run([exe, inp], check=True, capture_output=True, text=True).stdout.split("\n")
    w = [np.array(sp1["w"], dtype=np.float64), None if same else np.array(sp2["w"], dtype=np.float64)]
    spent = [np.zeros(len(sp1["w"]), dtype=bool), None if same else np.zeros(len(sp2["w"]), dtype=bool)]
    prods = ([], [])
    pos = 0
    for c in order:
        for s, (idx, st, n) in enumerate(((idx1, st1, n1), (idx2, st2, n2))):
            if same and s == 1:
                continue
            for p in idx[st[c]:st[c] + n[c]]:
                v, flag = out[pos].split()
                pos += 1
                w[s][p], spent[s][p] = float(v), flag == "1"
        nev = int(out[pos]); pos += 1
        for _ in range(nev):
            v = out[pos].split(); pos += 1
            e1, e2 = int(v[1]), int(v[2])
            a, b = idx1[st1[c] + e1], (idx1[st1[c] + e2] if same else idx2[st2[c] + e2])
            wr, uA, uB = float(v[3]), [float(x) for x in v[4:7]], [float(x) for x in v[7:10]]
            s2 = sp1 if same else sp2
            for prod, u in ((prods[0], uA), (prods[1], uB)):
                for sp_, q in ((sp1, a), (s2, b)):
                    prod.append([sp_["x"][q], sp_["y"][q], sp_["z"][q], wr / 2.0] + u)
    P = [np.array(p, dtype=np.float64).reshape(-1, 7) for p in prods]
    return w[0], spent[0], w[1], spent[1], P[0], P[1]


def cases():
    import collision_cases as cc
    import fusion_cases as fc
    from warpx_b200 import abi
    g = fc.GEOM
    out = {}
    rng = np.random.default_rng(0)

    def cnt(seed, mean, big=0):
        n = np.random.default_rng(seed).poisson(mean, size=(4, 5, 6))
        if big:
            n[1, 1, 1] = big
        return n
    for ftype, name in ((abi.FUSION_DT_NHE4, "dt"), (abi.FUSION_DD_PT, "dd_pt"), (abi.FUSION_DD_NHE3, "dd_nhe3")):
        dd = 100.0 if ftype != abi.FUSION_DT_NHE4 else 1.0      # D-D cross sections are ~100 times smaller
        # (E* scale keV, multiplier, threshold, target, weight scale, dt): probabilities ~0.3 without the threshold;
        # above it with a multiplier that stays above 1, and with one the floor of 1 clamps; ~1e-16 (expm1)
        for E, mult, thr, target, w0, dt, tag in ((10.0, 1e8 * dd, 1e300, 0.002, 1e9, 1e-13, "kev"),
                                                  (2000.0, 1e8 * dd, 1e300, 0.002, 1e9, 1e-13, "mev"),
                                                  (30.0, 1e25, 0.02, 0.3, 1e9, 1e-9, "threshold"),
                                                  (30.0, 1.0, 0.02, 0.3, 1e21 * dd, 1e-9, "threshold_floor"),
                                                  (30.0, 1.0, 0.02, 0.002, 1e9, 1e-16, "tiny")):
            f = fc.spec(ftype, mult=mult, thr=thr, target=target, seed=int(rng.integers(1 << 40)),
                        cidx=int(rng.integers(4)))
            sp1 = fc.reactants(int(rng.integers(1 << 30)), cnt(1, 3.0, 37), f["m1"], E, weights="log", w0=w0)
            sp2 = None if f["same_species"] else fc.reactants(int(rng.integers(1 << 30)), cnt(2, 2.0, 21), f["m2"], E,
                                                              weights="log", id_offset=10 ** 6, w0=w0)
            out["%s_%s" % (name, tag)] = (sp1, sp2, f, dt, int(rng.integers(100)))
    # E* = 0: identical momenta of every pair (all at rest)
    f = fc.spec(abi.FUSION_DT_NHE4, mult=1e20)
    sp1 = fc.reactants(5, cnt(5, 3.0), f["m1"], 0.0)
    sp2 = fc.reactants(6, cnt(6, 3.0), f["m2"], 0.0, id_offset=10 ** 6)
    out["dt_rest"] = (sp1, sp2, f, 1e-9, 0)
    # spent mid-chain: probability ~ 1, unequal counts, n1 != n2, odd intra-species counts
    f = fc.spec(abi.FUSION_DT_NHE4, mult=1.0, thr=1e300)
    n1, n2 = np.zeros((4, 5, 6), dtype=int), np.zeros((4, 5, 6), dtype=int)
    n1[2, 2, 2], n2[2, 2, 2], n1[0, 1, 2], n2[0, 1, 2] = 3, 11, 9, 4
    sp1 = fc.reactants(7, n1, f["m1"], 60.0, weights="log", w0=1e39)
    sp2 = fc.reactants(8, n2, f["m2"], 60.0, weights="log", w0=1e39, id_offset=10 ** 6)
    out["dt_spent_midchain"] = (sp1, sp2, f, 1e-6, 3)
    f = fc.spec(abi.FUSION_DD_NHE3, mult=1.0, thr=1e300)
    n1 = np.zeros((4, 5, 6), dtype=int)
    n1[1, 2, 3], n1[3, 4, 5] = 7, 13
    out["dd_odd_spent"] = (fc.reactants(9, n1, f["m1"], 60.0, weights="log", w0=1e39), None, f, 1e-6, 1)
    # mildly relativistic pairs (|u| ~ 0.3 c)
    f = fc.spec(abi.FUSION_DT_NHE4, mult=1e20)
    sp1 = fc.reactants(10, cnt(10, 3.0), f["m1"], 50.0, drift_keV=1.0e5)
    sp2 = fc.reactants(11, cnt(11, 3.0), f["m2"], 50.0, id_offset=10 ** 6)
    f["fusion_multiplier"], f["fusion_probability_threshold"] = 1e8, 1e300
    out["dt_relativistic"] = (sp1, sp2, f, 1e-13, 2)
    del cc
    return out


def main(tree):
    import fusion_cases as fc
    z = {}
    with tempfile.TemporaryDirectory() as d:
        exe = build(tree, d)
        for name, (sp1, sp2, f, dt, step) in cases().items():
            w1, s1, w2, s2, pA, pB = run_case(exe, d, sp1, sp2, f, fc.GEOM, dt, step)
            p = name + "/"
            for k, v in sp1.items():
                z[p + "sp1_" + k] = v
            if sp2 is not None:
                for k, v in sp2.items():
                    z[p + "sp2_" + k] = v
                z[p + "w2"], z[p + "spent2"] = w2, s2
            z[p + "w1"], z[p + "spent1"] = w1, s1
            z[p + "prodA"], z[p + "prodB"] = pA, pB
            z[p + "spec"] = np.array([f["m1"], f["m2"], f["mA"], f["mB"], f["fusion_multiplier"],
                                      f["fusion_probability_threshold"], f["fusion_probability_target_value"], dt,
                                      f["q1"], f["q2"]])
            z[p + "ints"] = np.array([f["type"], f["seed"], f["collision_index"], f["same_species"], step], dtype=np.int64)
            print(name, "events", len(pA) // 2, "spent", int(s1.sum()) + (0 if s2 is None else int(s2.sum())))
    np.savez_compressed(os.path.join(HERE, "fusion_reference.npz"), **z)


if __name__ == "__main__":
    main(sys.argv[1])
