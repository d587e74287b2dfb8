#!/usr/bin/env python3
"""Regenerates tests/golden/proton_boron_reference.npz: what the reference's own proton-boron headers compute.

    python tests/golden/make_proton_boron_reference.py <WarpX source tree>

A small C++ program includes, from the given tree and unchanged, Source/Particles/Collision/BinaryCollision/
NuclearFusion/SingleNuclearFusionEvent.H (with ProtonBoronFusionCrossSection.H and BinaryCollisionUtils.H),
NuclearFusion/ProtonBoronFusionInitializeMomentum.H (with TwoProductFusionUtil.H) and ShuffleFisherYates.H.  It is built
against make_fusion_reference.py's stand-in (the AMReX macros and literals, PhysConst, RandomizeVelocity, the random
engine that replays this project's Philox4x64-10 streams), with amrex::Math::powi as AMReX defines it (x * powi<N-1>
for odd N, powi<2>(powi<N/2>) for even N) and a particle-tile type whose m_rdata rows are w, ux, uy, uz.  The cell loop is
make_fusion_reference.py's; the products of the cell's j-th event come from ProtonBoronFusionInitializeMomentum with the
stream of tag 2^62 | j, six alphas written as ParticleCreationFunc.H:170-200 writes them.

Cases: the cross section at E* = 0, around each fit boundary (400 keV, 668 keV, 9.76 MeV) and across the resonances;
events at keV and MeV energies and above the switch to Buck's fit, in the centre-of-momentum frame and in the boron
rest frame; the threshold branch; reactants at rest (E* = 0); boron as species 1 and as species 2; reactants spent
mid-chain; n1 != n2.  The zero-velocity branch of the 8Be* boost is not reachable through an event (the 8Be* recoils
from the first alpha) and is not covered."""
import importlib.util
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

_spec = importlib.util.spec_from_file_location("make_fusion_reference", os.path.join(HERE, "make_fusion_reference.py"))
_mfr = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_mfr)

SHIM = dict(_mfr.SHIM)
SHIM["AMReX_Math.H"] = _mfr.SHIM["AMReX_Math.H"].replace(
    "template <int N, class T> T powi(T x) { T r = x; for (int i = 1; i < N; ++i) r *= x; return r; }",
    "template <int N, class T> constexpr T powi(T x) {\n"
    "    if constexpr (N == 1) { return x; } else if constexpr (N == 2) { return x * x; }\n"
    "    else if constexpr (N % 2 == 0) { return powi<2>(powi<N / 2>(x)); } else { return x * powi<N - 1>(x); }\n}")
assert SHIM["AMReX_Math.H"] != _mfr.SHIM["AMReX_Math.H"]
SHIM["AMReX_DenseBins.H"] = "#pragma once\nnamespace amrex { template <class T> struct DenseBins { using index_type = unsigned int; }; }\n"
SHIM["Particles/WarpXParticleContainer.H"] = r'''#pragma once
#include "Particles/MultiParticleContainer.H"
struct PIdx { enum { w = 0, ux, uy, uz }; };
struct SoaTile { double* m_rdata[4]; };
struct WarpXParticleContainer {
    struct ParticleType {};
    struct ParticleTileType { using ParticleTileDataType = SoaTile; };
};
'''

PROGRAM = r'''
#include <cstdio>
#include <cstring>
#include <vector>
#include "Particles/Collision/BinaryCollision/NuclearFusion/SingleNuclearFusionEvent.H"
#include "Particles/Collision/BinaryCollision/NuclearFusion/ProtonBoronFusionInitializeMomentum.H"
#include "Particles/Collision/BinaryCollision/ShuffleFisherYates.H"
static amrex::RandomEngine engine(uint64_t seed, uint64_t step, uint64_t cell, uint64_t cidx, uint64_t tag) {
    amrex::RandomEngine e; e.seed = seed; e.c1 = step; e.c2 = cell; e.c3 = (1ull << 63) | (cidx << 32) | tag; return e;
}
int main(int argc, char** argv) {
    FILE* in = fopen(argv[1], "r");
    if (argc > 2 && !strcmp(argv[2], "xs")) {          // the cross section of each energy [J]
        double E;
        while (fscanf(in, "%lf", &E) == 1) printf("%.17g\n", ProtonBoronFusionCrossSection(E));
        return 0;
    }
    int same, type; double m1, m2, mA, mB, mult, thr, target, dt, dV; unsigned long long seed, step, cidx; int ncell;
    fscanf(in, "%d %d %lf %lf %lf %lf %lf %lf %lf %lf %lf %llu %llu %llu %d", &same, &type, &m1, &m2, &mA, &mB, &mult,
           &thr, &target, &dt, &dV, &seed, &step, &cidx, &ncell);
    const NuclearFusionType ft = NuclearFusionType::ProtonBoronToAlphas;
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
        std::vector<int> I1(n1), I2(n2);
        for (int i = 0; i < n1; ++i) I1[i] = i;
        for (int i = 0; i < n2; ++i) I2[i] = i;
        ShuffleFisherYates(I1.data(), 0, n1, engine(seed, step, cell, cidx, 0));   // BinaryCollision.H:613-730
        ShuffleFisherYates(I2.data(), 0, n2, engine(seed, step, cell, cidx, 1));
        const int NI1 = n1, NI2 = n2;
        const int max_N = std::max(NI1, NI2), min_N = std::min(NI1, NI2);
        const int multiplier_ratio = min_N;
        std::vector<int> mask(max_N, 0), p1(max_N), p2(max_N);
        std::vector<double> wr(max_N, 0.0);
        for (int ci = 0; ci < min_N; ++ci) {      // NuclearFusionFunc::Executor, one independent chain
            const amrex::RandomEngine eng = engine(seed, step, cell, cidx, 2 + ci);
            int i1 = ci, i2 = ci;
            for (int k = ci; k < max_N; k += min_N) {
                const int e1 = I1[i1], e2 = I2[i2];
                p1[k] = e1; p2[k] = e2;
                if (id[0][e1] == amrex::ParticleIdCpus::Invalid || id[1][e2] == amrex::ParticleIdCpus::Invalid) {
                    mask[k] = 0;
                } else {
                    SingleNuclearFusionEvent(a[0][1][e1], a[0][2][e1], a[0][3][e1], a[1][1][e2], a[1][2][e2],
                                             a[1][3][e2], m1, m2, a[0][0][e1], a[1][0][e2], dt, dV, k, mask.data(),
                                             wr.data(), mult, multiplier_ratio, thr, target, ft, eng);
                    if (mask[k]) {
                        BinaryCollisionUtils::remove_weight_from_colliding_particle(a[0][0][e1], id[0][e1], wr[k]);
                        BinaryCollisionUtils::remove_weight_from_colliding_particle(a[1][0][e2], id[1][e2], wr[k]);
                    }
                }
                if (max_N == NI1) { i1 += min_N; }
                if (max_N == NI2) { i2 += min_N; }
            }
        }
        for (int s = 0; s < 2; ++s)
            for (int i = 0; i < (s ? n2 : n1); ++i)
                printf("%.17g %d\n", a[s][0][i], id[s][i] == amrex::ParticleIdCpus::Invalid ? 1 : 0);
        int nev = 0;
        for (int k = 0; k < max_N; ++k) nev += mask[k] ? 1 : 0;
        printf("%d\n", nev);
        int j = 0;
        for (int k = 0; k < max_N; ++k) {
            if (!mask[k]) continue;
            const int e1 = p1[k], e2 = p2[k];
            SoaTile s1, s2, sa;
            std::vector<double> alpha[4];
            for (int r = 0; r < 4; ++r) {
                s1.m_rdata[r] = a[0][r].data(); s2.m_rdata[r] = a[1][r].data();
                alpha[r].assign(6, 0.0); sa.m_rdata[r] = alpha[r].data();
            }
            ProtonBoronFusionInitializeMomentum(s1, s2, sa, e1, e2, 0, m1, m2,
                                                engine(seed, step, cell, cidx, (1ull << 62) | (uint64_t)j));
            printf("%d %d %d %.17g", k, e1, e2, wr[k]);
            for (int q = 0; q < 6; ++q) printf(" %.17g %.17g %.17g", alpha[1][q], alpha[2][q], alpha[3][q]);
            printf("\n");
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
    subprocess.run(["g++", "-std=c++17", "-O0", "-ffp-contract=off", "-I", os.path.join(d, "shim"), "-I",
                    os.path.join(tree, "Source"), src, "-o", exe], check=True)
    return exe


def cross_sections(exe, d, E):
    inp = os.path.join(d, "xs.txt")
    with open(inp, "w") as fh:
        fh.write("\n".join("%.17g" % v for v in E) + "\n")
    out = subprocess.run([exe, inp, "xs"], check=True, capture_output=True, text=True).stdout.split()
    return np.array([float(v) for v in out])


def run_case(exe, d, sp1, sp2, f, geom, dt, step, tile=(8, 8, 8)):
    """the reference on one particle set: (w1, spent1, w2, spent2, alphas [6 per event, x y z w ux uy uz])"""
    import fusion_oracle as fo
    dxs = [(geom["prob_hi"][k] - geom["prob_lo"][k]) / geom["n_cell"][k] for k in range(3)]
    dV = dxs[0] * dxs[1] * dxs[2]
    idx1, c1, st1, n1 = fo._live_canonical(sp1, geom)
    idx2, c2, st2, n2 = fo._live_canonical(sp2, geom)
    cells, i1, i2 = np.intersect1d(c1, c2, assume_unique=True, return_indices=True)
    st1, n1, st2, n2 = st1[i1], n1[i1], st2[i2], n2[i2]
    order = np.argsort(fo.bins_of(cells, geom, tile), kind="stable")
    lines = ["0 3 %.17g %.17g %.17g 0 %.17g %.17g %.17g %.17g %.17g %d %d %d %d" % (
        f["m1"], f["m2"], f["mA"], f["fusion_multiplier"], f["fusion_probability_threshold"],
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
    w = [np.array(sp1["w"], dtype=np.float64), np.array(sp2["w"], dtype=np.float64)]
    spent = [np.zeros(len(sp1["w"]), dtype=bool), np.zeros(len(sp2["w"]), dtype=bool)]
    alphas = []
    pos = 0
    for c in order:
        for s, (idx, st, n) in enumerate(((idx1, st1, n1), (idx2, st2, n2))):
            for p in idx[st[c]:st[c] + n[c]]:
                v, flag = out[pos].split()
                pos += 1
                w[s][p], spent[s][p] = float(v), flag == "1"
        nev = int(out[pos]); pos += 1
        for _ in range(nev):
            v = out[pos].split(); pos += 1
            a, b = idx1[st1[c] + int(v[1])], idx2[st2[c] + int(v[2])]
            wr = float(v[3])
            u = np.array([float(x) for x in v[4:]]).reshape(6, 3)
            for q in range(6):
                sp_, r = (sp1, a) if q % 2 == 0 else (sp2, b)
                alphas.append([sp_["x"][r], sp_["y"][r], sp_["z"][r], wr / 2.0] + list(u[q]))
    return w[0], spent[0], w[1], spent[1], np.array(alphas, dtype=np.float64).reshape(-1, 7)


def _tuned(sp1, sp2, f, dt, p_target=0.3):
    """the multiplier that brings the median first-pair probability of the set to about p_target (no threshold)"""
    import proton_boron_oracle as po
    n = min(len(sp1["x"]), len(sp2["x"]), 400)
    u1 = [sp1[k][:n] for k in ("ux", "uy", "uz")]
    u2 = [sp2[k][:n] for k in ("ux", "uy", "uz")]
    dxs = [(_GEOM()["prob_hi"][k] - _GEOM()["prob_lo"][k]) / _GEOM()["n_cell"][k] for k in range(3)]
    prob, _ = po.event_probability(u1, u2, f["m1"], f["m2"], sp1["w"][:n], sp2["w"][:n], dt, dxs[0] * dxs[1] * dxs[2],
                                   1.0, np.full(n, 3), 1e300, 0.002)
    pe = -np.log1p(-np.clip(prob, 0.0, 1.0 - 1e-16))
    return float(p_target / np.median(pe[pe > 0]))


def _GEOM():
    import fusion_cases as fc
    return fc.GEOM


def cases():
    import fusion_cases as fc
    import proton_boron_cases as pc
    out = {}
    rng = np.random.default_rng(1)

    def cnt(seed, mean, big=0):
        n = np.random.default_rng(seed).poisson(mean, size=(4, 5, 6))
        if big:
            n[1, 1, 1] = big
        return n

    def pair(boron_first, E1, E2, drift1=0.0, big=(37, 21)):
        f = pc.spec(boron_first, seed=int(rng.integers(1 << 40)), cidx=int(rng.integers(4)))
        sp1 = fc.reactants(int(rng.integers(1 << 30)), cnt(1, 3.0, big[0]), f["m1"], E1, weights="log", drift_keV=drift1)
        sp2 = fc.reactants(int(rng.integers(1 << 30)), cnt(2, 2.0, big[1]), f["m2"], E2, weights="log",
                           id_offset=10 ** 6)
        return f, sp1, sp2
    dt = 1e-13
    # (tag, E of species 1 / 2 [keV], drift of species 1 [keV]): thermal pairs near their centre of momentum; a proton
    # beam on boron at rest (boron rest frame)
    for bf in (False, True):
        side = "b1" if bf else "p1"
        for tag, E1, E2, drift in (("kev", 30.0, 30.0, 0.0), ("resonance", 400.0, 400.0, 0.0),
                                   ("mev", 3000.0, 3000.0, 0.0), ("buck", 2.0e4, 2.0e4, 0.0)):
            f, sp1, sp2 = pair(bf, E1, E2, drift)
            f["fusion_multiplier"], f["fusion_probability_threshold"] = _tuned(sp1, sp2, f, dt), 1e300
            out["pb_%s_%s" % (side, tag)] = (sp1, sp2, f, dt, int(rng.integers(100)))
        # the boron at rest, the protons a 150 keV / 2 MeV beam with a small spread
        for tag, drift in (("beam_kev", 150.0), ("beam_mev", 2000.0)):
            f = pc.spec(bf, seed=int(rng.integers(1 << 40)))
            mp, mb = (f["m2"], f["m1"]) if bf else (f["m1"], f["m2"])
            p = fc.reactants(int(rng.integers(1 << 30)), cnt(3, 3.0), mp, 1.0, weights="log", drift_keV=drift)
            b = fc.reactants(int(rng.integers(1 << 30)), cnt(4, 2.0), mb, 0.0, weights="log", id_offset=10 ** 6)
            sp1, sp2 = (b, p) if bf else (p, b)
            f["fusion_multiplier"], f["fusion_probability_threshold"] = _tuned(sp1, sp2, f, dt), 1e300
            out["pb_%s_%s" % (side, tag)] = (sp1, sp2, f, dt, int(rng.integers(100)))
    # the threshold branch with the multiplier's floor and without
    for tag, scale in (("threshold", 1e3), ("threshold_floor", 1e-30)):
        f, sp1, sp2 = pair(False, 400.0, 400.0)
        f["fusion_multiplier"] = _tuned(sp1, sp2, f, dt) * scale
        f["fusion_probability_threshold"], f["fusion_probability_target_value"] = 0.02, 0.3
        if scale < 1:
            sp1["w"], sp2["w"] = sp1["w"] * 1e33, sp2["w"] * 1e33
        out["pb_" + tag] = (sp1, sp2, f, dt, 7)
    # E* = 0: every reactant at rest
    f, sp1, sp2 = pair(False, 0.0, 0.0)
    f["fusion_multiplier"] = 1e30
    out["pb_rest"] = (sp1, sp2, f, dt, 0)
    # spent mid-chain: probability ~ 1, n1 != n2 in each cell
    for bf in (False, True):
        f = pc.spec(bf, mult=1.0, thr=1e300, seed=int(rng.integers(1 << 40)))
        n1, n2 = np.zeros((4, 5, 6), dtype=int), np.zeros((4, 5, 6), dtype=int)
        n1[2, 2, 2], n2[2, 2, 2], n1[0, 1, 2], n2[0, 1, 2] = 3, 11, 9, 4
        sp1 = fc.reactants(int(rng.integers(1 << 30)), n1, f["m1"], 500.0, weights="log", w0=1e39)
        sp2 = fc.reactants(int(rng.integers(1 << 30)), n2, f["m2"], 500.0, weights="log", w0=1e39, id_offset=10 ** 6)
        out["pb_%s_spent_midchain" % ("b1" if bf else "p1")] = (sp1, sp2, f, 1e-6, 3)
    return out


def xs_energies():
    """E* [J]: 0, around 400 keV, 668 keV and 9.76 MeV, the resonances, and a log sweep"""
    keV = 1.0e3 * 1.602176634e-19
    pts = [0.0, 1e-3, 1.0, 10.0, 100.0, 148.0, 640.9, 1211.0, 2340.0, 3294.0]
    for b in (400.0, 668.0, 9760.0):
        pts += [b * (1 - 1e-12), b, b * (1 + 1e-12), b - 1.0, b + 1.0]
    pts += list(np.geomspace(1.0, 1.0e5, 400))
    return np.array(pts) * keV


def main(tree):
    import fusion_cases as fc
    z = {}
    with tempfile.TemporaryDirectory() as d:
        exe = build(tree, d)
        E = xs_energies()
        z["xs/E"], z["xs/sigma"] = E, cross_sections(exe, d, E)
        for name, (sp1, sp2, f, dt, step) in cases().items():
            w1, s1, w2, s2, al = run_case(exe, d, sp1, sp2, f, fc.GEOM, dt, step)
            p = name + "/"
            for k, v in sp1.items():
                z[p + "sp1_" + k] = v
            for k, v in sp2.items():
                z[p + "sp2_" + k] = v
            z[p + "w1"], z[p + "spent1"], z[p + "w2"], z[p + "spent2"], z[p + "alphas"] = w1, s1, w2, s2, al
            z[p + "spec"] = np.array([f["m1"], f["m2"], f["mA"], f["fusion_multiplier"], f["fusion_probability_threshold"],
                                      f["fusion_probability_target_value"], dt, f["q1"], f["q2"]])
            z[p + "ints"] = np.array([f["seed"], f["collision_index"], step], dtype=np.int64)
            print(name, "events", len(al) // 6, "spent", int(s1.sum()) + int(s2.sum()))
    np.savez_compressed(os.path.join(HERE, "proton_boron_reference.npz"), **z)


if __name__ == "__main__":
    main(sys.argv[1])
