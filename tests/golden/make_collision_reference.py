#!/usr/bin/env python3
"""Regenerates tests/golden/collision_reference.npz: what the reference's own collision leaf headers compute.

    python tests/golden/make_collision_reference.py <WarpX source tree>

A small C++ program includes Source/Particles/Collision/BinaryCollision/Coulomb/ElasticCollisionPerez.H (with the
UpdateMomentumPerezElastic.H it includes), Coulomb/ComputeTemperature.H and ShuffleFisherYates.H from the given tree,
unchanged, against a stand-in written here: the AMReX macros and max / min / Math::abs, PhysConst / MathConst with the
values of Source/ablastr/constant.H, a PIdx / SoA view with m_rdata, and an amrex::RandomEngine that replays this
project's Philox4x64-10 stream of (seed, step, global cell, collision index, tag) with its conversions
(amrex::Random = ((w >> 11) + 1) 2^-53, Random_int(n) = floor(((w >> 11) 2^-53) n)).  Its loops have the shape of
BinaryCollision::doCollisionsWithinTile's two ParallelFors (BinaryCollision.H:383-472 intra-species, :613-730
inter-species): per cell the density, the temperature when CoulombLog < 0, ShuffleFisherYates; then per independent
pair ElasticCollisionPerez.  All physics is in the headers.  The particles of a cell are handed over in this project's
canonical order (ascending id), the one thing the contract adds.

Cases: every s12 branch (dt from 1e-17 to 1e-11), a forced redraw (cos < -1: a step whose first chain draw is below
exp(-2/s12), found by searching), computed Coulomb logs with the classical and the quantum minimum impact parameter and
at the floor of 2, identical momenta, p* along z, relativistic pairs (|u| ~ 10 c), unequal weights, odd intra-species
counts and n1 != n2 inter-species.  The fixture stores inputs and outputs."""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

SHIM = {
    "AMReX_Random.H": r'''#pragma once
#include <cstdint>
#include "AMReX_Math.H"
namespace amrex {
struct RandomEngine { uint64_t seed, c1, c2, c3; mutable uint64_t drawn = 0; };
inline uint64_t stand_in_mulhi(uint64_t a, uint64_t b) { return (uint64_t)(((unsigned __int128)a * b) >> 64); }
inline uint64_t stand_in_word(const RandomEngine& e) {
    uint64_t c0 = e.drawn / 4 + 1, c1 = e.c1, c2 = e.c2, c3 = e.c3, k0 = e.seed, k1 = 0;
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
        const uint64_t hi0 = stand_in_mulhi(0xD2E7470EE14C6C93ull, c0), lo0 = 0xD2E7470EE14C6C93ull * c0;
        const uint64_t hi1 = stand_in_mulhi(0xCA5A826395121157ull, c2), lo1 = 0xCA5A826395121157ull * c2;
        const uint64_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    }
    const uint64_t w[4] = {c0, c1, c2, c3};
    return w[e.drawn++ % 4];
}
inline double Random(const RandomEngine& e) { return (double)((stand_in_word(e) >> 11) + 1) * (1.0 / 9007199254740992.0); }
inline unsigned int Random_int(unsigned int n, const RandomEngine& e) {
    return (unsigned int)(((double)(stand_in_word(e) >> 11) * (1.0 / 9007199254740992.0)) * n);
}
}
''',
    "AMReX_Math.H": r'''#pragma once
#include <cmath>
#include <algorithm>
#define AMREX_GPU_HOST_DEVICE
#define AMREX_INLINE inline
#define AMREX_FORCE_INLINE inline
#define AMREX_RESTRICT __restrict__
#define AMREX_ASSERT(x) ((void)0)
namespace amrex {
template <class T> const T& max(const T& a, const T& b) { return std::max(a, b); }
template <class T> const T& min(const T& a, const T& b) { return std::min(a, b); }
namespace Math { template <class T> T abs(T v) { return std::abs(v); } }
}
''',
    "Utils/WarpXConst.H": "#pragma once\nnamespace PhysConst { constexpr double c = 299792458.0; "
                          "constexpr double ep0 = 8.8541878128e-12; constexpr double hbar = 1.054571817e-34; }\n"
                          "namespace MathConst { constexpr double pi = 3.14159265358979323846; }\n",
    "Particles/WarpXParticleContainer.H": "#pragma once\nstruct PIdx { enum { w = 0, ux, uy, uz }; };\n"
                                          "struct StandInSoA { double* m_rdata[4]; };\n",
}

PROGRAM = r'''
#include <cstdio>
#include <vector>
#include "Particles/Collision/BinaryCollision/Coulomb/ElasticCollisionPerez.H"
#include "Particles/Collision/BinaryCollision/Coulomb/ComputeTemperature.H"
#include "Particles/Collision/BinaryCollision/ShuffleFisherYates.H"
static amrex::RandomEngine engine(uint64_t seed, uint64_t step, uint64_t cell, uint64_t cidx, uint64_t tag) {
    amrex::RandomEngine e; e.seed = seed; e.c1 = step; e.c2 = cell; e.c3 = (1ull << 63) | (cidx << 32) | tag; return e;
}
int main(int argc, char** argv) {
    FILE* in = fopen(argv[1], "r");
    if (argv[2][0] == 's') {        // search <in> s: "seed cell cidx thr first" -> first step with Random < thr
        unsigned long long seed, cell, cidx, first; double thr;
        fscanf(in, "%llu %llu %llu %lf %llu", &seed, &cell, &cidx, &thr, &first);
        for (uint64_t st = first;; ++st) if (amrex::Random(engine(seed, st, cell, cidx, 2)) < thr) { printf("%llu\n", (unsigned long long)st); return 0; }
    }
    int same; double q1, m1, q2, m2, L, dt, dV; unsigned long long seed, step, cidx; int ncell;
    fscanf(in, "%d %lf %lf %lf %lf %lf %lf %lf %llu %llu %llu %d", &same, &q1, &m1, &q2, &m2, &L, &dt, &dV, &seed, &step,
           &cidx, &ncell);
    for (int c = 0; c < ncell; ++c) {
        unsigned long long cell; int n1, n2;
        fscanf(in, "%llu %d %d", &cell, &n1, &n2);
        std::vector<double> a[2][4];
        for (int s = 0; s < 2; ++s)
            for (int i = 0; i < (s ? n2 : n1); ++i)
                for (int k = 0; k < 4; ++k) { double v; fscanf(in, "%lf", &v); a[s][k].push_back(v); }
        StandInSoA soa[2];
        for (int s = 0; s < 2; ++s) for (int k = 0; k < 4; ++k) soa[s].m_rdata[k] = a[s][k].data();
        std::vector<int> I1(n1), I2(n2);
        for (int i = 0; i < n1; ++i) I1[i] = i;
        for (int i = 0; i < n2; ++i) I2[i] = i;
        const bool computeT = L < 0.0;
        if (same) {                                    // BinaryCollision.H:383-472
            if (n1 > 1) {
                double wt = 0.0;
                for (int i = 0; i < n1; ++i) wt += a[0][0][I1[i]];
                const double n = wt / (dV * 1.0);
                const double T = computeT ? ComputeTemperature(0, n1, I1.data(), a[0][0].data(), a[0][1].data(),
                                                               a[0][2].data(), a[0][3].data(), m1) : 0.0;
                ShuffleFisherYates(I1.data(), 0, n1, engine(seed, step, cell, cidx, 0));
                const int half = n1 / 2;
                for (int k = 0; k < n1 / 2; ++k)
                    ElasticCollisionPerez(0, half, half, n1, I1.data(), I1.data(), soa[0], soa[0], n, n, T, T, q1, q1, m1,
                                          m1, dt, L, dV * 1.0, engine(seed, step, cell, cidx, 2 + k), true, k);
            }
        } else {                                       // BinaryCollision.H:613-730
            double w1 = 0.0, w2 = 0.0;
            for (int i = 0; i < n1; ++i) w1 += a[0][0][I1[i]];
            for (int i = 0; i < n2; ++i) w2 += a[1][0][I2[i]];
            const double nn1 = w1 / (dV * 1.0), nn2 = w2 / (dV * 1.0);
            double T1 = 0.0, T2 = 0.0;
            if (computeT) {
                T1 = ComputeTemperature(0, n1, I1.data(), a[0][0].data(), a[0][1].data(), a[0][2].data(), a[0][3].data(), m1);
                T2 = ComputeTemperature(0, n2, I2.data(), a[1][0].data(), a[1][1].data(), a[1][2].data(), a[1][3].data(), m2);
            }
            if (n1 >= 1 && n2 >= 1) {
                ShuffleFisherYates(I1.data(), 0, n1, engine(seed, step, cell, cidx, 0));
                ShuffleFisherYates(I2.data(), 0, n2, engine(seed, step, cell, cidx, 1));
                for (int k = 0; k < (n1 < n2 ? n1 : n2); ++k)
                    ElasticCollisionPerez(0, n1, 0, n2, I1.data(), I2.data(), soa[0], soa[1], nn1, nn2, T1, T2, q1, q2,
                                          m1, m2, dt, L, dV * 1.0, engine(seed, step, cell, cidx, 2 + k), false, k);
            }
        }
        for (int i = 0; i < n1; ++i) printf("%d ", I1[i]);
        printf("\n");
        for (int i = 0; i < n2; ++i) printf("%d ", I2[i]);
        printf("\n");
        for (int s = 0; s < 2; ++s)
            for (int i = 0; i < (s ? n2 : n1); ++i) printf("%.17g %.17g %.17g\n", a[s][1][i], a[s][2][i], a[s][3][i]);
    }
    return 0;
}
'''


def build(tree, d):
    for name, text in SHIM.items():
        path = os.path.join(d, "shim", name)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        open(path, "w").write(text)
    src = os.path.join(d, "prog.cpp")
    open(src, "w").write(PROGRAM)
    exe = os.path.join(d, "prog")
    # the stand-in headers first: they shadow Source/Utils/WarpXConst.H and Particles/WarpXParticleContainer.H
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wno-unused-result", "-I", os.path.join(d, "shim"), "-I",
                    os.path.join(tree, "Source"), src, "-o", exe], check=True)
    return exe


def canonical_cells(sp, geom):
    import collision_oracle as co
    g = co.cells_of(sp, geom)
    order = np.lexsort((sp["id"], g))
    return g, order


def run_case(exe, d, sp1, sp2, coll, geom, dt, step):
    """the reference headers on one collision call: returns (u1, u2) in storage order and the shuffles per cell"""
    same = bool(coll["same_species"])
    dxs = [(geom["prob_hi"][k] - geom["prob_lo"][k]) / geom["n_cell"][k] for k in range(3)]
    dV = dxs[0] * dxs[1] * dxs[2]
    g1, o1 = canonical_cells(sp1, geom)
    g2, o2 = canonical_cells(sp2, geom) if not same else (np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64))
    cells = np.union1d(g1, g2)
    lines = ["%d %.17g %.17g %.17g %.17g %.17g %.17g %.17g %d %d %d %d" % (
        int(same), coll["q1"], coll["m1"], coll["q2"], coll["m2"], coll["coulomb_log"], dt, dV, coll["seed"], step,
        coll["collision_index"], len(cells))]
    members = []
    for c in cells:
        m1 = o1[g1[o1] == c]
        m2 = o2[g2[o2] == c] if not same else np.zeros(0, dtype=np.int64)
        members.append((m1, m2))
        lines.append("%d %d %d" % (c, len(m1), len(m2)))
        for sp, m in ((sp1, m1), (sp2, m2)):
            for i in m:
                lines.append("%.17g %.17g %.17g %.17g" % (sp["w"][i], sp["ux"][i], sp["uy"][i], sp["uz"][i]))
    path = os.path.join(d, "in.txt")
    open(path, "w").write("\n".join(lines) + "\n")
    out = subprocess.run([exe, path, "r"], check=True, capture_output=True, text=True).stdout.split("\n")
    u1 = np.stack([sp1["ux"], sp1["uy"], sp1["uz"]]).copy()
    u2 = None if same else np.stack([sp2["ux"], sp2["uy"], sp2["uz"]]).copy()
    shuffles, k = [], 0
    for (m1, m2) in members:
        s1 = [int(v) for v in out[k].split()]
        s2 = [int(v) for v in out[k + 1].split()]
        shuffles.append((s1, s2))
        k += 2
        for u, m in ((u1, m1), (u2, m2)):
            for i in m:
                u[:, i] = [float(v) for v in out[k].split()]
                k += 1
    return u1, u2, shuffles


def search_redraw(exe, d, seed, cell, cidx, thr):
    path = os.path.join(d, "s.txt")
    open(path, "w").write("%d %d %d %.17g 0\n" % (seed, cell, cidx, thr))
    return int(subprocess.run([exe, path, "s"], check=True, capture_output=True, text=True).stdout)


def cases(exe, d):
    import collision_cases as cc
    import collision_oracle as co
    from warpx_b200 import workloads
    C = workloads.C
    out = []
    rng = np.random.default_rng(77)

    def counts(mean, big):
        n = rng.poisson(mean, size=(4, 5, 6))
        n[0, 0, 0:4] = (0, 1, 2, 3)
        n[1, 1, 1] = big
        n[2, 2, 2] = 5                                    # odd
        return n
    for dt in (1e-17, 3e-15, 3e-14, 1e-11):
        out.append(("ee_fixed_%g" % dt, cc.particle_set(21, cc.GEOM, counts(4.0, 70), (0.01, 0.02, 0.01)), None,
                    cc.ee_spec(L=15.9), dt, 4))
        out.append(("ei_computed_%g" % dt,
                    cc.particle_set(22, cc.GEOM, counts(5.0, 90), (0.01, 0.02, 0.01), weights="log"),
                    cc.particle_set(23, cc.GEOM, counts(2.0, 40), (0.004, 0.004, 0.004), u_m=(0.01, 0, 0), weights="log",
                                    id_offset=10 ** 6), cc.ei_spec(L=-1.0), dt, 7))
    # computed Coulomb log: slow pairs (b0/2 > hbar/2p), fast pairs (quantum), dense and cold (the floor of 2)
    out.append(("ee_classical", cc.particle_set(24, cc.GEOM, 6.0, (1e-4, 1e-4, 1e-4)), None, cc.ee_spec(L=-1.0), 1e-12, 1))
    out.append(("ee_quantum", cc.particle_set(25, cc.GEOM, 6.0, (0.2, 0.2, 0.2)), None, cc.ee_spec(L=-1.0), 1e-14, 1))
    out.append(("ee_floor", cc.particle_set(26, cc.GEOM, 6.0, (1e-3, 1e-3, 1e-3), w0=1e14), None, cc.ee_spec(L=-1.0),
                1e-18, 1))
    out.append(("ee_relativistic", cc.particle_set(27, cc.GEOM, 6.0, (10.0, 10.0, 10.0), weights="log"), None,
                cc.ee_spec(L=-1.0), 1e-13, 2))
    # identical momenta in one cell, p* along z in another
    sp = cc.particle_set(28, cc.GEOM, 4.0, (0.01, 0.01, 0.01))
    cell = co.cells_of(sp, cc.GEOM)
    cs = np.unique(cell)
    a = np.flatnonzero(cell == cs[0])
    for k in ("ux", "uy", "uz"):
        sp[k][a] = sp[k][a[0]]
    b = np.flatnonzero(cell == cs[1])
    sp["ux"][b] = 0.0
    sp["uy"][b] = 0.0
    out.append(("ee_identical_and_axis", sp, None, cc.ee_spec(L=15.9), 3e-15, 3))
    # a forced redraw: one pair, s12 just under 0.1, a step whose first draw of chain 0 lies below exp(-2/s12)
    geom1 = dict(n_cell=(1, 1, 1), prob_lo=(0.0, 0.0, 0.0), prob_hi=(1e-6, 1e-6, 1e-6), box_lo=(0, 0, 0), box_hi=(0, 0, 0))
    pair = dict(x=np.array([2e-7, 6e-7]), y=np.array([3e-7, 5e-7]), z=np.array([4e-7, 1e-7]), w=np.array([1e9, 1e9]),
                ux=np.array([0.01 * C, -0.004 * C]), uy=np.array([0.002 * C, 0.0]), uz=np.array([0.0, 0.003 * C]),
                id=np.array([0, 1], dtype=np.int64))
    spec = cc.ee_spec(L=15.9, seed=3, cidx=0)
    co.collide({k: v.copy() for k, v in pair.items()}, None, spec, geom1, 1.0, 0)
    dt = 0.099 / float(co.LAST_S12[0][0])
    thr = np.exp(-2.0 / 0.099)
    step = search_redraw(exe, d, spec["seed"], 0, 0, thr)
    out.append(("ee_redraw", pair, None, spec, dt, step, geom1))
    return out


def main():
    tree = sys.argv[1]
    store = {}
    with tempfile.TemporaryDirectory() as d:
        exe = build(tree, d)
        import collision_cases as cc
        for case in cases(exe, d):
            name, sp1, sp2, coll, dt, step = case[:6]
            geom = case[6] if len(case) > 6 else cc.GEOM
            u1, u2, _ = run_case(exe, d, sp1, sp2, coll, geom, dt, step)
            p = name + "/"
            for k, v in sp1.items():
                store[p + "sp1_" + k] = v
            store[p + "u1"] = u1
            if sp2 is not None:
                for k, v in sp2.items():
                    store[p + "sp2_" + k] = v
                store[p + "u2"] = u2
            store[p + "coll"] = np.array([coll[k] for k in ("q1", "m1", "q2", "m2", "coulomb_log")] + [dt, step])
            store[p + "ints"] = np.array([coll["seed"], coll["collision_index"], coll["same_species"]], dtype=np.int64)
            store[p + "geom"] = np.array(list(geom["n_cell"]) + list(geom["prob_lo"]) + list(geom["prob_hi"]) +
                                         list(geom["box_lo"]) + list(geom["box_hi"]), dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "collision_reference.npz"), **store)
    print("wrote", len({k.split("/")[0] for k in store}), "cases")


if __name__ == "__main__":
    main()
