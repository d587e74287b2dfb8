#!/usr/bin/env python3
"""Regenerates tests/golden/flux_reference.npz: what the reference's own Gaussian-flux sampler computes.

    python tests/golden/make_flux_reference.py <WarpX source tree>

A small C++ program includes Source/Initialization/SampleGaussianFluxDistribution.H from the given tree, unchanged,
against a one-file stand-in for <AMReX_Random.H> written here: amrex::Real, the literals, AMREX_FORCE_INLINE /
AMREX_GPU_HOST_DEVICE, and an amrex::RandomEngine that replays this project's Philox4x64-10 streams (key (seed, 0),
counter (j + 1, step, cell, 2^63 | 2^61 | injector index << 32 | tag), the flux-injection counters of
csrc/flux_injection.cu) with amrex::Random = ((w >> 11) + 1) 2^-53 and amrex::RandomNormal = Box-Muller on two
consecutive uniforms, the cosine branch -- the project's definitions.  Sample i of a case draws
generateGaussianFluxDist(u_m, u_th) from the stream of cell i; the fixture stores the samples and how many words each
took.

Cases: u_m = 0; both rejection branches at 0.59 and 0.61 u_th; negative u_m in either branch; u_th = 0; long rejection
runs (u_m far below zero, where the normal draws of the second branch are mostly negative)."""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

SHIM = r'''#pragma once
#include <cstdint>
#include <cmath>
#define AMREX_GPU_HOST_DEVICE
#define AMREX_FORCE_INLINE inline
namespace amrex {
using Real = double;
namespace literals {
constexpr double operator""_rt(long double x) { return double(x); }
constexpr double operator""_rt(unsigned long long x) { return double(x); }
}
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
inline double RandomNormal(double mean, double stddev, const RandomEngine& e) {
    const double u1 = Random(e);
    const double u2 = Random(e);
    return mean + stddev * (std::sqrt(-2.0 * std::log(u1)) * std::cos(2.0 * 3.14159265358979323846 * u2));
}
}
'''

PROGRAM = r'''
#include <cstdio>
#include <cstdlib>
#include "Initialization/SampleGaussianFluxDistribution.H"
int main(int argc, char** argv) {
    // u_m u_th seed step index tag n
    const double u_m = atof(argv[1]), u_th = atof(argv[2]);
    const uint64_t seed = strtoull(argv[3], nullptr, 10), step = strtoull(argv[4], nullptr, 10);
    const uint64_t index = strtoull(argv[5], nullptr, 10), tag = strtoull(argv[6], nullptr, 10);
    const long n = atol(argv[7]);
    for (long i = 0; i < n; ++i) {
        amrex::RandomEngine e;
        e.seed = seed; e.c1 = step; e.c2 = (uint64_t)i; e.c3 = (1ull << 63) | (1ull << 61) | (index << 32) | tag;
        const double u = generateGaussianFluxDist(u_m, u_th, e);
        printf("%.17g %llu\n", u, (unsigned long long)e.drawn);
    }
    return 0;
}
'''

# name: (u_m, u_th, seed, step, injector index, tag, samples)
CASES = {
    "um_zero": (0.0, 0.1, 11, 0, 0, 1, 4000),
    "branch1_below_0p6": (0.059, 0.1, 12, 3, 1, 2, 4000),
    "branch2_above_0p6": (0.061, 0.1, 13, 7, 0, 1, 4000),
    "negative_branch1": (-0.05, 0.1, 14, 1, 2, 3, 4000),
    "negative_branch2": (-0.07, 0.1, 15, 2, 0, 1, 4000),
    "large_um": (1.5, 0.2, 16, 4, 3, 5, 2000),
    "u_th_zero": (0.3, 0.0, 17, 0, 0, 1, 50),
    "long_rejection_runs": (-0.3, 0.1, 18, 9, 1, 4, 40),
}


def build(tree, d):
    os.makedirs(os.path.join(d, "shim"), exist_ok=True)
    with open(os.path.join(d, "shim", "AMReX_Random.H"), "w") as f:
        f.write(SHIM)
    src = os.path.join(d, "flux_reference.cpp")
    with open(src, "w") as f:
        f.write(PROGRAM)
    exe = os.path.join(d, "flux_reference")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(d, "shim"), "-I",
                    os.path.join(tree, "Source"), src, "-o", exe], check=True)
    return exe


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    tree = sys.argv[1]
    out = {}
    with tempfile.TemporaryDirectory() as d:
        exe = build(tree, d)
        for name, (u_m, u_th, seed, step, index, tag, n) in CASES.items():
            text = subprocess.run([exe, repr(u_m), repr(u_th), str(seed), str(step), str(index), str(tag), str(n)],
                                  check=True, capture_output=True, text=True).stdout.split()
            vals = np.array(text, dtype=object).reshape(-1, 2)
            out[name + "/params"] = np.array([u_m, u_th], dtype=np.float64)
            out[name + "/ints"] = np.array([seed, step, index, tag, n], dtype=np.int64)
            out[name + "/u"] = np.array([float(v) for v in vals[:, 0]], dtype=np.float64)
            out[name + "/words"] = np.array([int(v) for v in vals[:, 1]], dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "flux_reference.npz"), **out)
    print("wrote", os.path.join(HERE, "flux_reference.npz"), "with", len(CASES), "cases")


if __name__ == "__main__":
    main()
