#!/usr/bin/env python3
"""Regenerates tests/golden/fluid_reference_stages.npz: what the reference's own fluid leaf headers compute.

    python tests/golden/make_fluid_reference.py <WarpX source tree>

A small C++ program includes Source/Fluids/MusclHancockUtils.H and Source/Particles/Pusher/UpdateMomentumHigueraCary.H
from the given tree, unchanged, against a minimal AMReX stand-in written here (Array4, Box::contains, Real literals;
PhysConst::c from Source/ablastr/constant.H's value).  Its two loops have the shape of
WarpXFluidContainer::AdvectivePush_Muscl (Source/Fluids/WarpXFluidContainer.cpp:538-805): the prediction loop over
the valid nodes grown by one writes the six edge temporaries through compute_U_edges, positivity_limiter and
set_U_edges_to_zero, with their box checks, and the update loop applies dF.  All branch logic is in the headers; the
loops only call them.  The program also applies UpdateMomentumHigueraCary to given momenta and fields.

Inputs: seeded states of tests/fluid_cases.py and tests/fluid_oracle.py, one of them a vacuum edge at the step where
the positivity limiter acts.  The fixture stores inputs and outputs; the tests feed the inputs to the numpy
restatement and to the product's kernels and compare bit for bit."""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

SHIM = {
    "AMReX.H": "#pragma once\n#include <cmath>\n#include <algorithm>\n#define AMREX_GPU_HOST_DEVICE\n#define AMREX_FORCE_INLINE inline\n"
               "#define AMREX_INLINE inline\nnamespace amrex { using Real = double;\n"
               "namespace literals { constexpr double operator\"\"_rt(long double v) { return double(v); }\n"
               "constexpr double operator\"\"_rt(unsigned long long v) { return double(v); }\n"
               "constexpr double operator\"\"_prt(long double v) { return double(v); }\n"
               "constexpr double operator\"\"_prt(unsigned long long v) { return double(v); } }\n"
               "struct Box { int lo[3], hi[3];\n  bool contains(int i, int j, int k) const { return i >= lo[0] && i <= hi[0] && "
               "j >= lo[1] && j <= hi[1] && k >= lo[2] && k <= hi[2]; } };\n"
               "template <class T> struct Array4 { T* p; int lo[3], n[3], nc;\n"
               "  T& operator()(int i, int j, int k, int c = 0) const { return p[(i - lo[0]) + (long)n[0] * ((j - lo[1]) + "
               "(long)n[1] * ((k - lo[2]) + (long)n[2] * c))]; } };\n"
               "inline void ignore_unused(...) {} }\n",
    "AMReX_Array4.H": "#pragma once\n#include \"AMReX.H\"\n",
    "AMReX_Gpu.H": "#pragma once\n#include \"AMReX.H\"\n",
    "AMReX_REAL.H": "#pragma once\n#include \"AMReX.H\"\n",
    "AMReX_FArrayBox.H": "#pragma once\n#include \"AMReX.H\"\n",
    "Utils/WarpXConst.H": "#pragma once\nnamespace PhysConst { constexpr double c = 299792458.0; }\n",
}

PROGRAM = r'''
#include <cstdio>
#include <vector>
#include "Fluids/MusclHancockUtils.H"
#include "Particles/Pusher/UpdateMomentumHigueraCary.H"
using amrex::Array4; using amrex::Box;
static Array4<double> view(std::vector<double>& v, const int lo[3], const int hi[3], int nc) {
    Array4<double> a; a.p = v.data(); a.nc = nc;
    for (int d = 0; d < 3; ++d) { a.lo[d] = lo[d]; a.n[d] = hi[d] - lo[d] + 1; }
    return a;
}
int main(int argc, char** argv) {
    // advect <in> <out>: header "vlo0 vlo1 vlo2 vhi0 vhi1 vhi2 dx dy dz dt" then N NUx NUy NUz over vlo-2..vhi+2
    if (std::string(argv[1]) == "advect") {
        FILE* f = fopen(argv[2], "rb");
        int vlo[3], vhi[3]; double dx[3], dt;
        fread(vlo, 4, 3, f); fread(vhi, 4, 3, f); fread(dx, 8, 3, f); fread(&dt, 8, 1, f);
        int alo[3], ahi[3]; long n = 1;
        for (int d = 0; d < 3; ++d) { alo[d] = vlo[d] - 2; ahi[d] = vhi[d] + 2; n *= ahi[d] - alo[d] + 1; }
        std::vector<double> s[4];
        for (int c = 0; c < 4; ++c) { s[c].resize(n); fread(s[c].data(), 8, n, f); }
        fclose(f);
        auto N = view(s[0], alo, ahi, 1), NUx = view(s[1], alo, ahi, 1), NUy = view(s[2], alo, ahi, 1), NUz = view(s[3], alo, ahi, 1);
        const double clight = PhysConst::c;
        // edge temporaries: valid box grown by 1, converted to the edge index type (one 4-component array per side)
        Box bx[3]; std::vector<double> mem[6]; Array4<double> Um[3], Up[3];
        for (int d = 0; d < 3; ++d) {
            int lo[3], hi[3];
            for (int e = 0; e < 3; ++e) { lo[e] = vlo[e] - 1; hi[e] = vhi[e] + 1 - (e == d ? 1 : 0); bx[d].lo[e] = lo[e]; bx[d].hi[e] = hi[e]; }
            long m = 4; for (int e = 0; e < 3; ++e) m *= hi[e] - lo[e] + 1;
            mem[2 * d].assign(m, 0.0); mem[2 * d + 1].assign(m, 0.0);
            Um[d] = view(mem[2 * d], lo, hi, 4); Up[d] = view(mem[2 * d + 1], lo, hi, 4);
        }
        const double dt_over_dx = (dt/dx[0]), dt_over_dy = (dt/dx[1]), dt_over_dz = (dt/dx[2]);
        const double dt_over_dx_half = 0.5*(dt/dx[0]), dt_over_dy_half = 0.5*(dt/dx[1]), dt_over_dz_half = 0.5*(dt/dx[2]);
        for (int k = vlo[2] - 1; k <= vhi[2] + 1; ++k) for (int j = vlo[1] - 1; j <= vhi[1] + 1; ++j) for (int i = vlo[0] - 1; i <= vhi[0] + 1; ++i) {
            if (N(i,j,k) > 0.0) {
                double Ux = (NUx(i,j,k) / N(i,j,k)), Uy = (NUy(i,j,k) / N(i,j,k)), Uz = (NUz(i,j,k) / N(i,j,k));
                const double c_sq = clight*clight;
                const double gamma = std::sqrt(1.0 + (Ux*Ux + Uy*Uy + Uz*Uz)/(c_sq));
                const double inv_c2_gamma3 = 1./(c_sq*gamma*gamma*gamma);
                const double Vx = Ux/gamma, Vy = Uy/gamma, Vz = Uz/gamma;
                const double J00x = Vx, J01x = N(i,j,k)*(1/gamma)*(1-Vx*Vx/c_sq), J02x = -N(i,j,k)*Uy*Ux*inv_c2_gamma3, J03x = -N(i,j,k)*Uz*Ux*inv_c2_gamma3;
                const double J00y = Vy, J01y = -N(i,j,k)*Ux*Uy*inv_c2_gamma3, J02y = N(i,j,k)*(1/gamma)*(1-Vy*Vy/c_sq), J03y = -N(i,j,k)*Uz*Uy*inv_c2_gamma3;
                const double J00z = Vz, J01z = -N(i,j,k)*Ux*Uz*inv_c2_gamma3, J02z = -N(i,j,k)*Uy*Uz*inv_c2_gamma3, J03z = N(i,j,k)*(1/gamma)*(1-Vz*Vz/c_sq);
                const double dU0x = ave(DownDx_N(N,i,j,k), UpDx_N(N,i,j,k)), dU1x = ave(DownDx_U(N,NUx,Ux,i,j,k), UpDx_U(N,NUx,Ux,i,j,k));
                const double dU2x = ave(DownDx_U(N,NUy,Uy,i,j,k), UpDx_U(N,NUy,Uy,i,j,k)), dU3x = ave(DownDx_U(N,NUz,Uz,i,j,k), UpDx_U(N,NUz,Uz,i,j,k));
                const double dU0y = ave(DownDy_N(N,i,j,k), UpDy_N(N,i,j,k)), dU1y = ave(DownDy_U(N,NUx,Ux,i,j,k), UpDy_U(N,NUx,Ux,i,j,k));
                const double dU2y = ave(DownDy_U(N,NUy,Uy,i,j,k), UpDy_U(N,NUy,Uy,i,j,k)), dU3y = ave(DownDy_U(N,NUz,Uz,i,j,k), UpDy_U(N,NUz,Uz,i,j,k));
                const double dU0z = ave(DownDz_N(N,i,j,k), UpDz_N(N,i,j,k)), dU1z = ave(DownDz_U(N,NUx,Ux,i,j,k), UpDz_U(N,NUx,Ux,i,j,k));
                const double dU2z = ave(DownDz_U(N,NUy,Uy,i,j,k), UpDz_U(N,NUy,Uy,i,j,k)), dU3z = ave(DownDz_U(N,NUz,Uz,i,j,k), UpDz_U(N,NUz,Uz,i,j,k));
                const double JdU0x = J00x*dU0x + J01x*dU1x + J02x*dU2x + J03x*dU3x, JdU1x = Vx*dU1x, JdU2x = Vx*dU2x, JdU3x = Vx*dU3x;
                const double JdU0y = J00y*dU0y + J01y*dU1y + J02y*dU2y + J03y*dU3y, JdU1y = Vy*dU1y, JdU2y = Vy*dU2y, JdU3y = Vy*dU3y;
                const double JdU0z = J00z*dU0z + J01z*dU1z + J02z*dU2z + J03z*dU3z, JdU1z = Vz*dU1z, JdU2z = Vz*dU2z, JdU3z = Vz*dU3z;
                const double U_tilde0 = N(i,j,k) - dt_over_dx_half*JdU0x - dt_over_dy_half*JdU0y - dt_over_dz_half*JdU0z;
                const double U_tilde1 = Ux - dt_over_dx_half*JdU1x - dt_over_dy_half*JdU1y - dt_over_dz_half*JdU1z;
                const double U_tilde2 = Uy - dt_over_dx_half*JdU2x - dt_over_dy_half*JdU2y - dt_over_dz_half*JdU2z;
                const double U_tilde3 = Uz - dt_over_dx_half*JdU3x - dt_over_dy_half*JdU3y - dt_over_dz_half*JdU3z;
                compute_U_edges(Um[0], Up[0], i, j, k, bx[0], U_tilde0, U_tilde1, U_tilde2, U_tilde3, dU0x, dU1x, dU2x, dU3x, 0);
                positivity_limiter(Up[0], Um[0], N, i, j, k, bx[0], Ux, Uy, Uz, 0);
                compute_U_edges(Um[1], Up[1], i, j, k, bx[1], U_tilde0, U_tilde1, U_tilde2, U_tilde3, dU0y, dU1y, dU2y, dU3y, 1);
                positivity_limiter(Up[1], Um[1], N, i, j, k, bx[1], Ux, Uy, Uz, 1);
                compute_U_edges(Um[2], Up[2], i, j, k, bx[2], U_tilde0, U_tilde1, U_tilde2, U_tilde3, dU0z, dU1z, dU2z, dU3z, 2);
                positivity_limiter(Up[2], Um[2], N, i, j, k, bx[2], Ux, Uy, Uz, 2);
            } else {
                for (int d = 0; d < 3; ++d) set_U_edges_to_zero(Um[d], Up[d], i, j, k, bx[d], d);
            }
        }
        std::vector<double> o[4];
        for (int c = 0; c < 4; ++c) o[c] = s[c];
        auto oN = view(o[0], alo, ahi, 1), oX = view(o[1], alo, ahi, 1), oY = view(o[2], alo, ahi, 1), oZ = view(o[3], alo, ahi, 1);
        for (int k = vlo[2]; k <= vhi[2]; ++k) for (int j = vlo[1]; j <= vhi[1]; ++j) for (int i = vlo[0]; i <= vhi[0]; ++i) {
            oN(i,j,k) = N(i,j,k) - dt_over_dx*dF(Um[0],Up[0],i,j,k,clight,0,0) - dt_over_dy*dF(Um[1],Up[1],i,j,k,clight,0,1) - dt_over_dz*dF(Um[2],Up[2],i,j,k,clight,0,2);
            oX(i,j,k) = NUx(i,j,k) - dt_over_dx*dF(Um[0],Up[0],i,j,k,clight,1,0) - dt_over_dy*dF(Um[1],Up[1],i,j,k,clight,1,1) - dt_over_dz*dF(Um[2],Up[2],i,j,k,clight,1,2);
            oY(i,j,k) = NUy(i,j,k) - dt_over_dx*dF(Um[0],Up[0],i,j,k,clight,2,0) - dt_over_dy*dF(Um[1],Up[1],i,j,k,clight,2,1) - dt_over_dz*dF(Um[2],Up[2],i,j,k,clight,2,2);
            oZ(i,j,k) = NUz(i,j,k) - dt_over_dx*dF(Um[0],Up[0],i,j,k,clight,3,0) - dt_over_dy*dF(Um[1],Up[1],i,j,k,clight,3,1) - dt_over_dz*dF(Um[2],Up[2],i,j,k,clight,3,2);
        }
        f = fopen(argv[3], "wb");
        for (int c = 0; c < 4; ++c) fwrite(o[c].data(), 8, n, f);
        fclose(f);
    } else {   // hc <in> <out>: "n q m dt" then ux uy uz Ex Ey Ez Bx By Bz (n each)
        FILE* f = fopen(argv[2], "rb");
        long n; double q, m, dt;
        fread(&n, 8, 1, f); fread(&q, 8, 1, f); fread(&m, 8, 1, f); fread(&dt, 8, 1, f);
        std::vector<double> a(9 * n);
        fread(a.data(), 8, 9 * n, f);
        fclose(f);
        for (long p = 0; p < n; ++p)
            UpdateMomentumHigueraCary(a[p], a[n + p], a[2 * n + p], a[3 * n + p], a[4 * n + p], a[5 * n + p], a[6 * n + p],
                                      a[7 * n + p], a[8 * n + p], q, m, dt);
        f = fopen(argv[3], "wb");
        fwrite(a.data(), 8, 3 * n, f);
        fclose(f);
    }
    return 0;
}
'''


def build(ref, d):
    for name, text in SHIM.items():
        p = os.path.join(d, "shim", name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        open(p, "w").write(text)
    src = os.path.join(d, "fluid_ref.cpp")
    open(src, "w").write("#include <string>\n" + PROGRAM)
    exe = os.path.join(d, "fluid_ref")
    subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-DWARPX_DIM_3D", "-w", "-I", os.path.join(d, "shim"), "-I",
                    os.path.join(ref, "Source"), src, "-o", exe], check=True)
    return exe


def run_advect(exe, d, state, desc, dx, dt):
    vlo = [desc.lo[k] + 2 for k in range(3)]
    vhi = [desc.hi[k] - 2 for k in range(3)]
    fin, fout = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(fin, "wb") as f:
        f.write(np.array(vlo + vhi, dtype=np.int32).tobytes() + np.array(list(dx) + [dt]).tobytes())
        for a in state:
            f.write(np.ascontiguousarray(a).tobytes())
    subprocess.run([exe, "advect", fin, fout], check=True)
    return np.fromfile(fout).reshape((4,) + state[0].shape)


def cases():
    """(name, state, descriptor, dx, dt): seeded advection inputs, guards filled."""
    import math
    import fluid_cases
    import fluid_oracle as fo
    from oracle import oracle as orc
    out = []
    for kind, box in (("vacuum", ((8, 4, 12), (15, 11, 19))), ("drift", ((0, 0, 0), (7, 7, 7)))):
        desc, st, dx = fluid_cases.make_state(kind, (24,) * 3, *box)
        dt = 0.99 / (fluid_cases.workloads.C * math.sqrt(sum(1.0 / v ** 2 for v in dx)))
        out.append((kind, st, desc, dx, dt))
    # a vacuum edge evolved until the positivity limiter acts: the input of that step's advection
    density, momentum, _ = fluid_cases._inputs("vacuum", (16,) * 3, u=0.3)
    run = fo.FluidRun(orc, (16,) * 3, (-fluid_cases.LX / 2,) * 3, (fluid_cases.LX / 2,) * 3)
    run.add_fluid(-fluid_cases.workloads.Q_E, fluid_cases.workloads.M_E, density, momentum)
    fl = run.fluids[0]
    captured = []
    orig = fo.advect

    def spy(state, desc, dx, dt, counters=None):
        c = {}
        orig(state, desc, dx, dt, c)
        if c["limited"] > 0 and not captured:
            captured.append([a.copy() for a in state])
        return orig(state, desc, dx, dt, counters)
    fo.advect = spy
    try:
        for _ in range(12):
            run.step(False)
            if captured:
                break
    finally:
        fo.advect = orig
    assert captured, "the limiter never acted"
    out.append(("vacuum_limited", captured[0], fl["desc"], run.dx, run.dt))
    return out


def main():
    ref = sys.argv[1]
    data = {}
    with tempfile.TemporaryDirectory() as d:
        exe = build(ref, d)
        for name, st, desc, dx, dt in cases():
            data[name + "/in"] = np.stack(st)
            data[name + "/out"] = run_advect(exe, d, st, desc, dx, dt)
            data[name + "/desc"] = np.array([desc.lo[k] for k in range(3)] + [desc.hi[k] for k in range(3)])
            data[name + "/dxdt"] = np.array(list(dx) + [dt])
        rng = np.random.default_rng(7)
        n = 4096
        u = rng.uniform(-20, 20, (3, n)) * 299792458.0
        e = rng.uniform(-1e13, 1e13, (3, n))
        b = rng.uniform(-3e4, 3e4, (3, n))
        q, m, dt = -1.602176634e-19, 9.1093837015e-31, 1e-15
        fin, fout = os.path.join(d, "hin.bin"), os.path.join(d, "hout.bin")
        with open(fin, "wb") as f:
            f.write(np.array([n], dtype=np.int64).tobytes() + np.array([q, m, dt]).tobytes())
            f.write(np.concatenate([u, e, b]).tobytes())
        subprocess.run([exe, "hc", fin, fout], check=True)
        data["hc/in"] = np.concatenate([u, e, b])
        data["hc/qmdt"] = np.array([q, m, dt])
        data["hc/out"] = np.fromfile(fout).reshape(3, n)
    np.savez_compressed(os.path.join(HERE, "fluid_reference_stages.npz"), **data)


if __name__ == "__main__":
    main()
