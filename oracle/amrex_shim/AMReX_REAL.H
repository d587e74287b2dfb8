// Minimal stand-in for AMReX (un-vendored dependency of the reference, pinned at
// 62c2a81eac7862d526e5861ef2befc00b7f5b759, >= 24.10) -- TEST INFRASTRUCTURE ONLY.
// It provides just enough of the AMReX vocabulary for a handful of WarpX *leaf* headers
// (shape factors, pushers, FDTD stencil policies, constants) to be compiled VERBATIM from
// a WarpX source tree so that the oracle's restated arithmetic can be checked against the real
// thing.  Double precision build (WarpX_PRECISION=DOUBLE, CMakeLists.txt:110,117).
#ifndef SHIM_AMREX_REAL_H_
#define SHIM_AMREX_REAL_H_
#include <cmath>
namespace amrex {
using Real = double;
using ParticleReal = double;
using Long = long;
inline namespace literals {
constexpr Real operator"" _rt(long double x) { return static_cast<Real>(x); }
constexpr Real operator"" _rt(unsigned long long x) { return static_cast<Real>(x); }
constexpr ParticleReal operator"" _prt(long double x) { return static_cast<ParticleReal>(x); }
constexpr ParticleReal operator"" _prt(unsigned long long x) { return static_cast<ParticleReal>(x); }
}
}
#endif
