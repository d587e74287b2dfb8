// Nuclear fusion (collisions.collision_names, <name>.type = nuclearfusion) over the rank's box: two-product reactions and
// proton-boron.
//
// Restates, for one tile = the rank's box (paths relative to Source/Particles/Collision/BinaryCollision/):
//   fuse_cell / chains   <- BinaryCollision::doCollisionsWithinTile  BinaryCollision.H:383-472 (intra-species, halves),
//                           :613-730 (inter-species), with NuclearFusionFunc::Executor  NuclearFusion/NuclearFusionFunc.H:127-234
//   collision_parameters <- BinaryCollisionUtils::get_collision_parameters             BinaryCollisionUtils.H
//   bosch_hale           <- BoschHaleFusionCrossSection                                NuclearFusion/BoschHaleFusionCrossSection.H
//   fusion_event         <- SingleNuclearFusionEvent                                   NuclearFusion/SingleNuclearFusionEvent.H
//   product_momenta      <- TwoProductFusionComputeProductMomenta + RandomizeVelocity  NuclearFusion/TwoProductFusionUtil.H,
//                                                                                      Utils/ParticleUtils.H:137-175
//   create_kernel        <- ParticleCreationFunc::operator() for two products          ParticleCreationFunc.H:120-230
//   proton_boron         <- ProtonBoronFusionCrossSection (Tentori + Buck)             NuclearFusion/ProtonBoronFusionCrossSection.H
//   alpha_momenta        <- ProtonBoronFusionInitializeMomentum                        NuclearFusion/ProtonBoronFusionInitializeMomentum.H
//   create_kernel<true>  <- ParticleCreationFunc::operator() for p + B11 -> 3 alpha    ParticleCreationFunc.H:170-200
//
// Determinism: the result is a function of (the particles of each cell by id, seed, collision index, step, global cell)
// and nothing else -- not of the storage order or the thread mapping.  The Coulomb pass's contract (collision.cu), with:
//   * canonical order: a cell's live particles of each species (id != PIC_SPENT_ID) in ascending id order.  Particles an
//     earlier fusion of the step spent are left out, as the reference's deleteInvalidParticles after each collision
//     leaves them out (BinaryCollision.H:212-218);
//   * random streams: key (seed, 0), counter (j + 1, step, global cell, 2^63 | collision index << 32 | tag): tags 0 and
//     1 shuffle species 1 and 2, tag 2 + c is pair chain c and draws ONE uniform per pair that reaches
//     SingleNuclearFusionEvent (pairs with a spent reactant draw nothing, NuclearFusionFunc.H:181-184).  The momenta of
//     the products of the cell's j-th event (in pair order) come from the stream with bit 62 also set in the last word:
//     (2^63 | 2^62 | collision index << 32 | j), two uniforms (RandomizeVelocity's theta, then z); for proton-boron
//     four (one Philox4x64 block): theta and z of the alpha + 8Be* emission, then theta and z of the 8Be* decay;
//   * product order: event e of the call counts events bin by bin (the supercell-major order of pic_bins), then by
//     pair index inside the cell (the chain position k of NuclearFusionFunc.H's pair_index); a two-product event
//     writes slots 2e, 2e + 1 of each product, a proton-boron event slots 6e + 2k, 6e + 2k + 1 of alpha k = 0, 1, 2;
//   * the file is compiled without FMA contraction.
//
// Event pass: one pass over the bins with the Coulomb pass's grouping -- a warp per cell of at most SMALL_CAP
// particles, a 256-thread block per cell of at most LARGE_CAP, and beyond that a block that keeps only the cell's
// canonical order in the caller's per-slot scratch.  A cell's pairs go to records at its own slots (cell_start of
// species 1 plus that of species 2), its pair and event counts to per-bin arrays: no global atomics.  Product pass:
// an exclusive scan of the event counts, one host read of the total, a warp per bin writing its events' products in
// pair order.
#include "binary_collision.cuh"
#include <cub/device/device_scan.cuh>

namespace pic {

namespace fus {

using coll::Stream;
using coll::dmax;
using coll::dmin;
using coll::DBL_MIN_;
using coll::PI;

constexpr double Q_E = 1.602176634e-19;         // PhysConst::q_e
constexpr double ALPHA = 0.007297352573748943;  // PhysConst::alpha
constexpr double M_U = 1.66053906660e-27;      // PhysConst::m_u
constexpr double EP0 = 8.8541878128e-12;       // PhysConst::ep0
constexpr double HBAR = 1.054571817e-34;       // PhysConst::hbar
constexpr double C_SQ = C_LIGHT * C_LIGHT;
constexpr double INV_CSQ = 1.0 / C_SQ;

constexpr int SMALL_CAP = 64;
constexpr int SMALL_WARPS = 4;
constexpr int LARGE_CAP = 2048;
constexpr int LARGE_THREADS = 256;
constexpr int LARGE_SCAN = 32;
constexpr uint64_t PRODUCT_TAG = 1ull << 62;

static size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// the workspace: per pair (at the cell's slots) the two reactants' storage indices, the reaction weight and the event
// flag; per bin the number of pairs and of events, the scan of the events, the scan's temporary storage
struct Work {
    int *slot1, *slot2;
    double* wr;
    unsigned char* mask;
    int *npairs, *events, *offsets;
    void* temp;
    size_t temp_bytes;
};

static size_t scan_bytes(long n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int*)nullptr, (int*)nullptr, (int)n);
    return bytes;
}

static Work carve(void* base, long pc, long nbins, size_t* total = nullptr) {
    Work w;
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char* q = p ? p + off : nullptr; off += align256(bytes); return q; };
    const size_t npc = (size_t)(pc > 0 ? pc : 1);
    w.slot1 = (int*)take(npc * 4);
    w.slot2 = (int*)take(npc * 4);
    w.wr = (double*)take(npc * 8);
    w.mask = (unsigned char*)take(npc);
    w.npairs = (int*)take((size_t)(nbins + 1) * 4);
    w.events = (int*)take((size_t)(nbins + 1) * 4);
    w.offsets = (int*)take((size_t)(nbins + 1) * 4);
    w.temp_bytes = scan_bytes(nbins + 1);
    w.temp = take(w.temp_bytes);
    if (total) *total = off;
    return w;
}

struct Args {
    SoaView P1, P2;
    uint64_t* id1; uint64_t* id2;
    const int* src1; const int* src2;
    int* scr1; int* scr2;
    BinsView b1, b2;
    int gn[2];
    double m1, m2, dt, dV;
    double mult, thr, target;
    int type;
    uint64_t seed, cidx, step;
    int same;
    Work wk;
    int* status;
};

// BinaryCollisionUtils::get_collision_parameters: kinetic energy and relative velocity in the centre-of-momentum frame,
// and the ratio of its Lorentz factors to the lab frame's
__host__ __device__ __forceinline__ void collision_parameters(double u1x, double u1y, double u1z, double u2x, double u2y,
                                                              double u2z, double m1, double m2, double& E_kin,
                                                              double& v_rel, double& lab_to_com) {
    const double m1_sq = m1 * m1, m2_sq = m2 * m2;
    const double g1 = sqrt(1.0 + (u1x * u1x + u1y * u1y + u1z * u1z) * INV_CSQ);
    const double g2 = sqrt(1.0 + (u2x * u2x + u2y * u2y + u2z * u2z) * INV_CSQ);
    const double p1x = u1x * m1, p1y = u1y * m1, p1z = u1z * m1;
    const double p2x = u2x * m2, p2y = u2y * m2, p2z = u2z * m2;
    const double sx = p1x + p2x, sy = p1y + p2y, sz = p1z + p2z;
    const double p_total_sq = sx * sx + sy * sy + sz * sz;
    const double E_lab = (m1 * g1 + m2 * g2) * C_SQ;
    const double E_star_sq = E_lab * E_lab - C_SQ * p_total_sq;
    const double E_star = sqrt(E_star_sq);
    E_kin = E_star - (m1 + m2) * C_SQ;
    const double E_ratio = E_star / ((m1 + m2) * C_SQ);
    const double dm = m1 - m2, er = E_ratio - 1.0 / E_ratio;
    const double p_star_sq = m1 * m2 * C_SQ * (E_ratio * E_ratio - 1.0) + dm * dm * C_SQ / 4.0 * (er * er);
    const double g1s = sqrt(1.0 + p_star_sq / (m1_sq * C_SQ));
    const double g2s = sqrt(1.0 + p_star_sq / (m2_sq * C_SQ));
    v_rel = sqrt(p_star_sq) * (1.0 / (m1 * g1s) + 1.0 / (m2 * g2s));
    lab_to_com = g1s * g2s / (g1 * g2);
}

// BoschHaleFusionCrossSection [m^2] of the centre-of-momentum kinetic energy E [J]
__host__ __device__ __forceinline__ double bosch_hale(double E, int type, double m1, double m2) {
    constexpr double joule_to_keV = 1.e-3 / Q_E;
    const double E_keV = E * joule_to_keV;
    if (E_keV == 0.0) return 0.0;
    const double m_reduced = m1 / (1.0 + m1 / m2);
    const double B_G = PI * ALPHA * sqrt(2.0 * m_reduced * C_LIGHT * C_LIGHT * joule_to_keV);
    double A1, A2, A3, A4, A5, B1, B2, B3, B4;
    if (type == PIC_FUSION_DT_NHE4) {
        A1 = 6.927e4; A2 = 7.454e8; A3 = 2.050e6; A4 = 5.2002e4; A5 = 0.0;
        B1 = 6.38e1; B2 = -9.95e-1; B3 = 6.981e-5; B4 = 1.728e-4;
    } else if (type == PIC_FUSION_DD_PT) {
        A1 = 5.5576e4; A2 = 2.1054e2; A3 = -3.2638e-2; A4 = 1.4987e-6; A5 = 1.8181e-10;
        B1 = 0.0; B2 = 0.0; B3 = 0.0; B4 = 0.0;
    } else {
        A1 = 5.3701e4; A2 = 3.3027e2; A3 = -1.2706e-1; A4 = 2.9327e-5; A5 = -2.5151e-9;
        B1 = 0.0; B2 = 0.0; B3 = 0.0; B4 = 0.0;
    }
    const double astrophysical_factor = (A1 + E_keV * (A2 + E_keV * (A3 + E_keV * (A4 + E_keV * A5)))) /
                                        (1.0 + E_keV * (B1 + E_keV * (B2 + E_keV * (B3 + E_keV * B4))));
    constexpr double millibarn_to_sqm = 1.e-31;
    return millibarn_to_sqm * astrophysical_factor / E_keV * exp(-B_G / sqrt(E_keV));
}

// ProtonBoronFusionCrossSectionTentori [barn] of the centre-of-momentum kinetic energy in keV (0 < E < 9.76 MeV)
__host__ __device__ __forceinline__ double pb_tentori(double E_keV) {
    if (E_keV == 0.0) return 0.0;
    const double E_MeV = E_keV * 1.e-3;
    constexpr double joule_to_MeV = 1.e-6 / Q_E;
    constexpr double one_pr = 1.0;
    constexpr double Z_boron = 5.0;
    constexpr double m_boron = 11.00930536 * M_U;
    constexpr double m_hydrogen = 1.00782503223 * M_U;
    constexpr double m_reduced = m_boron / (one_pr + m_boron / m_hydrogen);
    constexpr double gamow_factor = m_reduced / 2.0 * (Q_E * Q_E * Z_boron / (2.0 * EP0 * HBAR)) *
                                    (Q_E * Q_E * Z_boron / (2.0 * EP0 * HBAR)) * joule_to_MeV;
    double astrophysical_factor;
    if (E_keV < 400.0) {
        constexpr double C0 = 197.0, C1 = 0.269, C2 = 2.54e-4, AL = 1.82e4, EL = 148.0, dEL_sq = 2.35 * 2.35;
        astrophysical_factor = C0 + C1 * E_keV + C2 * (E_keV * E_keV) + AL / ((E_keV - EL) * (E_keV - EL) + dEL_sq);
    } else if (E_keV < 668.0) {
        constexpr double D0 = 346.0, D1 = 150.0, D2 = -59.9, D5 = -0.460;
        const double E_norm = (E_keV - 400.0) * 1.e-2;
        const double E_norm_sq = E_norm * E_norm;
        // amrex::Math::powi<5>(x) = x * powi<2>(powi<2>(x))
        astrophysical_factor = D0 + D1 * E_norm + D2 * E_norm_sq + D5 * (E_norm * (E_norm_sq * E_norm_sq));
    } else {
        constexpr double A0 = 1.98e6, A1 = 3.89e6, A2 = 1.36e6, A3 = 3.71e6;
        constexpr double E0 = 640.9, E1 = 1211.0, E2 = 2340.0, E3 = 3294.0;
        constexpr double dE0_sq = 85.5 * 85.5, dE1_sq = 414.0 * 414.0, dE2_sq = 221.0 * 221.0, dE3_sq = 351.0 * 351.0;
        constexpr double B = 0.381;
        astrophysical_factor = A0 / ((E_keV - E0) * (E_keV - E0) + dE0_sq) + A1 / ((E_keV - E1) * (E_keV - E1) + dE1_sq) +
                               A2 / ((E_keV - E2) * (E_keV - E2) + dE2_sq) + A3 / ((E_keV - E3) * (E_keV - E3) + dE3_sq) + B;
    }
    return astrophysical_factor / E_MeV * exp(-sqrt(gamow_factor / E_MeV));
}

// ProtonBoronFusionCrossSection [m^2] of the centre-of-momentum kinetic energy E [J]: Tentori up to 9.76 MeV, Buck's
// power law above
__host__ __device__ __forceinline__ double proton_boron(double E) {
    constexpr double joule_to_keV = 1.e-3 / Q_E;
    const double E_keV = E * joule_to_keV;
    const double cross_section_b = E_keV <= 9760.0 ? pb_tentori(E_keV)
                                                   : 0.01277998 * pow(E_keV / 9760.0, -2.661840717596765);
    return cross_section_b * 1.e-28;
}

// SingleNuclearFusionEvent: one uniform; returns the reaction weight w_min / multiplier_eff, or 0 without an event
__host__ __device__ __forceinline__ bool fusion_event(double u1x, double u1y, double u1z, double u2x, double u2y,
                                                     double u2z, double m1, double m2, double w1, double w2, double dt,
                                                     double dV, double mult, int multiplier_ratio, double thr,
                                                     double target, int type, Stream& rng, double* wr) {
    double E_coll, v_coll, lab_to_com;
    collision_parameters(u1x, u1y, u1z, u2x, u2y, u2z, m1, m2, E_coll, v_coll, lab_to_com);
    const double w_min = dmin(w1, w2);
    const double w_max = dmax(w1, w2);
    const double sigma = type == PIC_FUSION_PB_3HE4 ? proton_boron(E_coll) : bosch_hale(E_coll, type, m1, m2);
    double pe = multiplier_ratio * mult * lab_to_com * w_max * sigma * v_coll * dt / dV;
    double mult_eff = mult;
    if (pe > thr) {
        mult_eff = dmax(mult * target / pe, 1.0);
        pe *= mult_eff / mult;
    }
    const double probability = -expm1(-pe);
    const double r = rng.uniform();
    if (r < probability) { *wr = w_min / mult_eff; return true; }
    return false;
}

// TwoProductFusionComputeProductMomenta with RandomizeVelocity: u of product A (u1) and B (u2)
__host__ __device__ __forceinline__ void product_momenta(double u1x, double u1y, double u1z, double m1, double u2x,
                                                         double u2y, double u2z, double m2, double mA, double mB,
                                                         double E_fusion, Stream& rng, double* uA, double* uB) {
    const double E_rest_in = (m1 + m2) * C_SQ;
    const double E_rest_out = (mA + mB) * C_SQ;
    const double g1 = sqrt(1.0 + (u1x * u1x + u1y * u1y + u1z * u1z) * INV_CSQ);
    const double g2 = sqrt(1.0 + (u2x * u2x + u2y * u2y + u2z * u2z) * INV_CSQ);
    const double p1x = u1x * m1, p1y = u1y * m1, p1z = u1z * m1;
    const double p2x = u2x * m2, p2y = u2y * m2, p2z = u2z * m2;
    const double sx = p1x + p2x, sy = p1y + p2y, sz = p1z + p2z;
    const double p_total_sq = sx * sx + sy * sy + sz * sz;
    const double E_lab = (m1 * g1 + m2 * g2) * C_SQ;
    const double E_star_sq = E_lab * E_lab - C_SQ * p_total_sq;
    const double ef = sqrt(E_star_sq) - E_rest_in + E_rest_out + E_fusion;
    const double E_star_f_sq = ef * ef;
    const double E_ratio = sqrt(E_star_f_sq) / ((mA + mB) * C_SQ);
    const double dm = mA - mB, er = E_ratio - 1.0 / E_ratio;
    const double p_star_f_sq = mA * mB * C_SQ * (E_ratio * E_ratio - 1.0) + dm * dm * C_SQ * 0.25 * (er * er);
    // RandomizeVelocity(px*, py*, pz*, |p*|): getRandomVector draws theta, then z
    const double vp = sqrt(p_star_f_sq);
    const double theta = rng.uniform() * 2.0 * PI;
    const double z = 2.0 * rng.uniform() - 1.0;
    const double xy = sqrt(1.0 - z * z);
    double st, ct;
#ifdef __CUDA_ARCH__
    sincos(theta, &st, &ct);
#else
    st = sin(theta); ct = cos(theta);
#endif
    const double px = xy * ct * vp, py = xy * st * vp, pz = z * vp;
    const double mass_g = m1 * g1 + m2 * g2;
    const double vcx = sx / mass_g, vcy = sy / mass_g, vcz = sz / mass_g;
    const double vc_sq = vcx * vcx + vcy * vcy + vcz * vcz;
    double qx = px, qy = py, qz = pz;
    if (vc_sq > DBL_MIN_) {
        const double gc = 1.0 / sqrt(1.0 - vc_sq * INV_CSQ);
        const double g_star = sqrt(1.0 + p_star_f_sq / (mA * mA * C_SQ));
        const double vcDps = vcx * px + vcy * py + vcz * pz;
        const double factor0 = (gc - 1.0) / vc_sq;
        const double factor = factor0 * vcDps + mA * g_star * gc;
        qx = px + vcx * factor; qy = py + vcy * factor; qz = pz + vcz * factor;
    }
    uA[0] = qx / mA; uA[1] = qy / mA; uA[2] = qz / mA;
    uB[0] = (p1x + p2x - qx) / mB; uB[1] = (p1y + p2y - qy) / mB; uB[2] = (p1z + p2z - qz) / mB;
}

__host__ __device__ __forceinline__ double fusion_energy(int type) {   // ParticleCreationFunc.H:205-217
    return type == PIC_FUSION_DT_NHE4 ? 17.5893e6 * Q_E : (type == PIC_FUSION_DD_PT ? 4.032667e6 * Q_E : 3.268911e6 * Q_E);
}

// ProtonBoronFusionInitializeMomentum: p + B11 -> alpha + 8Be* (isotropic in the centre-of-momentum frame), then
// 8Be* -> 2 alpha (isotropic in its rest frame, boosted back with Perez eq. 13).  u[k] is alpha k's momentum.
__host__ __device__ __forceinline__ void alpha_momenta(double u1x, double u1y, double u1z, double m1, double u2x,
                                                       double u2y, double u2z, double m2, Stream& rng, double u[3][3]) {
    constexpr double mev_to_joule = Q_E * 1.e6;
    constexpr double E_fusion = 5.55610759 * mev_to_joule;
    constexpr double E_decay = 3.12600414 * mev_to_joule;
    constexpr double m_alpha = M_U * 4.00260325413;
    constexpr double m_beryllium = M_U * (8.0053095729 + 0.00325283863);
    constexpr double mBe_sq = m_beryllium * m_beryllium;
    double uBe[3];
    product_momenta(u1x, u1y, u1z, m1, u2x, u2y, u2z, m2, m_alpha, m_beryllium, E_fusion, rng, u[0], uBe);
    const double px_Be = m_beryllium * uBe[0], py_Be = m_beryllium * uBe[1], pz_Be = m_beryllium * uBe[2];
    constexpr double gamma_Bestar = 1.0 + 0.5 * E_decay / (m_alpha * C_SQ);
    constexpr double gamma_Bestar_sq_minus_one = gamma_Bestar * gamma_Bestar - 1.0;
    const double p_Bestar = m_alpha * C_LIGHT * sqrt(gamma_Bestar_sq_minus_one);
    // RandomizeVelocity(px*, py*, pz*, p_Bestar): theta, then z
    const double theta = rng.uniform() * 2.0 * PI;
    const double z = 2.0 * rng.uniform() - 1.0;
    const double xy = sqrt(1.0 - z * z);
    double st, ct;
#ifdef __CUDA_ARCH__
    sincos(theta, &st, &ct);
#else
    st = sin(theta); ct = cos(theta);
#endif
    const double px_s = xy * ct * p_Bestar, py_s = xy * st * p_Bestar, pz_s = z * p_Bestar;
    const double p_Be_sq = px_Be * px_Be + py_Be * py_Be + pz_Be * pz_Be;
    const double g_Be = sqrt(1.0 + p_Be_sq / (mBe_sq * C_SQ));
    const double mg_Be = m_beryllium * g_Be;
    const double vx = px_Be / mg_Be, vy = py_Be / mg_Be, vz = pz_Be / mg_Be;
    const double v_Be_sq = vx * vx + vy * vy + vz * vz;
    double px2 = px_s, py2 = py_s, pz2 = pz_s;
    if (v_Be_sq > DBL_MIN_) {
        const double vcDps = vx * px_s + vy * py_s + vz * pz_s;
        const double factor0 = (g_Be - 1.0) / v_Be_sq;
        const double factor = factor0 * vcDps + m_alpha * gamma_Bestar * g_Be;
        px2 = px_s + vx * factor; py2 = py_s + vy * factor; pz2 = pz_s + vz * factor;
    }
    u[1][0] = px2 / m_alpha; u[1][1] = py2 / m_alpha; u[1][2] = pz2 / m_alpha;
    u[2][0] = (px_Be - px2) / m_alpha; u[2][1] = (py_Be - py2) / m_alpha; u[2][2] = (pz_Be - pz2) / m_alpha;
}

// first record slot of the bin's pairs: [cs1 + cs2, + n1 + n2) of one bin never overlaps another's
__device__ __forceinline__ long pair_base(const Args& a, long bin) {
    return a.b1.cell_start[bin] + (a.same ? 0 : a.b2.cell_start[bin]);
}

// particles of the cell's species 1 (and 2), spent ones included; 0 when fewer than a pair's worth are stored
__device__ __forceinline__ int cell_load(const Args& a, long bin, long* cs1, int* n1, long* cs2, int* n2) {
    *cs1 = a.b1.cell_start[bin];
    *n1 = a.b1.cell_start[bin + 1] - (int)*cs1;
    if (a.same) { *cs2 = *cs1; *n2 = 0; return *n1 >= 2 ? *n1 : 0; }
    *cs2 = a.b2.cell_start[bin];
    *n2 = a.b2.cell_start[bin + 1] - (int)*cs2;
    return (*n1 >= 1 && *n2 >= 1) ? *n1 + *n2 : 0;
}

__device__ __forceinline__ void shuffle(const Args& a, int* sh, int n, uint64_t gcell, int tag) {
    Stream rng(a.seed, a.step, gcell, (a.cidx << 32) | (uint64_t)tag);
    for (int i = n - 1; i >= 1; --i) {
        const int j = rng.random_int(i + 1);
        const int t = sh[i]; sh[i] = sh[j]; sh[j] = t;
    }
}

// The pair chains of one cell (NuclearFusionFunc::Executor), chain c by thread c, c + G, ...: pairs (I1[i1], I2[i2])
// of the index sets into w1 / w2 and u1 / u2, whose spent flags are dead1 / dead2 (entries of the same arrays for an
// intra-species collision); pos1 / pos2 give a particle's storage index.  Pair k of the cell goes to record base + k.
// Returns this thread's number of events.
template <int G>
__device__ int chains(const Args& a, int t, uint64_t gcell, long base, const int* I1, const int* I2, int NI1, int NI2,
                      double* w1, const double* u1x, const double* u1y, const double* u1z, unsigned char* dead1,
                      const int* pos1, double* w2, const double* u2x, const double* u2y, const double* u2z,
                      unsigned char* dead2, const int* pos2) {
    const int maxN = NI1 > NI2 ? NI1 : NI2, minN = NI1 < NI2 ? NI1 : NI2;
    const int multiplier_ratio = a.same ? minN + maxN - 1 : minN;
    const double m2 = a.same ? a.m1 : a.m2;
    int events = 0;
    for (int c = t; c < minN; c += G) {
        Stream rng(a.seed, a.step, gcell, (a.cidx << 32) | (uint64_t)(2 + c));
        int i1 = c, i2 = c;
        for (int k = c; k < maxN; k += minN) {
            const int e1 = I1[i1], e2 = I2[i2];
            bool ev = false;
            double wr = 0.0;
            if (!dead1[e1] && !dead2[e2]) {
                ev = fusion_event(u1x[e1], u1y[e1], u1z[e1], u2x[e2], u2y[e2], u2z[e2], a.m1, m2, w1[e1], w2[e2], a.dt,
                                  a.dV, a.mult, multiplier_ratio, a.thr, a.target, a.type, rng, &wr);
                if (ev) {                      // BinaryCollisionUtils::remove_weight_from_colliding_particle
                    w1[e1] = w1[e1] + -wr;
                    if (w1[e1] <= DBL_MIN_) dead1[e1] = 1;
                    w2[e2] = w2[e2] + -wr;
                    if (w2[e2] <= DBL_MIN_) dead2[e2] = 1;
                    ++events;
                }
            }
            const long r = base + k;
            a.wk.slot1[r] = pos1[e1]; a.wk.slot2[r] = pos2[e2];
            a.wk.wr[r] = wr; a.wk.mask[r] = ev ? 1 : 0;
            if (maxN == NI1) i1 += minN;
            if (maxN == NI2) i2 += minN;
        }
    }
    return events;
}

// Shared memory of one group for `cap` particles: w ux uy uz (canonical order), ids (load order), storage index (load
// order), storage index (canonical order), shuffled positions, spent flags (canonical order), 2 counters.
__host__ __device__ constexpr size_t group_bytes(int cap) { return (size_t)cap * (4 * 8 + 8 + 3 * 4 + 1) + 16; }

struct Group {
    double *w, *ux, *uy, *uz;
    uint64_t* key;
    int *lp, *pp, *sh, *cnt;
    unsigned char* dead;
    __device__ Group(char* base, int cap) {
        double* d = reinterpret_cast<double*>(base);
        w = d; ux = d + cap; uy = d + 2 * cap; uz = d + 3 * cap;
        key = reinterpret_cast<uint64_t*>(d + 4 * cap);
        lp = reinterpret_cast<int*>(key + cap); pp = lp + cap; sh = pp + cap; cnt = sh + cap;
        dead = reinterpret_cast<unsigned char*>(cnt + 4);
    }
};

// One cell with n = n1 + n2 stored particles (n1 for intra-species), 0 < n <= cap, by a group of G threads.
template <int G>
__device__ void fuse_cell(const Args& a, long bin, int t, char* smem, int cap, long cs1, int n1, long cs2, int n2) {
    Group s(smem, cap);
    const int n = n1 + n2;
    if (t == 0) { s.cnt[0] = 0; s.cnt[1] = 0; s.cnt[2] = 0; }
    for (int e = t; e < n; e += G) {
        const int p = coll::storage_index(a, e, n1, cs1, cs2);
        s.key[e] = (e >= n1 ? a.id2 : a.id1)[p];
        s.lp[e] = p;
    }
    coll::group_sync<G>();
    // canonical order of the live particles: rank by id inside each species; spent ids (the largest value) rank last
    for (int e = t; e < n; e += G) {
        const bool two = e >= n1;
        const int lo = two ? n1 : 0, hi = two ? n : n1;
        const uint64_t k = s.key[e];
        if (k == PIC_SPENT_ID) continue;
        atomicAdd(&s.cnt[two ? 1 : 0], 1);                     // shared memory only
        int r = lo;
        for (int f = lo; f < hi; ++f) { const uint64_t kf = s.key[f]; r += (kf < k) || (kf == k && f < e); }
        const int p = s.lp[e];
        const SoaView& P = two ? a.P2 : a.P1;
        s.pp[r] = p;
        s.w[r] = P.w[p]; s.ux[r] = P.ux[p]; s.uy[r] = P.uy[p]; s.uz[r] = P.uz[p];
        s.dead[r] = 0;
        s.sh[r] = r;
    }
    coll::group_sync<G>();
    const int L1 = s.cnt[0], L2 = s.cnt[1];
    coll::group_sync<G>();                                     // read by all before the next cell resets them
    if (a.same ? L1 < 2 : (L1 < 1 || L2 < 1)) return;          // uniform over the group
    const uint64_t gcell = coll::global_cell(a, bin);
    constexpr int second = G == 32 ? 1 : 32;
    if (t == 0) shuffle(a, s.sh, L1, gcell, 0);
    if (t == second && !a.same) shuffle(a, s.sh + n1, L2, gcell, 1);
    coll::group_sync<G>();
    const int half = L1 / 2;
    const int NI1 = a.same ? half : L1, NI2 = a.same ? L1 - half : L2;
    const int ev = chains<G>(a, t, gcell, pair_base(a, bin), s.sh, a.same ? s.sh + half : s.sh + n1, NI1, NI2, s.w, s.ux,
                             s.uy, s.uz, s.dead, s.pp, s.w, s.ux, s.uy, s.uz, s.dead, s.pp);
    if (ev) atomicAdd(&s.cnt[2], ev);
    coll::group_sync<G>();
    if (t == 0) { a.wk.npairs[bin] = NI1 > NI2 ? NI1 : NI2; a.wk.events[bin] = s.cnt[2]; }
    const int nl = a.same ? L1 : n1 + L2;
    for (int e = t; e < nl; e += G) {
        if (e >= L1 && e < n1) continue;
        const bool two = e >= n1;
        const SoaView& P = two ? a.P2 : a.P1;
        const int p = s.pp[e];
        P.w[p] = s.w[e];
        if (s.dead[e]) (two ? a.id2 : a.id1)[p] = PIC_SPENT_ID;
    }
    coll::group_sync<G>();
}

// A cell beyond LARGE_CAP by a block on the particles in place: the canonical order of each species' live particles
// goes to the caller's scratch at the cell's own slots; a reactant is spent when its id says so.
__device__ void fuse_cell_global(const Args& a, long bin, int t, int* cnt, long cs1, int n1, long cs2, int n2) {
    constexpr int G = LARGE_THREADS;
    const int n = n1 + n2;
    int* I1 = a.scr1 + cs1;
    int* I2 = a.same ? nullptr : a.scr2 + cs2;
    if (t == 0) { cnt[0] = 0; cnt[1] = 0; cnt[2] = 0; }
    __syncthreads();
    for (int e = t; e < n; e += G) {
        const bool two = e >= n1;
        const int lo = two ? n1 : 0, hi = two ? n : n1;
        const uint64_t* id = two ? a.id2 : a.id1;
        const int p = coll::storage_index(a, e, n1, cs1, cs2);
        const uint64_t k = id[p];
        if (k == PIC_SPENT_ID) continue;
        atomicAdd(&cnt[two ? 1 : 0], 1);
        int r = 0;
        for (int f = lo; f < hi; ++f) {
            const uint64_t kf = id[coll::storage_index(a, f, n1, cs1, cs2)];
            r += (kf < k) || (kf == k && f < e);
        }
        (two ? I2 : I1)[r] = p;
    }
    __syncthreads();
    const int L1 = cnt[0], L2 = cnt[1];
    __syncthreads();
    if (a.same ? L1 < 2 : (L1 < 1 || L2 < 1)) return;
    const uint64_t gcell = coll::global_cell(a, bin);
    if (t == 0) shuffle(a, I1, L1, gcell, 0);
    if (t == 32 && !a.same) shuffle(a, I2, L2, gcell, 1);
    __syncthreads();
    const int half = L1 / 2;
    const int NI1 = a.same ? half : L1, NI2 = a.same ? L1 - half : L2;
    // storage indices index the particle arrays directly; "spent" is the particle's id.  The ids are written only
    // through the spent flag below, one particle per pair chain, so no chain reads an id another one writes.
    const int ev = [&] {
        const int maxN = NI1 > NI2 ? NI1 : NI2, minN = NI1 < NI2 ? NI1 : NI2;
        const int multiplier_ratio = a.same ? minN + maxN - 1 : minN;
        const double m2 = a.same ? a.m1 : a.m2;
        const SoaView& Q = a.same ? a.P1 : a.P2;
        uint64_t* id2 = a.same ? a.id1 : a.id2;
        const int* J1 = I1;
        const int* J2 = a.same ? I1 + half : I2;
        const long base = pair_base(a, bin);
        int events = 0;
        for (int c = t; c < minN; c += G) {
            Stream rng(a.seed, a.step, gcell, (a.cidx << 32) | (uint64_t)(2 + c));
            int i1 = c, i2 = c;
            for (int k = c; k < maxN; k += minN) {
                const int p1 = J1[i1], p2 = J2[i2];
                bool evk = false;
                double wr = 0.0;
                if (a.id1[p1] != PIC_SPENT_ID && id2[p2] != PIC_SPENT_ID) {
                    evk = fusion_event(a.P1.ux[p1], a.P1.uy[p1], a.P1.uz[p1], Q.ux[p2], Q.uy[p2], Q.uz[p2], a.m1, m2,
                                       a.P1.w[p1], Q.w[p2], a.dt, a.dV, a.mult, multiplier_ratio, a.thr, a.target,
                                       a.type, rng, &wr);
                    if (evk) {
                        a.P1.w[p1] = a.P1.w[p1] + -wr;
                        if (a.P1.w[p1] <= DBL_MIN_) a.id1[p1] = PIC_SPENT_ID;
                        Q.w[p2] = Q.w[p2] + -wr;
                        if (Q.w[p2] <= DBL_MIN_) id2[p2] = PIC_SPENT_ID;
                        ++events;
                    }
                }
                const long r = base + k;
                a.wk.slot1[r] = p1; a.wk.slot2[r] = p2;
                a.wk.wr[r] = wr; a.wk.mask[r] = evk ? 1 : 0;
                if (maxN == NI1) i1 += minN;
                if (maxN == NI2) i2 += minN;
            }
        }
        return events;
    }();
    if (ev) atomicAdd(&cnt[2], ev);
    __syncthreads();
    if (t == 0) { a.wk.npairs[bin] = NI1 > NI2 ? NI1 : NI2; a.wk.events[bin] = cnt[2]; }
    __syncthreads();
}

__global__ void __launch_bounds__(SMALL_WARPS * 32) fuse_small_kernel(Args a, long nbins) {
    PIC_STATIC_SMEM(double, smem, SMALL_WARPS * group_bytes(SMALL_CAP) / 8);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    char* mine = reinterpret_cast<char*>(smem) + warp * group_bytes(SMALL_CAP);
    const long stride = (long)gridDim.x * SMALL_WARPS;
    for (long bin = (long)blockIdx.x * SMALL_WARPS + warp; bin < nbins; bin += stride) {
        long cs1, cs2; int n1, n2;
        const int n = cell_load(a, bin, &cs1, &n1, &cs2, &n2);
        if (n == 0 || n > SMALL_CAP) continue;
        fuse_cell<32>(a, bin, lane, mine, SMALL_CAP, cs1, n1, cs2, n2);
    }
}

__global__ void __launch_bounds__(LARGE_THREADS) fuse_large_kernel(Args a, long nbins) {
    PIC_DYNAMIC_SMEM(double, smem);
    PIC_STATIC_SMEM(int, list, LARGE_SCAN + 1);
    PIC_STATIC_SMEM(int, cnt, 4);
    const int t = threadIdx.x;
    for (long base = (long)blockIdx.x * LARGE_SCAN; base < nbins; base += (long)gridDim.x * LARGE_SCAN) {
        if (t == 0) list[LARGE_SCAN] = 0;
        __syncthreads();
        const long bin = base + t;
        if (t < LARGE_SCAN && bin < nbins) {
            long cs1, cs2; int n1, n2;
            if (cell_load(a, bin, &cs1, &n1, &cs2, &n2) > SMALL_CAP) list[atomicAdd(&list[LARGE_SCAN], 1)] = t;   // shared memory only
        }
        __syncthreads();
        const int nl = list[LARGE_SCAN];
        for (int k = 0; k < nl; ++k) {
            const long b = base + list[k];
            long cs1, cs2; int n1, n2;
            const int n = cell_load(a, b, &cs1, &n1, &cs2, &n2);
            if (n <= LARGE_CAP) fuse_cell<LARGE_THREADS>(a, b, t, reinterpret_cast<char*>(smem), LARGE_CAP, cs1, n1, cs2, n2);
            else if (a.scr1 && (a.same || a.scr2)) fuse_cell_global(a, b, t, cnt, cs1, n1, cs2, n2);
            else if (t == 0) *a.status = 1;
        }
        __syncthreads();
    }
}

struct CreateArgs {
    SoaView P1, P2, PA, PB;
    uint64_t *idA, *idB;
    BinsView b1, b2;
    int gn[2];
    int same, type;
    double m1, m2, mA, mB;
    uint64_t seed, cidx, step;
    uint64_t next_idA, next_idB;
    Work wk;
};

// a warp per bin: the bin's events in pair order, event e of the call at offsets[bin] + (its rank in the bin).  PB: the
// proton-boron reaction, six alphas per event in product A.
template <bool PB>
__global__ void __launch_bounds__(128) create_kernel(CreateArgs a, long nbins) {
    const int lane = threadIdx.x & 31;
    const long stride = (long)gridDim.x * 4;
    const double E_fusion = fusion_energy(a.type);
    for (long bin = (long)blockIdx.x * 4 + (threadIdx.x >> 5); bin < nbins; bin += stride) {
        if (a.wk.events[bin] == 0) continue;
        const long base = a.b1.cell_start[bin] + (a.same ? 0 : a.b2.cell_start[bin]);
        const int np = a.wk.npairs[bin];
        const uint64_t gcell = coll::global_cell(a, bin);
        int seen = 0;
        for (int k0 = 0; k0 < np; k0 += 32) {
            const int k = k0 + lane;
            const bool ev = k < np && a.wk.mask[base + k];
            const unsigned m = __ballot_sync(0xffffffffu, ev);
            if (ev) {
                const int j = seen + __popc(m & ((1u << lane) - 1u));
                const long e = (long)a.wk.offsets[bin] + j;
                const int p1 = a.wk.slot1[base + k], p2 = a.wk.slot2[base + k];
                const SoaView& Q = a.same ? a.P1 : a.P2;
                const double m2 = a.same ? a.m1 : a.m2;
                Stream rng(a.seed, a.step, gcell, PRODUCT_TAG | (a.cidx << 32) | (uint64_t)j);
                const double wh = a.wk.wr[base + k] / 2.0;
                if constexpr (PB) {
                    double u[3][3];
                    alpha_momenta(a.P1.ux[p1], a.P1.uy[p1], a.P1.uz[p1], a.m1, Q.ux[p2], Q.uy[p2], Q.uz[p2], m2, rng, u);
                    for (int al = 0; al < 3; ++al)
                        for (int side = 0; side < 2; ++side) {
                            const long o = 6 * e + 2 * al + side;          // PA's pointers start at its old np
                            const SoaView& S = side ? Q : a.P1;
                            const int p = side ? p2 : p1;
                            a.PA.x[o] = S.x[p]; a.PA.y[o] = S.y[p]; a.PA.z[o] = S.z[p];
                            a.PA.ux[o] = u[al][0]; a.PA.uy[o] = u[al][1]; a.PA.uz[o] = u[al][2];
                            a.PA.w[o] = wh;
                            a.idA[o] = a.next_idA + (uint64_t)o;
                        }
                } else {
                    double uA[3], uB[3];
                    product_momenta(a.P1.ux[p1], a.P1.uy[p1], a.P1.uz[p1], a.m1, Q.ux[p2], Q.uy[p2], Q.uz[p2], m2, a.mA,
                                    a.mB, E_fusion, rng, uA, uB);
                    for (int prod = 0; prod < 2; ++prod) {
                        const SoaView& P = prod ? a.PB : a.PA;
                        uint64_t* id = prod ? a.idB : a.idA;
                        const double* u = prod ? uB : uA;
                        const uint64_t first = prod ? a.next_idB : a.next_idA;
                        for (int side = 0; side < 2; ++side) {
                            const long o = 2 * e + side;                       // P's pointers start at its old np
                            const SoaView& S = side ? Q : a.P1;
                            const int p = side ? p2 : p1;
                            P.x[o] = S.x[p]; P.y[o] = S.y[p]; P.z[o] = S.z[p];
                            P.ux[o] = u[0]; P.uy[o] = u[1]; P.uz[o] = u[2];
                            P.w[o] = wh;
                            id[o] = first + (uint64_t)o;
                        }
                    }
                }
            }
            seen += __popc(m);
        }
    }
}

__global__ void mark_spent_kernel(const uint64_t* __restrict__ id, long np, int* __restrict__ count, int* __restrict__ list,
                                  int cap) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= np || id[i] != PIC_SPENT_ID) return;
    const int k = atomicAdd(count, 1);
    if (k < cap) list[k] = (int)i;
}

}  // namespace fus
}  // namespace pic

using namespace pic;

extern "C" long pic_fusion_workspace_bytes(long pair_capacity, long nbins) {
    size_t total = 0;
    fus::carve(nullptr, pair_capacity, nbins, &total);
    return (long)total;
}

static int check_fusion(const char* what, const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1,
                        const pic_soa* p2, const pic_bins* b2) {
    PIC_REQUIRE(c && p1 && b1, "%s: null argument", what);
    PIC_REQUIRE(b1->cell_start && b1->np_binned == p1->np, "%s: species 1 needs current bins", what);
    PIC_REQUIRE(p1->idcpu && p1->w, "%s: species 1 needs ids and weights", what);
    PIC_REQUIRE(c->type == PIC_FUSION_DT_NHE4 || c->type == PIC_FUSION_DD_PT || c->type == PIC_FUSION_DD_NHE3 ||
                c->type == PIC_FUSION_PB_3HE4, "%s: unknown fusion type %d", what, c->type);
    PIC_REQUIRE(c->m1 > 0.0 && (c->same_species || c->m2 > 0.0) && c->mA > 0.0 &&
                (c->type == PIC_FUSION_PB_3HE4 || c->mB > 0.0), "%s: masses must be positive", what);
    PIC_REQUIRE(c->fusion_multiplier > 0.0, "%s: the fusion multiplier must be positive", what);
    if (!c->same_species) {
        PIC_REQUIRE(p2 && b2 && b2->cell_start && b2->np_binned == p2->np && p2->idcpu && p2->w,
                    "%s: species 2 needs current bins, ids and weights", what);
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(b1->box_lo[d] == b2->box_lo[d] && b1->box_hi[d] == b2->box_hi[d] && b1->tile[d] == b2->tile[d],
                        "%s: the two species' bins must describe the same box and tiles", what);
    }
    return 0;
}

extern "C" int pic_collide_nuclear_fusion(const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1,
                                          const int* src1, const pic_soa* p2, const pic_bins* b2, const int* src2,
                                          const pic_geom* g, double dt, long step, int* scratch1, int* scratch2,
                                          void* work, long pair_capacity, int* status, void* stream) {
    if (int rc = check_fusion("pic_collide_nuclear_fusion", c, p1, b1, p2, b2)) return rc;
    PIC_REQUIRE(g && status && work, "pic_collide_nuclear_fusion: null argument");
    PIC_REQUIRE(step >= 0, "pic_collide_nuclear_fusion: negative step");
    const long need = c->same_species ? p1->np : p1->np + p2->np;
    PIC_REQUIRE(pair_capacity >= need, "pic_collide_nuclear_fusion: the workspace holds %ld pairs, the reactants %ld",
                pair_capacity, need);
    fus::Args a;
    a.P1 = make_soa(*p1, 0); a.id1 = p1->idcpu; a.src1 = src1; a.b1 = make_bins(*b1);
    if (c->same_species) { a.P2 = a.P1; a.id2 = a.id1; a.src2 = a.src1; a.b2 = a.b1; }
    else { a.P2 = make_soa(*p2, 0); a.id2 = p2->idcpu; a.src2 = src2; a.b2 = make_bins(*b2); }
    a.gn[0] = g->n_cell[0]; a.gn[1] = g->n_cell[1];
    double dx[3];
    for (int d = 0; d < 3; ++d) dx[d] = (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
    a.dV = dx[0] * dx[1] * dx[2];
    a.m1 = c->m1; a.m2 = c->m2; a.dt = dt;
    a.mult = c->fusion_multiplier; a.thr = c->fusion_probability_threshold; a.target = c->fusion_probability_target_value;
    a.type = c->type;
    a.seed = c->seed; a.cidx = (uint64_t)(uint32_t)c->collision_index; a.step = (uint64_t)step; a.same = c->same_species;
    a.scr1 = scratch1; a.scr2 = c->same_species ? nullptr : scratch2;
    a.status = status;
    const long nbins = bins_count(a.b1);
    a.wk = fus::carve(work, pair_capacity, nbins);
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(a.wk.npairs, 0, sizeof(int) * (size_t)(nbins + 1), s);
    cudaMemsetAsync(a.wk.events, 0, sizeof(int) * (size_t)(nbins + 1), s);
    if (p1->np == 0 || (!c->same_species && p2->np == 0)) return 0;
    const long small_blocks = (nbins + fus::SMALL_WARPS - 1) / fus::SMALL_WARPS;
    fus::fuse_small_kernel<<<(unsigned)(small_blocks < 2147483647L ? small_blocks : 2147483647L), fus::SMALL_WARPS * 32,
                             0, s>>>(a, nbins);
    count_launch();
    static const size_t large_smem = fus::group_bytes(fus::LARGE_CAP);
    static bool attr = [] {
        return cudaFuncSetAttribute(fus::fuse_large_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)large_smem) == cudaSuccess;
    }();
    PIC_REQUIRE(attr, "pic_collide_nuclear_fusion: cannot reserve %zu bytes of shared memory", large_smem);
    const long large_rounds = (nbins + fus::LARGE_SCAN - 1) / fus::LARGE_SCAN;
    const long large_blocks = large_rounds < 16L * NUM_SMS ? large_rounds : 16L * NUM_SMS;
    fus::fuse_large_kernel<<<(unsigned)large_blocks, fus::LARGE_THREADS, large_smem, s>>>(a, nbins);
    count_launch();
    return check_launch("pic_collide_nuclear_fusion") ? 0 : 1;
}

extern "C" int pic_fusion_create_products(const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1,
                                          const pic_soa* p2, const pic_bins* b2, const pic_geom* g, long step,
                                          void* work, long pair_capacity, const pic_soa* pA, long capA,
                                          uint64_t next_idA, const pic_soa* pB, long capB, uint64_t next_idB,
                                          long* n_events, void* stream) {
    if (int rc = check_fusion("pic_fusion_create_products", c, p1, b1, p2, b2)) return rc;
    const bool pb = c->type == PIC_FUSION_PB_3HE4;
    PIC_REQUIRE(g && work && pA && (pb || pB) && n_events, "pic_fusion_create_products: null argument");
    PIC_REQUIRE(pA->idcpu && pA->w && (pb || (pB->idcpu && pB->w)),
                "pic_fusion_create_products: products need ids and weights");
    *n_events = 0;
    fus::CreateArgs a;
    a.b1 = make_bins(*b1);
    a.b2 = c->same_species ? a.b1 : make_bins(*b2);
    const long nbins = bins_count(a.b1);
    a.wk = fus::carve(work, pair_capacity, nbins);
    cudaStream_t s = (cudaStream_t)stream;
    cub::DeviceScan::ExclusiveSum(a.wk.temp, a.wk.temp_bytes, a.wk.events, a.wk.offsets, (int)(nbins + 1), s);
    count_launch();
    int total = 0;
    cudaMemcpyAsync(&total, a.wk.offsets + nbins, sizeof(int), cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess)
        return fail("pic_fusion_create_products: %s", cudaGetErrorString(cudaGetLastError()));
    const long per_event = pb ? 6L : 2L;
    PIC_REQUIRE(pA->np + per_event * total <= capA,
                "pic_fusion_create_products: product A needs a capacity of %ld (has %ld)", pA->np + per_event * total, capA);
    PIC_REQUIRE(pb || pB->np + 2L * total <= capB,
                "pic_fusion_create_products: product B needs a capacity of %ld (has %ld)", pB->np + 2L * total, capB);
    *n_events = total;
    if (total == 0) return 0;
    a.P1 = make_soa(*p1, 0);
    a.P2 = c->same_species ? a.P1 : make_soa(*p2, 0);
    a.PA = make_soa(*pA, pA->np);
    a.idA = pA->idcpu + pA->np;
    if (!pb) { a.PB = make_soa(*pB, pB->np); a.idB = pB->idcpu + pB->np; }
    a.gn[0] = g->n_cell[0]; a.gn[1] = g->n_cell[1];
    a.same = c->same_species; a.type = c->type;
    a.m1 = c->m1; a.m2 = c->m2; a.mA = c->mA; a.mB = c->mB;
    a.seed = c->seed; a.cidx = (uint64_t)(uint32_t)c->collision_index; a.step = (uint64_t)step;
    a.next_idA = next_idA; a.next_idB = next_idB;
    const long blocks = (nbins + 3) / 4;
    const unsigned grid = (unsigned)(blocks < 2147483647L ? blocks : 2147483647L);
    if (pb) fus::create_kernel<true><<<grid, 128, 0, s>>>(a, nbins);
    else fus::create_kernel<false><<<grid, 128, 0, s>>>(a, nbins);
    count_launch();
    return check_launch("pic_fusion_create_products") ? 0 : 1;
}

extern "C" int pic_particles_mark_spent(const pic_soa* p, int* work, int cap, void* stream) {
    PIC_REQUIRE(p && work, "pic_particles_mark_spent: null argument");
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(work, 0, 4 * sizeof(int), s);
    if (p->np == 0) return 0;
    PIC_REQUIRE(p->idcpu, "pic_particles_mark_spent: no ids");
    fus::mark_spent_kernel<<<(unsigned)((p->np + 255) / 256), 256, 0, s>>>(p->idcpu, p->np, work, work + 4, cap);
    count_launch();
    return check_launch("pic_particles_mark_spent") ? 0 : 1;
}
