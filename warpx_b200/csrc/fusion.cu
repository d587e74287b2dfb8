// Nuclear fusion (collisions.collision_names, <name>.type = nuclearfusion) over the rank's box: two-product reactions and
// proton-boron.
//
// Restates, for one tile = the rank's box (paths relative to Source/Particles/Collision/BinaryCollision/):
//   the cell walk        <- BinaryCollision::doCollisionsWithinTile  BinaryCollision.H:383-472 (intra-species, halves),
//   (binary_collision.cuh)  :613-730 (inter-species)
//   NuclearFusion        <- NuclearFusionFunc::Executor                                NuclearFusion/NuclearFusionFunc.H:127-234
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
// Event pass: one pass of the cell walk of binary_collision.cuh over the bins, the Coulomb pass's walk, leaving spent
// particles out.  A cell's pairs go to records at its own slots (cell_start of species 1 plus that of species 2), its
// pair and event counts to per-bin arrays: no global atomics.  Product pass:
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
using coll::HBAR;
using coll::PI;

constexpr double Q_E = 1.602176634e-19;         // PhysConst::q_e
constexpr double ALPHA = 0.007297352573748943;  // PhysConst::alpha
constexpr double M_U = 1.66053906660e-27;      // PhysConst::m_u
constexpr double C_SQ = C_LIGHT * C_LIGHT;
constexpr double INV_CSQ = 1.0 / C_SQ;
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

// The cell walk's functor (binary_collision.cuh) for NuclearFusionFunc::Executor: pair k of a cell goes to the record
// base + k of the workspace, a reactant that an event leaves with w <= DBL_MIN is spent.
struct NuclearFusion {
    struct Args : coll::PairArgs {
        double mult, thr, target;
        int type;
        Work wk;
    };
    static constexpr bool skip_spent = true;
    struct Scalars { int live[2], events; };   // live particles of each species, events of the cell

    template <class V> __device__ static void species(const Args&, const V&, int, const int*, int, Scalars&) {}

    long base;                 // first record of the cell: [cs1 + cs2, + n1 + n2) of one bin never overlaps another's
    int multiplier_ratio, npairs, events;

    __device__ NuclearFusion(const Args& a, long bin, const Scalars&, int minN, int maxN)
        : base(a.b1.cell_start[bin] + (a.same ? 0 : a.b2.cell_start[bin])),
          multiplier_ratio(a.same ? minN + maxN - 1 : minN), npairs(maxN), events(0) {}

    // pairs with a spent reactant draw nothing (NuclearFusionFunc.H:181-184)
    template <class V>
    __device__ void pair(const Args& a, const V& v, int e1, int e2, int k, Stream& rng) {
        bool ev = false;
        double wr = 0.0;
        if (!v.spent(1, e1) && !v.spent(2, e2)) {
            ev = fusion_event(v.ux(1, e1), v.uy(1, e1), v.uz(1, e1), v.ux(2, e2), v.uy(2, e2), v.uz(2, e2), a.m1,
                              a.same ? a.m1 : a.m2, v.w(1, e1), v.w(2, e2), a.dt, a.dV, a.mult, multiplier_ratio, a.thr,
                              a.target, a.type, rng, &wr);
            if (ev) {                          // BinaryCollisionUtils::remove_weight_from_colliding_particle
                v.w(1, e1) = v.w(1, e1) + -wr;
                if (v.w(1, e1) <= DBL_MIN_) v.spend(1, e1);
                v.w(2, e2) = v.w(2, e2) + -wr;
                if (v.w(2, e2) <= DBL_MIN_) v.spend(2, e2);
                ++events;
            }
        }
        const long r = base + k;
        a.wk.slot1[r] = v.storage(1, e1); a.wk.slot2[r] = v.storage(2, e2);
        a.wk.wr[r] = wr; a.wk.mask[r] = ev ? 1 : 0;
    }

    template <int G> __device__ void end_cell(const Args& a, long bin, int t, Scalars& x) const {
        if (events) atomicAdd(&x.events, events);   // shared memory only
        coll::group_sync<G>();
        if (t == 0) { a.wk.npairs[bin] = npairs; a.wk.events[bin] = x.events; }
    }

    template <class V>
    __device__ static void store(const Args& a, const V& v, int sp, int e) {
        const SoaView& P = sp == 1 ? a.P1 : a.P2;
        const int p = v.storage(sp, e);
        P.w[p] = v.w(sp, e);
        if (v.spent(sp, e)) (sp == 1 ? a.id1 : a.id2)[p] = PIC_SPENT_ID;
    }
};

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

// the refusals about the reaction that both passes make
static int check_fusion(const char* what, const pic_fusion_collision* c) {
    PIC_REQUIRE(c->type == PIC_FUSION_DT_NHE4 || c->type == PIC_FUSION_DD_PT || c->type == PIC_FUSION_DD_NHE3 ||
                c->type == PIC_FUSION_PB_3HE4, "%s: unknown fusion type %d", what, c->type);
    PIC_REQUIRE(c->m1 > 0.0 && (c->same_species || c->m2 > 0.0) && c->mA > 0.0 &&
                (c->type == PIC_FUSION_PB_3HE4 || c->mB > 0.0), "%s: masses must be positive", what);
    PIC_REQUIRE(c->fusion_multiplier > 0.0, "%s: the fusion multiplier must be positive", what);
    return 0;
}

extern "C" int pic_collide_nuclear_fusion(const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1,
                                          const int* src1, const pic_soa* p2, const pic_bins* b2, const int* src2,
                                          const pic_geom* g, double dt, long step, int* scratch1, int* scratch2,
                                          void* work, long pair_capacity, int* status, void* stream) {
    const char* what = "pic_collide_nuclear_fusion";
    fus::NuclearFusion::Args a;
    if (int rc = coll::pair_args(what, c, p1, b1, src1, p2, b2, src2, g, dt, step, scratch1, scratch2, status, a))
        return rc;
    if (int rc = check_fusion(what, c)) return rc;
    PIC_REQUIRE(work, "%s: null argument", what);
    const long need = c->same_species ? p1->np : p1->np + p2->np;
    PIC_REQUIRE(pair_capacity >= need, "%s: the workspace holds %ld pairs, the reactants %ld", what, pair_capacity, need);
    a.mult = c->fusion_multiplier; a.thr = c->fusion_probability_threshold; a.target = c->fusion_probability_target_value;
    a.type = c->type;
    const long nbins = bins_count(a.b1);
    a.wk = fus::carve(work, pair_capacity, nbins);
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(a.wk.npairs, 0, sizeof(int) * (size_t)(nbins + 1), s);
    cudaMemsetAsync(a.wk.events, 0, sizeof(int) * (size_t)(nbins + 1), s);
    if (p1->np == 0 || (!c->same_species && p2->np == 0)) return 0;
    return coll::launch<fus::NuclearFusion>(what, a, s);
}

extern "C" int pic_fusion_create_products(const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1,
                                          const pic_soa* p2, const pic_bins* b2, const pic_geom* g, long step,
                                          void* work, long pair_capacity, const pic_soa* pA, long capA,
                                          uint64_t next_idA, const pic_soa* pB, long capB, uint64_t next_idB,
                                          long* n_events, void* stream) {
    PIC_REQUIRE(c && p1 && b1, "pic_fusion_create_products: null argument");
    if (int rc = coll::check_species("pic_fusion_create_products", c->same_species, p1, b1, p2, b2)) return rc;
    if (int rc = check_fusion("pic_fusion_create_products", c)) return rc;
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
