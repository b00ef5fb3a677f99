// pwpp_math.cuh — scalar math of the ground-segmentation path, shared by every kernel.
//
// Everything here is __host__ __device__ so that tests/host_twin.cu (tests/test_host_twin.py) can run the exact same
// code on the CPU (nvcc host pass) against the oracle before it ever runs on a GPU.
//
// Arithmetic contract ("CANON64", DESIGN.md §3): the reference's formulas
// (cpp/patchworkpp/src/patchworkpp.cpp, "S:") evaluated in IEEE double with every operation
// rounded separately (no FMA contraction: __dmul_rn/__dadd_rn/... on the device, -ffp-contract=off
// on the host), so that given identical inputs the device and the CPU oracle produce identical bits.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define PW_HD __host__ __device__ __forceinline__
#else
#define PW_HD inline
#endif

namespace pwpp {

// ---- separately rounded double ops ---------------------------------------------------------------
PW_HD double dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
PW_HD double dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
PW_HD double dsub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
PW_HD double ddiv(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
PW_HD double dsqrt(double a) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(a);
#else
  return sqrt(a);
#endif
}
PW_HD float fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
PW_HD float fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
PW_HD float fsqrt(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}

// Smallest float >= t (NaN stays NaN). For every float z, ±inf and NaN included:  (double) z < t  <=>  z < float_ru(t).
// If float_ru(t) == t both sides compare the same value. Otherwise no float lies in [t, float_ru(t)), so a float is
// below t exactly when it is below float_ru(t). NaN on either side makes both compares false. The fit kernels compute
// it once per round, so that the per-point tests against a double threshold are one fp32 compare instead of a
// float->double conversion (a quarter of the FP64 rate on sm_90) plus a double compare.
PW_HD float float_ru(double t) {
  float f = (float) t;   // round to nearest, then step up to the next float if that went below t
  if ((double) f < t) {  // f is finite or -inf here
    uint32_t b;
    memcpy(&b, &f, sizeof b);
    b = (f == 0.0f) ? 1u : (f > 0.0f ? b + 1u : b - 1u);
    memcpy(&f, &b, sizeof f);
  }
  return f;
}

#define PW_PI 3.14159265358979323846 /* M_PI, reference patchworkpp.h:4-6 */

// double atan2 of the exact (rare) paths: kept out of line on the device so that the unrolled hot loops of the
// binning kernel do not carry eight inlined copies of it (instruction-cache footprint)
#if defined(__CUDACC__)
__host__ __device__ __noinline__ inline double atan2_exact(double y, double x) { return atan2(y, x); }
#else
inline double atan2_exact(double y, double x) { return atan2(y, x); }
#endif

// ---- concentric-zone geometry + thresholds (reference Params, H:42-112, and ctor H:120-134) -------
struct Geometry {
  double min_ranges[4];    // H:122-125
  double ring_sizes[4];    // H:127-130
  double sector_sizes[4];  // H:131-134
  double max_range, min_range;
  int num_rings[4], num_sectors[4];
  int bin_base[5];         // first bin id of each zone in (zone, ring, sector) order
  int concentric_base[5];  // first concentric ring index of each zone
  int nbins;               // 504 with the defaults
  // float copies for the filtered fast path of bin_of_point()
  float f_min_ranges[4], f_ring_sizes[4], f_sector_sizes[4], f_max_range;
  float f_inv_ring[4], f_inv_sector[4];  // reciprocals (the fp32 filter multiplies instead of dividing)
};

struct AlgoParams {
  double RNR_ver_angle_thr, RNR_intensity_thr;
  double th_seeds, th_seeds_v, th_dist, th_dist_v;
  double uprightness_thr, adaptive_seed_selection_margin;
  int num_iter, num_lpr, num_min_pts, num_rings_of_interest;
  int enable_RNR, enable_RVPF, enable_TGR;
  int max_flatness_storage, max_elevation_storage;
  float f_RNR_intensity_thr;   // float_ru(RNR_intensity_thr): rnr_hit's intensity test in fp32, exact
};
static_assert(sizeof(AlgoParams) == 104, "f_RNR_intensity_thr sits in what was tail padding: AlgoParamSets keeps its size");

// Pseudo-bins after the nbins real ones (see include/pwpp.h pwpp_copy_bin_ids)
#define PW_BIN_RNR(nb) ((nb))        /* reflected noise, S:391-396 -> nonground            */
#define PW_BIN_OOR(nb) ((nb) + 1)    /* outside (min_range, max_range], S:617-619 -> nonground */
#define PW_BIN_DROP(nb) ((nb) + 2)   /* input z == FLT_MIN: vanishes from both outputs, S:591  */
#define PW_NUM_PSEUDO 3

// reflected_noise_removal predicate, S:385-391. r is computed in float like the reference does.
PW_HD bool rnr_hit(float x, float y, float z, float intensity, double sensor_height, const AlgoParams& ap) {
  // cheap conjuncts first (pure predicates, order does not matter): S:391
  if (!(intensity < ap.f_RNR_intensity_thr)) return false;   // (double) intensity < RNR_intensity_thr (float_ru)
  const double zd = (double) z;
  if (!(zd < dsub(-sensor_height, 0.8))) return false;
  const float rf = fsqrt(fadd(fmul(x, x), fmul(y, y)));          // S:387 (float ops, std::sqrt(float))
  const double ang = ddiv(dmul(atan2_exact(zd, (double) rf), 180.0), PW_PI);  // S:389
  return ang < ap.RNR_ver_angle_thr;
}

// pc2czm for one point, S:587-619 in double exactly as written. Returns the bin id, or
// PW_BIN_OOR(nbins) when the point is outside (min_range, max_range] or has a non-finite z
// (defined behaviour where the reference would sort NaNs, see oracle/pwpp_oracle.c header).
PW_HD int bin_of_point_exact(float x, float y, float z, const Geometry& g) {
  const double xd = (double) x, yd = (double) y;
  const double r = dsqrt(dadd(dmul(xd, xd), dmul(yd, yd)));  // xy2radius S:573-576
  if (!((r <= g.max_range) && (r > g.min_range)) || !(fabsf(z) <= FLT_MAX)) return PW_BIN_OOR(g.nbins);
  double theta = atan2_exact(yd, xd);                        // xy2theta S:568-571
  theta = theta > 0 ? theta : dadd(2 * PW_PI, theta);
  const int k = (r < g.min_ranges[1]) ? 0 : (r < g.min_ranges[2]) ? 1 : (r < g.min_ranges[3]) ? 2 : 3;
  int ring = (int) ddiv(dsub(r, g.min_ranges[k]), g.ring_sizes[k]);
  ring = ring < g.num_rings[k] - 1 ? ring : g.num_rings[k] - 1;
  int sector = (int) ddiv(theta, g.sector_sizes[k]);
  sector = sector < g.num_sectors[k] - 1 ? sector : g.num_sectors[k] - 1;
  return g.bin_base[k] + ring * g.num_sectors[k] + sector;
}

// atan2 in [-pi, pi] with |error| < 2.5e-6 rad: odd polynomial of atan on [0,1] (degree 11, max error 1.7e-6,
// checked numerically) evaluated in float with an approximate division, + octant reduction. Only used by the filter below, which treats
// anything within 2e-4 sector widths (>= 2.3e-5 rad) of a boundary as ambiguous.
PW_HD float atan2_filter(float y, float x) {
  const float ax = fabsf(x), ay = fabsf(y);
  const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
#if defined(__CUDA_ARCH__)
  const float q = __fdividef(mn, mx);
#else
  const float q = mn / mx;
#endif
  const float t = q * q;
  float r = -0.0117212f;
  r = r * t + 0.05265332f;
  r = r * t - 0.11643287f;
  r = r * t + 0.19354346f;
  r = r * t - 0.33262347f;
  r = r * t + 0.99997726f;
  r = r * q;
  if (ay > ax) r = 1.57079632679f - r;
  if (x < 0.f) r = 3.14159265359f - r;
  return y < 0.f ? -r : r;
}

// Same decision through an fp32 filter: float radius / polynomial atan2 decide the bin whenever the float values
// are farther from every decision boundary than a guard band that is >= 6x the worst-case float error (radius:
// < 3e-5 m at 80 m vs 2e-4 m; ring coordinate: < 2e-5 vs 2e-4; angle: < 2.5e-6 rad, i.e. < 2.2e-5 sector widths
// for up to 128 sectors, vs 2e-4); only points inside a guard band (~1e-3 of a KITTI scan) pay for the double
// sqrt/atan2/div of the exact path. The result is identical to bin_of_point_exact by construction (and checked
// point by point in tests/test_host_twin.py). Zone boundaries need no separate test: they are ring boundaries
// (u = 0 or u = num_rings) of the neighbouring zones, so the ring-coordinate guard covers them.
PW_HD int bin_of_point(float x, float y, float z, const Geometry& g) {
  const float GUARD_R = 2e-4f;   // metres
  const float GUARD_U = 2e-4f;   // ring / sector units
  const float r2 = x * x + y * y;
  const float rf = sqrtf(r2);
  if (!(rf < 1e6f) || !(fabsf(z) <= FLT_MAX)) return bin_of_point_exact(x, y, z, g);  // NaN/Inf/huge
  if (rf > g.f_max_range + GUARD_R || rf < g.f_min_ranges[0] - GUARD_R) return PW_BIN_OOR(g.nbins);
  const int k = (rf < g.f_min_ranges[1]) ? 0 : (rf < g.f_min_ranges[2]) ? 1 : (rf < g.f_min_ranges[3]) ? 2 : 3;
  const float uf = (rf - g.f_min_ranges[k]) * g.f_inv_ring[k];
  bool amb = fabsf(uf - rintf(uf)) <= GUARD_U;
  float tf = atan2_filter(y, x);
  amb = amb || fabsf(tf) <= 1e-4f;
  tf = tf > 0.f ? tf : tf + 6.28318530717958647692f;
  const float sf = tf * g.f_inv_sector[k];
  amb = amb || fabsf(sf - rintf(sf)) <= GUARD_U;
  if (amb) return bin_of_point_exact(x, y, z, g);
  int ring = (int) uf;
  ring = ring < g.num_rings[k] - 1 ? ring : g.num_rings[k] - 1;
  int sector = (int) sf;
  sector = sector < g.num_sectors[k] - 1 ? sector : g.num_sectors[k] - 1;
  return g.bin_base[k] + ring * g.num_sectors[k] + sector;
}

// ---- plane of a point set -------------------------------------------------------------------------
struct Plane {
  double mean[3];    // pc_mean_           S:59-60
  double normal[3];  // normal_, z >= 0    S:66-68
  double sv[3];      // singular_values_, descending  S:63
  double d;          // d_                 S:74
};

// rotation in the plane (Eigen/src/Jacobi/Jacobi.h apply_rotation_in_the_plane), restated as in
// oracle/pwpp_oracle.c DEFINE_JSVD: x_i <- c x_i + s y_i ; y_i <- -s x_i + c y_i
#define PW_ROT(X, Y, C, S)                                         \
  {                                                                \
    const double _xi = (X), _yi = (Y);                             \
    (X) = dadd(dmul((C), _xi), dmul((S), _yi));                    \
    (Y) = dadd(-dmul((S), _xi), dmul((C), _yi));                   \
  }

// 3x3 two-sided Jacobi SVD in double, the algorithm published for Eigen 3.4.0's JacobiSVD that the
// reference calls at S:62 (there in float), operation for operation the same as jsvd3d() in
// oracle/pwpp_oracle.c. cov is symmetric and given by its 6 unique entries.
// Outputs singular values (descending) and U's third column (the least singular vector).
PW_HD void jacobi_svd3(double cxx, double cxy, double cxz, double cyy, double cyz, double czz, double sv[3], double ucol2[3]) {
  // W(i,j) and U(i,j) kept in scalars so the whole thing lives in registers on the device
  double W00 = cxx, W01 = cxy, W02 = cxz, W10 = cxy, W11 = cyy, W12 = cyz, W20 = cxz, W21 = cyz, W22 = czz;
  double U00 = 1, U01 = 0, U02 = 0, U10 = 0, U11 = 1, U12 = 0, U20 = 0, U21 = 0, U22 = 1;
  double scale = 0.0;
  bool finite = true;
  {
    const double a[6] = {fabs(cxx), fabs(cxy), fabs(cxz), fabs(cyy), fabs(cyz), fabs(czz)};
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      if (!(a[i] <= DBL_MAX)) finite = false;
      if (a[i] > scale) scale = a[i];
    }
  }
  if (!finite) {  // S:57 with one point: 0/0. Defined as U = I, singular values NaN (oracle header).
    sv[0] = sv[1] = sv[2] = NAN;
    ucol2[0] = 0; ucol2[1] = 0; ucol2[2] = 1;
    return;
  }
  if (scale == 0.0) scale = 1.0;
  W00 = ddiv(W00, scale); W01 = ddiv(W01, scale); W02 = ddiv(W02, scale);
  W10 = ddiv(W10, scale); W11 = ddiv(W11, scale); W12 = ddiv(W12, scale);
  W20 = ddiv(W20, scale); W21 = ddiv(W21, scale); W22 = ddiv(W22, scale);
  const double precision = 2 * DBL_EPSILON, considerAsZero = DBL_MIN;
  double maxDiag = fmax(fabs(W00), fmax(fabs(W11), fabs(W22)));

// one (p,q) step; Wpp.. are lvalues naming the entries; R* are the third index r (the row/col not in {p,q})
#define PW_JSTEP(Wpp, Wpq, Wqp, Wqq, Wpr, Wqr, Wrp, Wrq, Upp_, Upq_, Uqp_, Uqq_, Urp_, Urq_)                     \
  {                                                                                                               \
    double thr = dmul(precision, maxDiag);                                                                        \
    if (considerAsZero > thr) thr = considerAsZero;                                                               \
    if (fabs(Wpq) > thr || fabs(Wqp) > thr) {                                                                     \
      finished = false;                                                                                           \
      double m00 = Wpp, m01 = Wpq, m10 = Wqp, m11 = Wqq;                                                          \
      double r1c, r1s;                                                                                            \
      const double t = dadd(m00, m11), dd = dsub(m10, m01);                                                       \
      if (fabs(dd) < DBL_MIN) { r1s = 0.0; r1c = 1.0; }                                                           \
      else { const double u = ddiv(t, dd); const double tmp = dsqrt(dadd(1.0, dmul(u, u))); r1s = ddiv(1.0, tmp); r1c = ddiv(u, tmp); } \
      if (!(r1c == 1.0 && r1s == 0.0)) { PW_ROT(m00, m10, r1c, r1s); PW_ROT(m01, m11, r1c, r1s); }                \
      double jrc, jrs;                                                                                            \
      const double deno = dmul(2.0, fabs(m01));                                                                   \
      if (deno < DBL_MIN) { jrc = 1.0; jrs = 0.0; }                                                               \
      else {                                                                                                      \
        const double tau = ddiv(dsub(m00, m11), deno);                                                            \
        const double w = dsqrt(dadd(dmul(tau, tau), 1.0));                                                        \
        const double tn = (tau > 0.0) ? ddiv(1.0, dadd(tau, w)) : ddiv(1.0, dsub(tau, w));                        \
        const double sign_t = tn > 0.0 ? 1.0 : -1.0;                                                              \
        const double nn = ddiv(1.0, dsqrt(dadd(dmul(tn, tn), 1.0)));                                              \
        jrs = dmul(dmul(dmul(-sign_t, ddiv(m01, fabs(m01))), fabs(tn)), nn);                                      \
        jrc = nn;                                                                                                 \
      }                                                                                                           \
      const double oc = jrc, os = -jrs;                                                                           \
      const double jlc = dsub(dmul(r1c, oc), dmul(r1s, os)), jls = dadd(dmul(r1c, os), dmul(r1s, oc));            \
      if (!(jlc == 1.0 && jls == 0.0)) {                                                                          \
        /* W.applyOnTheLeft(p,q,j_left): rows p,q, columns in index order */                                      \
        PW_ROWS_PQ(jlc, jls)                                                                                      \
        /* U.applyOnTheRight(p,q,j_left^T): columns p,q of U, rows in index order */                              \
        PW_UCOLS_PQ(jlc, jls)                                                                                     \
      }                                                                                                           \
      if (!(jrc == 1.0 && (-jrs) == 0.0)) {                                                                       \
        /* W.applyOnTheRight(p,q,j_right): columns p,q of W with (c,-s) */                                        \
        PW_WCOLS_PQ(jrc, -jrs)                                                                                    \
      }                                                                                                           \
      const double a1 = fabs(Wpp), a2 = fabs(Wqq);                                                                \
      const double mx = a1 > a2 ? a1 : a2;                                                                        \
      if (mx > maxDiag) maxDiag = mx;                                                                             \
    }                                                                                                             \
  }

  bool finished = false;
  while (!finished) {
    finished = true;
    // (p,q) = (1,0)
#define PW_ROWS_PQ(C, S) PW_ROT(W10, W00, C, S) PW_ROT(W11, W01, C, S) PW_ROT(W12, W02, C, S)
#define PW_UCOLS_PQ(C, S) PW_ROT(U01, U00, C, S) PW_ROT(U11, U10, C, S) PW_ROT(U21, U20, C, S)
#define PW_WCOLS_PQ(C, S) PW_ROT(W01, W00, C, S) PW_ROT(W11, W10, C, S) PW_ROT(W21, W20, C, S)
    PW_JSTEP(W11, W10, W01, W00, W12, W02, W21, W20, U11, U10, U01, U00, U21, U20)
#undef PW_ROWS_PQ
#undef PW_UCOLS_PQ
#undef PW_WCOLS_PQ
    // (p,q) = (2,0)
#define PW_ROWS_PQ(C, S) PW_ROT(W20, W00, C, S) PW_ROT(W21, W01, C, S) PW_ROT(W22, W02, C, S)
#define PW_UCOLS_PQ(C, S) PW_ROT(U02, U00, C, S) PW_ROT(U12, U10, C, S) PW_ROT(U22, U20, C, S)
#define PW_WCOLS_PQ(C, S) PW_ROT(W02, W00, C, S) PW_ROT(W12, W10, C, S) PW_ROT(W22, W20, C, S)
    PW_JSTEP(W22, W20, W02, W00, W21, W01, W12, W10, U22, U20, U02, U00, U12, U10)
#undef PW_ROWS_PQ
#undef PW_UCOLS_PQ
#undef PW_WCOLS_PQ
    // (p,q) = (2,1)
#define PW_ROWS_PQ(C, S) PW_ROT(W20, W10, C, S) PW_ROT(W21, W11, C, S) PW_ROT(W22, W12, C, S)
#define PW_UCOLS_PQ(C, S) PW_ROT(U02, U01, C, S) PW_ROT(U12, U11, C, S) PW_ROT(U22, U21, C, S)
#define PW_WCOLS_PQ(C, S) PW_ROT(W02, W01, C, S) PW_ROT(W12, W11, C, S) PW_ROT(W22, W21, C, S)
    PW_JSTEP(W22, W21, W12, W11, W20, W10, W02, W01, U22, U21, U12, U11, U02, U01)
#undef PW_ROWS_PQ
#undef PW_UCOLS_PQ
#undef PW_WCOLS_PQ
  }
#undef PW_JSTEP

  // |diag| * scale, flip U columns of negative diagonal entries
  double s0 = fabs(W00), s1 = fabs(W11), s2 = fabs(W22);
  if (W00 < 0.0) { U00 = dmul(U00, -1.0); U10 = dmul(U10, -1.0); U20 = dmul(U20, -1.0); }
  if (W11 < 0.0) { U01 = dmul(U01, -1.0); U11 = dmul(U11, -1.0); U21 = dmul(U21, -1.0); }
  if (W22 < 0.0) { U02 = dmul(U02, -1.0); U12 = dmul(U12, -1.0); U22 = dmul(U22, -1.0); }
  s0 = dmul(s0, scale); s1 = dmul(s1, scale); s2 = dmul(s2, scale);
  // selection sort descending with U columns swapped (only column 2 is needed at the end, but the
  // swaps move columns around, so track all three)
  double c0[3] = {U00, U10, U20}, c1[3] = {U01, U11, U21}, c2[3] = {U02, U12, U22};
  // i = 0: max over (s0,s1,s2); first maximal position wins (strict >)
  {
    int pos = 0; double mx = s0;
    if (s1 > mx) { mx = s1; pos = 1; }
    if (s2 > mx) { mx = s2; pos = 2; }
    if (mx == 0.0) { sv[0] = s0; sv[1] = s1; sv[2] = s2; ucol2[0] = c2[0]; ucol2[1] = c2[1]; ucol2[2] = c2[2]; return; }
    if (pos == 1) { double t = s0; s0 = s1; s1 = t; for (int k = 0; k < 3; ++k) { double u = c0[k]; c0[k] = c1[k]; c1[k] = u; } }
    else if (pos == 2) { double t = s0; s0 = s2; s2 = t; for (int k = 0; k < 3; ++k) { double u = c0[k]; c0[k] = c2[k]; c2[k] = u; } }
  }
  // i = 1: max over (s1,s2)
  {
    int pos = 0; double mx = s1;
    if (s2 > mx) { mx = s2; pos = 1; }
    if (mx != 0.0 && pos == 1) { double t = s1; s1 = s2; s2 = t; for (int k = 0; k < 3; ++k) { double u = c1[k]; c1[k] = c2[k]; c2[k] = u; } }
    // i = 2: single element, nothing to swap (and mx == 0 would only break out)
  }
  sv[0] = s0; sv[1] = s1; sv[2] = s2;
  ucol2[0] = c2[0]; ucol2[1] = c2[1]; ucol2[2] = c2[2];
}

// ---- closed-form symmetric 3x3 eigen-solver ----------------------------------------------------------------
// The Jacobi iteration above is a chain of ~1200 dependent double operations on one lane, which is
// what bounded the fit kernels. For the covariance of S:57 (symmetric positive semi-definite) the same quantities —
// singular values = |eigenvalues| in descending order and the eigenvector of the smallest one — follow from the
// trigonometric solution of the characteristic cubic plus cross products of rows of (A - lambda I), evaluated the
// numerically careful way published by D. Eberly ("A Robust Eigensolver for 3x3 Symmetric Matrices"): scale by the
// largest |entry|, shift by trace/3, pick the better-isolated extreme eigenvalue first and build the remaining
// vectors in its orthogonal complement. ~200 double operations with short dependency chains. The oracle keeps the
// Jacobi SVD; tests/test_host_twin.py checks this solver against it on every patch of the fixtures
// (|delta normal| <= 1e-9), so the two implementations cross-validate each other.
PW_HD void cross3(const double a[3], const double b[3], double r[3]) {
  r[0] = a[1] * b[2] - a[2] * b[1]; r[1] = a[2] * b[0] - a[0] * b[2]; r[2] = a[0] * b[1] - a[1] * b[0];
}
// Reciprocal and reciprocal square root for the plane solve: the hardware seed (MUFU.RCP64H / RSQ64H, ~2^-19) plus two
// Newton steps, ~1 ulp, no slow-path subroutine. Operands here are sums of squares / counts in the normal range;
// 0 -> inf seed -> NaN after the Newton step, which every caller treats like the reference's 0/0 (degenerate patch).
PW_HD double rcp_d(double x) {
#if defined(__CUDA_ARCH__)
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  r = fma(fma(-x, r, 1.0), r, r);
  r = fma(fma(-x, r, 1.0), r, r);
  return r;
#else
  return 1.0 / x;
#endif
}
PW_HD double rsqrt_d(double x) {
#if defined(__CUDA_ARCH__)
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double hx = 0.5 * x;
  y = fma(fma(-hx * y, y, 0.5), y, y);
  y = fma(fma(-hx * y, y, 0.5), y, y);
  return y;
#else
  return 1.0 / sqrt(x);
#endif
}
PW_HD float rcp_f(float x) {   // ~1e-7 relative; only steers a Newton iteration
#if defined(__CUDA_ARCH__)
  return __fdividef(1.0f, x);
#else
  return 1.0f / x;
#endif
}
// unit vector in the null space of (A - lambda I): the largest cross product of two rows (scalar selects only, so
// everything stays in registers)
PW_HD void eigvec_by_rows(double a00, double a01, double a02, double a11, double a12, double a22, double lambda, double v[3]) {
  const double r00 = a00 - lambda, r11 = a11 - lambda, r22 = a22 - lambda;
  // rows r0 = (r00, a01, a02), r1 = (a01, r11, a12), r2 = (a02, a12, r22)
  const double x01 = a01 * a12 - a02 * r11, y01 = a02 * a01 - r00 * a12, z01 = r00 * r11 - a01 * a01;   // r0 x r1
  const double x02 = a01 * r22 - a02 * a12, y02 = a02 * a02 - r00 * r22, z02 = r00 * a12 - a01 * a02;   // r0 x r2
  const double x12 = r11 * r22 - a12 * a12, y12 = a12 * a02 - a01 * r22, z12 = a01 * a12 - r11 * a02;   // r1 x r2
  const double d01 = x01 * x01 + y01 * y01 + z01 * z01;
  const double d02 = x02 * x02 + y02 * y02 + z02 * z02;
  const double d12 = x12 * x12 + y12 * y12 + z12 * z12;
  double bx = x01, by = y01, bz = z01, dmax = d01;
  if (d02 > dmax) { dmax = d02; bx = x02; by = y02; bz = z02; }
  if (d12 > dmax) { dmax = d12; bx = x12; by = y12; bz = z12; }
  if (dmax > 0.0) { const double inv = rsqrt_d(dmax); v[0] = bx * inv; v[1] = by * inv; v[2] = bz * inv; }
  else { v[0] = 0.0; v[1] = 0.0; v[2] = 1.0; }
}
// unit vectors u, w with {u, w, v} orthonormal (branch-free: one reciprocal square root)
PW_HD void orthogonal_complement(const double v[3], double u[3], double w[3]) {
  const bool x_big = fabs(v[0]) > fabs(v[1]);
  const double a = x_big ? v[0] : v[1];
  const double inv = rsqrt_d(a * a + v[2] * v[2]);
  const double s = v[2] * inv, t = a * inv;
  u[0] = x_big ? -s : 0.0; u[1] = x_big ? 0.0 : s; u[2] = x_big ? t : -t;
  cross3(v, u, w);
}
PW_HD double pow2_biased(int biased_exponent) {   // 2^(biased_exponent - 1023), 1 <= biased_exponent <= 2046
  const long long bits = (long long) biased_exponent << 52;
#if defined(__CUDA_ARCH__)
  return __longlong_as_double(bits);
#else
  double d; memcpy(&d, &bits, sizeof d); return d;
#endif
}
PW_HD int biased_exponent_of(double x) {
#if defined(__CUDA_ARCH__)
  return (int) ((__double_as_longlong(x) >> 52) & 0x7ff);
#else
  long long bits; memcpy(&bits, &x, sizeof bits); return (int) ((bits >> 52) & 0x7ff);
#endif
}
// Largest root of  l^3 - 3 l - x = 0  for x in [0, 2]  (= 2 cos(acos(x/2)/3), in [sqrt 3, 2]).
// The root is simple with f' = 3 l^2 - 3 in [6, 9], so Newton's iteration is quadratically convergent from the
// degree-4 fit below (|error| <= 1.9e-5 over the interval): 2e-5 -> 3e-10 -> 1e-17 -> done; the slope's reciprocal only
// needs single precision for that. ~30 instructions instead of the double-precision acos + cos (~600 with their
// slow paths), and the same arithmetic on host and device.
PW_HD double cubic_top_root(double x) {
  const float t = (float) x - 1.0f;
  const float l0 = fmaf(fmaf(fmaf(fmaf(-5.08044654e-04f, t, 2.34362113e-03f), t, -1.28488787e-02f), t, 1.31615076e-01f), t, 1.87938457f);
  double l = (double) l0;
  for (int k = 0; k < 3; ++k) {
    const double f = fma(fma(l, l, -3.0), l, -x);
    const double fp = fma(3.0 * l, l, -3.0);
    const double r = (double) rcp_f((float) fp);
    l = fma(-f, r, l);
  }
  return l;
}
// Same contract as jacobi_svd3(): sv descending, ucol2 = unit eigenvector of the smallest singular value.
// Steps: (1) scale by the power of two that brings the largest |entry| into [1, 2) (exact); (2) the extreme eigenvalue
// that is better isolated (the largest if det(B) >= 0, else the smallest) as the simple root of the characteristic
// cubic in its trigonometric normal form (cubic_top_root) — that root is well conditioned, unlike the clustered pair;
// (3) its eigenvector from the rows of (A - lambda I); (4) the other two eigenpairs EXACTLY from the 2x2 problem in
// the orthogonal complement (one Jacobi rotation).
// Measured accuracy of the returned vector: <= 8 eps * lambda_max / (lambda_mid - lambda_min) over 2e5 random
// matrices including clustered spectra, i.e. the conditioning limit of the problem itself (tests/test_host_twin.py).
PW_HD void sym_eig3(double cxx, double cxy, double cxz, double cyy, double cyz, double czz, double sv[3], double ucol2[3]) {
  const double amax = fmax(fmax(fabs(cxx), fabs(cxy)), fmax(fmax(fabs(cxz), fabs(cyy)), fmax(fabs(cyz), fabs(czz))));
  const double chk = (cxx + cxy) + (cxz + cyy) + (cyz + czz);   // fmax() skips NaN operands; the sum does not
  if (!(amax <= DBL_MAX) || chk != chk) {  // S:57 with one point: 0/0. Defined as U = I, singular values NaN (oracle header).
    sv[0] = sv[1] = sv[2] = NAN;
    ucol2[0] = 0; ucol2[1] = 0; ucol2[2] = 1;
    return;
  }
  if (amax == 0.0) { sv[0] = sv[1] = sv[2] = 0.0; ucol2[0] = 0; ucol2[1] = 0; ucol2[2] = 1; return; }
  int be = biased_exponent_of(amax);
  be = be < 1 ? 1 : (be > 2045 ? 2045 : be);
  const double inv = pow2_biased(2046 - be), unscale = pow2_biased(be);
  const double a00 = cxx * inv, a01 = cxy * inv, a02 = cxz * inv, a11 = cyy * inv, a12 = cyz * inv, a22 = czz * inv;
  const double norm = a01 * a01 + a02 * a02 + a12 * a12;
  const double q = (a00 + a11 + a22) * (1.0 / 3.0);   // any shift near trace/3 works
  const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
  const double p2 = (b00 * b00 + b11 * b11 + b22 * b22 + norm * 2.0) * (1.0 / 6.0);
  const double rp = rsqrt_d(p2), rp3 = rp * rp * rp;   // p2 == 0 -> inf, rejected below
  double e0, e1, e2;  // ascending
  double v0[3];
  if (norm > 0.0 && rp3 <= DBL_MAX) {
    const double c00 = b11 * b22 - a12 * a12, c01 = a01 * b22 - a12 * a02, c02 = a01 * a12 - b11 * a02;
    const double det = b00 * c00 - a01 * c01 + a02 * c02;   // det(B); det(B / p) = 2 cos(3 theta) in [-2, 2]
    double x = fabs(det) * rp3;
    x = x > 2.0 ? 2.0 : x;
    const bool top = det >= 0.0;  // isolate the largest eigenvalue, else the smallest
    const double pl = p2 * rp * cubic_top_root(x);
    const double e_iso = top ? q + pl : q - pl;
    double v[3];
    eigvec_by_rows(a00, a01, a02, a11, a12, a22, e_iso, v);
    const double av[3] = {a00 * v[0] + a01 * v[1] + a02 * v[2], a01 * v[0] + a11 * v[1] + a12 * v[2], a02 * v[0] + a12 * v[1] + a22 * v[2]};
    const double l_iso = v[0] * av[0] + v[1] * av[1] + v[2] * av[2];  // Rayleigh quotient
    double u[3], w[3];
    orthogonal_complement(v, u, w);
    const double au[3] = {a00 * u[0] + a01 * u[1] + a02 * u[2], a01 * u[0] + a11 * u[1] + a12 * u[2], a02 * u[0] + a12 * u[1] + a22 * u[2]};
    const double aw[3] = {a00 * w[0] + a01 * w[1] + a02 * w[2], a01 * w[0] + a11 * w[1] + a12 * w[2], a02 * w[0] + a12 * w[1] + a22 * w[2]};
    const double m00 = u[0] * au[0] + u[1] * au[1] + u[2] * au[2];
    const double m01 = u[0] * aw[0] + u[1] * aw[1] + u[2] * aw[2];
    const double m11 = w[0] * aw[0] + w[1] * aw[1] + w[2] * aw[2];
    // Jacobi rotation of [[m00, m01], [m01, m11]]: t = tan(phi) = sign(d) m01 / (|d| + hypot(d, m01)), d = (m11 - m00)/2
    double c = 1.0, sn = 0.0, la = m00, lb = m11;
    const double dl = (m11 - m00) * 0.5;
    const double h2 = dl * dl + m01 * m01;
    if (m01 != 0.0 && h2 > 0.0) {
      const double t = (dl >= 0.0 ? m01 : -m01) * rcp_d(fabs(dl) + h2 * rsqrt_d(h2));
      c = rsqrt_d(1.0 + t * t);
      sn = t * c;
      la = m00 - t * m01;
      lb = m11 + t * m01;
    }
    // eigenvectors in the complement: la <-> c u - s w, lb <-> s u + c w
    const bool a_small = la <= lb;
    const double l_lo = a_small ? la : lb, l_hi = a_small ? lb : la;
    if (top) {
      e2 = l_iso; e1 = l_hi; e0 = l_lo;
      for (int k = 0; k < 3; ++k) v0[k] = a_small ? (c * u[k] - sn * w[k]) : (sn * u[k] + c * w[k]);
    } else {
      e0 = l_iso; e1 = l_lo; e2 = l_hi;
      for (int k = 0; k < 3; ++k) v0[k] = v[k];
    }
  } else {  // (numerically) diagonal
    e0 = a00; e1 = a11; e2 = a22;
    int imin = 0;
    double emin = a00;
    if (a11 < emin) { emin = a11; imin = 1; }
    if (a22 < emin) { emin = a22; imin = 2; }
    v0[0] = imin == 0 ? 1.0 : 0.0; v0[1] = imin == 1 ? 1.0 : 0.0; v0[2] = imin == 2 ? 1.0 : 0.0;
    if (e0 > e1) { const double t = e0; e0 = e1; e1 = t; }
    if (e1 > e2) { const double t = e1; e1 = e2; e2 = t; }
    if (e0 > e1) { const double t = e0; e0 = e1; e1 = t; }
  }
  double s0 = fabs(e2) * unscale, s1 = fabs(e1) * unscale, s2 = fabs(e0) * unscale;
  if (s1 > s0) { const double t = s0; s0 = s1; s1 = t; }
  if (s2 > s1) { const double t = s1; s1 = s2; s2 = t; }
  if (s1 > s0) { const double t = s0; s0 = s1; s1 = t; }
  sv[0] = s0; sv[1] = s1; sv[2] = s2;
  ucol2[0] = v0[0]; ucol2[1] = v0[1]; ucol2[2] = v0[2];
}

// Moment sums of a point set taken relative to a reference point c (shifted one-pass covariance):
//   s1[k] = sum (p_k - c_k),  s2 = sum (p_j - c_j)(p_k - c_k)  in order xx xy xz yy yz zz.
struct Moments {
  double s1[3];
  double s2[6];
  int n;
};

// estimate_plane (S:47-75) from the moment sums. n == 0 must be handled by the caller (S:49: keep
// the previous plane). mean = c + s1/n ; cov = (s2 - s1 s1^T / n) / (n-1).
PW_HD void plane_from_moments(const Moments& m, const double c[3], Plane& pl) {
  const double inv_n = rcp_d((double) m.n);
  const double m0 = m.s1[0] * inv_n, m1 = m.s1[1] * inv_n, m2 = m.s1[2] * inv_n;
  pl.mean[0] = c[0] + m0; pl.mean[1] = c[1] + m1; pl.mean[2] = c[2] + m2;
  // n == 1: 0 * inf = NaN covariance, like the 0/0 of S:57
  const double inv_dn = rcp_d((double) (m.n - 1));
  const double cxx = (m.s2[0] - m.s1[0] * m0) * inv_dn;
  const double cxy = (m.s2[1] - m.s1[0] * m1) * inv_dn;
  const double cxz = (m.s2[2] - m.s1[0] * m2) * inv_dn;
  const double cyy = (m.s2[3] - m.s1[1] * m1) * inv_dn;
  const double cyz = (m.s2[4] - m.s1[1] * m2) * inv_dn;
  const double czz = (m.s2[5] - m.s1[2] * m2) * inv_dn;
  double u2[3];
#if defined(PWPP_USE_JACOBI)
  jacobi_svd3(cxx, cxy, cxz, cyy, cyz, czz, pl.sv, u2);
#else
  sym_eig3(cxx, cxy, cxz, cyy, cyz, czz, pl.sv, u2);
#endif
  if (u2[2] < 0.0) { u2[0] = -u2[0]; u2[1] = -u2[1]; u2[2] = -u2[2]; }  // S:68
  pl.normal[0] = u2[0]; pl.normal[1] = u2[1]; pl.normal[2] = u2[2];
  // d = -(normal . mean), association x0 + (x1 + x2) (S:74 through Eigen's unrolled redux)
  pl.d = -(u2[0] * pl.mean[0] + (u2[1] * pl.mean[1] + u2[2] * pl.mean[2]));
}

// calc_point_to_plane_d (S:551-554) in double: ((n0*x + n1*y) + n2*z) + d
PW_HD double point_plane_distance(const Plane& pl, float x, float y, float z) {
  const double a = dmul(pl.normal[0], (double) x), b = dmul(pl.normal[1], (double) y), c = dmul(pl.normal[2], (double) z);
  return dadd(dadd(dadd(a, b), c), pl.d);
}

}  // namespace pwpp
