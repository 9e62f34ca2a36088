// Per-cell flow-metric device functions shared by the materialising kernels (FM_D8 /
// FM_Tarboton -> 9 floats per cell) and the fused accumulation path (compact code per cell).
#pragma once
#include "common.cuh"

namespace rdb {

constexpr float kNoFlowGen = -1.0f;   // reference common/constants.hpp:83
constexpr float kHasFlowGen = 0.0f;   // :84
constexpr float kNoDataGen = -2.0f;   // :85

// Compact per-cell flow code used by the fused accumulation:
//   0        no receiver (no-flow cell, raster-edge cell)
//   1..8     one receiver in D8 direction n, proportion 1
//   16|n     two receivers: n with proportion p1 and nwrap(n+1) with proportion p2 (D-infinity)
//   255      NoData cell
constexpr uint8_t kCodeNoData = 255;
constexpr uint8_t kCodeTwo = 16;

__device__ __forceinline__ int nwrap(int n) { return n == 9 ? 1 : n; }
__device__ __forceinline__ int d8_inverse(int n) { return n == 0 ? 0 : ((n + 3) & 7) + 1; }  // {0,5,6,7,8,1,2,3,4}

// The per-cell functions below take the elevation type T of the reference's templates: float, or double for the
// rdb200_*_f64 entry points.  Where the two differ the difference is written out; everything else is the same code.
template <class T> __device__ __forceinline__ T elev_max();  // numeric_limits<T>::max()
template <> __device__ __forceinline__ float elev_max<float>() { return 3.402823466e+38f; }
template <> __device__ __forceinline__ double elev_max<double>() { return 1.7976931348623157e+308; }
// e - ne as the reference computes it in E and widens to double: exact for floats, one rounding for doubles
__device__ __forceinline__ double elev_diff(float a, float b) { return (double)__fsub_rn(a, b); }
__device__ __forceinline__ double elev_diff(double a, double b) { return __dsub_rn(a, b); }

// FM_OCallaghan<D8> for one cell (reference flowmet/OCallaghan1984.hpp:37-75).
// returns kCodeNoData, 0 (no flow) or the receiver direction 1..8.
template <class T>
__device__ __forceinline__ int fm_d8_cell(const T *__restrict__ dem, int x, int y, int W, int H, T nodata) {
  const size_t i = (size_t)y * W + x;
  const T e = __ldg(dem + i);
  if (e == nodata) return kCodeNoData;                          // :37-40
  if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return 0;  // :42-43
  int lowest_n = 0;
  T lowest = elev_max<T>();  // numeric_limits<T>::max(), :48
#pragma unroll
  for (int n = 1; n <= 8; n++) {
    const T ne = __ldg(dem + (size_t)(y + d8dy(n)) * W + (x + d8dx(n)));
    if (ne == nodata) continue;  // :53-54
    if (ne >= e) continue;       // :58-59
    if (ne < lowest) {           // :61-64  strict: the first minimum wins
      lowest = ne;
      lowest_n = n;
    }
  }
  return lowest_n;
}

// FM_OCallaghan<D4> for one cell (reference flowmet/OCallaghan1984.hpp:37-75 with the D4 offset tables
// common/constants.hpp:53-54: 1 = W, 2 = N, 3 = E, 4 = S).  Returns kCodeNoData, 0 or the D4 index 1..4 --
// the reference stores the proportion in THAT slot of the 9-slot cell (and its generic accumulation then
// reads slots as D8 directions, flow_accumulation_generic.hpp:53-56); both are reproduced as they are.
template <class T>
__device__ __forceinline__ int fm_d4_cell(const T *__restrict__ dem, int x, int y, int W, int H, T nodata) {
  const size_t i = (size_t)y * W + x;
  const T e = __ldg(dem + i);
  if (e == nodata) return kCodeNoData;
  if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return 0;
  int lowest_n = 0;
  T lowest = elev_max<T>();
#pragma unroll
  for (int n = 1; n <= 4; n++) {
    const int dx = n == 1 ? -1 : (n == 3 ? 1 : 0), dy = n == 2 ? -1 : (n == 4 ? 1 : 0);
    const T ne = __ldg(dem + (size_t)(y + dy) * W + (x + dx));
    if (ne == nodata) continue;
    if (ne >= e) continue;
    if (ne < lowest) {
      lowest = ne;
      lowest_n = n;
    }
  }
  return lowest_n;
}

// FM_Holmgren (HOLMGREN = true; reference flowmet/Holmgren1994.hpp:33-80; FM_Quinn is xparam = 1,
// Quinn1991.hpp:15) and FM_Freeman (HOLMGREN = false; flowmet/Freeman1991.hpp:28-77) for one cell.
// p[0..8] arrives filled with NO_FLOW_GEN.  The reference's mixed precision is kept step by step:
// rise is e - ne in E widened to double (elev_diff), the gradient and the power are double; Holmgren rounds
// each power to float BEFORE summing (it sums props(x,y,n)), Freeman sums the unrounded doubles;
// normalisation multiplies the stored float by the double 1/C and rounds once.  pow(g, 1.0) is g in
// glibc, so the exponent-1 case takes the value itself instead of the device pow (<= 2 ulp).
template <bool HOLMGREN, class T>
__device__ __forceinline__ void fm_mfd_cell(const T *__restrict__ dem, int x, int y, int W, int H, T nodata,
                                            double xparam, float (&p)[9]) {
  const size_t i = (size_t)y * W + x;
  const T e = __ldg(dem + i);
  if (e == nodata) {
    p[0] = kNoDataGen;
    return;
  }
  if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return;
  double C = 0;
#pragma unroll
  for (int n = 1; n <= 8; n++) {
    const T ne = __ldg(dem + (size_t)(y + d8dy(n)) * W + (x + d8dx(n)));
    if (ne == nodata) continue;
    if (ne < e) {
      const double rise = elev_diff(e, ne);
      const double run = (n & 1) ? 1.0 : 1.414213562373095048801688724209698078569671875376948;
      double g = __ddiv_rn(rise, run);
      if (HOLMGREN) g = __dmul_rn(g, (n & 1) ? 0.5 : 0.354);
      const double cval = xparam == 1.0 ? g : pow(g, xparam);
      p[n] = (float)cval;
      C = __dadd_rn(C, HOLMGREN ? (double)p[n] : cval);
    }
  }
  if (C > 0) {
    p[0] = kHasFlowGen;
    C = __ddiv_rn(1.0, C);
#pragma unroll
    for (int n = 1; n <= 8; n++) p[n] = p[n] > 0 ? (float)__dmul_rn((double)p[n], C) : 0.0f;
  }
}

// FM_Tarboton for one cell (reference flowmet/Tarboton1997.hpp:62-141).
// returns kCodeNoData, 0 (no flow) or nmax in 1..8 with *rmax_out = rmax after the facet-parity
// flip (:121-126).  All double arithmetic uses explicit round-to-nearest intrinsics so that no
// FMA contraction happens (the CPU reference is compiled without it).

// which of the reference's three cases a facet falls into (:95-107): 0: r < 1e-7, 1: r > dang - 1e-7, 2: in between.
// r = atan2(s2, s1) only matters through these two threshold tests and, for the steepest facet, as rmax.  The tests are
// decided from the signs and the ratio s2 / s1 (atan2 is monotone in it) whenever the ratio is clear of tan(1e-7) and
// tan(dang - 1e-7) by a relative 1e-9 -- ten million ulps, far beyond any atan2's error -- and by the function itself
// otherwise; the one atan2 a cell needs is taken at the end.  (8 double atan2 per cell were 77 of the 575 ms of FA_Dinf
// at 32768^2.)  `ratio` false skips the shortcut and decides by atan2 alone, the reference's own sequence: a double
// facet whose s1 or s2 lies outside dinf_in_range below, where the products can be subnormal and lose the margin.
__device__ __forceinline__ int tarboton_facet_case(double s1, double s2, double dangd, bool ratio = true) {
  if (ratio) {
    if (s2 < 0.0 || (s2 == 0.0 && s1 >= 0.0)) return 0;  // angles in (-pi, 0], and atan2(0, 0) = 0
    if (s1 <= 0.0) return 1;                              // s2 > 0 (or s2 == 0 with s1 < 0): angles in [pi/2, pi]
    const double tlo = 1.0000000000000033e-07, thi = 0.9999998437114023;  // tan(1e-7), tan(dang - 1e-7)
    const double eps = 1e-9;
    if (s2 < s1 * (tlo * (1.0 - eps))) return 0;
    if (s2 > s1 * (thi * (1.0 + eps))) return 1;
    if (s2 > s1 * (tlo * (1.0 + eps)) && s2 < s1 * (thi * (1.0 - eps))) return 2;
  }
  const double ra = atan2(s2, s1);
  return ra < 1e-7 ? 0 : (ra > __dsub_rn(dangd, 1e-7) ? 1 : 2);
}
// the facet's slope as the reference computes it
__device__ __forceinline__ double tarboton_facet_slope(int fcase, double s1, double s2, double e0_minus_e2) {
  if (fcase == 0) return s1;                                               // :99-101
  if (fcase == 1) return __ddiv_rn(e0_minus_e2, 1.4142135623730951);       // :102-104, sqrt(d1*d1+d2*d2) = sqrt(2.0)
  return __dsqrt_rn(__dadd_rn(__dmul_rn(s1, s1), __dmul_rn(s2, s2)));      // :106
}
// Both shortcuts are proven for differences of floats, which lie in [2^-149, 2^129].  Differences of doubles are
// rounded and unbounded: a square overflows above 2^512 and underflows below 2^-511, a ratio-test product is subnormal
// below about 2^-999.  Inside [2^-500, 2^500] every square, sum of squares and product is a normal double, so the
// relative margins (1e-12, 1e-9) hold as for floats; 0, +-inf and NaN take the float path's rules (DESIGN §0.2).
__device__ __forceinline__ bool dinf_in_range(double x) {
  const double a = fabs(x);
  return !((a > 0.0 && a < 0x1p-500) || (a > 0x1p500 && a <= 1.7976931348623157e+308));
}

// `filter`: choose the steepest facet from the SQUARED slopes first (no square root, no division per facet: in a warp
// whose lanes sit in different cases every facet otherwise costs both) and evaluate the reference's slope for the winner
// only.  Squaring is monotone, so the facet with the largest square has the largest slope unless another facet's square
// is within a relative 1e-12 of it (several thousand ulps); an exact tie inside one case means an exactly equal slope and
// the first facet wins as in the reference; anything else near the maximum sends the cell through the reference's own
// sequence of comparisons.  Identical result either way (rdb200_set_param("flowmet_tarboton_filter", 0) turns it off).
// T = double: s1, s2 and e0 - e2 are rounded differences, as in the reference's double template.  A cell with a finite,
// nonzero difference outside dinf_in_range leaves the filter for the reference's sequence, and a facet with such an s1 or
// s2 has its case decided by atan2 alone; the checks fold away for T = float.
template <class T>
__device__ __forceinline__ int fm_tarboton_cell(const T *__restrict__ dem, int x, int y, int W, int H,
                                                T nodata, float *rmax_out, bool filter = true) {
  constexpr bool F64 = sizeof(T) == 8;
  const size_t i = (size_t)y * W + x;
  const T e0f = __ldg(dem + i);
  if (e0f == nodata) return kCodeNoData;
  if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return 0;
  // facet tables, :48-53 (remapped facets 1..8)
  //  dy_e1 = {0, 0,-1,-1, 0, 0, 1, 1, 0}   dx_e1 = {0,-1, 0, 0, 1, 1, 0, 0,-1}
  //  dy_e2 = {0,-1,-1,-1,-1, 1, 1, 1, 1}   dx_e2 = {0,-1,-1, 1, 1, 1, 1,-1,-1}
  //  af    = {0,-1, 1,-1, 1,-1, 1,-1, 1}
  const float dang = 0.78539818525314331f;  // float(atan2(1,1)), :29
  const double dangd = (double)dang;
  const double e0 = (double)e0f;
  // the eight neighbours once: cardinal W, N, E, S and diagonal NW, NE, SE, SW (interior cell: all in the grid)
  const T cw = __ldg(dem + i - 1), cn = __ldg(dem + i - W), ce = __ldg(dem + i + 1), cs = __ldg(dem + i + W);
  const T dnw = __ldg(dem + i - W - 1), dne = __ldg(dem + i - W + 1), dse = __ldg(dem + i + W + 1), dsw = __ldg(dem + i + W - 1);
  // facet n: e1 = its cardinal neighbour, e2 = its diagonal one
  const T e1s[9] = {T(0), cw, cn, cn, ce, ce, cs, cs, cw};
  const T e2s[9] = {T(0), dnw, dnw, dne, dne, dse, dse, dsw, dsw};
  int nmax = -1, bmax = 0;
  double smax = 0, s1max = 0, s2max = 0;
  bool decided = false;
  if (filter) {
    double qbest = 0, qsecond = 0;  // largest squared slope and the largest one of any OTHER facet that is not its exact twin
    int nb = -1, cb = 0;
    double s1b = 0, s2b = 0, tb = 0;
    bool outside = false;  // a double difference outside dinf_in_range (always false for T = float)
#pragma unroll
    for (int n = 1; n <= 8; n++) {
      const T e1f = e1s[n], e2f = e2s[n];
      if (e1f == nodata || e2f == nodata) continue;  // :76-83
      const double e1 = (double)e1f, e2 = (double)e2f;
      const double s1 = __dsub_rn(e0, e1), s2 = __dsub_rn(e1, e2), t = __dsub_rn(e0, e2);  // exact for floats
      if (F64 && !(dinf_in_range(s1) && dinf_in_range(s2) && dinf_in_range(t))) {
        outside = true;  // leave the filter: the reference's sequence decides this cell
        break;
      }
      const int fc = tarboton_facet_case(s1, s2, dangd);
      double q;  // the slope's square; 0 for a slope that is not positive (it can never beat smax = 0)
      if (fc == 0) q = s1 > 0.0 ? __dmul_rn(s1, s1) : 0.0;
      else if (fc == 1) q = t > 0.0 ? __dmul_rn(__dmul_rn(t, t), 0.5) : 0.0;
      else q = __dadd_rn(__dmul_rn(s1, s1), __dmul_rn(s2, s2));
      if (q > qbest) {
        if (qbest > qsecond) qsecond = qbest;  // the previous leader becomes a rival
        qbest = q;
        nb = n;
        cb = fc;
        s1b = s1;
        s2b = s2;
        tb = t;
      } else if (q == qbest && fc == cb) {
        // an exact twin of the leader in the same case: exactly the same slope, the earlier facet keeps the lead
      } else if (q > qsecond) {
        qsecond = q;
      }
    }
    if (nb == -1 && !outside) return 0;  // no facet slopes down (:115-116; every q is 0)
    if (!outside && qsecond < qbest * (1.0 - 1e-12)) {
      nmax = nb;
      bmax = cb;
      s1max = s1b;
      s2max = s2b;
      smax = tarboton_facet_slope(cb, s1b, s2b, tb);
      decided = true;
    }
  }
  if (!decided) {
    nmax = -1;
#pragma unroll
    for (int n = 1; n <= 8; n++) {
      const T e1f = e1s[n], e2f = e2s[n];
      if (e1f == nodata || e2f == nodata) continue;
      const double e1 = (double)e1f, e2 = (double)e2f;
      const double s1 = __dsub_rn(e0, e1);  // (e0-e1)/d1, d1 = 1
      const double s2 = __dsub_rn(e1, e2);
      const int fc = tarboton_facet_case(s1, s2, dangd, !F64 || (dinf_in_range(s1) && dinf_in_range(s2)));
      const double s = tarboton_facet_slope(fc, s1, s2, __dsub_rn(e0, e2));
      if (s > smax) {  // :109-113
        smax = s;
        nmax = n;
        bmax = fc;
        s1max = s1;
        s2max = s2;
      }
    }
  }
  if (nmax == -1) return 0;
  float rmax = bmax == 0 ? 0.0f : (bmax == 1 ? (float)dangd : (float)atan2(s2max, s1max));
  const bool af_pos = (nmax & 1) == 0;  // af[n] == +1 for even n
  if (af_pos && rmax == 0.0f) rmax = dang;
  else if (af_pos && rmax == dang) rmax = 0.0f;
  else if (af_pos) rmax = (float)__dsub_rn(0.78539816339744830962, (double)rmax);  // M_PI/4 - rmax
  *rmax_out = rmax;
  return nmax;
}

// proportions written by FM_Tarboton, :134-141
__device__ __forceinline__ void tarboton_props(float rmax, float *p1, float *p2) {
  const double q = __ddiv_rn((double)rmax, 0.78539816339744830962);
  *p1 = (float)q;
  *p2 = (float)__dsub_rn(1.0, q);
}
constexpr float kDang = 0.78539818525314331f;

}  // namespace rdb
