// Terrain attributes (slope, aspect, curvatures): independent 3x3 stencils over the elevation raster, one
// float out per cell (reference methods/terrain_attributes.hpp:154-538).  HBM-bound at 8 B/cell; the
// arithmetic is the reference's, in double, one rounding per operation and in the reference's order (no
// fused multiply-adds: the reference's stock x86-64 build has none), so slopes and curvatures come out
// bit-identical and only the attributes that go through atan / atan2 can differ in the last float bit.
//
// A block stages a (128+2) x (16+2) window in shared memory; a thread owns one column of it and walks the
// 16 rows, carrying the 3x3 neighbourhood's previous two rows in registers.
#include "common.cuh"

#include <cmath>

namespace rdb {

namespace {

constexpr int kTW = 128, kTH = 16;

struct Nbhd {  // reference naming (terrain_attributes.hpp:163-169):  a b c / d e f / g h i, already z-scaled
  double a, b, c, d, e, f, g, h, i;
};

// A division by a power of two is the multiplication by its (exact) reciprocal -- same correctly rounded result, a
// fraction of the double-precision instructions.  The 2, 4 and 8 of the formulas always are; a cell length is checked on
// the host (1 x 1 cells, the geotransform pyrichdem assumes when there is none, are).
struct CellLen {
  double len, inv;  // inv = 1 / len when that is exact, else 0
};
__device__ __forceinline__ double over(double x, const CellLen &l) {
  return l.inv != 0.0 ? __dmul_rn(x, l.inv) : __ddiv_rn(x, l.len);
}

// Horn (1981) gradients, terrain_attributes.hpp:225-227,244-246
__device__ __forceinline__ void horn(const Nbhd &t, const CellLen &lx, const CellLen &ly, double *dzdx, double *dzdy) {
  const double right = __dadd_rn(__dadd_rn(t.c, __dmul_rn(2.0, t.f)), t.i);
  const double left = __dadd_rn(__dadd_rn(t.a, __dmul_rn(2.0, t.d)), t.g);
  const double down = __dadd_rn(__dadd_rn(t.g, __dmul_rn(2.0, t.h)), t.i);
  const double up = __dadd_rn(__dadd_rn(t.a, __dmul_rn(2.0, t.b)), t.c);
  *dzdx = over(__dmul_rn(__dsub_rn(right, left), 0.125), lx);
  *dzdy = over(__dmul_rn(__dsub_rn(down, up), 0.125), ly);
}

struct Curves {  // Zevenbergen & Thorne (1987) coefficients, terrain_attributes.hpp:198-213
  double D, E, F, G, H;
};
__device__ __forceinline__ Curves curves(const Nbhd &t, const CellLen &L) {
  Curves p;
  p.D = over(over(__dsub_rn(__dmul_rn(__dadd_rn(t.d, t.f), 0.5), t.e), L), L);
  p.E = over(over(__dsub_rn(__dmul_rn(__dadd_rn(t.b, t.h), 0.5), t.e), L), L);
  p.F = over(over(__dmul_rn(__dsub_rn(__dadd_rn(__dadd_rn(-t.a, t.c), t.g), t.i), 0.25), L), L);
  p.G = over(__dmul_rn(__dadd_rn(-t.d, t.f), 0.5), L);
  p.H = over(__dmul_rn(__dsub_rn(t.b, t.h), 0.5), L);
  return p;
}

template <int ATTR>
__device__ __forceinline__ double attribute(const Nbhd &t, const CellLen &lx, const CellLen &ly) {
  constexpr double kPi = 3.14159265358979323846;
  if (ATTR <= RDB200_TA_SLOPE_RADIANS) {
    double dzdx, dzdy;
    horn(t, lx, ly, &dzdx, &dzdy);
    const double rr = sqrt(__dadd_rn(__dmul_rn(dzdx, dzdx), __dmul_rn(dzdy, dzdy)));  // :247
    if (ATTR == RDB200_TA_SLOPE_RISERUN) return rr;
    if (ATTR == RDB200_TA_SLOPE_PERCENTAGE) return __dmul_rn(rr, 100.0);                        // :301
    if (ATTR == RDB200_TA_SLOPE_DEGREES) return __ddiv_rn(__dmul_rn(atan(rr), 180.0), kPi);     // :319
    return atan(rr);                                                                             // :310
  }
  if (ATTR == RDB200_TA_ASPECT) {  // :222-236
    double dzdx, dzdy;
    horn(t, lx, ly, &dzdx, &dzdy);
    const double asp = __dmul_rn(180.0 / kPi, atan2(dzdy, -dzdx));
    if (asp < 0) return __dsub_rn(90.0, asp);
    if (asp > 90.0) return __dadd_rn(__dsub_rn(360.0, asp), 90.0);
    return __dsub_rn(90.0, asp);
  }
  const Curves p = curves(t, lx);
  if (ATTR == RDB200_TA_CURVATURE) return __dmul_rn(__dmul_rn(-2.0, __dadd_rn(p.D, p.E)), 100.0);  // :257
  if (p.G == 0 && p.H == 0) return 0;
  const double gg = __dmul_rn(p.G, p.G), hh = __dmul_rn(p.H, p.H), den = __dadd_rn(gg, hh);
  const double fgh = __dmul_rn(__dmul_rn(p.F, p.G), p.H);
  if (ATTR == RDB200_TA_PLANFORM_CURVATURE) {  // :271
    const double num = __dsub_rn(__dadd_rn(__dmul_rn(__dmul_rn(p.D, p.H), p.H), __dmul_rn(__dmul_rn(p.E, p.G), p.G)), fgh);
    return __dmul_rn(__ddiv_rn(__dmul_rn(-2.0, num), den), 100.0);
  }
  const double num = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(p.D, p.G), p.G), __dmul_rn(__dmul_rn(p.E, p.H), p.H)), fgh);  // :285
  return __dmul_rn(__ddiv_rn(__dmul_rn(2.0, num), den), 100.0);
}

// T: float, or double for rdb200_terrain_attribute_f64 (the reference reads T into its double neighbourhood,
// terrain_attributes.hpp:172-190; only the window and the NoData test change type, the window to 18.7 KB)
template <int ATTR, class T>
__global__ void __launch_bounds__(kTW) terrain_attribute_kernel(const T *__restrict__ dem, float *__restrict__ out, int W, int H,
                                                                T nodata_in, float nodata_out, float zscale, CellLen lx,
                                                                CellLen ly) {
  __shared__ T s[kTH + 2][kTW + 2];
  const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
  // window load: cells outside the raster are marked by a flag row/column test at use, their slot is never read
  for (int r = 0; r < kTH + 2; r++) {
    const int y = y0 + r - 1;
    if (y < 0 || y >= H) continue;
    for (int cidx = threadIdx.x; cidx < kTW + 2; cidx += kTW) {
      const int x = x0 + cidx - 1;
      if (x >= 0 && x < W) s[r][cidx] = dem[(size_t)y * W + x];
    }
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= W) return;
  const int cx = threadIdx.x + 1;
  const bool has_l = x > 0, has_r = x + 1 < W;
  const double zs = (double)zscale;
  for (int r = 1; r <= kTH; r++) {
    const int y = y0 + r - 1;
    if (y >= H) break;
    const T ef = s[r][cx];
    float o;
    if (ef == nodata_in) {  // terrain_attributes.hpp:349-350
      o = nodata_out;
    } else {
      const bool has_u = y > 0, has_d = y + 1 < H;
      // neighbours outside the raster or NoData take the centre's value (:172-181)
      auto pick = [&](bool in, int rr, int cc) -> double {
        T v = ef;
        if (in) {
          const T nv = s[rr][cc];
          if (nv != nodata_in) v = nv;
        }
        return __dmul_rn((double)v, zs);
      };
      Nbhd t;
      t.a = pick(has_l && has_u, r - 1, cx - 1);
      t.b = pick(has_u, r - 1, cx);
      t.c = pick(has_r && has_u, r - 1, cx + 1);
      t.d = pick(has_l, r, cx - 1);
      t.e = __dmul_rn((double)ef, zs);
      t.f = pick(has_r, r, cx + 1);
      t.g = pick(has_l && has_d, r + 1, cx - 1);
      t.h = pick(has_d, r + 1, cx);
      t.i = pick(has_r && has_d, r + 1, cx + 1);
      o = (float)attribute<ATTR>(t, lx, ly);
    }
    out[(size_t)y * W + x] = o;
  }
}

template <int ATTR, class T>
void launch(const T *d_dem, float *d_out, int w, int h, T nodata_in, float nodata_out, float zscale, double cell_x, double cell_y) {
  Ctx &c = ctx();
  auto cell = [](double len) {
    int e = 0;
    CellLen l;
    l.len = len;
    l.inv = (std::frexp(len, &e) == 0.5 && e > -1000 && e < 1000) ? 1.0 / len : 0.0;  // a power of two: 1 / len is exact
    return l;
  };
  const CellLen lx = cell(cell_x), ly = cell(cell_y);
  const dim3 grd((w + kTW - 1) / kTW, (h + kTH - 1) / kTH);
  terrain_attribute_kernel<ATTR, T><<<grd, kTW, 0, c.stream>>>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, lx, ly);
  RDB_CK(cudaGetLastError());
  count_launch();
}

// attribute: RDB200_TA_* (include/richdem_b200.h); cell_x / cell_y = |geotransform[1]|, |geotransform[5]|
template <class T>
void terrain_attribute_any(int attribute_id, const T *d_dem, float *d_out, int w, int h, T nodata_in, float nodata_out,
                           float zscale, double cell_x, double cell_y) {
  if (!(cell_x > 0) || !(cell_y > 0)) fail("terrain attribute: cell lengths must be positive (got %g x %g)", cell_x, cell_y);
  switch (attribute_id) {
    case RDB200_TA_SLOPE_RISERUN: launch<RDB200_TA_SLOPE_RISERUN>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_SLOPE_PERCENTAGE: launch<RDB200_TA_SLOPE_PERCENTAGE>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_SLOPE_DEGREES: launch<RDB200_TA_SLOPE_DEGREES>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_SLOPE_RADIANS: launch<RDB200_TA_SLOPE_RADIANS>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_ASPECT: launch<RDB200_TA_ASPECT>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_CURVATURE: launch<RDB200_TA_CURVATURE>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_PLANFORM_CURVATURE: launch<RDB200_TA_PLANFORM_CURVATURE>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    case RDB200_TA_PROFILE_CURVATURE: launch<RDB200_TA_PROFILE_CURVATURE>(d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y); break;
    default: fail("unknown terrain attribute %d", attribute_id);
  }
}

}  // namespace

void terrain_attribute_dev(int attribute_id, const float *d_dem, float *d_out, int w, int h, float nodata_in, float nodata_out,
                           float zscale, double cell_x, double cell_y) {
  terrain_attribute_any(attribute_id, d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
}
void terrain_attribute_dev(int attribute_id, const double *d_dem, float *d_out, int w, int h, double nodata_in,
                           float nodata_out, float zscale, double cell_x, double cell_y) {
  terrain_attribute_any(attribute_id, d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
}

}  // namespace rdb
