// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or executed from the product path.
//
// extern "C" entry points over the UNMODIFIED reference flow metrics (FM_*), accumulations (FA_*) and terrain attributes
// (TA_*), each instantiated with E / T = double and = float, the fixtures of the float64 D-infinity / MFD / attribute path
// (tests/golden/make_f64_flowmet.py).  Built by oracle/f64_flowmet.py into oracle/_ref/libref_f64_flowmet.so
// (git-ignored).  Plain row-major host buffers (i = y*W + x) are wrapped unowned in richdem::Array2D / Array3D, as
// ref_shim.cpp does.  method as the C ABI numbers it: 0 D8, 1 Tarboton, 2 D4, 3 Holmgren (xparam 1: Quinn,
// Quinn1991.hpp:15), 4 Freeman; attribute as RDB200_TA_*.
#include <richdem/common/Array2D.hpp>
#include <richdem/common/Array3D.hpp>
#include <richdem/methods/flow_accumulation.hpp>
#include <richdem/methods/terrain_attributes.hpp>

#include <cstring>

using namespace richdem;

namespace {

// flowmet/*.hpp into a 9-float-per-cell buffer ([y][x][9], Array3D.hpp:203-206)
template <class T>
void fm(int method, const T *dem, int w, int h, T nodata, double xparam, float *props) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata);
  Array3D<float> p(props, w, h);
  switch (method) {
    case 0: FM_D8(a, p); break;
    case 1: FM_Tarboton(a, p); break;
    case 2: FM_D4(a, p); break;
    case 3: if (xparam == 1.0) FM_Quinn(a, p); else FM_Holmgren(a, p, xparam); break;
    default: FM_Freeman(a, p, xparam); break;
  }
}

// methods/flow_accumulation.hpp:16-20,27-28 with the caller's weights in accum
template <class T>
void fa(int method, const T *dem, int w, int h, T nodata, double xparam, double *accum) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata);
  Array2D<double> acc(accum, w, h);
  switch (method) {
    case 0: FA_D8(a, acc); break;
    case 1: FA_Tarboton(a, acc); break;
    case 2: FA_D4(a, acc); break;
    case 3: if (xparam == 1.0) FA_Quinn(a, acc); else FA_Holmgren(a, acc, xparam); break;
    default: FA_Freeman(a, acc, xparam); break;
  }
}

// methods/terrain_attributes.hpp:370-538; the output keeps its own NoData (:344)
template <class T>
void ta(int attribute, const T *dem, int w, int h, T nodata_in, float nodata_out, float zscale, double cell_x, double cell_y,
        float *out) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata_in);
  a.geotransform = {0.0, cell_x, 0.0, 0.0, 0.0, -cell_y};
  Array2D<float> o;
  o.setNoData(nodata_out);
  switch (attribute) {
    case 0: TA_slope_riserun(a, o, zscale); break;
    case 1: TA_slope_percentage(a, o, zscale); break;
    case 2: TA_slope_degrees(a, o, zscale); break;
    case 3: TA_slope_radians(a, o, zscale); break;
    case 4: TA_aspect(a, o, zscale); break;
    case 5: TA_curvature(a, o, zscale); break;
    case 6: TA_planform_curvature(a, o, zscale); break;
    default: TA_profile_curvature(a, o, zscale); break;
  }
  std::memcpy(out, o.data(), sizeof(float) * (size_t)w * h);
}

}  // namespace

#define INSTANTIATE(T, S)                                                                                               \
  void ref_fm_##S(int m, const T *dem, int w, int h, T nd, double xp, float *props) { fm<T>(m, dem, w, h, nd, xp, props); } \
  void ref_fa_##S(int m, const T *dem, int w, int h, T nd, double xp, double *accum) { fa<T>(m, dem, w, h, nd, xp, accum); } \
  void ref_ta_##S(int at, const T *dem, int w, int h, T nd, float ndo, float zs, double cx, double cy, float *out) {  \
    ta<T>(at, dem, w, h, nd, ndo, zs, cx, cy, out);                                                                   \
  }

extern "C" {
INSTANTIATE(double, f64)
INSTANTIATE(float, f32)
}  // extern "C"
