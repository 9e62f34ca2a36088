// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or executed from the product path.
//
// extern "C" entry points over the UNMODIFIED reference templates of the direction-grid pipeline, instantiated with
// T = double and T = float: barnes_flat_resolution_d8<T, uint8_t> (flats/flat_resolution.hpp:588-607, both alter modes),
// GetFlatMask<T> (flats/Barnes2014.hpp:398-467) and d8_flow_accum<uint8_t, int32_t> (methods/d8_methods.hpp:47-139).
// Built by oracle/f64_flowdirs.py into oracle/_ref/libref_f64_flowdirs.so (git-ignored).  Plain row-major host buffers
// (i = y*W + x) are wrapped unowned in richdem::Array2D, as ref_shim.cpp does.
#include <richdem/common/Array2D.hpp>
#include <richdem/flats/Barnes2014.hpp>
#include <richdem/flats/flat_resolution.hpp>
#include <richdem/methods/d8_methods.hpp>

#include <cstdint>
#include <cstring>

using namespace richdem;

namespace {

// dem is altered in place when alter != 0
template <class T>
void flowdirs_flats(T *dem, int w, int h, T nodata, int alter, uint8_t *out) {
  Array2D<T> a(dem, w, h);
  a.setNoData(nodata);
  Array2D<uint8_t> d(w, h);
  d.setNoData(255);
  barnes_flat_resolution_d8(a, d, alter != 0);
  std::memcpy(out, d.data(), (size_t)w * h);
}

template <class T>
void flat_mask(const T *dem, int w, int h, T nodata, int32_t *mask, int32_t *labels) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata);
  Array2D<int32_t> m, l;
  GetFlatMask(a, m, l);
  std::memcpy(mask, m.data(), sizeof(int32_t) * (size_t)w * h);
  std::memcpy(labels, l.data(), sizeof(int32_t) * (size_t)w * h);
}

}  // namespace

extern "C" {
void ref_flowdirs_flats_f64(double *dem, int w, int h, double nd, int alter, uint8_t *out) { flowdirs_flats(dem, w, h, nd, alter, out); }
void ref_flowdirs_flats_f32(float *dem, int w, int h, float nd, int alter, uint8_t *out) { flowdirs_flats(dem, w, h, nd, alter, out); }
void ref_flat_mask_f64(const double *dem, int w, int h, double nd, int32_t *m, int32_t *l) { flat_mask(dem, w, h, nd, m, l); }
void ref_flat_mask_f32(const float *dem, int w, int h, float nd, int32_t *m, int32_t *l) { flat_mask(dem, w, h, nd, m, l); }
void ref_d8_flow_accum(const uint8_t *dirs, int w, int h, int32_t *area) {
  Array2D<uint8_t> d(const_cast<uint8_t *>(dirs), w, h);
  d.setNoData(255);
  Array2D<int32_t> a;
  d8_flow_accum(d, a);
  std::memcpy(area, a.data(), sizeof(int32_t) * (size_t)w * h);
}
}  // extern "C"
