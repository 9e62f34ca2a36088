// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or executed from the product path.
//
// extern "C" entry points over the UNMODIFIED reference templates, each instantiated with T = double and T = float, so
// that the float64 path's argument -- reference<double>(Z) == kappa^-1(reference<float>(kappa(Z))) -- can be checked
// against the reference itself.  Built by oracle/f64.py into oracle/_ref/libref_f64.so (git-ignored) next to
// ref_shim.cpp's library.  Plain row-major host buffers (i = y*W + x) are wrapped unowned in richdem::Array2D, as
// ref_shim.cpp does.  topo: 0 D8, 1 D4.
#include <richdem/common/Array2D.hpp>
#include <richdem/common/Array3D.hpp>
#include <richdem/depressions/depressions.hpp>
#include <richdem/depressions/Zhou2016.hpp>
#include <richdem/depressions/Barnes2014.hpp>
#include <richdem/flats/flats.hpp>
#include <richdem/flowmet/d8_flowdirs.hpp>
#include <richdem/methods/flow_accumulation.hpp>

#include <cstdint>
#include <cstring>

using namespace richdem;

namespace {

// depressions/depressions.hpp:13-21 -> Zhou2016.hpp:125-191 (D8) / Barnes2014.hpp:230-304 (D4)
template <class T>
void fill(int topo, T *dem, int w, int h) {
  Array2D<T> a(dem, w, h);
  if (topo) FillDepressions<Topology::D4>(a);
  else FillDepressions<Topology::D8>(a);
}

// depressions/Barnes2014.hpp:593-676
template <class T>
void mask(int topo, T *dem, int w, int h, T nodata, uint8_t *out) {
  Array2D<T> a(dem, w, h);
  a.setNoData(nodata);
  Array2D<uint8_t> m;
  if (topo) pit_mask<Topology::D4>(a, m);
  else pit_mask<Topology::D8>(a, m);
  std::memcpy(out, m.data(), (size_t)w * h);
}

// depressions/Barnes2014.hpp:43-104
template <class T>
int has(int topo, T *dem, int w, int h) {
  Array2D<T> a(dem, w, h);
  return topo ? HasDepressions<Topology::D4>(a) : HasDepressions<Topology::D8>(a);
}

// flats/flats.hpp:21-28
template <class T>
void resolve(T *dem, int w, int h, T nodata) {
  Array2D<T> a(dem, w, h);
  a.setNoData(nodata);
  ResolveFlatsEpsilon(a);
}

// flats/Barnes2014.hpp:398-467: the increment mask ResolveFlatsEpsilon applies
template <class T>
void flat_mask(const T *dem, int w, int h, T nodata, int32_t *out) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata);
  Array2D<int32_t> m, l;
  GetFlatMask(a, m, l);
  std::memcpy(out, m.data(), sizeof(int32_t) * (size_t)w * h);
}

// flowmet/d8_flowdirs.hpp:96-123
template <class T>
void dirs(const T *dem, int w, int h, T nodata, uint8_t *out) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata);
  Array2D<uint8_t> d;
  d8_flow_directions(a, d);
  std::memcpy(out, d.data(), (size_t)w * h);
}

// methods/flow_accumulation.hpp:27 (FA_D8) / :28 (FA_D4); accum holds the weights on entry
template <class T>
void fa(int topo, const T *dem, int w, int h, T nodata, double *accum) {
  Array2D<T> a(const_cast<T *>(dem), w, h);
  a.setNoData(nodata);
  Array2D<double> acc(accum, w, h);
  if (topo) FA_D4(a, acc);
  else FA_D8(a, acc);
}

}  // namespace

#define INSTANTIATE(T, S)                                                                                                 \
  void ref_fill_##S(int topo, T *dem, int w, int h) { fill<T>(topo, dem, w, h); }                                       \
  void ref_pit_mask_##S(int topo, T *dem, int w, int h, T nd, uint8_t *out) { mask<T>(topo, dem, w, h, nd, out); }      \
  int ref_has_depressions_##S(int topo, T *dem, int w, int h) { return has<T>(topo, dem, w, h); }                       \
  void ref_resolve_flats_##S(T *dem, int w, int h, T nd) { resolve<T>(dem, w, h, nd); }                                 \
  void ref_flat_mask_##S(const T *dem, int w, int h, T nd, int32_t *out) { flat_mask<T>(dem, w, h, nd, out); }          \
  void ref_d8_flow_directions_##S(const T *dem, int w, int h, T nd, uint8_t *out) { dirs<T>(dem, w, h, nd, out); }      \
  void ref_fa_##S(int topo, const T *dem, int w, int h, T nd, double *accum) { fa<T>(topo, dem, w, h, nd, accum); }

extern "C" {
INSTANTIATE(double, f64)
INSTANTIATE(float, f32)
}  // extern "C"
