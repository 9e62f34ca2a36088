// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or executed from the product path.
//
// extern "C" entry points over the UNMODIFIED reference templates pit_mask<topo> and HasDepressions<topo>
// (include/richdem/depressions/Barnes2014.hpp:593-676, :43-104), built by oracle/depressions.py into
// oracle/_ref/libref_depressions.so (git-ignored) next to ref_shim.cpp's library.  Plain row-major host buffers
// (i = y*W + x) are wrapped unowned in richdem::Array2D, as ref_shim.cpp does.
#include <richdem/common/Array2D.hpp>
#include <richdem/depressions/Barnes2014.hpp>

#include <cstdint>
#include <cstring>

using namespace richdem;

extern "C" {

// topo: 0 D8, 1 D4.  mask receives the reference's output raster as it leaves pit_mask (resize, setNoData(3), writes).
void ref_pit_mask_f32(int topo, float *dem, int w, int h, float nodata, uint8_t *mask) {
  Array2D<float> a(dem, w, h);
  a.setNoData(nodata);
  Array2D<uint8_t> m;
  if (topo) pit_mask<Topology::D4>(a, m);
  else pit_mask<Topology::D8>(a, m);
  std::memcpy(mask, m.data(), (size_t)w * h);
}

int ref_has_depressions_f32(int topo, float *dem, int w, int h) {
  Array2D<float> a(dem, w, h);
  return topo ? HasDepressions<Topology::D4>(a) : HasDepressions<Topology::D8>(a);
}

}  // extern "C"
