// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or executed from the product path.
//
// extern "C" entry point over the UNMODIFIED reference template PriorityFloodEpsilon_Barnes2014<topo, float>
// (include/richdem/depressions/Barnes2014.hpp:336-420), built by oracle/epsilon_fill.py into
// oracle/_ref/libref_epsilon_fill.so (git-ignored).  The row-major host buffer (i = y*W + x) is wrapped unowned in
// richdem::Array2D, as ref_shim.cpp does, with the caller's NoData value set on it.
#include <richdem/common/Array2D.hpp>
#include <richdem/depressions/Barnes2014.hpp>

using namespace richdem;

extern "C" {

// topo: 0 D8, 1 D4.  dem is filled in place.
void ref_epsilon_fill_f32(int topo, float *dem, int w, int h, float nodata) {
  Array2D<float> a(dem, w, h);
  a.setNoData(nodata);
  if (topo) PriorityFloodEpsilon_Barnes2014<Topology::D4>(a);
  else PriorityFloodEpsilon_Barnes2014<Topology::D8>(a);
}

}  // extern "C"
