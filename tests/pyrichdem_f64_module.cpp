// tests/pyrichdem_f64_module.cpp -- the reference's OWN pybind11 module (`_richdem`) with the float64 specialisations of
// the drop-in layer switched on (RICHDEM_B200_F64).  Same translation unit as tests/pyrichdem_module.cpp otherwise: the
// header first, then the unmodified reference binding source.  richdem/__init__.py then runs FillDepressions,
// ResolveFlats and FlowAccumulation (D8, D4) on float64 rasters on the GPU as well.  Built by __graft_entry__.build()
// into tests/_bin/pyrichdem_f64/; it is also a package `richdem` with a module `_richdem`, so tests import it in a
// subprocess of its own.
#define RICHDEM_B200_F64
#include <richdem_b200.hpp>

#include <pywrapper.cpp>
