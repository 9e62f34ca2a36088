// tests/pyrichdem_epsilon_module.cpp -- the reference's OWN pybind11 module (`_richdem`) with the epsilon-fill
// specialisations of the drop-in layer switched on (RICHDEM_B200_EPSILON).  Same translation unit as
// tests/pyrichdem_module.cpp otherwise: the header first, then the unmodified reference binding source.  The reference's
// richdem.FillDepressions(dem, epsilon=True) (rdPFepsilonD8 / rdPFepsilonD4) then runs on the GPU for float32 rasters.
// Built by __graft_entry__.build() into tests/_bin/pyrichdem_epsilon/; it is also a package `richdem` with a module
// `_richdem`, so tests import it in a subprocess of its own.
#define RICHDEM_B200_EPSILON
#include <richdem_b200.hpp>

#include <pywrapper.cpp>
