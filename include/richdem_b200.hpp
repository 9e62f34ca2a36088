// richdem_b200.hpp -- C++ drop-in layer over the C ABI (include/richdem_b200.h).
//
// Include this header INSTEAD OF (or before any use of) the RichDEM algorithm headers it covers,
// with RichDEM's include/ directory on the include path.  It pulls in
//
//     <richdem/depressions/depressions.hpp>   <richdem/flats/flats.hpp>
//     <richdem/methods/flow_accumulation.hpp> <richdem/flowmet/d8_flowdirs.hpp>
//     <richdem/methods/d8_methods.hpp>         <richdem/methods/terrain_attributes.hpp>
//
// itself and then declares the explicit specialisations, so they are seen before any implicit
// instantiation.  Without RichDEM on the include path only the duck-typed helpers in namespace
// richdem_b200 are available.
//
// It provides explicit specialisations of the reference's function templates for the dtypes of
// the hot path (elevations float, accumulation double, proportions float, direction grids uint8,
// areas int32), so existing callers -- `richdem::FillDepressions<Topology::D8>(dem)`,
// `richdem::FA_D8(dem, accum)`, pyrichdem's `&FA_D8<float,double>` bindings -- run on the H100
// without source changes; every other instantiation keeps using the reference's CPU templates.
// Errors surface as std::runtime_error, as in the reference (e.g. depressions.hpp:20,
// flow_accumulation_generic.hpp:42-43).  Link with -lrichdem_b200.
//
// Nothing here is copied from the reference: each specialisation forwards the raster's
// data()/width()/height()/noData() to the C ABI entry point that names the function it replaces.
#pragma once

#include <cstdint>
#include <stdexcept>
#include <string>

#include "richdem_b200.h"

namespace richdem_b200 {

inline void check(int rc) {
  if (rc != 0) throw std::runtime_error(std::string("richdem_b200: ") + rdb200_last_error());
}

// Duck-typed forwarding helpers: A2 is any row-major raster with data()/width()/height()/noData()
// (richdem::Array2D<T> qualifies: include/richdem/common/Array2D.hpp:89-1416).
template <class A2>
void fill_depressions_d8(A2 &dem) {
  check(rdb200_fill_depressions_d8_f32(dem.data(), dem.width(), dem.height()));
}
template <class A2>
void fill_depressions_d4(A2 &dem) {
  check(rdb200_fill_depressions_d4_f32(dem.data(), dem.width(), dem.height()));
}
// FillDepressions(epsilon=True): the order-free surface of rdb200_fill_depressions_epsilon_d8_f32 (never above the
// reference's PriorityFloodEpsilon_Barnes2014, not bit-identical to it); cells equal to dem.noData() are pinned
template <class A2>
void fill_depressions_epsilon_d8(A2 &dem) {
  check(rdb200_fill_depressions_epsilon_d8_f32(dem.data(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2>
void fill_depressions_epsilon_d4(A2 &dem) {
  check(rdb200_fill_depressions_epsilon_d4_f32(dem.data(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2>
void resolve_flats_epsilon(A2 &dem) {
  check(rdb200_resolve_flats_epsilon_f32(dem.data(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class D2>
void d8_flow_directions(const A2 &dem, D2 &dirs) {
  check(rdb200_d8_flow_directions_f32(dem.data(), dirs.data(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class D2, class I2>
void d8_flow_accum(const D2 &dirs, I2 &area) {
  check(rdb200_d8_flow_accum_u8_i32(dirs.data(), area.data(), dirs.width(), dirs.height()));
}
template <class A2, class P3>
void fm_d8(const A2 &dem, P3 &props) {
  check(rdb200_fm_d8_f32(dem.data(), props.getData(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class P3>
void fm_tarboton(const A2 &dem, P3 &props) {
  check(rdb200_fm_tarboton_f32(dem.data(), props.getData(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class P3>
void fm_d4(const A2 &dem, P3 &props) {
  check(rdb200_fm_d4_f32(dem.data(), props.getData(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class P3>
void fm_quinn(const A2 &dem, P3 &props) {
  check(rdb200_fm_quinn_f32(dem.data(), props.getData(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class P3>
void fm_holmgren(const A2 &dem, P3 &props, double xparam) {
  check(rdb200_fm_holmgren_f32(dem.data(), props.getData(), dem.width(), dem.height(), (float)dem.noData(), xparam));
}
template <class A2, class P3>
void fm_freeman(const A2 &dem, P3 &props, double xparam) {
  check(rdb200_fm_freeman_f32(dem.data(), props.getData(), dem.width(), dem.height(), (float)dem.noData(), xparam));
}
// attribute: RDB200_TA_*; `out` must already have the raster's size (TerrainProcessor resizes it, terrain_attributes.hpp:344)
template <class A2, class O2>
void terrain_attribute(int attribute, const A2 &dem, O2 &out, float zscale) {
  check(rdb200_terrain_attribute_f32(attribute, dem.data(), out.data(), dem.width(), dem.height(), (float)dem.noData(),
                                     (float)out.noData(), zscale, dem.getCellLengthX(), dem.getCellLengthY()));
}
template <class P3, class C2>
void flow_accumulation(P3 &props, C2 &accum) {
  check(rdb200_flow_accumulation_props_f64(props.getData(), accum.data(), accum.width(), accum.height()));
}
template <class A2, class C2>
void fa_d8(const A2 &dem, C2 &accum) {
  check(rdb200_fa_d8_f32_f64(dem.data(), accum.data(), dem.width(), dem.height(), (float)dem.noData(), 0));
}
template <class A2, class C2>
void fa_d4(const A2 &dem, C2 &accum) {
  check(rdb200_fa_d4_f32_f64(dem.data(), accum.data(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class C2>
void fa_quinn(const A2 &dem, C2 &accum) {
  check(rdb200_fa_quinn_f32_f64(dem.data(), accum.data(), dem.width(), dem.height(), (float)dem.noData()));
}
template <class A2, class C2>
void fa_holmgren(const A2 &dem, C2 &accum, double xparam) {
  check(rdb200_fa_holmgren_f32_f64(dem.data(), accum.data(), dem.width(), dem.height(), (float)dem.noData(), xparam));
}
template <class A2, class C2>
void fa_freeman(const A2 &dem, C2 &accum, double xparam) {
  check(rdb200_fa_freeman_f32_f64(dem.data(), accum.data(), dem.width(), dem.height(), (float)dem.noData(), xparam));
}
template <class A2, class C2>
void fa_tarboton(const A2 &dem, C2 &accum) {
  check(rdb200_fa_tarboton_f32_f64(dem.data(), accum.data(), dem.width(), dem.height(), (float)dem.noData(), 0));
}

}  // namespace richdem_b200

// ---- explicit specialisations of the reference templates (only when its headers are present) ----
#if defined(__has_include)
#if __has_include(<richdem/common/Array2D.hpp>)
#define RICHDEM_B200_HAVE_RICHDEM 1
#endif
#endif

#ifdef RICHDEM_B200_HAVE_RICHDEM
#include <richdem/depressions/depressions.hpp>
#include <richdem/flats/flat_resolution.hpp>
#include <richdem/flats/flats.hpp>
#include <richdem/flowmet/d8_flowdirs.hpp>
#include <richdem/methods/d8_methods.hpp>
#include <richdem/methods/flow_accumulation.hpp>
#include <richdem/methods/terrain_attributes.hpp>

namespace richdem {

#if 1
// depressions/depressions.hpp:13-21 (D8 -> PriorityFlood_Zhou2016, Zhou2016.hpp:125-191)
template <>
inline void FillDepressions<Topology::D8, float>(Array2D<float> &dem) {
  richdem_b200::fill_depressions_d8(dem);
}
// depressions/depressions.hpp:16-17 (D4 -> PriorityFlood_Barnes2014<D4>, Barnes2014.hpp:230-304; pyrichdem binds the
// latter as rdFillDepressionsD4, pywrapper.hpp:33)
template <>
inline void FillDepressions<Topology::D4, float>(Array2D<float> &dem) {
  richdem_b200::fill_depressions_d4(dem);
}
template <>
inline void PriorityFlood_Barnes2014<Topology::D4, float>(Array2D<float> &dem) {
  richdem_b200::fill_depressions_d4(dem);
}
// depressions/Zhou2016.hpp:125-191 -- what FillDepressions<D8> dispatches to, and what pyrichdem binds directly as
// rdFillDepressionsD8 (wrappers/pyrichdem/src/pywrapper.hpp:32)
template <>
inline void PriorityFlood_Zhou2016<float>(Array2D<float> &dem) {
  richdem_b200::fill_depressions_d8(dem);
}
#endif

#if 1
// depressions/Barnes2014.hpp:593-676: the output is resized as the reference does (every cell 0) and gets NoData 3; the
// call then writes every cell, and the ones the reference never writes come out 0 as they do there
template <>
inline void pit_mask<Topology::D8, float>(const Array2D<float> &elevations, Array2D<uint8_t> &mask) {
  mask.resize(elevations.width(), elevations.height());
  mask.setNoData(3);
  richdem_b200::check(rdb200_pit_mask_d8_f32(elevations.data(), mask.data(), elevations.width(), elevations.height(),
                                             elevations.noData()));
}
template <>
inline void pit_mask<Topology::D4, float>(const Array2D<float> &elevations, Array2D<uint8_t> &mask) {
  mask.resize(elevations.width(), elevations.height());
  mask.setNoData(3);
  richdem_b200::check(rdb200_pit_mask_d4_f32(elevations.data(), mask.data(), elevations.width(), elevations.height(),
                                             elevations.noData()));
}
// depressions/Barnes2014.hpp:43-104
template <>
inline bool HasDepressions<Topology::D8, float>(const Array2D<float> &elevations) {
  int32_t any = 0;
  richdem_b200::check(rdb200_has_depressions_d8_f32(elevations.data(), elevations.width(), elevations.height(), &any));
  return any != 0;
}
template <>
inline bool HasDepressions<Topology::D4, float>(const Array2D<float> &elevations) {
  int32_t any = 0;
  richdem_b200::check(rdb200_has_depressions_d4_f32(elevations.data(), elevations.width(), elevations.height(), &any));
  return any != 0;
}
#endif

#if 1
// flats/flats.hpp:21-28
template <>
inline void ResolveFlatsEpsilon<float>(Array2D<float> &elevations) {
  richdem_b200::resolve_flats_epsilon(elevations);
}
#endif

#if 1
// flowmet/d8_flowdirs.hpp:96-123 ; the output is (re)sized like the reference does (:107-109)
template <>
inline void d8_flow_directions<float, uint8_t>(const Array2D<float> &elevations, Array2D<uint8_t> &flowdirs) {
  flowdirs.resize(elevations);
  flowdirs.setNoData(FLOWDIR_NO_DATA);
  richdem_b200::d8_flow_directions(elevations, flowdirs);
}
#endif

#if 1
// flats/flat_resolution.hpp:588-607 (apps/rd_d8_flowdirs.cpp:18): D8 directions with the flats resolved through the
// increment mask (alter = false) or by altering the elevations (alter = true)
template <>
inline void barnes_flat_resolution_d8<float, uint8_t>(Array2D<float> &elevations, Array2D<uint8_t> &flowdirs, bool alter) {
  flowdirs.resize(elevations);
  flowdirs.setNoData(FLOWDIR_NO_DATA);
  richdem_b200::check(rdb200_d8_flow_directions_flats_f32(elevations.data(), flowdirs.data(), elevations.width(),
                                                          elevations.height(), (float)elevations.noData(), alter ? 1 : 0));
  flowdirs.templateCopy(elevations);
}
#endif

#if 1
// methods/d8_methods.hpp:47-139 ; direction NoData is FLOWDIR_NO_DATA (255)
template <>
inline void d8_flow_accum<uint8_t, int32_t>(const Array2D<uint8_t> &flowdirs, Array2D<int32_t> &area) {
  area.resize(flowdirs, 0);
  area.setNoData(-1);
  richdem_b200::d8_flow_accum(flowdirs, area);
}
#endif

#if 1
// flowmet/OCallaghan1984.hpp:81-84 and flowmet/Tarboton1997.hpp:14-17,146-149
template <>
inline void FM_D8<float>(const Array2D<float> &elevations, Array3D<float> &props) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_d8(elevations, props);
}
template <>
inline void FM_Tarboton<float>(const Array2D<float> &elevations, Array3D<float> &props) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_tarboton(elevations, props);
}
template <>
inline void FM_Dinfinity<float>(const Array2D<float> &elevations, Array3D<float> &props) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_tarboton(elevations, props);
}
// flowmet/OCallaghan1984.hpp:89-91, Quinn1991.hpp:12-16, Holmgren1994.hpp:13-83, Freeman1991.hpp:13-80
template <>
inline void FM_D4<float>(const Array2D<float> &elevations, Array3D<float> &props) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_d4(elevations, props);
}
template <>
inline void FM_Quinn<float>(const Array2D<float> &elevations, Array3D<float> &props) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_quinn(elevations, props);
}
template <>
inline void FM_Holmgren<float>(const Array2D<float> &elevations, Array3D<float> &props, const double xparam) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_holmgren(elevations, props, xparam);
}
template <>
inline void FM_Freeman<float>(const Array2D<float> &elevations, Array3D<float> &props, const double xparam) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::fm_freeman(elevations, props, xparam);
}
// methods/flow_accumulation_generic.hpp:33-100
template <>
inline void FlowAccumulation<double>(const Array3D<float> &props, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != props.width() || accum.height() != props.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::flow_accumulation(const_cast<Array3D<float> &>(props), accum);
}
// methods/flow_accumulation.hpp:27,16,17 -- fused on the device: no 36 B/cell temporary
template <>
inline void FA_D8<float, double>(const Array2D<float> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_d8(elevations, accum);
}
template <>
inline void FA_Tarboton<float, double>(const Array2D<float> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_tarboton(elevations, accum);
}
template <>
inline void FA_Dinfinity<float, double>(const Array2D<float> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_tarboton(elevations, accum);
}
// methods/flow_accumulation.hpp:28,19,18,20 -- the 36 B/cell proportions stay in HBM
template <>
inline void FA_D4<float, double>(const Array2D<float> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_d4(elevations, accum);
}
template <>
inline void FA_Quinn<float, double>(const Array2D<float> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_quinn(elevations, accum);
}
template <>
inline void FA_Holmgren<float, double>(const Array2D<float> &elevations, Array2D<double> &accum, double xparam) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_holmgren(elevations, accum, xparam);
}
template <>
inline void FA_Freeman<float, double>(const Array2D<float> &elevations, Array2D<double> &accum, double xparam) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::fa_freeman(elevations, accum, xparam);
}
// methods/terrain_attributes.hpp:370-538 (pyrichdem binds &TA_x<float>, pywrapper.hpp:46-53).  As in TerrainProcessor
// (:336-354) the output is resized to the elevations' shape and keeps its own NoData value.
#define RICHDEM_B200_TA(NAME, ID)                                                                              \
  template <>                                                                                                 \
  inline void NAME<float>(const Array2D<float> &elevations, Array2D<float> &output, float zscale) {           \
    output.resize(elevations);                                                                                \
    richdem_b200::terrain_attribute(ID, elevations, output, zscale);                                          \
  }
RICHDEM_B200_TA(TA_slope_riserun, RDB200_TA_SLOPE_RISERUN)
RICHDEM_B200_TA(TA_slope_percentage, RDB200_TA_SLOPE_PERCENTAGE)
RICHDEM_B200_TA(TA_slope_degrees, RDB200_TA_SLOPE_DEGREES)
RICHDEM_B200_TA(TA_slope_radians, RDB200_TA_SLOPE_RADIANS)
RICHDEM_B200_TA(TA_aspect, RDB200_TA_ASPECT)
RICHDEM_B200_TA(TA_curvature, RDB200_TA_CURVATURE)
RICHDEM_B200_TA(TA_planform_curvature, RDB200_TA_PLANFORM_CURVATURE)
RICHDEM_B200_TA(TA_profile_curvature, RDB200_TA_PROFILE_CURVATURE)
#undef RICHDEM_B200_TA
#endif

#ifdef RICHDEM_B200_F64
// float64 elevations (opt-in: `#define RICHDEM_B200_F64` before this include).  Without the macro Array2D<double> keeps
// the reference's CPU templates.  Each specialisation below forwards to the rdb200_*_f64 entry point of the same
// reference function; the results are the double templates' bit for bit, the fill's zero sign aside (DESIGN §0.1).
// depressions/depressions.hpp:13-21 -> Zhou2016.hpp:125-191 (D8) / Barnes2014.hpp:230-304 (D4)
template <>
inline void FillDepressions<Topology::D8, double>(Array2D<double> &dem) {
  richdem_b200::check(rdb200_fill_depressions_d8_f64(dem.data(), dem.width(), dem.height()));
}
template <>
inline void FillDepressions<Topology::D4, double>(Array2D<double> &dem) {
  richdem_b200::check(rdb200_fill_depressions_d4_f64(dem.data(), dem.width(), dem.height()));
}
template <>
inline void PriorityFlood_Zhou2016<double>(Array2D<double> &dem) {
  richdem_b200::check(rdb200_fill_depressions_d8_f64(dem.data(), dem.width(), dem.height()));
}
template <>
inline void PriorityFlood_Barnes2014<Topology::D4, double>(Array2D<double> &dem) {
  richdem_b200::check(rdb200_fill_depressions_d4_f64(dem.data(), dem.width(), dem.height()));
}
// depressions/Barnes2014.hpp:593-676 and :43-104
template <>
inline void pit_mask<Topology::D8, double>(const Array2D<double> &elevations, Array2D<uint8_t> &mask) {
  mask.resize(elevations.width(), elevations.height());
  mask.setNoData(3);
  richdem_b200::check(rdb200_pit_mask_d8_f64(elevations.data(), mask.data(), elevations.width(), elevations.height(),
                                             elevations.noData()));
}
template <>
inline void pit_mask<Topology::D4, double>(const Array2D<double> &elevations, Array2D<uint8_t> &mask) {
  mask.resize(elevations.width(), elevations.height());
  mask.setNoData(3);
  richdem_b200::check(rdb200_pit_mask_d4_f64(elevations.data(), mask.data(), elevations.width(), elevations.height(),
                                             elevations.noData()));
}
template <>
inline bool HasDepressions<Topology::D8, double>(const Array2D<double> &elevations) {
  int32_t any = 0;
  richdem_b200::check(rdb200_has_depressions_d8_f64(elevations.data(), elevations.width(), elevations.height(), &any));
  return any != 0;
}
template <>
inline bool HasDepressions<Topology::D4, double>(const Array2D<double> &elevations) {
  int32_t any = 0;
  richdem_b200::check(rdb200_has_depressions_d4_f64(elevations.data(), elevations.width(), elevations.height(), &any));
  return any != 0;
}
// flats/flats.hpp:21-28
template <>
inline void ResolveFlatsEpsilon<double>(Array2D<double> &elevations) {
  richdem_b200::check(rdb200_resolve_flats_epsilon_f64(elevations.data(), elevations.width(), elevations.height(),
                                                       elevations.noData()));
}
// flowmet/d8_flowdirs.hpp:96-123
template <>
inline void d8_flow_directions<double, uint8_t>(const Array2D<double> &elevations, Array2D<uint8_t> &flowdirs) {
  flowdirs.resize(elevations);
  flowdirs.setNoData(FLOWDIR_NO_DATA);
  richdem_b200::check(rdb200_d8_flow_directions_f64(elevations.data(), flowdirs.data(), elevations.width(),
                                                    elevations.height(), elevations.noData()));
}
// flats/flat_resolution.hpp:588-607; with alter the doubles take the reference's nextafterf steps
template <>
inline void barnes_flat_resolution_d8<double, uint8_t>(Array2D<double> &elevations, Array2D<uint8_t> &flowdirs, bool alter) {
  flowdirs.resize(elevations);
  flowdirs.setNoData(FLOWDIR_NO_DATA);
  richdem_b200::check(rdb200_d8_flow_directions_flats_f64(elevations.data(), flowdirs.data(), elevations.width(),
                                                          elevations.height(), elevations.noData(), alter ? 1 : 0));
  flowdirs.templateCopy(elevations);
}
// methods/flow_accumulation.hpp:27,28; accum holds the weights, as for float
template <>
inline void FA_D8<double, double>(const Array2D<double> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::check(rdb200_fa_d8_f64_f64(elevations.data(), accum.data(), elevations.width(), elevations.height(),
                                           elevations.noData(), 0));
}
template <>
inline void FA_D4<double, double>(const Array2D<double> &elevations, Array2D<double> &accum) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::check(rdb200_fa_d4_f64_f64(elevations.data(), accum.data(), elevations.width(), elevations.height(),
                                           elevations.noData()));
}
// flowmet/OCallaghan1984.hpp:81-91, Tarboton1997.hpp:14-149, Quinn1991.hpp:12-16, Holmgren1994.hpp:13-83,
// Freeman1991.hpp:13-80 with E = double: the double instantiations of the float kernels (no keys; DESIGN §0.2)
#define RICHDEM_B200_FM64(NAME, CALL)                                                                          \
  template <>                                                                                                 \
  inline void NAME<double>(const Array2D<double> &elevations, Array3D<float> &props) {                        \
    props.setNoData(NO_DATA_GEN);                                                                             \
    richdem_b200::check(CALL(elevations.data(), props.getData(), elevations.width(), elevations.height(),     \
                             elevations.noData()));                                                           \
  }
RICHDEM_B200_FM64(FM_D8, rdb200_fm_d8_f64)
RICHDEM_B200_FM64(FM_D4, rdb200_fm_d4_f64)
RICHDEM_B200_FM64(FM_Tarboton, rdb200_fm_tarboton_f64)
RICHDEM_B200_FM64(FM_Dinfinity, rdb200_fm_tarboton_f64)
RICHDEM_B200_FM64(FM_Quinn, rdb200_fm_quinn_f64)
#undef RICHDEM_B200_FM64
template <>
inline void FM_Holmgren<double>(const Array2D<double> &elevations, Array3D<float> &props, const double xparam) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::check(rdb200_fm_holmgren_f64(elevations.data(), props.getData(), elevations.width(), elevations.height(),
                                             elevations.noData(), xparam));
}
template <>
inline void FM_Freeman<double>(const Array2D<double> &elevations, Array3D<float> &props, const double xparam) {
  props.setNoData(NO_DATA_GEN);
  richdem_b200::check(rdb200_fm_freeman_f64(elevations.data(), props.getData(), elevations.width(), elevations.height(),
                                            elevations.noData(), xparam));
}
// methods/flow_accumulation.hpp:16-20 with E = double; accum holds the weights, as for float
#define RICHDEM_B200_FA64(NAME, CALL)                                                                          \
  template <>                                                                                                 \
  inline void NAME<double, double>(const Array2D<double> &elevations, Array2D<double> &accum) {               \
    accum.setNoData(ACCUM_NO_DATA);                                                                           \
    if (accum.width() != elevations.width() || accum.height() != elevations.height())                         \
      throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");         \
    CALL;                                                                                                     \
  }
RICHDEM_B200_FA64(FA_Tarboton, richdem_b200::check(rdb200_fa_tarboton_f64_f64(elevations.data(), accum.data(),
                  elevations.width(), elevations.height(), elevations.noData(), 0)))
RICHDEM_B200_FA64(FA_Dinfinity, richdem_b200::check(rdb200_fa_tarboton_f64_f64(elevations.data(), accum.data(),
                  elevations.width(), elevations.height(), elevations.noData(), 0)))
RICHDEM_B200_FA64(FA_Quinn, richdem_b200::check(rdb200_fa_quinn_f64_f64(elevations.data(), accum.data(),
                  elevations.width(), elevations.height(), elevations.noData())))
#undef RICHDEM_B200_FA64
template <>
inline void FA_Holmgren<double, double>(const Array2D<double> &elevations, Array2D<double> &accum, double xparam) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::check(rdb200_fa_holmgren_f64_f64(elevations.data(), accum.data(), elevations.width(), elevations.height(),
                                                 elevations.noData(), xparam));
}
template <>
inline void FA_Freeman<double, double>(const Array2D<double> &elevations, Array2D<double> &accum, double xparam) {
  accum.setNoData(ACCUM_NO_DATA);
  if (accum.width() != elevations.width() || accum.height() != elevations.height())
    throw std::runtime_error("Accumulation array must have same dimensions as proportions array!");
  richdem_b200::check(rdb200_fa_freeman_f64_f64(elevations.data(), accum.data(), elevations.width(), elevations.height(),
                                                elevations.noData(), xparam));
}
// methods/terrain_attributes.hpp:370-538 with T = double; as for float the output is resized and keeps its own NoData
#define RICHDEM_B200_TA64(NAME, ID)                                                                            \
  template <>                                                                                                 \
  inline void NAME<double>(const Array2D<double> &elevations, Array2D<float> &output, float zscale) {         \
    output.resize(elevations);                                                                                \
    richdem_b200::check(rdb200_terrain_attribute_f64(ID, elevations.data(), output.data(), elevations.width(), \
                                                     elevations.height(), elevations.noData(), output.noData(), \
                                                     zscale, elevations.getCellLengthX(),                     \
                                                     elevations.getCellLengthY()));                           \
  }
RICHDEM_B200_TA64(TA_slope_riserun, RDB200_TA_SLOPE_RISERUN)
RICHDEM_B200_TA64(TA_slope_percentage, RDB200_TA_SLOPE_PERCENTAGE)
RICHDEM_B200_TA64(TA_slope_degrees, RDB200_TA_SLOPE_DEGREES)
RICHDEM_B200_TA64(TA_slope_radians, RDB200_TA_SLOPE_RADIANS)
RICHDEM_B200_TA64(TA_aspect, RDB200_TA_ASPECT)
RICHDEM_B200_TA64(TA_curvature, RDB200_TA_CURVATURE)
RICHDEM_B200_TA64(TA_planform_curvature, RDB200_TA_PLANFORM_CURVATURE)
RICHDEM_B200_TA64(TA_profile_curvature, RDB200_TA_PROFILE_CURVATURE)
#undef RICHDEM_B200_TA64
#endif  // RICHDEM_B200_F64

#ifdef RICHDEM_B200_EPSILON
// the epsilon fill (opt-in: `#define RICHDEM_B200_EPSILON` before this include), depressions/Barnes2014.hpp:336-420, also
// reached through FillDepressionsEpsilon<topo> (depressions/depressions.hpp:23).  Opt-in because the GPU's surface is
// not the reference's bit for bit: it is the order-free one, never above the reference's and a few ulps below it in
// rare cells (include/richdem_b200.h, rdb200_fill_depressions_epsilon_d8_f32).  Without the macro these keep the
// reference's CPU template.
template <>
inline void PriorityFloodEpsilon_Barnes2014<Topology::D8, float>(Array2D<float> &elevations) {
  richdem_b200::fill_depressions_epsilon_d8(elevations);
}
template <>
inline void PriorityFloodEpsilon_Barnes2014<Topology::D4, float>(Array2D<float> &elevations) {
  richdem_b200::fill_depressions_epsilon_d4(elevations);
}
#endif  // RICHDEM_B200_EPSILON

}  // namespace richdem

#endif
