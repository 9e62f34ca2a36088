/*
 * richdem_b200.h -- C ABI of librichdem_b200.so (H100 / sm_90a).
 *
 * This is the drop-in boundary for RichDEM's depression-filling / flat-resolution /
 * flow-routing hot path.  Every entry point below replaces one reference function template
 * (cited as file:line relative to the RichDEM source tree) for the dtypes the Python API
 * uses on this path: elevations float32, accumulation float64, proportions float32 x 9,
 * direction grids uint8.  Buffers are plain row-major rasters, i = y*width + x
 * (reference include/richdem/common/Array2D.hpp:592-595) -- i.e. exactly what
 * richdem::Array2D<T>::data() or a C-contiguous numpy array hands over.
 *
 * Conventions
 *   - All functions return 0 on success, non-zero on failure; rdb200_last_error() then
 *     returns a static, thread-local, human-readable message (CUDA errors included).
 *     There is NO CPU fallback: without a usable sm_90 device every compute call fails.
 *   - "Host" entry points take host pointers, copy to the device, compute, and copy the
 *     result back before returning; nothing is retained after return (same ownership rules
 *     as the reference: caller-owned, mutated in place).
 *   - "dev" entry points take device pointers on the current device and run on the
 *     library's stream; they let callers chain stages without leaving HBM.
 *   - Calls are synchronous from the caller's point of view and must be made from one
 *     thread at a time (the reference holds the GIL for the whole call as well).
 *   - D8 neighbour numbering is the reference's (include/richdem/common/constants.hpp:44-45):
 *         2 3 4
 *         1 0 5
 *         8 7 6
 */
#ifndef RICHDEM_B200_H_
#define RICHDEM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RDB200_VERSION 100 /* 0.1.0 */

#if defined(__GNUC__)
#define RDB200_API __attribute__((visibility("default")))
#else
#define RDB200_API
#endif

/* ---- library lifetime ------------------------------------------------------------- */

/* Selects CUDA device `device` (>=0) for this process, creates the stream and workspace.
 * Idempotent for the same device.  Compute calls lazily do rdb200_init(current device). */
RDB200_API int rdb200_init(int device);
/* Releases the workspace, stream and cached descriptors. */
RDB200_API void rdb200_shutdown(void);
RDB200_API const char *rdb200_last_error(void);
RDB200_API int rdb200_version(void);

/* Run all subsequent work on the caller's CUDA stream (a cudaStream_t; NULL restores the
 * library's own stream).  Lets a caller bracket calls with its own CUDA events. */
RDB200_API int rdb200_set_stream(void *cuda_stream);

/* Counters of the most recent call (for benchmarks / roofline accounting). */
typedef struct rdb200_stats {
  int64_t cells;             /* width*height of the raster processed                       */
  int64_t kernel_launches;   /* CUDA kernels launched by the call                          */
  int64_t fill_rounds;       /* fill: global sweep rounds (one persistent launch each)     */
  int64_t fill_tile_visits;  /* fill: tiles loaded+relaxed, summed over rounds             */
  int64_t fill_tile_cells;   /* fill: cells per tile (visits*tile_cells = cells swept)     */
  int64_t fill_tile_iters;   /* fill: in-shared-memory relaxation passes, summed           */
  int64_t accum_rounds;      /* accumulation: frontier rounds                              */
  int64_t flat_bfs_levels;   /* flats: BFS levels (away + towards)                         */
  int64_t flat_cells_raised; /* flats: cells whose elevation changed                       */
  double ms_total;           /* device time of the whole call (CUDA events)                */
  double ms_main_kernel;     /* device time summed over launches of the dominant kernel    */
  double ms_h2d, ms_d2h;     /* host entry points only                                     */
} rdb200_stats;
RDB200_API int rdb200_get_stats(rdb200_stats *out);

/* Tunables (algorithm switches and debug aids; see struct Params in csrc/common.cuh for the list and the
 * defaults).  "reset_defaults" restores every one of them; "trim_workspace" returns the cached device scratch (kept
 * between calls so that repeated calls do not pay cudaMalloc) to the driver.  They are process-wide and survive
 * rdb200_shutdown / re-init.  The library is single-threaded by contract (see above). */
RDB200_API int rdb200_set_param(const char *name, int64_t value);

/* ---- host entry points: the reference functions they replace ----------------------- */

/* richdem::FillDepressions<Topology::D8>(Array2D<float>&)
 *   include/richdem/depressions/depressions.hpp:13-21 -> PriorityFlood_Zhou2016,
 *   include/richdem/depressions/Zhou2016.hpp:125-191 (pyrichdem: rdFillDepressionsD8,
 *   wrappers/pyrichdem/src/pywrapper.hpp:32).  In place.  NoData is not special (as in the
 *   reference).  Result is bit-identical to the reference. */
RDB200_API int rdb200_fill_depressions_d8_f32(float *dem, int32_t width, int32_t height);

/* richdem::FillDepressions<Topology::D4>(Array2D<float>&)
 *   include/richdem/depressions/depressions.hpp:16-17 -> PriorityFlood_Barnes2014<Topology::D4>,
 *   include/richdem/depressions/Barnes2014.hpp:230-304 (pyrichdem: rdFillDepressionsD4, pywrapper.hpp:33).
 *   Same engine with the 4-neighbour stencil; bit-identical. */
RDB200_API int rdb200_fill_depressions_d4_f32(float *dem, int32_t width, int32_t height);

/* richdem::PriorityFloodEpsilon_Barnes2014<Topology::D8 / D4>(Array2D<float>&) -- FillDepressions(epsilon=True)
 *   include/richdem/depressions/Barnes2014.hpp:336-420 (pyrichdem: rdPFepsilonD8 / rdPFepsilonD4, pywrapper.hpp:34-35).
 *   In place.  With up(x) = nextafterf(x, +inf), the result W is the unique solution of
 *       W(c) = Z(c)                                               on the raster's border and where Z(c) == nodata,
 *       W(c) = max(Z(c), min over the neighbours n of up(W(n)))   elsewhere (8 neighbours for D8, 4 for D4).
 *   NoData cells are never raised and offer up(nodata) to their neighbours; a NaN nodata pins nothing; NaN elevations are
 *   not supported.  The reference's result depends on the order in which its priority queue breaks ties, so this is NOT
 *   bit-identical to it: W is order-free and never above the reference's surface anywhere (on NoData-free rasters a few
 *   ulps below it in under 1 % of cells; next to NoData cells inside depressions it can be lower by more).  Without NoData
 *   every interior cell of W has a strictly lower neighbour, so W has no depressions and no flats.
 *   Stats: fill_rounds, fill_tile_visits. */
RDB200_API int rdb200_fill_depressions_epsilon_d8_f32(float *dem, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_fill_depressions_epsilon_d4_f32(float *dem, int32_t width, int32_t height, float nodata);

/* richdem::pit_mask<Topology::D8 / D4>(const Array2D<float>&, Array2D<uint8_t>&)
 *   include/richdem/depressions/Barnes2014.hpp:593-676 (app rd_depressions_mask).  mask (width x height, written in
 *   full): 3 where dem == nodata, 1 where the cell lies below the depression-filled surface of dem (the fill above,
 *   NoData an ordinary value), 0 elsewhere -- edge cells and cells at their filled level included, which the reference
 *   leaves as its resize() set them.  dem is not modified.  Bit-identical. */
RDB200_API int rdb200_pit_mask_d8_f32(const float *dem, uint8_t *mask, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_pit_mask_d4_f32(const float *dem, uint8_t *mask, int32_t width, int32_t height, float nodata);

/* richdem::HasDepressions<Topology::D8 / D4>(const Array2D<float>&)
 *   include/richdem/depressions/Barnes2014.hpp:43-104 (app rd_depressions_has).  *out = 1 if some cell lies below the
 *   filled surface, else 0 (NoData is not special, as in the reference).  A stencil pass that finds a strict pit answers
 *   without filling. */
RDB200_API int rdb200_has_depressions_d8_f32(const float *dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_has_depressions_d4_f32(const float *dem, int32_t width, int32_t height, int32_t *out);

/* richdem::ResolveFlatsEpsilon(Array2D<float>&)
 *   include/richdem/flats/flats.hpp:21-28 (GetFlatMask + ResolveFlatsEpsilon_Barnes2014,
 *   include/richdem/flats/Barnes2014.hpp:398-467, 496-550); pyrichdem rdResolveFlatsEpsilon
 *   (pywrapper.hpp:37).  In place; bit-identical. */
RDB200_API int rdb200_resolve_flats_epsilon_f32(float *dem, int32_t width, int32_t height, float nodata);

/* richdem::GetFlatMask (include/richdem/flats/Barnes2014.hpp:398-467): the int32 increment
 * mask and a flat id per cell (0 = not in a drainable flat; ids are arbitrary but equal
 * within one flat -- the reference's ids are traversal-order dependent too). */
RDB200_API int rdb200_get_flat_mask_f32(const float *dem, int32_t *flat_mask, int32_t *labels, int32_t width,
                             int32_t height, float nodata);

/* richdem::d8_flow_directions(const Array2D<float>&, Array2D<uint8_t>&)
 *   include/richdem/flowmet/d8_flowdirs.hpp:96-123 (+ d8_FlowDir :32-74).  Codes 0..8,
 *   255 = NoData (include/richdem/common/constants.hpp:76).  Bit-identical. */
RDB200_API int rdb200_d8_flow_directions_f32(const float *dem, uint8_t *flowdirs, int32_t width,
                                  int32_t height, float nodata);

/* richdem::barnes_flat_resolution_d8(Array2D<float>&, Array2D<uint8_t>&, bool alter)
 *   include/richdem/flats/flat_resolution.hpp:588-607 (apps/rd_d8_flowdirs.cpp:18 ships it with alter = false):
 *   d8_flow_directions, then the increment mask / labels of the flats the DIRECTION grid shows (resolve_flats_barnes,
 *   :448-515) and either directions inside the flats from the mask (d8_flow_flats, :97-116; dem untouched) or, with
 *   alter != 0, the elevations altered by the mask (d8_flats_alter_dem, :540-586; dem updated in place) and the
 *   directions recomputed.  Bit-identical. */
RDB200_API int rdb200_d8_flow_directions_flats_f32(float *dem, uint8_t *flowdirs, int32_t width, int32_t height,
                                                   float nodata, int32_t alter);

/* richdem::d8_flow_accum(const Array2D<uint8_t>&, Array2D<int32_t>&)
 *   include/richdem/methods/d8_methods.hpp:47-139.  NoData direction = 255 -> area -1. */
RDB200_API int rdb200_d8_flow_accum_u8_i32(const uint8_t *flowdirs, int32_t *area, int32_t width,
                                int32_t height);

/* richdem::FM_D8 / FM_OCallaghan<D8>(const Array2D<float>&, Array3D<float>&)
 *   include/richdem/flowmet/OCallaghan1984.hpp:13-77,81-84.  props9 is [y][x][9] float
 *   (include/richdem/common/Array3D.hpp:203-206).  Bit-identical. */
RDB200_API int rdb200_fm_d8_f32(const float *dem, float *props9, int32_t width, int32_t height, float nodata);

/* richdem::FM_Tarboton / FM_Dinfinity  include/richdem/flowmet/Tarboton1997.hpp:14-149.
 * Facet choice identical; proportions within 1 float ulp (device atan2 vs libm). */
RDB200_API int rdb200_fm_tarboton_f32(const float *dem, float *props9, int32_t width, int32_t height,
                           float nodata);

/* richdem::FM_D4 = FM_OCallaghan<Topology::D4>  include/richdem/flowmet/OCallaghan1984.hpp:13-77,89-91.
 * As in the reference, the single receiver's proportion 1 is stored in slot n of the D4 numbering
 * (1 = W, 2 = N, 3 = E, 4 = S; common/constants.hpp:53-54).  Bit-identical. */
RDB200_API int rdb200_fm_d4_f32(const float *dem, float *props9, int32_t width, int32_t height, float nodata);
/* richdem::FM_Quinn  include/richdem/flowmet/Quinn1991.hpp:12-16 (= FM_Holmgren with exponent 1); bit-identical.
 * richdem::FM_Holmgren(elevations, props, xparam)  include/richdem/flowmet/Holmgren1994.hpp:13-83.
 * richdem::FM_Freeman(elevations, props, xparam)   include/richdem/flowmet/Freeman1991.hpp:13-80.
 * Same mixed float/double arithmetic as the reference; with an exponent other than 1 the device pow differs from
 * libm by <= 2 ulp (double), i.e. proportions within 1 float ulp. */
RDB200_API int rdb200_fm_quinn_f32(const float *dem, float *props9, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_fm_holmgren_f32(const float *dem, float *props9, int32_t width, int32_t height, float nodata,
                                      double xparam);
RDB200_API int rdb200_fm_freeman_f32(const float *dem, float *props9, int32_t width, int32_t height, float nodata,
                                     double xparam);

/* richdem::FA_D4 / FA_Quinn / FA_Holmgren / FA_Freeman(const Array2D<float>&, Array2D<double>&[, xparam])
 *   include/richdem/methods/flow_accumulation.hpp:28,19,18,20 (pyrichdem: pywrapper.hpp:65,58,57,59).
 *   FM_x into a device-resident proportions array (36 B/cell, never leaves HBM) + the generic accumulation below.
 *   accum_inout arrives holding the weights. */
RDB200_API int rdb200_fa_d4_f32_f64(const float *dem, double *accum_inout, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_fa_quinn_f32_f64(const float *dem, double *accum_inout, int32_t width, int32_t height,
                                       float nodata);
RDB200_API int rdb200_fa_holmgren_f32_f64(const float *dem, double *accum_inout, int32_t width, int32_t height,
                                          float nodata, double xparam);
RDB200_API int rdb200_fa_freeman_f32_f64(const float *dem, double *accum_inout, int32_t width, int32_t height,
                                         float nodata, double xparam);

/* float64 elevations: the same reference functions with T = double, bit for bit (the fill's zero sign aside, as for
 * float).  Each runs the float engine on kappa(dem), a strictly increasing map of the raster's doubles to float keys
 * (the cast to float when every value is a float already, else dense ranks by a radix sort), and maps the result back;
 * DESIGN §0 gives the argument.  NaN elevations carry no promise beyond what the float entry points make.
 *   fill_depressions_*_f64   depressions/depressions.hpp:13-21 -> Zhou2016.hpp:125-191 (D8), Barnes2014.hpp:230-304 (D4);
 *                            cells the fill does not raise keep their own bits
 *   pit_mask_*_f64           depressions/Barnes2014.hpp:593-676 (3 NoData, 1 depression, 0 otherwise)
 *   has_depressions_*_f64    depressions/Barnes2014.hpp:43-104
 *   resolve_flats_epsilon_f64  flats/flats.hpp:21-28: GetFlatMask (Barnes2014.hpp:398-467) of the keys, then k double
 *                            ulps (nextafter towards +inf) on the original values (:496-550)
 *   d8_flow_directions_f64   flowmet/d8_flowdirs.hpp:32-123, compared as doubles
 *   fa_d8_f64_f64            methods/flow_accumulation.hpp:27 (FA_D8<double, double>); accum_is_ones as rdb200_fa_d8_f32_f64
 *   fa_d4_f64_f64            methods/flow_accumulation.hpp:28 (FA_D4<double, double>); accum_inout holds the weights
 * Peak device memory per cell (beyond the float engine's own scratch): see INTEGRATION.md. */
RDB200_API int rdb200_fill_depressions_d8_f64(double *dem, int32_t width, int32_t height);
RDB200_API int rdb200_fill_depressions_d4_f64(double *dem, int32_t width, int32_t height);
RDB200_API int rdb200_pit_mask_d8_f64(const double *dem, uint8_t *mask, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_pit_mask_d4_f64(const double *dem, uint8_t *mask, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_has_depressions_d8_f64(const double *dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_has_depressions_d4_f64(const double *dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_resolve_flats_epsilon_f64(double *dem, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_d8_flow_directions_f64(const double *dem, uint8_t *flowdirs, int32_t width, int32_t height,
                                             double nodata);
RDB200_API int rdb200_fa_d8_f64_f64(const double *dem, double *accum_inout, int32_t width, int32_t height, double nodata,
                                    int32_t accum_is_ones);
/* GetFlatMask<double> (flats/Barnes2014.hpp:398-467) as rdb200_get_flat_mask_f32: the mask bit for bit, the labels equal
 * to the reference's as a partition of the cells. */
RDB200_API int rdb200_get_flat_mask_f64(const double *dem, int32_t *flat_mask, int32_t *labels, int32_t width, int32_t height,
                                        double nodata);
/* barnes_flat_resolution_d8<double, uint8_t> (flats/flat_resolution.hpp:588-607) as rdb200_d8_flow_directions_flats_f32:
 * directions of the doubles, the flats of that direction grid resolved on the keys, then d8_flow_flats, or with alter != 0
 * d8_flats_alter_dem and the directions of the altered doubles.  The reference alters a double with nextafterf
 * (:565-568): a labelled interior cell with increment count m > 0 becomes the double of m float-ulp steps towards +inf
 * from the double rounded to the nearest float (so +inf from any double above FLT_MAX), m = 0 leaves it as it is.  The
 * directions and the altered dem are bit-identical. */
RDB200_API int rdb200_d8_flow_directions_flats_f64(double *dem, uint8_t *flowdirs, int32_t width, int32_t height, double nodata,
                                                   int32_t alter);
RDB200_API int rdb200_fa_d4_f64_f64(const double *dem, double *accum_inout, int32_t width, int32_t height, double nodata);
/* DIAGNOSTIC, not part of the stable interface: the key encoding is an implementation detail of the entry points above
 * and may change between versions (tests use these two to check it).  kappa itself: keys (width x height floats), *nodata_key = kappa(nodata) (the key of a cell equal to nodata; else the
 * image of +-inf / +-DBL_MAX when nodata is one; else NaN), *ranked = 0 for the cast to float, 1 for dense ranks
 * (__uint_as_float(0x00800000 + rank); +-inf, +-DBL_MAX and NaN keep the images +-inf, +-FLT_MAX and NaN).
 * nodata_key and ranked may be null. */
RDB200_API int rdb200_f64_order_keys(const double *dem, float *keys, int32_t width, int32_t height, double nodata,
                                     float *nodata_key, int32_t *ranked);

/* richdem::TA_slope_riserun / TA_slope_percentage / TA_slope_degrees / TA_slope_radians / TA_aspect / TA_curvature /
 * TA_planform_curvature / TA_profile_curvature(const Array2D<float>&, Array2D<float>&, float zscale)
 *   include/richdem/methods/terrain_attributes.hpp:370-538 over TerrainProcessor (:336-354) and the per-cell
 *   formulas (:154-322); pyrichdem TerrainAttribute (wrappers/pyrichdem/richdem/__init__.py:735-794).
 *   NoData cells of the input (== nodata_in) become nodata_out (the output raster's own NoData, -9999 from
 *   pyrichdem); neighbours that are NoData or outside the raster take the centre's value.  cell_x / cell_y are
 *   |geotransform[1]| and |geotransform[5]| (Array2D.hpp:1387-1399).  Double arithmetic in the reference's order
 *   without fused multiply-adds: slopes (rise/run, percentage) and the three curvatures are bit-identical to a
 *   stock x86-64 build of the reference; the attributes through atan / atan2 (degrees, radians, aspect) are within
 *   1 float ulp (device libm differs from glibc by <= 2 ulp of the double). */
enum {
  RDB200_TA_SLOPE_RISERUN = 0,
  RDB200_TA_SLOPE_PERCENTAGE = 1,
  RDB200_TA_SLOPE_DEGREES = 2,
  RDB200_TA_SLOPE_RADIANS = 3,
  RDB200_TA_ASPECT = 4,
  RDB200_TA_CURVATURE = 5,
  RDB200_TA_PLANFORM_CURVATURE = 6,
  RDB200_TA_PROFILE_CURVATURE = 7
};
RDB200_API int rdb200_terrain_attribute_f32(int32_t attribute, const float *dem, float *out, int32_t width, int32_t height,
                                            float nodata_in, float nodata_out, float zscale, double cell_x, double cell_y);

/* richdem::FlowAccumulation(const Array3D<float>&, Array2D<double>&)
 *   include/richdem/methods/flow_accumulation_generic.hpp:33-100 (pyrichdem
 *   "FlowAccumulation", wrappers/pyrichdem/src/pywrapper.cpp:50).  accum arrives holding the
 *   per-cell weights and leaves holding the accumulation; NoData cells (props slot 0 == -2)
 *   become -1.  Flow out of raster-edge cells is ignored (the reference FM_* never emit it). */
RDB200_API int rdb200_flow_accumulation_props_f64(const float *props9, double *accum_inout, int32_t width,
                                       int32_t height);

/* richdem::FA_D8 / FA_Tarboton(=FA_Dinfinity)(const Array2D<float>&, Array2D<double>&)
 *   include/richdem/methods/flow_accumulation.hpp:27,16,17 (pywrapper.hpp:64,55,56).
 *   Fused: the 36 B/cell proportions array is never materialised.  accum_inout as above;
 *   pass accum_is_ones != 0 to promise that every weight is 1.0 (skips the upload). */
RDB200_API int rdb200_fa_d8_f32_f64(const float *dem, double *accum_inout, int32_t width, int32_t height,
                         float nodata, int32_t accum_is_ones);
RDB200_API int rdb200_fa_tarboton_f32_f64(const float *dem, double *accum_inout, int32_t width,
                               int32_t height, float nodata, int32_t accum_is_ones);

/* float64 elevations for the stages that do arithmetic on them: the reference's templates with E / T = double, run by
 * the double instantiations of the float kernels (no keys).  Arguments, checks and tolerances as the float entry points
 * above; NoData is a double.  s1, s2, e0 - e2 (D-infinity) and e - ne (Holmgren, Freeman) are rounded double
 * differences, as in the reference; DESIGN §0.2 gives the D-infinity fallback for differences outside [2^-500, 2^500].
 *   fm_*_f64                 flowmet/OCallaghan1984.hpp, Tarboton1997.hpp, Quinn1991.hpp, Holmgren1994.hpp, Freeman1991.hpp
 *   fa_tarboton_f64_f64      methods/flow_accumulation.hpp:16 (FA_Tarboton<double, double>): the fused engine of
 *                            rdb200_fa_tarboton_f32_f64 after a code pass on the doubles; accum_is_ones as there
 *   fa_{quinn,holmgren,freeman}_f64_f64  methods/flow_accumulation.hpp:18-20: FM_x on the doubles + the generic
 *                            accumulation; accum_inout holds the weights
 *   terrain_attribute_f64    methods/terrain_attributes.hpp:370-538 with T = double; float output */
RDB200_API int rdb200_fm_d8_f64(const double *dem, float *props9, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_fm_tarboton_f64(const double *dem, float *props9, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_fm_d4_f64(const double *dem, float *props9, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_fm_quinn_f64(const double *dem, float *props9, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_fm_holmgren_f64(const double *dem, float *props9, int32_t width, int32_t height, double nodata,
                                      double xparam);
RDB200_API int rdb200_fm_freeman_f64(const double *dem, float *props9, int32_t width, int32_t height, double nodata,
                                     double xparam);
RDB200_API int rdb200_fa_tarboton_f64_f64(const double *dem, double *accum_inout, int32_t width, int32_t height,
                                          double nodata, int32_t accum_is_ones);
RDB200_API int rdb200_fa_quinn_f64_f64(const double *dem, double *accum_inout, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_fa_holmgren_f64_f64(const double *dem, double *accum_inout, int32_t width, int32_t height,
                                          double nodata, double xparam);
RDB200_API int rdb200_fa_freeman_f64_f64(const double *dem, double *accum_inout, int32_t width, int32_t height,
                                         double nodata, double xparam);
RDB200_API int rdb200_terrain_attribute_f64(int32_t attribute, const double *dem, float *out, int32_t width, int32_t height,
                                            double nodata_in, float nodata_out, float zscale, double cell_x, double cell_y);

/* ---- device entry points (pointers into HBM of the current device) ----------------- */

/* Depression filling in place.  While the call runs, d_dem holds intermediate water levels (when width is a multiple
 * of 4 and d_dem is 16-byte aligned, the fill relaxes its water surface in the raster itself and keeps the elevations
 * in a scratch copy), so nothing else may read or write it meanwhile.  If the call returns an error, the contents of
 * d_dem are unspecified. */
RDB200_API int rdb200_dev_fill_depressions_d8_f32(float *d_dem, int32_t width, int32_t height);
RDB200_API int rdb200_dev_fill_depressions_d4_f32(float *d_dem, int32_t width, int32_t height);
/* The epsilon fill of rdb200_fill_depressions_epsilon_d8_f32 / _d4_f32 in place, with the same contract (never above the
 * reference's surface, not bit-identical to it) and the same rule for d_dem while the call runs. */
RDB200_API int rdb200_dev_fill_depressions_epsilon_d8_f32(float *d_dem, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_dev_fill_depressions_epsilon_d4_f32(float *d_dem, int32_t width, int32_t height, float nodata);
/* pit_mask / HasDepressions on device pointers (d_dem is not modified; *out is a host int) */
RDB200_API int rdb200_dev_pit_mask_d8_f32(const float *d_dem, uint8_t *d_mask, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_dev_pit_mask_d4_f32(const float *d_dem, uint8_t *d_mask, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_dev_has_depressions_d8_f32(const float *d_dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_dev_has_depressions_d4_f32(const float *d_dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_dev_resolve_flats_epsilon_f32(float *d_dem, int32_t width, int32_t height, float nodata);
RDB200_API int rdb200_dev_d8_flow_directions_f32(const float *d_dem, uint8_t *d_flowdirs, int32_t width,
                                      int32_t height, float nodata);
RDB200_API int rdb200_dev_d8_flow_directions_flats_f32(float *d_dem, uint8_t *d_flowdirs, int32_t width, int32_t height,
                                                       float nodata, int32_t alter);
RDB200_API int rdb200_dev_d8_flow_accum_u8_i32(const uint8_t *d_flowdirs, int32_t *d_area, int32_t width,
                                    int32_t height);
RDB200_API int rdb200_dev_fm_d8_f32(const float *d_dem, float *d_props9, int32_t width, int32_t height,
                         float nodata);
RDB200_API int rdb200_dev_fm_tarboton_f32(const float *d_dem, float *d_props9, int32_t width, int32_t height,
                               float nodata);
/* method: 0 FM_D8, 1 FM_Tarboton, 2 FM_D4, 3 FM_Holmgren (xparam; FM_Quinn = 1.0), 4 FM_Freeman (xparam) */
RDB200_API int rdb200_dev_fm_method_f32(int32_t method, const float *d_dem, float *d_props9, int32_t width,
                                        int32_t height, float nodata, double xparam);
RDB200_API int rdb200_dev_fa_method_f32_f64(int32_t method, const float *d_dem, double *d_accum_inout, int32_t width,
                                            int32_t height, float nodata, double xparam);
RDB200_API int rdb200_dev_terrain_attribute_f32(int32_t attribute, const float *d_dem, float *d_out, int32_t width,
                                                int32_t height, float nodata_in, float nodata_out, float zscale,
                                                double cell_x, double cell_y);
RDB200_API int rdb200_dev_flow_accumulation_props_f64(const float *d_props9, double *d_accum_inout,
                                           int32_t width, int32_t height);
RDB200_API int rdb200_dev_fa_d8_f32_f64(const float *d_dem, double *d_accum_inout, int32_t width,
                             int32_t height, float nodata, int32_t accum_is_ones);
RDB200_API int rdb200_dev_fa_tarboton_f32_f64(const float *d_dem, double *d_accum_inout, int32_t width,
                                   int32_t height, float nodata, int32_t accum_is_ones);
/* the float64 entry points on device pointers (d_dem of pit_mask / has_depressions / d8 / fa is not modified) */
RDB200_API int rdb200_dev_fill_depressions_d8_f64(double *d_dem, int32_t width, int32_t height);
RDB200_API int rdb200_dev_fill_depressions_d4_f64(double *d_dem, int32_t width, int32_t height);
RDB200_API int rdb200_dev_pit_mask_d8_f64(const double *d_dem, uint8_t *d_mask, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_dev_pit_mask_d4_f64(const double *d_dem, uint8_t *d_mask, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_dev_has_depressions_d8_f64(const double *d_dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_dev_has_depressions_d4_f64(const double *d_dem, int32_t width, int32_t height, int32_t *out);
RDB200_API int rdb200_dev_resolve_flats_epsilon_f64(double *d_dem, int32_t width, int32_t height, double nodata);
RDB200_API int rdb200_dev_d8_flow_directions_f64(const double *d_dem, uint8_t *d_flowdirs, int32_t width, int32_t height,
                                                 double nodata);
RDB200_API int rdb200_dev_d8_flow_directions_flats_f64(double *d_dem, uint8_t *d_flowdirs, int32_t width, int32_t height,
                                                       double nodata, int32_t alter);
RDB200_API int rdb200_dev_fa_d8_f64_f64(const double *d_dem, double *d_accum_inout, int32_t width, int32_t height,
                                        double nodata, int32_t accum_is_ones);
RDB200_API int rdb200_dev_fa_d4_f64_f64(const double *d_dem, double *d_accum_inout, int32_t width, int32_t height,
                                        double nodata);
/* method numbered as in rdb200_dev_fm_method_f32; rdb200_dev_fa_method_f64_f64 runs methods 0 and 2 as
 * rdb200_dev_fa_d8_f64_f64 (given weights) and rdb200_dev_fa_d4_f64_f64, the others through proportions */
RDB200_API int rdb200_dev_fm_method_f64(int32_t method, const double *d_dem, float *d_props9, int32_t width, int32_t height,
                                        double nodata, double xparam);
RDB200_API int rdb200_dev_fa_method_f64_f64(int32_t method, const double *d_dem, double *d_accum_inout, int32_t width,
                                            int32_t height, double nodata, double xparam);
RDB200_API int rdb200_dev_fa_tarboton_f64_f64(const double *d_dem, double *d_accum_inout, int32_t width, int32_t height,
                                              double nodata, int32_t accum_is_ones);
RDB200_API int rdb200_dev_terrain_attribute_f64(int32_t attribute, const double *d_dem, float *d_out, int32_t width,
                                                int32_t height, double nodata_in, float nodata_out, float zscale,
                                                double cell_x, double cell_y);
/* diagnostic, as rdb200_f64_order_keys */
RDB200_API int rdb200_dev_f64_order_keys(const double *d_dem, float *d_keys, int32_t width, int32_t height, double nodata,
                                         float *nodata_key, int32_t *ranked);

/* Seeded synthetic fractal DEM (value-noise fBm, float32, no NaN / NoData) generated in HBM;
 * benchmark input only (the reference's generate_perlin_terrain is single-octave/double:
 * src/terrain_generation/terrain_generation.cpp:11-24).  Cell (x,y) of the band is global
 * cell (x, y0+y) of a raster `full_height` rows tall, so row bands of one raster agree. */
RDB200_API int rdb200_dev_generate_fbm_f32(float *d_dem, int32_t width, int32_t height, int32_t y0,
                                uint32_t seed, int32_t octaves, float quantum);

/* ---- multi-GPU: one process per GPU, the raster cut into row bands ----------------------------------------------
 * (the reference's own distributed path is an MPI tile farm: programs/parallel_priority_flood/main.cpp:394-548.)
 * Rank r of `world` holds ghost_top + owned + ghost_bottom rows in HBM (ghost_top = r > 0, ghost_bottom = r < world-1;
 * the ghost rows of the elevation raster hold the neighbouring bands' edge rows).  The rdb200_mgpu_* calls are
 * collective: every rank calls them in the same order.  A communicator is either NCCL (the product path; libnccl.so.2
 * is opened at run time) or a pair of caller-supplied callbacks (how the CPU tests run the same C++ drivers over gloo).
 *
 *   rank 0:  rdb200_nccl_unique_id(id)   ... ship the 128 bytes to every rank (MPI_Bcast, a file, torch.distributed) ...
 *   all:     rdb200_init(local_gpu); rdb200_comm_create_nccl(&comm, rank, world, id);
 *            rdb200_mgpu_fill_depressions_d8_f32(comm, d_band, W, rows, gt, gb, row0, H, NULL);   (or ..._d4_f32)
 *            rdb200_mgpu_resolve_flats_epsilon_f32(comm, d_band, W, rows, nodata, gt, gb, NULL);
 *            rdb200_mgpu_fa_f32_f64(comm, d_band, d_accum, W, rows, nodata, gt, gb, 0, 1, NULL);
 *   or, for the direction-grid pipeline after the fill (uint8 directions and int32 upslope-cell counts):
 *            rdb200_mgpu_d8_flow_directions_flats_f32(comm, d_band, d_dirs, W, rows, nodata, gt, gb, 0, NULL);
 *            rdb200_mgpu_d8_flow_accum_u8_i32(comm, d_dirs, d_area, W, rows, gt, gb, NULL);
 *   or, for flow proportions, accumulation from them and terrain attributes of the band:
 *            rdb200_mgpu_fm_method_f32(comm, 3, d_band, d_props, W, rows, nodata, gt, gb, 1.0);   (FM_Quinn)
 *            rdb200_mgpu_flow_accumulation_props_f64(comm, d_props, d_accum, W, rows, gt, gb, NULL);
 *            rdb200_mgpu_terrain_attribute_f32(comm, RDB200_TA_SLOPE_DEGREES, d_band, d_out, W, rows, nodata, -9999.f,
 *                                              1.f, cell_x, cell_y, gt, gb);
 */
typedef struct rdb200_comm rdb200_comm;
enum { RDB200_MAX_F32 = 0, RDB200_MIN_F32 = 1, RDB200_MAX_I32 = 2, RDB200_SUM_I32 = 3 };
/* exchange `bytes` with rank-1 (send_up / recv_up) and rank+1 (send_dn / recv_dn); a side without a neighbour gets
 * null pointers.  Pointers are device pointers of the calling rank; the call returns when the data has arrived. */
typedef int (*rdb200_exchange_fn)(void *user, const void *send_up, void *recv_up, const void *send_dn, void *recv_dn,
                                  size_t bytes);
/* in-place all-reduce of `count` elements, op = one of RDB200_MAX_F32 ... */
typedef int (*rdb200_allreduce_fn)(void *user, void *buf, size_t count, int op);
RDB200_API int rdb200_nccl_unique_id(uint8_t *out128);
RDB200_API int rdb200_comm_create_nccl(rdb200_comm **comm, int32_t rank, int32_t world, const uint8_t *id128);
RDB200_API int rdb200_comm_create_callbacks(rdb200_comm **comm, int32_t rank, int32_t world, void *user,
                                            rdb200_exchange_fn exchange, rdb200_allreduce_fn allreduce);
RDB200_API int rdb200_comm_destroy(rdb200_comm *comm);

/* FillDepressions<D8> (include/richdem/depressions/depressions.hpp:13-21) over row bands, in place on `d_band`
 * (local_rows x width, ghost rows included; their contents are ignored on entry and hold the neighbours' filled edge
 * rows on return).  row0 = global row of local row 0, height = rows of the whole raster.  Same result as the single-GPU
 * call, bit for bit.  *exchange_rounds (optional): halo exchanges done. */
RDB200_API int rdb200_mgpu_fill_depressions_d8_f32(const rdb200_comm *comm, float *d_band, int32_t width, int32_t local_rows,
                                                   int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                   int32_t *exchange_rounds);
/* FillDepressions<D4> (include/richdem/depressions/depressions.hpp:16-17 -> PriorityFlood_Barnes2014<Topology::D4>,
 * include/richdem/depressions/Barnes2014.hpp:230-304) over row bands: the 4-neighbour counterpart of
 * rdb200_mgpu_fill_depressions_d8_f32, with the same arguments and band convention.  Same result as
 * rdb200_dev_fill_depressions_d4_f32 on one GPU, bit for bit. */
RDB200_API int rdb200_mgpu_fill_depressions_d4_f32(const rdb200_comm *comm, float *d_band, int32_t width, int32_t local_rows,
                                                   int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                   int32_t *exchange_rounds);
/* pit_mask<D8 / D4> over row bands.  d_band (local_rows x width, row0 and height as in the band fill) is not modified; its
 * ghost rows are not read.  The band fill runs on a copy of it, then the owned rows of d_band_mask (local_rows x width)
 * receive the single-GPU mask, bit for bit; its ghost rows are not written.  The band must own a row, have the ghost
 * rows its rank needs, and -- when the raster has interior cells -- hold at least three local rows, as the band fill
 * requires; these are checked before any communication. */
RDB200_API int rdb200_mgpu_pit_mask_d8_f32(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t width,
                                           int32_t local_rows, float nodata, int32_t ghost_top, int32_t ghost_bottom, int32_t row0,
                                           int32_t height);
RDB200_API int rdb200_mgpu_pit_mask_d4_f32(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t width,
                                           int32_t local_rows, float nodata, int32_t ghost_top, int32_t ghost_bottom, int32_t row0,
                                           int32_t height);
/* HasDepressions<D8 / D4> over row bands, arguments as rdb200_mgpu_pit_mask_*.  Every rank first looks for a strict pit
 * in its owned rows (on a copy whose ghost rows receive the neighbours' edge rows) and one OR all-reduce combines the
 * answers; the band fill and a second all-reduce run only if no rank found one.  *out (host): 1 or 0 on every rank, the
 * single-GPU answer. */
RDB200_API int rdb200_mgpu_has_depressions_d8_f32(const rdb200_comm *comm, const float *d_band, int32_t width, int32_t local_rows,
                                                  int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                  int32_t *out);
RDB200_API int rdb200_mgpu_has_depressions_d4_f32(const rdb200_comm *comm, const float *d_band, int32_t width, int32_t local_rows,
                                                  int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                  int32_t *out);
/* ResolveFlatsEpsilon (include/richdem/flats/flats.hpp:21-28) over row bands, in place on the owned rows of `d_band`
 * (local_rows x width; the ghost rows must hold the neighbours' edge rows on entry, as the fill leaves them, and hold
 * the neighbours' resolved edge rows on return, ready for rdb200_mgpu_fa_*).  Same result as the single-GPU call, bit for
 * bit.  comm and d_band must not be null; ghost_top / ghost_bottom must be exactly (rank > 0) / (rank < world - 1) and
 * the band must own at least one row -- these are checked before any communication.  *seam_iterations (optional): rounds
 * of the outlet-flag and flat-height merges across seams (0 for one band). */
RDB200_API int rdb200_mgpu_resolve_flats_epsilon_f32(const rdb200_comm *comm, float *d_band, int32_t width, int32_t local_rows,
                                                     float nodata, int32_t ghost_top, int32_t ghost_bottom,
                                                     int32_t *seam_iterations);
/* FA_D8 (dinf = 0) / FA_Tarboton (dinf = 1) (include/richdem/methods/flow_accumulation.hpp:27,16) over row bands.
 * d_band_dem: elevations incl. ghost rows (neighbours' rows); d_band_accum_inout: weights in / accumulation out on the
 * owned rows (the ghost rows are scratch); accum_is_ones as in rdb200_fa_d8_f32_f64. */
RDB200_API int rdb200_mgpu_fa_f32_f64(const rdb200_comm *comm, const float *d_band_dem, double *d_band_accum_inout,
                                      int32_t width, int32_t local_rows, float nodata, int32_t ghost_top,
                                      int32_t ghost_bottom, int32_t dinf, int32_t accum_is_ones, int32_t *exchange_rounds);
/* Any FlowAccumulation method over row bands; method numbered as in rdb200_dev_fa_method_f32_f64: 0 FA_D8,
 * 1 FA_Tarboton, 2 FA_D4, 3 FA_Holmgren (xparam; FA_Quinn = 1.0), 4 FA_Freeman (xparam).  Everything else as
 * rdb200_mgpu_fa_f32_f64, which is this call with method 0 / 1.  An unknown method, or a non-finite xparam for
 * methods 3 and 4, is an error. */
RDB200_API int rdb200_mgpu_fa_method_f32_f64(const rdb200_comm *comm, const float *d_band_dem, double *d_band_accum_inout,
                                             int32_t width, int32_t local_rows, float nodata, int32_t ghost_top,
                                             int32_t ghost_bottom, int32_t method, double xparam, int32_t accum_is_ones,
                                             int32_t *exchange_rounds);
/* barnes_flat_resolution_d8 (include/richdem/flats/flat_resolution.hpp:588-607) over row bands: writes the D8 directions
 * of the band into d_band_dirs (local_rows x width, like d_band_dem).  The ghost rows of d_band_dem must hold the
 * neighbours' edge rows on entry, as the band fill leaves them.  The owned rows equal the single-GPU
 * rdb200_d8_flow_directions_flats_f32 of the whole raster, bit for bit; with alter = 1 so do the owned rows of the altered
 * d_band_dem.  On return the ghost rows of d_band_dirs (and, with alter = 1, of d_band_dem) hold the neighbours' edge
 * rows.  Argument checks as rdb200_mgpu_resolve_flats_epsilon_f32, d_band_dirs included.  *seam_iterations (optional):
 * rounds of the outlet-flag and flat-height merges across seams (0 for one band). */
RDB200_API int rdb200_mgpu_d8_flow_directions_flats_f32(const rdb200_comm *comm, float *d_band_dem, uint8_t *d_band_dirs,
                                                        int32_t width, int32_t local_rows, float nodata, int32_t ghost_top,
                                                        int32_t ghost_bottom, int32_t alter, int32_t *seam_iterations);
/* d8_flow_accum (include/richdem/methods/d8_methods.hpp:47-139) of a uint8 D8 direction grid cut into row bands.  The
 * ghost rows of d_band_dirs are not read: the call exchanges the edge rows itself.  The owned rows of d_band_area equal
 * the single-GPU rdb200_d8_flow_accum_u8_i32 of the whole grid (NoData 255 -> -1; codes other than 0..8 / 255 carry no
 * flow); its ghost rows are scratch.  Argument checks as rdb200_mgpu_resolve_flats_epsilon_f32.  *exchange_rounds
 * (optional): walk rounds, each followed by one exchange of the flow that crossed a seam. */
RDB200_API int rdb200_mgpu_d8_flow_accum_u8_i32(const rdb200_comm *comm, const uint8_t *d_band_dirs, int32_t *d_band_area,
                                                int32_t width, int32_t local_rows, int32_t ghost_top, int32_t ghost_bottom,
                                                int32_t *exchange_rounds);
/* FM_D8 / FM_Tarboton / FM_D4 / FM_Holmgren (FM_Quinn = xparam 1.0) / FM_Freeman over row bands; method numbered as in
 * rdb200_dev_fm_method_f32.  The call first exchanges the edge rows of d_band_dem, so on return its ghost rows hold the
 * neighbours' edge rows; their contents on entry are ignored.  The owned rows of d_band_props9 (local_rows x width x 9)
 * equal rdb200_dev_fm_method_f32 of the whole raster, bit for bit; its ghost rows are scratch.  Argument checks as
 * rdb200_mgpu_resolve_flats_epsilon_f32, plus an unknown method, all before any communication. */
RDB200_API int rdb200_mgpu_fm_method_f32(const rdb200_comm *comm, int32_t method, float *d_band_dem, float *d_band_props9,
                                         int32_t width, int32_t local_rows, float nodata, int32_t ghost_top, int32_t ghost_bottom,
                                         double xparam);
/* TA_* (RDB200_TA_*) over row bands, with the arguments of rdb200_dev_terrain_attribute_f32.  The ghost rows of d_band_dem
 * are refreshed as in rdb200_mgpu_fm_method_f32.  The owned rows of d_band_out equal rdb200_dev_terrain_attribute_f32 of
 * the whole raster, bit for bit; its ghost rows are scratch.  An unknown attribute or a cell length that is not positive
 * is an error before any communication. */
RDB200_API int rdb200_mgpu_terrain_attribute_f32(const rdb200_comm *comm, int32_t attribute, float *d_band_dem, float *d_band_out,
                                                 int32_t width, int32_t local_rows, float nodata_in, float nodata_out, float zscale,
                                                 double cell_x, double cell_y, int32_t ghost_top, int32_t ghost_bottom);
/* FlowAccumulation(props, accum) (include/richdem/methods/flow_accumulation_generic.hpp:33-100) over row bands, with the
 * proportions supplied by the caller (local_rows x width x 9, as FM_* lay them out).  The ghost rows of d_band_props9 are
 * not trusted: the call overwrites them with the neighbours' owned edge rows (one exchange of 36 B per cell and seam).
 * d_band_accum_inout holds the weights on the owned rows on entry and the accumulation on return; its ghost rows are
 * scratch.  As in rdb200_flow_accumulation_props_f64: NoData cells (slot 0 == -2) become -1, a share sent to a NoData cell
 * is dropped, and flow out of raster-edge cells (global rows 0 and H-1, columns 0 and W-1) is ignored.  The owned rows equal
 * the single-GPU call on the whole raster up to the order of the floating-point additions (bit for bit where every sum is
 * exact, e.g. one-hot proportions with unit weights).  Argument checks as rdb200_mgpu_resolve_flats_epsilon_f32.
 * *exchange_rounds (optional): walk rounds, each followed by one exchange of the flow that crossed a seam. */
RDB200_API int rdb200_mgpu_flow_accumulation_props_f64(const rdb200_comm *comm, float *d_band_props9, double *d_band_accum_inout,
                                                       int32_t width, int32_t local_rows, int32_t ghost_top, int32_t ghost_bottom,
                                                       int32_t *exchange_rounds);

/* float64 bands: the entry points above with double elevations and a double NoData, same band convention, argument
 * checks (all before any communication) and result: the owned rows equal the single-GPU float64 entry point on the
 * whole raster (rdb200_dev_*_f64), bit for bit where the float32 band call is bit for bit against its single-GPU twin.
 * The fill, pit_mask, HasDepressions, ResolveFlatsEpsilon and FA_D8 / FA_D4 run the float32 band drivers on float keys
 * kappa_G that every band shares: the cast to float when every band is float-exact, else global ranks built over the
 * rank chain (DESIGN §0.1).  The ranks cap the distinct values of all bands together at 2^31 - 2^25; a raster above it
 * fails on every rank before any stage runs.  The flow metrics, D-infinity / MFD accumulation and the terrain
 * attributes run the double kernels on bands whose ghost rows were exchanged.
 *   fill_depressions_*_f64     ghost rows ignored on entry, the neighbours' filled edge rows on return
 *   pit_mask_*_f64, has_depressions_*_f64   d_band not modified, its ghost rows not read
 *   resolve_flats_epsilon_f64  ghost rows not read on entry, the neighbours' resolved edge rows on return
 *   fm_method_f64, terrain_attribute_f64   ghost rows of d_band_dem refreshed, as the float32 calls do
 *   fa_method_f64_f64          methods as rdb200_mgpu_fa_method_f32_f64; ghost rows of d_band_dem not read
 *   d8_flow_directions_flats_f64  as rdb200_mgpu_d8_flow_directions_flats_f32: the ghost rows of d_band_dem hold the
 *                              neighbours' edge rows on entry; the directions of the doubles, the flats on kappa_G, and
 *                              with alter = 1 the float steps of rdb200_d8_flow_directions_flats_f64 on the owned rows */
RDB200_API int rdb200_mgpu_fill_depressions_d8_f64(const rdb200_comm *comm, double *d_band, int32_t width, int32_t local_rows,
                                                   int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                   int32_t *exchange_rounds);
RDB200_API int rdb200_mgpu_fill_depressions_d4_f64(const rdb200_comm *comm, double *d_band, int32_t width, int32_t local_rows,
                                                   int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                   int32_t *exchange_rounds);
RDB200_API int rdb200_mgpu_pit_mask_d8_f64(const rdb200_comm *comm, const double *d_band, uint8_t *d_band_mask, int32_t width,
                                           int32_t local_rows, double nodata, int32_t ghost_top, int32_t ghost_bottom, int32_t row0,
                                           int32_t height);
RDB200_API int rdb200_mgpu_pit_mask_d4_f64(const rdb200_comm *comm, const double *d_band, uint8_t *d_band_mask, int32_t width,
                                           int32_t local_rows, double nodata, int32_t ghost_top, int32_t ghost_bottom, int32_t row0,
                                           int32_t height);
RDB200_API int rdb200_mgpu_has_depressions_d8_f64(const rdb200_comm *comm, const double *d_band, int32_t width, int32_t local_rows,
                                                  int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                  int32_t *out);
RDB200_API int rdb200_mgpu_has_depressions_d4_f64(const rdb200_comm *comm, const double *d_band, int32_t width, int32_t local_rows,
                                                  int32_t ghost_top, int32_t ghost_bottom, int32_t row0, int32_t height,
                                                  int32_t *out);
RDB200_API int rdb200_mgpu_resolve_flats_epsilon_f64(const rdb200_comm *comm, double *d_band, int32_t width, int32_t local_rows,
                                                     double nodata, int32_t ghost_top, int32_t ghost_bottom,
                                                     int32_t *seam_iterations);
RDB200_API int rdb200_mgpu_d8_flow_directions_flats_f64(const rdb200_comm *comm, double *d_band_dem, uint8_t *d_band_dirs,
                                                        int32_t width, int32_t local_rows, double nodata, int32_t ghost_top,
                                                        int32_t ghost_bottom, int32_t alter, int32_t *seam_iterations);
RDB200_API int rdb200_mgpu_fm_method_f64(const rdb200_comm *comm, int32_t method, double *d_band_dem, float *d_band_props9,
                                         int32_t width, int32_t local_rows, double nodata, int32_t ghost_top, int32_t ghost_bottom,
                                         double xparam);
RDB200_API int rdb200_mgpu_terrain_attribute_f64(const rdb200_comm *comm, int32_t attribute, double *d_band_dem, float *d_band_out,
                                                 int32_t width, int32_t local_rows, double nodata_in, float nodata_out, float zscale,
                                                 double cell_x, double cell_y, int32_t ghost_top, int32_t ghost_bottom);
RDB200_API int rdb200_mgpu_fa_method_f64_f64(const rdb200_comm *comm, const double *d_band_dem, double *d_band_accum_inout,
                                             int32_t width, int32_t local_rows, double nodata, int32_t ghost_top,
                                             int32_t ghost_bottom, int32_t method, double xparam, int32_t accum_is_ones,
                                             int32_t *exchange_rounds);
/* DIAGNOSTIC, not part of the stable interface (as rdb200_f64_order_keys): kappa_G of the owned rows into d_band_keys
 * (local_rows x width; its ghost rows receive the neighbours' keys), *nodata_key = kappa_G(nodata) (the key of a cell
 * equal to nodata in any band; else as rdb200_f64_order_keys), *ranked = 0 for the cast to float, 1 for global ranks
 * (__uint_as_float(0x00800000 + r), r(v) = sum over the bands of their distinct values below v).  Collective. */
RDB200_API int rdb200_mgpu_f64_order_keys(const rdb200_comm *comm, const double *d_band, float *d_band_keys, int32_t width,
                                          int32_t local_rows, double nodata, int32_t ghost_top, int32_t ghost_bottom,
                                          float *nodata_key, int32_t *ranked);

/* ---- row-band (multi-GPU) fill: one band per GPU, halo rows exchanged by the caller -- */
/* The band raster handed in is (band_rows + ghost rows) x width.  Its first and last rows are
 * boundary conditions that the solver never changes: a real raster border row, or a ghost
 * row holding the neighbouring band's current water level (+inf before the first exchange).
 * Protocol per GPU: begin -> { run ; read own edge rows ; exchange ; update ghost rows } until
 * no band changed anywhere -> finish.  See richdem_b200/sharded.py. */
typedef struct rdb200_fill_state rdb200_fill_state;
RDB200_API int rdb200_dev_fill_begin(rdb200_fill_state **state, const float *d_dem, int32_t width,
                          int32_t height);
/* Multigrid start for a band (parameter fill_multigrid): `d_coarse` is the FILLED k x k max-pooled raster of the
 * WHOLE raster (coarse_width columns; every GPU solves that small raster itself), `row_offset` the global row of the
 * band's row 0.  Interior cells start at their block's coarse water level (an upper bound of the answer) instead of
 * +inf; the caller presets ghost rows the same way.  Everything else as rdb200_dev_fill_begin. */
RDB200_API int rdb200_dev_fill_begin_lifted(rdb200_fill_state **state, const float *d_dem, int32_t width, int32_t height,
                                 const float *d_coarse, int32_t coarse_width, int32_t pool, int32_t row_offset);
/* k x k max-pooling of rows [row_offset, row_offset + height) of a raster into the rows of the full coarse raster
 * (coarse_width x coarse_height, pre-filled by the caller, e.g. with -inf) that they touch; entries are combined
 * with max, so bands that share a coarse row can be merged with a MAX all-reduce. */
/* Multigrid V-cycle pieces for bands (parameter fill_vcycle; see DESIGN.md section 7):
 *   blockmax : k x k block maxima of the band's current water surface over its rows [skip_top, height - skip_bottom)
 *              (the owned rows), max-combined into the full coarse array (pre-filled with -inf; bands merge by MAX);
 *   relax_from: depression filling of `d_dem` started from the upper bound in `d_w_inout` (receives the result);
 *   prolong  : every interior cell of the band drops to its block's coarse level where that is lower; the tiles
 *              touched are queued for the next run; *tiles_lowered = how many. */
RDB200_API int rdb200_dev_fill_blockmax(rdb200_fill_state *state, float *d_blockmax, int32_t coarse_width, int32_t coarse_height,
                             int32_t pool, int32_t row_offset, int32_t skip_top, int32_t skip_bottom);
RDB200_API int rdb200_dev_fill_relax_from_f32(const float *d_dem, float *d_w_inout, int32_t width, int32_t height);
RDB200_API int rdb200_dev_fill_prolong(rdb200_fill_state *state, const float *d_coarse, int32_t coarse_width, int32_t pool,
                            int32_t row_offset, int32_t *tiles_lowered);
RDB200_API int rdb200_dev_maxpool_rows_f32(const float *d_src, int32_t width, int32_t height, int32_t row_offset, int32_t pool,
                                float *d_coarse, int32_t coarse_width, int32_t coarse_height);
/* Relax to the local fixed point (or for about `fill_band_rounds` sweep rounds when that parameter
 * is set).  *changed_rows: bit0 = row 1 changed, bit1 = row height-2 changed during this call (the
 * rows a neighbouring band holds as ghosts); bit2 = tiles are still active (call again). */
RDB200_API int rdb200_dev_fill_run(rdb200_fill_state *state, int32_t *changed_rows);
/* Copy water-level row y (0..height-1) to d_row[width]. */
RDB200_API int rdb200_dev_fill_read_row(rdb200_fill_state *state, int32_t y, float *d_row);
/* Replace boundary row y (0 or height-1) by d_row (element-wise <= the old values). */
RDB200_API int rdb200_dev_fill_update_row(rdb200_fill_state *state, int32_t y, const float *d_row);
/* Write the filled band to d_out (height x width, boundary rows included) and free state. */
RDB200_API int rdb200_dev_fill_finish(rdb200_fill_state *state, float *d_out);

/* ---- row-band (multi-GPU) flow accumulation ---------------------------------------------- */
/* Same role as FA_D8 / FA_Tarboton (include/richdem/methods/flow_accumulation.hpp:27,16) for one
 * row band.  The local raster (elevations and accumulation) is ghost_top + owned + ghost_bottom
 * rows; ghost elevation rows must hold the neighbouring bands' rows.  The ghost rows of the
 * accumulation array are scratch (parking slots for flow that leaves the band).
 * d_dem and d_accum_inout must stay valid until finish (the unit-weight D8 path computes the flow codes of the whole
 * band in its first run, after the neighbours' edge codes have arrived).
 * Protocol per GPU: begin -> exchange edge codes (get_edge_codes / set_ghost_codes) ->
 *   repeat { run ; take_outflow per side ; exchange ; apply_inflow per side } until no rank sent
 *   anything -> finish.  See richdem_b200/sharded.py. */
typedef struct rdb200_facc_state rdb200_facc_state;
RDB200_API int rdb200_dev_facc_begin(rdb200_facc_state **state, const float *d_dem, double *d_accum_inout,
                                     int32_t width, int32_t height, float nodata, int32_t ghost_top,
                                     int32_t ghost_bottom, int32_t dinf, int32_t accum_is_ones);
/* rdb200_dev_facc_begin for any method (numbered as in rdb200_mgpu_fa_method_f32_f64); the other rdb200_dev_facc_*
 * steps work on either kind of state. */
RDB200_API int rdb200_dev_facc_begin_method(rdb200_facc_state **state, const float *d_dem, double *d_accum_inout,
                                            int32_t width, int32_t height, float nodata, int32_t ghost_top,
                                            int32_t ghost_bottom, int32_t method, double xparam, int32_t accum_is_ones);
/* which: 0 = top side, 1 = bottom side.  Flow codes (1 byte/cell, + float rmax for D-infinity) of
 * my first/last owned row, to be installed as the neighbour's ghost codes.  Methods 2-4 (proportions) send a seam donor
 * mask in the code bytes instead (bit j: the cell sends a share to the neighbour's column x + j - 1; rmax unused), and
 * set_ghost_codes adds the shares it announces to the donor counts of my edge row. */
RDB200_API int rdb200_dev_facc_get_edge_codes(rdb200_facc_state *state, int32_t which, uint8_t *d_code_row,
                                              float *d_rmax_row);
RDB200_API int rdb200_dev_facc_set_ghost_codes(rdb200_facc_state *state, int32_t which,
                                               const uint8_t *d_code_row, const float *d_rmax_row);
/* Walk from the current frontier (first call: from all sources).  sent_*: number of flow parcels
 * parked in the top / bottom ghost row by this run. */
RDB200_API int rdb200_dev_facc_run(rdb200_facc_state *state, int32_t *sent_top, int32_t *sent_bottom);
/* Move the parked flow of one ghost row out (sum per cell, number of parcels per cell) and clear it. */
RDB200_API int rdb200_dev_facc_take_outflow(rdb200_facc_state *state, int32_t which, double *d_sum_row,
                                            int32_t *d_cnt_row);
/* Add a neighbour's outflow to my first/last owned row and release the cells it completes. */
RDB200_API int rdb200_dev_facc_apply_inflow(rdb200_facc_state *state, int32_t which, const double *d_sum_row,
                                            const int32_t *d_cnt_row);
RDB200_API int rdb200_dev_facc_finish(rdb200_facc_state *state);

/* ---- row-band (multi-GPU) flat resolution -------------------------------------------------- */
/* Same role as ResolveFlatsEpsilon (include/richdem/flats/flats.hpp:21-28) for one row band; the
 * local elevation raster (ghost_top + owned + ghost_bottom rows, ghost rows = the neighbours' rows)
 * is modified in place on the owned rows.  The steps run the single-GPU kernels on the local
 * raster; between them the caller moves the seam rows (see the protocol in csrc/flats.cu, which
 * rdb200_mgpu_resolve_flats_epsilon_f32 runs in one collective call). */
typedef struct rdb200_flats_state rdb200_flats_state;
RDB200_API int rdb200_dev_flats_begin(rdb200_flats_state **state, float *d_dem, int32_t width, int32_t height,
                                      float nodata, int32_t ghost_top, int32_t ghost_bottom);
RDB200_API int rdb200_dev_flats_arrays(rdb200_flats_state *state, uint64_t *out6);
RDB200_API int rdb200_dev_flats_edges(rdb200_flats_state *state);
RDB200_API int rdb200_dev_flats_components(rdb200_flats_state *state);
RDB200_API int rdb200_dev_flats_labels(rdb200_flats_state *state);
/* The distance state returned here speaks the row-band fill protocol: rdb200_dev_fill_run /
 * _read_row / _update_row; hand it back to gradient_end (do not call rdb200_dev_fill_finish). */
RDB200_API int rdb200_dev_flats_gradient_begin(rdb200_flats_state *state, int32_t away,
                                               rdb200_fill_state **dist_state);
RDB200_API int rdb200_dev_flats_gradient_end(rdb200_flats_state *state, int32_t away,
                                             rdb200_fill_state *dist_state);
RDB200_API int rdb200_dev_flats_apply(rdb200_flats_state *state);
RDB200_API int rdb200_dev_flats_finish(rdb200_flats_state *state);

#ifdef __cplusplus
}
#endif
#endif /* RICHDEM_B200_H_ */
