// Shared host/device plumbing for librichdem_b200 (sm_90a only).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/richdem_b200.h"

struct rdb200_fill_state;

namespace rdb {

// ---- errors -----------------------------------------------------------------------------
struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};

[[noreturn]] inline void fail(const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw Error(buf);
}

#define RDB_CK(expr)                                                                        \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      ::rdb::fail("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(_e)); \
  } while (0)

void capi_set_error(const char *msg);  // the text rdb200_last_error() returns

// The error boundary of every extern "C" entry point: nothing thrown may cross the C ABI.  Runs body and returns 0, or 1
// with what was thrown as the last error.
template <class F>
int capi_call(F &&body) {
  try {
    body();
    return 0;
  } catch (const std::exception &e) {
    capi_set_error(e.what());
  } catch (...) {
    capi_set_error("unknown C++ exception");
  }
  return 1;
}

// ---- D8 tables (reference include/richdem/common/constants.hpp:44-45,65) ----------------
//   2 3 4
//   1 0 5
//   8 7 6
__host__ __device__ __forceinline__ int d8dx(int n) {
  // {0,-1,-1,0,1,1,1,0,-1} packed 2 bits each (+1 bias)
  return (int)((0x6a41u >> (2 * n)) & 3u) - 1;  // n:0->0,1->-1,2->-1,3->0,4->1,5->1,6->1,7->0,8->-1
}
__host__ __device__ __forceinline__ int d8dy(int n) {
  // {0,0,-1,-1,-1,0,1,1,1}
  return (int)((0x2a405u >> (2 * n)) & 3u) - 1;
}

// ---- context ----------------------------------------------------------------------------
struct Params {
  int64_t fill_max_iters = 0;   // 0 = relax every tile visit to its local fixed point
  int64_t fill_rounds_per_sync = 16;
  int64_t fill_use_tma = 1;     // 0: plain ld.global staging (debug aid)
  int64_t fill_external_z = 1;  // single-GPU fill: W relaxed in the caller's raster, round 1 staged from the lifted start (0: padded W and Z)
  int64_t fill_ordered = 1;       // admit tiles by rising water level (device-side feedback on the level)
  int64_t fill_order_rounds = 0;  // rounds the level schedule spans (0: 0.8 x tiles across the raster)
  int64_t fill_band_rounds = 0;   // row-band mode: rounds per rdb200_dev_fill_run call (0: to convergence)
  int64_t fill_profile = 0;     // 1: collect + print in-tile work counters (slower)
  int64_t fill_wake_filter = 1; // fill: wake a neighbouring tile only when the new edge can lower one of its cells (0: always)
  int64_t fill_trace = 0;       // 1: per-V-cycle timeline of the multigrid fill on stderr (adds stream syncs)
  int64_t fill_multigrid = 8;      // k >= 2: start the flood from the lifted fill of the k x k max-pooled raster (recursive)
  int64_t fill_vcycle = 8;         // with fill_multigrid: coarse-grid correction after every that many fine rounds (0: none)
  int64_t fill_band_multigrid = 0; // row-band driver: pooling factor of the replicated coarse level (0: automatic)
  int64_t fill_multigrid_min = 0;  // smallest raster side that still gets a coarse level (0: 1024)
  int64_t flowdirs_rolling = 1;  // d8_flow_directions with a rolling three-row register window (W % 4 == 0)
  int64_t flats_uf_tiled = 1;  // union-find: unite inside 64x16 tiles in shared memory first, then across tile seams
  int64_t flats_fused_classify = 1;  // FindFlats + FindFlatEdges in one shared-memory window pass (single-GPU path)
  int64_t flats_pair = 1;    // the two gradient solves run side by side on two streams
  int64_t flats_tiled = 1;   // flat-resolution gradients by the tile engine (0: one cooperative BFS launch each)
  int64_t accum_dinf_packed = 1;  // unit-weight D-infinity: 0 level-synchronous kernel, 1 packed fixed-point walk in phases, 2 packed only when > 5 % of the cells have no receiver
  int64_t flowmet_tarboton_filter = 1;  // FM_Tarboton: pick the steepest facet from squared slopes first (flowmet.cuh), 0: the reference's sequence for every cell
  int64_t accum_walk_ahead = 0;   // packed D8 walk (row bands): sources a warp keeps queued ahead of its lanes (0: 64; 32..128)
  int64_t accum_walk_scan = 0;    // packed D8 walk (row bands), source scan: 0 over the 8 B words, 1 over the flagged code bytes + L2 prefetch of the words, 2 without the prefetch
  int64_t accum_dinf_stats = 0;   // packed D-infinity: print what the warps spent their iterations on (diagnostics)
  int64_t accum_dinf_share = -1;  // packed D-infinity: ring entries above which a warp asks for a rebalancing phase once enough warps wait (-1: 1)
  int64_t accum_dinf_wait = 0;    // packed D-infinity: ... once 1 / this share of the warps wait at the barrier (0: 4)
  int64_t accum_packed = 1;  // unit-weight D8: one GPU by 64 x 64 tiles, row bands on packed words (0: the generic walk)
  int64_t accum_fused_prep = 1;   // unit-weight D8 (row bands): flow codes + donor counts + sole-donor bits in one rolling-window pass
  int64_t accum_walk_lanes = 1;   // unit-weight D8 walk (row bands): persistent always-busy lanes fed from per-warp source queues
  int64_t accum_threads = 256;
  int64_t accum_budget = 0;  // cells one thread follows per level in the multi-receiver accumulation (0: 4)
  int64_t f64_band_rank_cap = 0;  // float64 row bands: distinct values the bands may hold in all (0: 2^31 - 2^25)
};

struct WsBlock {
  void *ptr;
  size_t bytes;
  bool in_use;
};

struct Ctx {
  bool inited = false;
  int device = -1;
  int num_sms = 0;
  cudaStream_t stream = nullptr;      // stream all work runs on
  cudaStream_t own_stream = nullptr;  // the library's default stream
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
  cudaStream_t aux_stream[2] = {nullptr, nullptr};  // side streams for solves that run side by side (flat gradients)
  cudaEvent_t aux_event[3] = {nullptr, nullptr, nullptr};
  std::vector<WsBlock> ws;
  void *pinned = nullptr;  // small pinned scratch for read-backs
  size_t pinned_bytes = 0;
  rdb200_stats stats;
  Params params;
};

Ctx &ctx();
void ensure_init();
void *ws_alloc(size_t bytes);
void ws_free(void *p);
void ws_release_all();

// RAII device scratch buffer from the cached workspace
template <class T>
struct DevBuf {
  T *p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  explicit DevBuf(size_t count) { alloc(count); }
  void alloc(size_t count) {
    reset();
    n = count;
    p = (T *)ws_alloc((count ? count : 1) * sizeof(T));
  }
  void reset() {
    if (p) ws_free(p);
    p = nullptr;
    n = 0;
  }
  ~DevBuf() { reset(); }
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  operator T *() const { return p; }
};

inline void count_launch(int64_t k = 1) { ctx().stats.kernel_launches += k; }

// kernel timing helper for the "dominant kernel" accounting (events on the launch stream)
struct KernelTimer {
  bool active;
  explicit KernelTimer(bool on = true) : active(on) {
    if (active) RDB_CK(cudaEventRecord(ctx().evk0, ctx().stream));
  }
  void stop_async() {
    if (active) RDB_CK(cudaEventRecord(ctx().evk1, ctx().stream));
  }
  // call after a stream sync
  double ms() {
    float t = 0;
    if (active) RDB_CK(cudaEventElapsedTime(&t, ctx().evk0, ctx().evk1));
    return t;
  }
};

// ---- row-band communication (comm.cu) and the multi-GPU drivers ------------------------------
int comm_rank(const rdb200_comm *c);
int comm_world(const rdb200_comm *c);
void comm_exchange(const rdb200_comm *c, const void *send_up, void *recv_up, const void *send_dn, void *recv_dn, size_t bytes);
void comm_allreduce(const rdb200_comm *c, void *buf, size_t count, int op);
void check_band_args(const char *what, const rdb200_comm *comm, const void *d_band, int w, int hloc, int gt, int gb);
void exchange_band_rows(const rdb200_comm *comm, void *d_band, size_t elem, int w, int hloc, int gt, int gb);
void mgpu_fill_band(const rdb200_comm *comm, float *d_local, int w, int hloc, int gt, int gb, int row0, int H, int *xrounds,
                    bool topo4 = false);
void mgpu_fill_band(const rdb200_comm *comm, double *d_band, int w, int hloc, int gt, int gb, int row0, int H, int *xrounds,
                    bool topo4);
// method: 0 D8, 1 Tarboton, 2 D4, 3 Holmgren (xparam; Quinn = 1.0), 4 Freeman (xparam)
void mgpu_fa_band(const rdb200_comm *comm, const float *d_dem, double *d_accum, int w, int hloc, float nodata, int gt, int gb,
                  int method, double xparam, bool ones, int *xrounds);
void mgpu_fa_band(const rdb200_comm *comm, const double *d_dem, double *d_accum, int w, int hloc, double nodata, int gt, int gb,
                  int method, double xparam, bool ones, int *xrounds);
void check_fa_method(int method, double xparam);  // an unknown method, or a non-finite exponent, is an error
// FlowAccumulation(props, accum) of caller-supplied 9-float proportions; the ghost rows of d_props are overwritten with the
// neighbours' edge rows
void mgpu_flow_accumulation_props_band(const rdb200_comm *comm, float *d_props, double *d_accum, int w, int hloc, int gt, int gb,
                                       int *xrounds);
// d_mask_out (w x hloc, may be null): write the increment mask there and leave the elevations and their ghost rows alone
void mgpu_resolve_flats_band(const rdb200_comm *comm, float *d_local, int w, int hloc, float nodata, int gt, int gb,
                             int *seam_iters, int32_t *d_mask_out = nullptr);
void mgpu_resolve_flats_band(const rdb200_comm *comm, double *d_band, int w, int hloc, double nodata, int gt, int gb,
                             int *seam_iters);
void mgpu_d8_flow_directions_flats_band(const rdb200_comm *comm, float *d_dem, uint8_t *d_dirs, int w, int hloc, float nodata,
                                        int gt, int gb, bool alter, int *seam_iters);
void mgpu_d8_flow_directions_flats_band(const rdb200_comm *comm, double *d_band, uint8_t *d_dirs, int w, int hloc, double nodata,
                                        int gt, int gb, bool alter, int *seam_iters);
// the flats of a band's plain D8 directions resolved over the bands (barnes_flat_resolution_d8 between its two direction
// passes); with alter, d_mask_out (may be null) receives the increment mask instead of d_dem its float ulps
int mgpu_dir_flats_band(const rdb200_comm *comm, float *d_dem, uint8_t *d_dirs, int w, int hloc, float nodata, int gt, int gb,
                        bool alter, int32_t *d_mask_out);
void mgpu_d8_flow_accum_band(const rdb200_comm *comm, const uint8_t *d_dirs, int32_t *d_area, int w, int hloc, int gt, int gb,
                             int *xrounds);
// the band relaxation protocol over a state that holds its start; R sweep rounds between halo exchanges (0: none)
int mgpu_relax_band(const rdb200_comm *comm, rdb200_fill_state *state, int gt, int gb, int R);

// ---- stage entry points implemented in the .cu files (device pointers, ctx stream) -------
// A double overload runs the float engines on order-preserving float keys (f64.cu) where the stage only compares
// elevations, and the kernels' double instantiations where it does arithmetic on them.
void fill_depressions_dev(float *d_dem, int w, int h, bool topo4 = false);
void fill_depressions_dev(double *d_z, int w, int h, bool topo4 = false);
// FillDepressions(epsilon=True) of a float raster (fill.cu): cells equal to nodata are pinned, never raised
void fill_depressions_epsilon_dev(float *d_dem, int w, int h, bool topo4, float nodata);
void geodesic_distance_dev(const uint8_t *d_open, int open_bit, float *d_w_inout, int w, int h);
void geodesic_distance_pair_dev(const uint8_t *d_open, int open_bit, float *d_wa, float *d_wb, int w, int h);
rdb200_fill_state *new_band_distance_state(const uint8_t *d_open, int open_bit, const float *d_winit, int w, int h,
                                           int ghost_top, int ghost_bottom);
void finish_band_distance_state(rdb200_fill_state *s, float *d_out);
void resolve_flats_dev(float *d_dem, int w, int h, float nodata, int32_t *d_mask_out,
                       int32_t *d_labels_out, bool apply, const uint8_t *d_dirs = nullptr);
// ResolveFlatsEpsilon and GetFlatMask
inline void resolve_flats_epsilon_dev(float *d_dem, int w, int h, float nodata) {
  resolve_flats_dev(d_dem, w, h, nodata, nullptr, nullptr, true);
}
void resolve_flats_epsilon_dev(double *d_z, int w, int h, double nodata);
inline void get_flat_mask_dev(const float *d_dem, int32_t *d_mask, int32_t *d_labels, int w, int h, float nodata) {
  resolve_flats_dev(const_cast<float *>(d_dem), w, h, nodata, d_mask, d_labels, false);  // apply = false: d_dem is not written
}
void get_flat_mask_dev(const double *d_z, int32_t *d_mask, int32_t *d_labels, int w, int h, double nodata);
void d8_flow_directions_flats_dev(float *d_dem, uint8_t *d_dirs, int w, int h, float nodata, bool alter);
void d8_flow_directions_flats_dev(double *d_z, uint8_t *d_dirs, int w, int h, double nodata, bool alter);
void d8_flow_directions_dev(const float *d_dem, uint8_t *d_dirs, int w, int h, float nodata);
void d8_flow_directions_dev(const double *d_dem, uint8_t *d_dirs, int w, int h, double nodata);
// d8_flow_flats: interior NO_FLOW cells take the direction of their lowest same-label neighbour in the increment mask
void d8_flow_flats_dev(const int32_t *d_mask, const int32_t *d_labels, uint8_t *d_dirs, int w, int h);
void d8_flow_accum_dev(const uint8_t *d_dirs, int32_t *d_area, int w, int h);
// FM_x by the C ABI's method number: 0 FM_D8, 1 FM_Tarboton, 2 FM_D4, 3 FM_Holmgren (FM_Quinn = exponent 1), 4 FM_Freeman
// (T = float, double)
template <class T>
void fm_method_dev(int method, const T *d_dem, float *d_props, int w, int h, T nodata, double xparam);
void flow_accumulation_props_dev(const float *d_props, double *d_accum, int w, int h);
// FA_D8 (dinf false) / FA_Tarboton by the fused engines
void fa_fused_dev(const float *d_dem, double *d_accum, int w, int h, float nodata, bool ones, bool dinf);
void fa_fused_dev(const double *d_dem, double *d_accum, int w, int h, double nodata, bool ones, bool dinf);
void terrain_attribute_dev(int attribute_id, const float *d_dem, float *d_out, int w, int h, float nodata_in, float nodata_out,
                           float zscale, double cell_x, double cell_y);
void terrain_attribute_dev(int attribute_id, const double *d_dem, float *d_out, int w, int h, double nodata_in,
                           float nodata_out, float zscale, double cell_x, double cell_y);
void generate_fbm_dev(float *d_dem, int w, int h, int y0, uint32_t seed, int octaves, float quantum);
// pit_mask<topo> / HasDepressions<topo> (depressions.cu); d_dem is not modified
void pit_mask_dev(const float *d_dem, uint8_t *d_mask, int w, int h, float nodata, bool topo4);
void pit_mask_dev(const double *d_z, uint8_t *d_mask, int w, int h, double nodata, bool topo4);
bool has_depressions_dev(const float *d_dem, int w, int h, bool topo4);
bool has_depressions_dev(const double *d_z, int w, int h, bool topo4);
void mgpu_pit_mask_band(const rdb200_comm *comm, const float *d_band, uint8_t *d_mask, int w, int hloc, float nodata, int gt,
                        int gb, int row0, int H, bool topo4);
void mgpu_pit_mask_band(const rdb200_comm *comm, const double *d_band, uint8_t *d_mask, int w, int hloc, double nodata, int gt,
                        int gb, int row0, int H, bool topo4);
bool mgpu_has_depressions_band(const rdb200_comm *comm, const float *d_band, int w, int hloc, int gt, int gb, int row0, int H,
                               bool topo4);
bool mgpu_has_depressions_band(const rdb200_comm *comm, const double *d_band, int w, int hloc, int gt, int gb, int row0, int H,
                               bool topo4);
// pit_mask's compare pass (mask may be null) and the strict-pit stencil (T = float, double), OR-ed into the device flags
void pit_mask_compare_dev(const float *d_z, const float *d_l, uint8_t *d_mask, size_t n, float nodata, int *d_any);
template <class T>
void strict_pit_dev(const T *d_z, int w, int h, bool topo4, int *d_flag);

// ---- float64 rasters through order-preserving float keys (f64.cu) ---------------------------
// kappa(Z) of n doubles into d_key; returns kappa(nodata).  *ranked (may be null): 0 when kappa is the cast to float,
// 1 when it is the dense rank.  With table, case 2 allocates the kappa^-1 table of sorted distinct values (n doubles).
float f64_keys_dev(const double *d_z, float *d_key, size_t n, double nodata, DevBuf<double> *table, int *ranked);
void f64_apply_ulps_dev(double *d_z, const int32_t *d_mask, int w, int h);
// d8_flats_alter_dem on doubles: the reference's nextafterf, i.e. k float ulps of the double rounded to float
void f64_float_steps_dev(double *d_z, const int32_t *d_mask, int w, int h);
int32_t read_i32(const int32_t *d_value);  // one device int, read back after the library's stream

// ---- float64 row bands: kappa_G, one key map shared by every band (f64.cu), and the band drivers (f64_band.cu) ----
// What a band keeps of kappa_G for kappa_G^-1: D_b (vals: [count | values], cap + 1 slots, cap = max over the bands of
// |D_b|) and r(D_b) (keys, strictly increasing), m = |D_b|.  ranked = 0: the cast route, nothing kept.
struct BandKeys {
  bool ranked = false;
  size_t m = 0, cap = 0;
  DevBuf<double> vals;
  DevBuf<uint32_t> keys;
};
// kappa_G of the owned rows of a double band into d_band_keys (same layout); its ghost rows receive the neighbours' owned
// keys.  Collective.  Returns kappa_G(nodata); inv (may be null) receives what kappa_G^-1 needs, *ranked the route.
float mgpu_f64_keys_dev(const rdb200_comm *comm, const double *d_band, float *d_band_keys, int w, int hloc, int gt, int gb,
                        double nodata, BandKeys *inv, int *ranked);
// the fill's write-back over bands: owned cells whose key k0 -> kf was raised take kappa_G^-1(kf).  Collective.
void mgpu_f64_writeback_dev(const rdb200_comm *comm, const BandKeys &inv, double *d_band, const float *k0, const float *kf, int w,
                            int hloc, int gt, int gb);
void check_mask_band(const char *what, const rdb200_comm *comm, const void *d_band, int w, int hloc, int gt, int gb, int row0,
                     int H);

}  // namespace rdb
