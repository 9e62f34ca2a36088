// C ABI of librichdem_b200.so: context, workspace cache, host<->device staging and the
// extern "C" entry points declared in include/richdem_b200.h.
#include "common.cuh"

#include <algorithm>
#include <cstdlib>

namespace rdb {

static thread_local std::string g_last_error;

void capi_set_error(const char *msg) { g_last_error = msg ? msg : "unknown error"; }

Ctx &ctx() {
  static Ctx c;
  return c;
}

static void init_device(int device) {
  Ctx &c = ctx();
  if (c.inited && c.device == device) return;
  if (c.inited) fail("rdb200_init: already initialised on device %d (call rdb200_shutdown first)", c.device);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    fail("no CUDA device available (%s); librichdem_b200 has no CPU fallback",
         e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  if (device < 0 || device >= ndev) fail("rdb200_init: device %d out of range (0..%d)", device, ndev - 1);
  RDB_CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  RDB_CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    fail("device %d is sm_%d%d; librichdem_b200 is built for sm_90a (H100) only", device, prop.major,
         prop.minor);
  c.device = device;
  c.num_sms = prop.multiProcessorCount;
  // a *blocking* stream: it orders itself with the legacy default stream, so callers that prepare
  // device buffers there (cudaMemcpy, PyTorch's default stream, ...) need no explicit events
  RDB_CK(cudaStreamCreate(&c.own_stream));
  c.stream = c.own_stream;
  RDB_CK(cudaEventCreate(&c.ev0));
  RDB_CK(cudaEventCreate(&c.ev1));
  RDB_CK(cudaEventCreate(&c.evk0));
  RDB_CK(cudaEventCreate(&c.evk1));
  c.pinned_bytes = 1 << 16;
  RDB_CK(cudaMallocHost(&c.pinned, c.pinned_bytes));
  memset(&c.stats, 0, sizeof(c.stats));
  c.inited = true;
}

void ensure_init() {
  Ctx &c = ctx();
  if (c.inited) {
    RDB_CK(cudaSetDevice(c.device));
    return;
  }
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) dev = 0;
  init_device(dev);
}

// ---- workspace cache: grow-only list of device blocks reused across calls -------------------
void *ws_alloc(size_t bytes) {
  Ctx &c = ctx();
  bytes = (bytes + 511) & ~(size_t)511;
  int best = -1;
  for (int i = 0; i < (int)c.ws.size(); i++)
    if (!c.ws[i].in_use && c.ws[i].bytes >= bytes && (best < 0 || c.ws[i].bytes < c.ws[best].bytes)) best = i;
  if (best >= 0 && c.ws[best].bytes <= bytes + bytes / 4 + (1 << 20)) {
    c.ws[best].in_use = true;
    return c.ws[best].ptr;
  }
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    // drop idle cached blocks and retry once
    cudaGetLastError();
    for (auto it = c.ws.begin(); it != c.ws.end();) {
      if (!it->in_use) {
        cudaFree(it->ptr);
        it = c.ws.erase(it);
      } else {
        ++it;
      }
    }
    e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) fail("cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
  }
  c.ws.push_back({p, bytes, true});
  return p;
}

void ws_free(void *p) {
  for (auto &b : ctx().ws)
    if (b.ptr == p) {
      b.in_use = false;
      return;
    }
}

// frees every cached block that is not in use (rdb200_set_param("trim_workspace", 1)): the cache only grows otherwise
void ws_trim() {
  Ctx &c = ctx();
  for (auto it = c.ws.begin(); it != c.ws.end();) {
    if (!it->in_use) {
      cudaFree(it->ptr);
      it = c.ws.erase(it);
    } else {
      ++it;
    }
  }
}

void ws_release_all() {
  Ctx &c = ctx();
  for (auto &b : c.ws) cudaFree(b.ptr);
  c.ws.clear();
}

// ---- helpers for the host entry points -------------------------------------------------------
struct CallScope {  // resets stats, times the whole call
  explicit CallScope(int64_t cells) {
    ensure_init();
    Ctx &c = ctx();
    memset(&c.stats, 0, sizeof(c.stats));
    c.stats.cells = cells;
    RDB_CK(cudaEventRecord(c.ev0, c.stream));
  }
  void done() {
    Ctx &c = ctx();
    RDB_CK(cudaEventRecord(c.ev1, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    float ms = 0;
    RDB_CK(cudaEventElapsedTime(&ms, c.ev0, c.ev1));
    c.stats.ms_total = ms;
  }
};

static void check_dims(int w, int h) {
  if (w <= 0 || h <= 0) fail("raster dimensions must be positive (got %d x %d)", w, h);
  // cell indices are 32-bit; the source scans of the accumulation walks bump a shared cursor by 1024 cells per warp, which may
  // run past the last cell by one chunk per resident warp before every warp has seen the end: keep that inside an int
  if ((int64_t)w * h > ((int64_t)1 << 31) - ((int64_t)1 << 25))
    fail("rasters above 2^31 - 2^25 cells per GPU are not supported (got %d x %d); shard by rows", w, h);
}

template <class T>
static void h2d(T *dst, const T *src, size_t n) {
  Ctx &c = ctx();
  cudaEvent_t a = c.evk0, b = c.evk1;
  RDB_CK(cudaEventRecord(a, c.stream));
  RDB_CK(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, c.stream));
  RDB_CK(cudaEventRecord(b, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  float ms = 0;
  RDB_CK(cudaEventElapsedTime(&ms, a, b));
  c.stats.ms_h2d += ms;
}
template <class T>
static void d2h(T *dst, const T *src, size_t n) {
  Ctx &c = ctx();
  cudaEvent_t a = c.evk0, b = c.evk1;
  RDB_CK(cudaEventRecord(a, c.stream));
  RDB_CK(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaEventRecord(b, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  float ms = 0;
  RDB_CK(cudaEventElapsedTime(&ms, a, b));
  c.stats.ms_d2h += ms;
}

}  // namespace rdb

using namespace rdb;

#define CAPI_TRY try {
#define CAPI_END                    \
  }                                 \
  catch (const std::exception &e) { \
    capi_set_error(e.what());       \
    return 1;                       \
  }                                 \
  catch (...) {                     \
    capi_set_error("unknown C++ exception"); \
    return 1;                       \
  }                                 \
  return 0;

extern "C" {

int rdb200_init(int device) {
  CAPI_TRY
  init_device(device);
  CAPI_END
}

void rdb200_shutdown(void) {
  Ctx &c = ctx();
  if (!c.inited) return;
  cudaSetDevice(c.device);
  cudaStreamSynchronize(c.stream);
  ws_release_all();
  if (c.pinned) cudaFreeHost(c.pinned);
  cudaEventDestroy(c.ev0);
  cudaEventDestroy(c.ev1);
  cudaEventDestroy(c.evk0);
  cudaEventDestroy(c.evk1);
  cudaStreamDestroy(c.own_stream);
  for (int k = 0; k < 2; k++)
    if (c.aux_stream[k]) cudaStreamDestroy(c.aux_stream[k]);
  for (int k = 0; k < 3; k++)
    if (c.aux_event[k]) cudaEventDestroy(c.aux_event[k]);
  const Params keep = c.params;  // rdb200_set_param switches are process settings: they survive a re-init
  c = Ctx();
  c.params = keep;
}

const char *rdb200_last_error(void) { return g_last_error.c_str(); }
int rdb200_version(void) { return RDB200_VERSION; }

int rdb200_set_stream(void *cuda_stream) {
  CAPI_TRY
  ensure_init();
  Ctx &c = ctx();
  RDB_CK(cudaStreamSynchronize(c.stream));
  c.stream = cuda_stream ? (cudaStream_t)cuda_stream : c.own_stream;
  CAPI_END
}

int rdb200_get_stats(rdb200_stats *out) {
  CAPI_TRY
  if (!out) fail("rdb200_get_stats: null pointer");
  *out = ctx().stats;
  CAPI_END
}

int rdb200_set_param(const char *name, int64_t value) {
  CAPI_TRY
  if (!name) fail("rdb200_set_param: null name");
  Params &p = ctx().params;
  const std::string n(name);
  if (n == "reset_defaults") p = Params();
  else if (n == "trim_workspace") {
    if (ctx().inited) {
      RDB_CK(cudaStreamSynchronize(ctx().stream));
      ws_trim();
    }
  }
  else if (n == "fill_max_iters") p.fill_max_iters = value;
  else if (n == "fill_rounds_per_sync") p.fill_rounds_per_sync = value > 0 ? value : 16;
  else if (n == "fill_use_tma") p.fill_use_tma = value;
  else if (n == "fill_external_z") p.fill_external_z = value;
  else if (n == "fill_profile") p.fill_profile = value;
  else if (n == "fill_wake_filter") p.fill_wake_filter = value;
  else if (n == "fill_trace") p.fill_trace = value;
  else if (n == "fill_ordered") p.fill_ordered = value;
  else if (n == "fill_order_rounds") p.fill_order_rounds = value;
  else if (n == "fill_band_rounds") p.fill_band_rounds = value;
  else if (n == "accum_threads") p.accum_threads = value > 0 ? value : 256;
  else if (n == "accum_budget") p.accum_budget = value;
  else if (n == "accum_walk_lanes") p.accum_walk_lanes = value;
  else if (n == "accum_fused_prep") p.accum_fused_prep = value;
  else if (n == "flats_tiled") p.flats_tiled = value;
  else if (n == "flats_pair") p.flats_pair = value;
  else if (n == "flats_fused_classify") p.flats_fused_classify = value;
  else if (n == "fill_multigrid") p.fill_multigrid = value;
  else if (n == "fill_multigrid_min") p.fill_multigrid_min = value;
  else if (n == "fill_vcycle") p.fill_vcycle = value;
  else if (n == "fill_band_multigrid") p.fill_band_multigrid = value;
  else if (n == "flats_uf_tiled") p.flats_uf_tiled = value;
  else if (n == "flowdirs_rolling") p.flowdirs_rolling = value;
  else if (n == "accum_packed") p.accum_packed = value;
  else if (n == "accum_dinf_packed") p.accum_dinf_packed = value;
  else if (n == "accum_dinf_share") p.accum_dinf_share = value;
  else if (n == "flowmet_tarboton_filter") p.flowmet_tarboton_filter = value;
  else if (n == "accum_walk_scan") p.accum_walk_scan = value;
  else if (n == "accum_walk_ahead") p.accum_walk_ahead = value;
  else if (n == "accum_dinf_stats") p.accum_dinf_stats = value;
  else if (n == "accum_dinf_wait") p.accum_dinf_wait = value;
  else fail("rdb200_set_param: unknown parameter '%s'", name);
  CAPI_END
}

// ---- host entry points ------------------------------------------------------------------------

int rdb200_fill_depressions_d8_f32(float *dem, int32_t w, int32_t h) {
  CAPI_TRY
  if (!dem) fail("fill_depressions: null dem");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  h2d(d.p, dem, n);
  fill_depressions_dev(d.p, w, h);
  d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}

int rdb200_fill_depressions_d4_f32(float *dem, int32_t w, int32_t h) {
  CAPI_TRY
  if (!dem) fail("fill_depressions: null dem");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  h2d(d.p, dem, n);
  fill_depressions_dev(d.p, w, h, true);
  d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}

static int pit_mask_host(const float *dem, uint8_t *mask, int32_t w, int32_t h, float nodata, bool topo4) {
  CAPI_TRY
  if (!dem || !mask) fail("pit_mask: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  DevBuf<uint8_t> m(n);
  h2d(d.p, dem, n);
  pit_mask_dev(d.p, m.p, w, h, nodata, topo4);
  d2h(mask, m.p, n);
  cs.done();
  CAPI_END
}
int rdb200_pit_mask_d8_f32(const float *dem, uint8_t *mask, int32_t w, int32_t h, float nodata) {
  return pit_mask_host(dem, mask, w, h, nodata, false);
}
int rdb200_pit_mask_d4_f32(const float *dem, uint8_t *mask, int32_t w, int32_t h, float nodata) {
  return pit_mask_host(dem, mask, w, h, nodata, true);
}

static int has_depressions_host(const float *dem, int32_t w, int32_t h, int32_t *out, bool topo4) {
  CAPI_TRY
  if (!dem || !out) fail("has_depressions: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  h2d(d.p, dem, n);
  const bool any = has_depressions_dev(d.p, w, h, topo4);
  cs.done();
  *out = any ? 1 : 0;
  CAPI_END
}
int rdb200_has_depressions_d8_f32(const float *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions_host(dem, w, h, out, false);
}
int rdb200_has_depressions_d4_f32(const float *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions_host(dem, w, h, out, true);
}

int rdb200_resolve_flats_epsilon_f32(float *dem, int32_t w, int32_t h, float nodata) {
  CAPI_TRY
  if (!dem) fail("resolve_flats: null dem");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  h2d(d.p, dem, n);
  resolve_flats_dev(d.p, w, h, nodata, nullptr, nullptr, true);
  d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}

int rdb200_get_flat_mask_f32(const float *dem, int32_t *flat_mask, int32_t *labels, int32_t w, int32_t h,
                             float nodata) {
  CAPI_TRY
  if (!dem || !flat_mask || !labels) fail("get_flat_mask: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  DevBuf<int32_t> m(n), l(n);
  h2d(d.p, dem, n);
  resolve_flats_dev(d.p, w, h, nodata, m.p, l.p, false);
  d2h(flat_mask, m.p, n);
  d2h(labels, l.p, n);
  cs.done();
  CAPI_END
}

int rdb200_d8_flow_directions_f32(const float *dem, uint8_t *dirs, int32_t w, int32_t h, float nodata) {
  CAPI_TRY
  if (!dem || !dirs) fail("d8_flow_directions: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  DevBuf<uint8_t> o(n);
  h2d(d.p, dem, n);
  d8_flow_directions_dev(d.p, o.p, w, h, nodata);
  d2h(dirs, o.p, n);
  cs.done();
  CAPI_END
}

int rdb200_d8_flow_directions_flats_f32(float *dem, uint8_t *dirs, int32_t w, int32_t h, float nodata, int32_t alter) {
  CAPI_TRY
  if (!dem || !dirs) fail("d8_flow_directions_flats: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  DevBuf<uint8_t> o(n);
  h2d(d.p, dem, n);
  d8_flow_directions_flats_dev(d.p, o.p, w, h, nodata, alter != 0);
  d2h(dirs, o.p, n);
  if (alter) d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}

int rdb200_d8_flow_accum_u8_i32(const uint8_t *dirs, int32_t *area, int32_t w, int32_t h) {
  CAPI_TRY
  if (!dirs || !area) fail("d8_flow_accum: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<uint8_t> d(n);
  DevBuf<int32_t> o(n);
  h2d(d.p, dirs, n);
  d8_flow_accum_dev(d.p, o.p, w, h);
  d2h(area, o.p, n);
  cs.done();
  CAPI_END
}

// method: 0 FM_D8, 1 FM_Tarboton, 2 FM_D4, 3 FM_Holmgren (FM_Quinn = exponent 1), 4 FM_Freeman
static void fm_dispatch_dev(int method, const float *d_dem, float *d_props, int w, int h, float nodata, double xparam) {
  switch (method) {
    case 0: fm_d8_dev(d_dem, d_props, w, h, nodata); break;
    case 1: fm_tarboton_dev(d_dem, d_props, w, h, nodata); break;
    case 2: fm_d4_dev(d_dem, d_props, w, h, nodata); break;
    case 3: fm_holmgren_dev(d_dem, d_props, w, h, nodata, xparam); break;
    case 4: fm_freeman_dev(d_dem, d_props, w, h, nodata, xparam); break;
    default: fail("unknown flow metric %d", method);
  }
}

static int fm_host(const float *dem, float *props, int32_t w, int32_t h, float nodata, int method, double xparam = 0) {
  CAPI_TRY
  if (!dem || !props) fail("flow metric: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n), p(9 * n);
  h2d(d.p, dem, n);
  fm_dispatch_dev(method, d.p, p.p, w, h, nodata, xparam);
  d2h(props, p.p, 9 * n);
  cs.done();
  CAPI_END
}
int rdb200_fm_d8_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm_host(dem, props, w, h, nodata, 0);
}
int rdb200_fm_tarboton_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm_host(dem, props, w, h, nodata, 1);
}
int rdb200_fm_d4_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm_host(dem, props, w, h, nodata, 2);
}
int rdb200_fm_quinn_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm_host(dem, props, w, h, nodata, 3, 1.0);
}
int rdb200_fm_holmgren_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata, double xparam) {
  return fm_host(dem, props, w, h, nodata, 3, xparam);
}
int rdb200_fm_freeman_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata, double xparam) {
  return fm_host(dem, props, w, h, nodata, 4, xparam);
}

// TA_* (reference methods/terrain_attributes.hpp:370-538): one stencil pass, 4 B in + 4 B out per cell
int rdb200_terrain_attribute_f32(int32_t attribute, const float *dem, float *out, int32_t w, int32_t h, float nodata_in,
                                 float nodata_out, float zscale, double cell_x, double cell_y) {
  CAPI_TRY
  if (!dem || !out) fail("terrain attribute: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n), o(n);
  h2d(d.p, dem, n);
  terrain_attribute_dev(attribute, d.p, o.p, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
  d2h(out, o.p, n);
  cs.done();
  CAPI_END
}

// FA_<metric> = FM_<metric> into a device-side proportions array + the generic accumulation
// (reference methods/flow_accumulation.hpp:18-20,28: `Array3D<float> props(elevations); FM_x(...); FlowAccumulation(...)`)
static void fa_via_props_dev(int method, const float *d_dem, double *d_accum, int w, int h, float nodata, double xparam) {
  DevBuf<float> p(9 * (size_t)w * h);
  fm_dispatch_dev(method, d_dem, p.p, w, h, nodata, xparam);
  flow_accumulation_props_dev(p.p, d_accum, w, h);
}
static int fa_via_props_host(int method, const float *dem, double *accum, int32_t w, int32_t h, float nodata, double xparam) {
  CAPI_TRY
  if (!dem || !accum) fail("flow accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  DevBuf<double> a(n);
  h2d(d.p, dem, n);
  h2d(a.p, accum, n);
  fa_via_props_dev(method, d.p, a.p, w, h, nodata, xparam);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}
int rdb200_fa_d4_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata) {
  return fa_via_props_host(2, dem, accum, w, h, nodata, 0);
}
int rdb200_fa_quinn_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata) {
  return fa_via_props_host(3, dem, accum, w, h, nodata, 1.0);
}
int rdb200_fa_holmgren_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, double xparam) {
  return fa_via_props_host(3, dem, accum, w, h, nodata, xparam);
}
int rdb200_fa_freeman_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, double xparam) {
  return fa_via_props_host(4, dem, accum, w, h, nodata, xparam);
}

int rdb200_flow_accumulation_props_f64(const float *props, double *accum, int32_t w, int32_t h) {
  CAPI_TRY
  if (!props || !accum) fail("flow_accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> p(9 * n);
  DevBuf<double> a(n);
  h2d(p.p, props, 9 * n);
  h2d(a.p, accum, n);
  flow_accumulation_props_dev(p.p, a.p, w, h);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}

static int fa_host(const float *dem, double *accum, int32_t w, int32_t h, float nodata, int32_t ones,
                   bool dinf) {
  CAPI_TRY
  if (!dem || !accum) fail("flow accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<float> d(n);
  DevBuf<double> a(n);
  h2d(d.p, dem, n);
  if (!ones) h2d(a.p, accum, n);
  fa_fused_dev(d.p, a.p, w, h, nodata, ones != 0, dinf);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}
int rdb200_fa_d8_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, int32_t ones) {
  return fa_host(dem, accum, w, h, nodata, ones, false);
}
int rdb200_fa_tarboton_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata,
                               int32_t ones) {
  return fa_host(dem, accum, w, h, nodata, ones, true);
}

// ---- float64 rasters (f64.cu): the float engines on kappa(Z), kappa an order-preserving map to float keys ------------

// reference depressions/depressions.hpp:13-21 -> Zhou2016.hpp:125-191 (D8) / Barnes2014.hpp:230-304 (D4), T = double
int rdb200_fill_depressions_d8_f64(double *dem, int32_t w, int32_t h) {
  CAPI_TRY
  if (!dem) fail("fill_depressions: null dem");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  h2d(d.p, dem, n);
  fill_depressions_f64_dev(d.p, w, h, false);
  d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}
int rdb200_fill_depressions_d4_f64(double *dem, int32_t w, int32_t h) {
  CAPI_TRY
  if (!dem) fail("fill_depressions: null dem");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  h2d(d.p, dem, n);
  fill_depressions_f64_dev(d.p, w, h, true);
  d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}

// reference depressions/Barnes2014.hpp:593-676 (pit_mask<topo>, T = double)
static int pit_mask_f64_host(const double *dem, uint8_t *mask, int32_t w, int32_t h, double nodata, bool topo4) {
  CAPI_TRY
  if (!dem || !mask) fail("pit_mask: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  DevBuf<uint8_t> m(n);
  h2d(d.p, dem, n);
  pit_mask_f64_dev(d.p, m.p, w, h, nodata, topo4);
  d2h(mask, m.p, n);
  cs.done();
  CAPI_END
}
int rdb200_pit_mask_d8_f64(const double *dem, uint8_t *mask, int32_t w, int32_t h, double nodata) {
  return pit_mask_f64_host(dem, mask, w, h, nodata, false);
}
int rdb200_pit_mask_d4_f64(const double *dem, uint8_t *mask, int32_t w, int32_t h, double nodata) {
  return pit_mask_f64_host(dem, mask, w, h, nodata, true);
}

// reference depressions/Barnes2014.hpp:43-104 (HasDepressions<topo>, T = double)
static int has_depressions_f64_host(const double *dem, int32_t w, int32_t h, int32_t *out, bool topo4) {
  CAPI_TRY
  if (!dem || !out) fail("has_depressions: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  h2d(d.p, dem, n);
  const bool any = has_depressions_f64_dev(d.p, w, h, topo4);
  cs.done();
  *out = any ? 1 : 0;
  CAPI_END
}
int rdb200_has_depressions_d8_f64(const double *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions_f64_host(dem, w, h, out, false);
}
int rdb200_has_depressions_d4_f64(const double *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions_f64_host(dem, w, h, out, true);
}

// reference flats/flats.hpp:21-28 -> flats/Barnes2014.hpp:398-467 (GetFlatMask) + :496-550 (apply), T = double
int rdb200_resolve_flats_epsilon_f64(double *dem, int32_t w, int32_t h, double nodata) {
  CAPI_TRY
  if (!dem) fail("resolve_flats: null dem");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  h2d(d.p, dem, n);
  resolve_flats_f64_dev(d.p, w, h, nodata);
  d2h(dem, d.p, n);
  cs.done();
  CAPI_END
}

// reference flowmet/d8_flowdirs.hpp:32-123 (d8_flow_directions<double, uint8_t>)
int rdb200_d8_flow_directions_f64(const double *dem, uint8_t *dirs, int32_t w, int32_t h, double nodata) {
  CAPI_TRY
  if (!dem || !dirs) fail("d8_flow_directions: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  DevBuf<uint8_t> o(n);
  h2d(d.p, dem, n);
  d8_flow_directions_f64_dev(d.p, o.p, w, h, nodata);
  d2h(dirs, o.p, n);
  cs.done();
  CAPI_END
}

// reference methods/flow_accumulation.hpp:27 (FA_D8<double, double>: OCallaghan1984.hpp:13-91 + flow_accumulation_generic.hpp:33-100)
int rdb200_fa_d8_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  CAPI_TRY
  if (!dem || !accum) fail("flow accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n), a(n);
  h2d(d.p, dem, n);
  if (!ones) h2d(a.p, accum, n);
  fa_d8_f64_dev(d.p, a.p, w, h, nodata, ones != 0);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}

// reference methods/flow_accumulation.hpp:28 (FA_D4<double, double>: OCallaghan1984.hpp:89-91 + the generic accumulation)
static void fa_d4_f64_dev(const double *d_dem, double *d_accum, int w, int h, double nodata) {
  DevBuf<float> key((size_t)w * h);
  const float nd = f64_keys_dev(d_dem, key.p, (size_t)w * h, nodata, nullptr, nullptr);
  fa_via_props_dev(2, key.p, d_accum, w, h, nd, 0);
}
int rdb200_fa_d4_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata) {
  CAPI_TRY
  if (!dem || !accum) fail("flow accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n), a(n);
  h2d(d.p, dem, n);
  h2d(a.p, accum, n);
  fa_d4_f64_dev(d.p, a.p, w, h, nodata);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}

// ---- float64 D-infinity, MFD and terrain attributes: the float kernels' double instantiations (no keys: these stages do
// arithmetic on the elevations, DESIGN §0.2).  Argument order and checks as the float entry points above.

// reference flowmet/*.hpp with E = double; method numbered as fm_dispatch_dev
static int fm_f64_host(const double *dem, float *props, int32_t w, int32_t h, double nodata, int method, double xparam = 0) {
  CAPI_TRY
  if (!dem || !props) fail("flow metric: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  DevBuf<float> p(9 * n);
  h2d(d.p, dem, n);
  fm_method_f64_dev(method, d.p, p.p, w, h, nodata, xparam);
  d2h(props, p.p, 9 * n);
  cs.done();
  CAPI_END
}
int rdb200_fm_d8_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm_f64_host(dem, props, w, h, nodata, 0);
}
int rdb200_fm_tarboton_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm_f64_host(dem, props, w, h, nodata, 1);
}
int rdb200_fm_d4_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm_f64_host(dem, props, w, h, nodata, 2);
}
int rdb200_fm_quinn_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm_f64_host(dem, props, w, h, nodata, 3, 1.0);
}
int rdb200_fm_holmgren_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata, double xparam) {
  return fm_f64_host(dem, props, w, h, nodata, 3, xparam);
}
int rdb200_fm_freeman_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata, double xparam) {
  return fm_f64_host(dem, props, w, h, nodata, 4, xparam);
}

// methods/flow_accumulation.hpp:16-20 with E = double: FM_x on the doubles into device-side proportions + the generic
// accumulation; methods 0 and 2 take the key route of FA_D8 / FA_D4 (accum holds the weights)
static void fa_method_f64_dev(int method, const double *d_dem, double *d_accum, int w, int h, double nodata, double xparam) {
  if (method == 0) {
    fa_d8_f64_dev(d_dem, d_accum, w, h, nodata, false);
  } else if (method == 2) {
    fa_d4_f64_dev(d_dem, d_accum, w, h, nodata);
  } else {
    DevBuf<float> p(9 * (size_t)w * h);
    fm_method_f64_dev(method, d_dem, p.p, w, h, nodata, xparam);
    flow_accumulation_props_dev(p.p, d_accum, w, h);
  }
}
static int fa_method_f64_host(int method, const double *dem, double *accum, int32_t w, int32_t h, double nodata, double xparam) {
  CAPI_TRY
  if (!dem || !accum) fail("flow accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n), a(n);
  h2d(d.p, dem, n);
  h2d(a.p, accum, n);
  fa_method_f64_dev(method, d.p, a.p, w, h, nodata, xparam);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}
int rdb200_fa_quinn_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata) {
  return fa_method_f64_host(3, dem, accum, w, h, nodata, 1.0);
}
int rdb200_fa_holmgren_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, double xparam) {
  return fa_method_f64_host(3, dem, accum, w, h, nodata, xparam);
}
int rdb200_fa_freeman_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, double xparam) {
  return fa_method_f64_host(4, dem, accum, w, h, nodata, xparam);
}

// methods/flow_accumulation.hpp:16 (FA_Tarboton<double, double>): the fused D-infinity engine after a code pass on the
// doubles; accum_is_ones as rdb200_fa_tarboton_f32_f64
int rdb200_fa_tarboton_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  CAPI_TRY
  if (!dem || !accum) fail("flow accumulation: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n), a(n);
  h2d(d.p, dem, n);
  if (!ones) h2d(a.p, accum, n);
  fa_tarboton_f64_dev(d.p, a.p, w, h, nodata, ones != 0);
  d2h(accum, a.p, n);
  cs.done();
  CAPI_END
}

// methods/terrain_attributes.hpp:370-538 with T = double: 8 B in + 4 B out per cell
int rdb200_terrain_attribute_f64(int32_t attribute, const double *dem, float *out, int32_t w, int32_t h, double nodata_in,
                                 float nodata_out, float zscale, double cell_x, double cell_y) {
  CAPI_TRY
  if (!dem || !out) fail("terrain attribute: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  DevBuf<float> o(n);
  h2d(d.p, dem, n);
  terrain_attribute_f64_dev(attribute, d.p, o.p, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
  d2h(out, o.p, n);
  cs.done();
  CAPI_END
}

// kappa itself: the float keys the entry points above run the float engines on, kappa(nodata) and which case ran
int rdb200_f64_order_keys(const double *dem, float *keys, int32_t w, int32_t h, double nodata, float *nodata_key,
                          int32_t *ranked) {
  CAPI_TRY
  if (!dem || !keys) fail("f64_order_keys: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const size_t n = (size_t)w * h;
  DevBuf<double> d(n);
  DevBuf<float> k(n);
  h2d(d.p, dem, n);
  int r = 0;
  const float nd = f64_keys_dev(d.p, k.p, n, nodata, nullptr, &r);
  d2h(keys, k.p, n);
  cs.done();
  if (nodata_key) *nodata_key = nd;
  if (ranked) *ranked = r;
  CAPI_END
}

// ---- device entry points ------------------------------------------------------------------------

#define DEV_ENTRY(cells, body) \
  CAPI_TRY                     \
  CallScope cs(cells);         \
  body;                        \
  cs.done();                   \
  CAPI_END

int rdb200_dev_fill_depressions_d8_f32(float *d_dem, int32_t w, int32_t h) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fill_depressions_dev(d_dem, w, h)))
}
int rdb200_dev_fill_depressions_d4_f32(float *d_dem, int32_t w, int32_t h) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fill_depressions_dev(d_dem, w, h, true)))
}
static int dev_pit_mask(const float *d_dem, uint8_t *d_mask, int32_t w, int32_t h, float nodata, bool topo4) {
  CAPI_TRY
  if (!d_dem || !d_mask) fail("pit_mask: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  pit_mask_dev(d_dem, d_mask, w, h, nodata, topo4);
  cs.done();
  CAPI_END
}
int rdb200_dev_pit_mask_d8_f32(const float *d_dem, uint8_t *d_mask, int32_t w, int32_t h, float nodata) {
  return dev_pit_mask(d_dem, d_mask, w, h, nodata, false);
}
int rdb200_dev_pit_mask_d4_f32(const float *d_dem, uint8_t *d_mask, int32_t w, int32_t h, float nodata) {
  return dev_pit_mask(d_dem, d_mask, w, h, nodata, true);
}
static int dev_has_depressions(const float *d_dem, int32_t w, int32_t h, int32_t *out, bool topo4) {
  CAPI_TRY
  if (!d_dem || !out) fail("has_depressions: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const bool any = has_depressions_dev(d_dem, w, h, topo4);
  cs.done();
  *out = any ? 1 : 0;
  CAPI_END
}
int rdb200_dev_has_depressions_d8_f32(const float *d_dem, int32_t w, int32_t h, int32_t *out) {
  return dev_has_depressions(d_dem, w, h, out, false);
}
int rdb200_dev_has_depressions_d4_f32(const float *d_dem, int32_t w, int32_t h, int32_t *out) {
  return dev_has_depressions(d_dem, w, h, out, true);
}
int rdb200_dev_resolve_flats_epsilon_f32(float *d_dem, int32_t w, int32_t h, float nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), resolve_flats_dev(d_dem, w, h, nodata, nullptr, nullptr, true)))
}
int rdb200_dev_d8_flow_directions_f32(const float *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, float nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), d8_flow_directions_dev(d_dem, d_dirs, w, h, nodata)))
}
int rdb200_dev_d8_flow_directions_flats_f32(float *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, float nodata, int32_t alter) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), d8_flow_directions_flats_dev(d_dem, d_dirs, w, h, nodata, alter != 0)))
}
int rdb200_dev_d8_flow_accum_u8_i32(const uint8_t *d_dirs, int32_t *d_area, int32_t w, int32_t h) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), d8_flow_accum_dev(d_dirs, d_area, w, h)))
}
int rdb200_dev_fm_d8_f32(const float *d_dem, float *d_props, int32_t w, int32_t h, float nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fm_d8_dev(d_dem, d_props, w, h, nodata)))
}
int rdb200_dev_fm_tarboton_f32(const float *d_dem, float *d_props, int32_t w, int32_t h, float nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fm_tarboton_dev(d_dem, d_props, w, h, nodata)))
}
int rdb200_dev_fm_method_f32(int32_t method, const float *d_dem, float *d_props, int32_t w, int32_t h, float nodata,
                             double xparam) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fm_dispatch_dev(method, d_dem, d_props, w, h, nodata, xparam)))
}
int rdb200_dev_fa_method_f32_f64(int32_t method, const float *d_dem, double *d_accum, int32_t w, int32_t h, float nodata,
                                 double xparam) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_via_props_dev(method, d_dem, d_accum, w, h, nodata, xparam)))
}
int rdb200_dev_flow_accumulation_props_f64(const float *d_props, double *d_accum, int32_t w, int32_t h) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), flow_accumulation_props_dev(d_props, d_accum, w, h)))
}
int rdb200_dev_fa_d8_f32_f64(const float *d_dem, double *d_accum, int32_t w, int32_t h, float nodata,
                             int32_t ones) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_fused_dev(d_dem, d_accum, w, h, nodata, ones != 0, false)))
}
int rdb200_dev_fa_tarboton_f32_f64(const float *d_dem, double *d_accum, int32_t w, int32_t h, float nodata,
                                   int32_t ones) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_fused_dev(d_dem, d_accum, w, h, nodata, ones != 0, true)))
}
int rdb200_dev_terrain_attribute_f32(int32_t attribute, const float *d_dem, float *d_out, int32_t w, int32_t h, float nodata_in,
                                     float nodata_out, float zscale, double cell_x, double cell_y) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), terrain_attribute_dev(attribute, d_dem, d_out, w, h, nodata_in, nodata_out, zscale,
                                                                    cell_x, cell_y)))
}
// float64 twins of the host entry points above, on device pointers (the reference lines are cited there)
int rdb200_dev_fill_depressions_d8_f64(double *d_dem, int32_t w, int32_t h) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fill_depressions_f64_dev(d_dem, w, h, false)))
}
int rdb200_dev_fill_depressions_d4_f64(double *d_dem, int32_t w, int32_t h) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fill_depressions_f64_dev(d_dem, w, h, true)))
}
static int dev_pit_mask_f64(const double *d_dem, uint8_t *d_mask, int32_t w, int32_t h, double nodata, bool topo4) {
  CAPI_TRY
  if (!d_dem || !d_mask) fail("pit_mask: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  pit_mask_f64_dev(d_dem, d_mask, w, h, nodata, topo4);
  cs.done();
  CAPI_END
}
int rdb200_dev_pit_mask_d8_f64(const double *d_dem, uint8_t *d_mask, int32_t w, int32_t h, double nodata) {
  return dev_pit_mask_f64(d_dem, d_mask, w, h, nodata, false);
}
int rdb200_dev_pit_mask_d4_f64(const double *d_dem, uint8_t *d_mask, int32_t w, int32_t h, double nodata) {
  return dev_pit_mask_f64(d_dem, d_mask, w, h, nodata, true);
}
static int dev_has_depressions_f64(const double *d_dem, int32_t w, int32_t h, int32_t *out, bool topo4) {
  CAPI_TRY
  if (!d_dem || !out) fail("has_depressions: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  const bool any = has_depressions_f64_dev(d_dem, w, h, topo4);
  cs.done();
  *out = any ? 1 : 0;
  CAPI_END
}
int rdb200_dev_has_depressions_d8_f64(const double *d_dem, int32_t w, int32_t h, int32_t *out) {
  return dev_has_depressions_f64(d_dem, w, h, out, false);
}
int rdb200_dev_has_depressions_d4_f64(const double *d_dem, int32_t w, int32_t h, int32_t *out) {
  return dev_has_depressions_f64(d_dem, w, h, out, true);
}
int rdb200_dev_resolve_flats_epsilon_f64(double *d_dem, int32_t w, int32_t h, double nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), resolve_flats_f64_dev(d_dem, w, h, nodata)))
}
int rdb200_dev_d8_flow_directions_f64(const double *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, double nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), d8_flow_directions_f64_dev(d_dem, d_dirs, w, h, nodata)))
}
int rdb200_dev_fa_d8_f64_f64(const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_d8_f64_dev(d_dem, d_accum, w, h, nodata, ones != 0)))
}
int rdb200_dev_fa_d4_f64_f64(const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_d4_f64_dev(d_dem, d_accum, w, h, nodata)))
}
int rdb200_dev_fm_method_f64(int32_t method, const double *d_dem, float *d_props, int32_t w, int32_t h, double nodata,
                             double xparam) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fm_method_f64_dev(method, d_dem, d_props, w, h, nodata, xparam)))
}
int rdb200_dev_fa_method_f64_f64(int32_t method, const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata,
                                 double xparam) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_method_f64_dev(method, d_dem, d_accum, w, h, nodata, xparam)))
}
int rdb200_dev_fa_tarboton_f64_f64(const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), fa_tarboton_f64_dev(d_dem, d_accum, w, h, nodata, ones != 0)))
}
int rdb200_dev_terrain_attribute_f64(int32_t attribute, const double *d_dem, float *d_out, int32_t w, int32_t h,
                                     double nodata_in, float nodata_out, float zscale, double cell_x, double cell_y) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), terrain_attribute_f64_dev(attribute, d_dem, d_out, w, h, nodata_in, nodata_out,
                                                                        zscale, cell_x, cell_y)))
}
int rdb200_dev_f64_order_keys(const double *d_dem, float *d_keys, int32_t w, int32_t h, double nodata, float *nodata_key,
                              int32_t *ranked) {
  CAPI_TRY
  if (!d_dem || !d_keys) fail("f64_order_keys: null pointer");
  check_dims(w, h);
  CallScope cs((int64_t)w * h);
  int r = 0;
  const float nd = f64_keys_dev(d_dem, d_keys, (size_t)w * h, nodata, nullptr, &r);
  cs.done();
  if (nodata_key) *nodata_key = nd;
  if (ranked) *ranked = r;
  CAPI_END
}

int rdb200_dev_generate_fbm_f32(float *d_dem, int32_t w, int32_t h, int32_t y0, uint32_t seed, int32_t octaves,
                                float quantum) {
  DEV_ENTRY((int64_t)w * h, (check_dims(w, h), generate_fbm_dev(d_dem, w, h, y0, seed, octaves, quantum)))
}

int rdb200_mgpu_fill_depressions_d8_f32(const rdb200_comm *comm, float *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                        int32_t row0, int32_t height, int32_t *exchange_rounds) {
  int xr = 0;
  CAPI_TRY
  if (!d_band) fail("mgpu_fill: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_fill_band(comm, d_band, w, rows, gt, gb, row0, height, &xr);
  cs.done();
  if (exchange_rounds) *exchange_rounds = xr;
  CAPI_END
}

int rdb200_mgpu_fill_depressions_d4_f32(const rdb200_comm *comm, float *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                        int32_t row0, int32_t height, int32_t *exchange_rounds) {
  int xr = 0;
  CAPI_TRY
  if (!d_band) fail("mgpu_fill: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_fill_band(comm, d_band, w, rows, gt, gb, row0, height, &xr, true);
  cs.done();
  if (exchange_rounds) *exchange_rounds = xr;
  CAPI_END
}

static int mgpu_pit_mask(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows, float nodata,
                         int32_t gt, int32_t gb, int32_t row0, int32_t height, bool topo4) {
  CAPI_TRY
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_pit_mask_band(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, topo4);
  cs.done();
  CAPI_END
}
int rdb200_mgpu_pit_mask_d8_f32(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows,
                                float nodata, int32_t gt, int32_t gb, int32_t row0, int32_t height) {
  return mgpu_pit_mask(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, false);
}
int rdb200_mgpu_pit_mask_d4_f32(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows,
                                float nodata, int32_t gt, int32_t gb, int32_t row0, int32_t height) {
  return mgpu_pit_mask(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, true);
}
static int mgpu_has_depressions(const rdb200_comm *comm, const float *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                int32_t row0, int32_t height, int32_t *out, bool topo4) {
  CAPI_TRY
  if (!out) fail("mgpu_has_depressions: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  const bool any = mgpu_has_depressions_band(comm, d_band, w, rows, gt, gb, row0, height, topo4);
  cs.done();
  *out = any ? 1 : 0;
  CAPI_END
}
int rdb200_mgpu_has_depressions_d8_f32(const rdb200_comm *comm, const float *d_band, int32_t w, int32_t rows, int32_t gt,
                                       int32_t gb, int32_t row0, int32_t height, int32_t *out) {
  return mgpu_has_depressions(comm, d_band, w, rows, gt, gb, row0, height, out, false);
}
int rdb200_mgpu_has_depressions_d4_f32(const rdb200_comm *comm, const float *d_band, int32_t w, int32_t rows, int32_t gt,
                                       int32_t gb, int32_t row0, int32_t height, int32_t *out) {
  return mgpu_has_depressions(comm, d_band, w, rows, gt, gb, row0, height, out, true);
}

int rdb200_mgpu_fa_f32_f64(const rdb200_comm *comm, const float *d_dem, double *d_accum, int32_t w, int32_t rows, float nodata,
                           int32_t gt, int32_t gb, int32_t dinf, int32_t ones, int32_t *exchange_rounds) {
  int xr = 0;
  CAPI_TRY
  if (!d_dem || !d_accum) fail("mgpu_fa: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_fa_band(comm, d_dem, d_accum, w, rows, nodata, gt, gb, dinf ? 1 : 0, 0.0, ones != 0, &xr);
  cs.done();
  if (exchange_rounds) *exchange_rounds = xr;
  CAPI_END
}

int rdb200_mgpu_fa_method_f32_f64(const rdb200_comm *comm, const float *d_dem, double *d_accum, int32_t w, int32_t rows,
                                  float nodata, int32_t gt, int32_t gb, int32_t method, double xparam, int32_t ones,
                                  int32_t *exchange_rounds) {
  int xr = 0;
  CAPI_TRY
  if (!d_dem || !d_accum) fail("mgpu_fa: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_fa_band(comm, d_dem, d_accum, w, rows, nodata, gt, gb, method, xparam, ones != 0, &xr);
  cs.done();
  if (exchange_rounds) *exchange_rounds = xr;
  CAPI_END
}

// FM_x and TA_x over row bands: one exchange of the DEM's edge rows gives every owned cell its whole 3 x 3 neighbourhood,
// and a local edge row is a raster edge row exactly when it is not a ghost row, so the single-GPU kernel on the local raster
// gives the owned rows the single-GPU bits.  The arguments are checked before the exchange: a rank that fails must not
// leave its neighbours waiting.
int rdb200_mgpu_fm_method_f32(const rdb200_comm *comm, int32_t method, float *d_band_dem, float *d_band_props9, int32_t w,
                              int32_t rows, float nodata, int32_t gt, int32_t gb, double xparam) {
  CAPI_TRY
  const char *what = "mgpu_fm_method";
  if (!d_band_props9) fail("%s: null pointer", what);
  check_band_args(what, comm, d_band_dem, w, rows, gt, gb);
  check_dims(w, rows);
  if (method < 0 || method > 4) fail("unknown flow metric %d", method);
  CallScope cs((int64_t)w * rows);
  exchange_band_rows(comm, d_band_dem, sizeof(float), w, rows, gt, gb);
  fm_dispatch_dev(method, d_band_dem, d_band_props9, w, rows, nodata, xparam);
  cs.done();
  CAPI_END
}

int rdb200_mgpu_terrain_attribute_f32(const rdb200_comm *comm, int32_t attribute, float *d_band_dem, float *d_band_out, int32_t w,
                                      int32_t rows, float nodata_in, float nodata_out, float zscale, double cell_x, double cell_y,
                                      int32_t gt, int32_t gb) {
  CAPI_TRY
  const char *what = "mgpu_terrain_attribute";
  if (!d_band_out) fail("%s: null pointer", what);
  check_band_args(what, comm, d_band_dem, w, rows, gt, gb);
  check_dims(w, rows);
  if (attribute < RDB200_TA_SLOPE_RISERUN || attribute > RDB200_TA_PROFILE_CURVATURE) fail("unknown terrain attribute %d", attribute);
  if (!(cell_x > 0) || !(cell_y > 0)) fail("terrain attribute: cell lengths must be positive (got %g x %g)", cell_x, cell_y);
  CallScope cs((int64_t)w * rows);
  exchange_band_rows(comm, d_band_dem, sizeof(float), w, rows, gt, gb);
  terrain_attribute_dev(attribute, d_band_dem, d_band_out, w, rows, nodata_in, nodata_out, zscale, cell_x, cell_y);
  cs.done();
  CAPI_END
}

int rdb200_mgpu_flow_accumulation_props_f64(const rdb200_comm *comm, float *d_band_props9, double *d_band_accum_inout, int32_t w,
                                            int32_t rows, int32_t gt, int32_t gb, int32_t *exchange_rounds) {
  int xr = 0;
  CAPI_TRY
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_flow_accumulation_props_band(comm, d_band_props9, d_band_accum_inout, w, rows, gt, gb, &xr);
  cs.done();
  if (exchange_rounds) *exchange_rounds = xr;
  CAPI_END
}

int rdb200_mgpu_resolve_flats_epsilon_f32(const rdb200_comm *comm, float *d_band, int32_t w, int32_t rows, float nodata,
                                          int32_t gt, int32_t gb, int32_t *seam_iterations) {
  int it = 0;
  CAPI_TRY
  if (!comm || !d_band) fail("mgpu_resolve_flats: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_resolve_flats_band(comm, d_band, w, rows, nodata, gt, gb, &it);
  cs.done();
  if (seam_iterations) *seam_iterations = it;
  CAPI_END
}

int rdb200_mgpu_d8_flow_directions_flats_f32(const rdb200_comm *comm, float *d_band_dem, uint8_t *d_band_dirs, int32_t w,
                                             int32_t rows, float nodata, int32_t gt, int32_t gb, int32_t alter,
                                             int32_t *seam_iterations) {
  int it = 0;
  CAPI_TRY
  if (!comm || !d_band_dem || !d_band_dirs) fail("mgpu_d8_flow_directions_flats: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_d8_flow_directions_flats_band(comm, d_band_dem, d_band_dirs, w, rows, nodata, gt, gb, alter != 0, &it);
  cs.done();
  if (seam_iterations) *seam_iterations = it;
  CAPI_END
}

int rdb200_mgpu_d8_flow_accum_u8_i32(const rdb200_comm *comm, const uint8_t *d_band_dirs, int32_t *d_band_area, int32_t w,
                                     int32_t rows, int32_t gt, int32_t gb, int32_t *exchange_rounds) {
  int xr = 0;
  CAPI_TRY
  if (!comm || !d_band_dirs || !d_band_area) fail("mgpu_d8_flow_accum: null pointer");
  check_dims(w, rows);
  CallScope cs((int64_t)w * rows);
  mgpu_d8_flow_accum_band(comm, d_band_dirs, d_band_area, w, rows, gt, gb, &xr);
  cs.done();
  if (exchange_rounds) *exchange_rounds = xr;
  CAPI_END
}

}  // extern "C"
