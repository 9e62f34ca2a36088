// C ABI of librichdem_b200.so: context, workspace cache, host<->device staging and the
// extern "C" entry points declared in include/richdem_b200.h.
#include "common.cuh"

#include <algorithm>
#include <cstdlib>
#include <type_traits>

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

// ---- the scope of every entry point on a raster ---------------------------------------------------------------------
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

// a copy on the library's stream, waited for; its time is added to ms (stats.ms_h2d or stats.ms_d2h)
static void timed_copy(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, double &ms) {
  Ctx &c = ctx();
  RDB_CK(cudaEventRecord(c.evk0, c.stream));
  RDB_CK(cudaMemcpyAsync(dst, src, bytes, kind, c.stream));
  RDB_CK(cudaEventRecord(c.evk1, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  float t = 0;
  RDB_CK(cudaEventElapsedTime(&t, c.evk0, c.evk1));
  ms += t;
}

enum class Side { host, device };  // where the arrays an entry point is given live

// The arrays of one entry point.  On the host side they are staged in device workspace: in() uploads, out() only
// allocates, inout() uploads, and copy_back() downloads every out / inout array.  On the device side the caller's
// pointers pass through unchanged.
class Arrays {
 public:
  explicit Arrays(Side side) : host_(side == Side::host) {}
  ~Arrays() {
    for (void *p : bufs_) ws_free(p);
  }
  Arrays(const Arrays &) = delete;
  Arrays &operator=(const Arrays &) = delete;

  template <class T>
  T *in(T *p, size_t n) {
    if (!host_) return p;
    void *d = alloc(n * sizeof(T));
    timed_copy(d, p, n * sizeof(T), cudaMemcpyHostToDevice, ctx().stats.ms_h2d);
    return static_cast<T *>(d);
  }
  template <class T>
  T *out(T *p, size_t n) {
    if (!host_) return p;
    T *d = static_cast<T *>(alloc(n * sizeof(T)));
    back_.push_back({p, d, n * sizeof(T)});
    return d;
  }
  template <class T>
  T *inout(T *p, size_t n) {
    T *d = in(p, n);
    if (host_) back_.push_back({p, d, n * sizeof(T)});
    return d;
  }
  void copy_back() {
    for (const Back &b : back_) timed_copy(b.host, b.dev, b.bytes, cudaMemcpyDeviceToHost, ctx().stats.ms_d2h);
  }

 private:
  struct Back {
    void *host;
    const void *dev;
    size_t bytes;
  };
  void *alloc(size_t bytes) {
    bufs_.push_back(ws_alloc(bytes));
    return bufs_.back();
  }
  bool host_;
  std::vector<void *> bufs_;
  std::vector<Back> back_;
};

// Every entry point on a raster (or a row band of one) runs through here.  Its pointers (null_msg when one is null), its
// further checks and the dimensions are checked before the device is touched, so that a bad call fails alike with and
// without a GPU, and before a band entry point's first exchange, so that a failing rank leaves no neighbour waiting.
// The body then runs in a CallScope on the entry point's Arrays, which are back on the host before the call is timed.
template <class Check, class F>
static int raster_call(Side side, const char *null_msg, std::initializer_list<const void *> ptrs, int w, int h, Check &&check,
                       F &&body) {
  return capi_call([&] {
    for (const void *p : ptrs)
      if (!p) fail("%s", null_msg);
    check();
    check_dims(w, h);
    CallScope cs((int64_t)w * h);
    Arrays a(side);
    body(a, (size_t)w * h);
    a.copy_back();
    cs.done();
  });
}
template <class F>
static int raster_call(Side side, const char *null_msg, std::initializer_list<const void *> ptrs, int w, int h, F &&body) {
  return raster_call(side, null_msg, ptrs, w, h, [] {}, body);
}

// ---- the stages, each for host and device arrays and T = float or double elevations -------------------------------
// A float64 stage runs the float engines on order-preserving float keys (f64.cu) where it only compares elevations, and
// the kernels' double instantiations where it does arithmetic on them (DESIGN §0.1, §0.2).

// reference depressions/depressions.hpp:13-21 -> Zhou2016.hpp:125-191 (D8) / Barnes2014.hpp:230-304 (D4)
template <class T>
static int fill_depressions(Side side, T *dem, int32_t w, int32_t h, bool topo4) {
  return raster_call(side, "fill_depressions: null dem", {dem}, w, h,
                     [&](Arrays &a, size_t n) { fill_depressions_dev(a.inout(dem, n), w, h, topo4); });
}

// reference depressions/Barnes2014.hpp:336-420 (PriorityFloodEpsilon_Barnes2014<topo>): the order-free surface, never
// above the reference's (DESIGN.md section 0, f3)
static int fill_depressions_epsilon(Side side, float *dem, int32_t w, int32_t h, float nodata, bool topo4) {
  return raster_call(side, "fill_depressions_epsilon: null dem", {dem}, w, h,
                     [&](Arrays &a, size_t n) { fill_depressions_epsilon_dev(a.inout(dem, n), w, h, topo4, nodata); });
}

// reference depressions/Barnes2014.hpp:593-676 (pit_mask<topo>)
template <class T>
static int pit_mask(Side side, const T *dem, uint8_t *mask, int32_t w, int32_t h, T nodata, bool topo4) {
  return raster_call(side, "pit_mask: null pointer", {dem, mask}, w, h,
                     [&](Arrays &a, size_t n) { pit_mask_dev(a.in(dem, n), a.out(mask, n), w, h, nodata, topo4); });
}

// reference depressions/Barnes2014.hpp:43-104 (HasDepressions<topo>)
template <class T>
static int has_depressions(Side side, const T *dem, int32_t w, int32_t h, int32_t *out, bool topo4) {
  bool any = false;
  const int rc = raster_call(side, "has_depressions: null pointer", {dem, out}, w, h,
                             [&](Arrays &a, size_t n) { any = has_depressions_dev(a.in(dem, n), w, h, topo4); });
  if (rc == 0) *out = any ? 1 : 0;
  return rc;
}

// reference flats/flats.hpp:21-28 -> flats/Barnes2014.hpp:398-467 (GetFlatMask) + :496-550 (apply)
template <class T>
static int resolve_flats_epsilon(Side side, T *dem, int32_t w, int32_t h, T nodata) {
  return raster_call(side, "resolve_flats: null dem", {dem}, w, h,
                     [&](Arrays &a, size_t n) { resolve_flats_epsilon_dev(a.inout(dem, n), w, h, nodata); });
}

// reference flats/Barnes2014.hpp:398-467 (GetFlatMask)
template <class T>
static int get_flat_mask(Side side, const T *dem, int32_t *flat_mask, int32_t *labels, int32_t w, int32_t h, T nodata) {
  return raster_call(side, "get_flat_mask: null pointer", {dem, flat_mask, labels}, w, h, [&](Arrays &a, size_t n) {
    get_flat_mask_dev(a.in(dem, n), a.out(flat_mask, n), a.out(labels, n), w, h, nodata);
  });
}

// reference flowmet/d8_flowdirs.hpp:32-123 (d8_flow_directions)
template <class T>
static int d8_flow_directions(Side side, const T *dem, uint8_t *dirs, int32_t w, int32_t h, T nodata) {
  return raster_call(side, "d8_flow_directions: null pointer", {dem, dirs}, w, h,
                     [&](Arrays &a, size_t n) { d8_flow_directions_dev(a.in(dem, n), a.out(dirs, n), w, h, nodata); });
}

// reference flats/flat_resolution.hpp:588-607 (barnes_flat_resolution_d8); dem is written only with alter
template <class T>
static int d8_flow_directions_flats(Side side, T *dem, uint8_t *dirs, int32_t w, int32_t h, T nodata, int32_t alter) {
  return raster_call(side, "d8_flow_directions_flats: null pointer", {dem, dirs}, w, h, [&](Arrays &a, size_t n) {
    d8_flow_directions_flats_dev(alter ? a.inout(dem, n) : a.in(dem, n), a.out(dirs, n), w, h, nodata, alter != 0);
  });
}

static int d8_flow_accum(Side side, const uint8_t *dirs, int32_t *area, int32_t w, int32_t h) {
  return raster_call(side, "d8_flow_accum: null pointer", {dirs, area}, w, h,
                     [&](Arrays &a, size_t n) { d8_flow_accum_dev(a.in(dirs, n), a.out(area, n), w, h); });
}

// method: 0 FM_D8, 1 FM_Tarboton, 2 FM_D4, 3 FM_Holmgren (FM_Quinn = exponent 1), 4 FM_Freeman
template <class T>
static int fm(Side side, int method, const T *dem, float *props, int32_t w, int32_t h, T nodata, double xparam = 0) {
  return raster_call(side, "flow metric: null pointer", {dem, props}, w, h, [&](Arrays &a, size_t n) {
    fm_method_dev(method, a.in(dem, n), a.out(props, 9 * n), w, h, nodata, xparam);
  });
}

// TA_* (reference methods/terrain_attributes.hpp:370-538): one stencil pass, sizeof(T) B in + 4 B out per cell
template <class T>
static int terrain_attribute(Side side, int32_t attribute, const T *dem, float *out, int32_t w, int32_t h, T nodata_in,
                             float nodata_out, float zscale, double cell_x, double cell_y) {
  return raster_call(side, "terrain attribute: null pointer", {dem, out}, w, h, [&](Arrays &a, size_t n) {
    terrain_attribute_dev(attribute, a.in(dem, n), a.out(out, n), w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
  });
}

// FA_<metric> = FM_<metric> into a device-side proportions array + the generic accumulation
// (reference methods/flow_accumulation.hpp:18-20,28: `Array3D<float> props(elevations); FM_x(...); FlowAccumulation(...)`).
// On doubles, D8 and D4 compare elevations only and take the key route: FA_D8 by the fused engine, FA_D4 by the float
// FM_D4 of the keys (accum holds the weights).
template <class T>
static void fa_via_props_dev(int method, const T *d_dem, double *d_accum, int w, int h, T nodata, double xparam) {
  if constexpr (std::is_same_v<T, double>) {
    if (method == 0) return fa_fused_dev(d_dem, d_accum, w, h, nodata, false, false);
    if (method == 2) {
      DevBuf<float> key((size_t)w * h);
      const float nd = f64_keys_dev(d_dem, key.p, (size_t)w * h, nodata, nullptr, nullptr);
      return fa_via_props_dev(2, key.p, d_accum, w, h, nd, 0.0);
    }
  }
  DevBuf<float> p(9 * (size_t)w * h);
  fm_method_dev(method, d_dem, p.p, w, h, nodata, xparam);
  flow_accumulation_props_dev(p.p, d_accum, w, h);
}
template <class T>
static int fa_via_props(Side side, int method, const T *dem, double *accum, int32_t w, int32_t h, T nodata, double xparam) {
  return raster_call(side, "flow accumulation: null pointer", {dem, accum}, w, h, [&](Arrays &a, size_t n) {
    fa_via_props_dev(method, a.in(dem, n), a.inout(accum, n), w, h, nodata, xparam);
  });
}

static int flow_accumulation_props(Side side, const float *props, double *accum, int32_t w, int32_t h) {
  return raster_call(side, "flow_accumulation: null pointer", {props, accum}, w, h, [&](Arrays &a, size_t n) {
    flow_accumulation_props_dev(a.in(props, 9 * n), a.inout(accum, n), w, h);
  });
}

// FA_D8 / FA_Tarboton by the fused engines; with ones the accumulator is not read, only written
template <class T>
static int fa_fused(Side side, const T *dem, double *accum, int32_t w, int32_t h, T nodata, int32_t ones, bool dinf) {
  return raster_call(side, "flow accumulation: null pointer", {dem, accum}, w, h, [&](Arrays &a, size_t n) {
    fa_fused_dev(a.in(dem, n), ones ? a.out(accum, n) : a.inout(accum, n), w, h, nodata, ones != 0, dinf);
  });
}

// kappa itself: the float keys the float64 stages run the float engines on, kappa(nodata) and which case ran
static int f64_order_keys(Side side, const double *dem, float *keys, int32_t w, int32_t h, double nodata, float *nodata_key,
                          int32_t *ranked) {
  float nd = 0;
  int r = 0;
  const int rc = raster_call(side, "f64_order_keys: null pointer", {dem, keys}, w, h, [&](Arrays &a, size_t n) {
    nd = f64_keys_dev(a.in(dem, n), a.out(keys, n), n, nodata, nullptr, &r);
  });
  if (rc == 0 && nodata_key) *nodata_key = nd;
  if (rc == 0 && ranked) *ranked = r;
  return rc;
}

// ---- row bands: the drivers take device pointers and check the band geometry themselves; the float64 drivers check
// every argument before kappa_G's first collective ------------------------------------------------------------------

template <class T>
static int mgpu_fill(const rdb200_comm *comm, T *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb, int32_t row0,
                     int32_t height, int32_t *exchange_rounds, bool topo4) {
  int xr = 0;
  const int rc = raster_call(Side::device, "mgpu_fill: null pointer", {d_band}, w, rows, [&](Arrays &, size_t) {
    mgpu_fill_band(comm, d_band, w, rows, gt, gb, row0, height, &xr, topo4);
  });
  if (rc == 0 && exchange_rounds) *exchange_rounds = xr;
  return rc;
}

template <class T>
static int mgpu_pit_mask(const rdb200_comm *comm, const T *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows, T nodata,
                         int32_t gt, int32_t gb, int32_t row0, int32_t height, bool topo4) {
  return raster_call(Side::device, "mgpu_pit_mask: null pointer", {comm, d_band, d_band_mask}, w, rows, [&](Arrays &, size_t) {
    mgpu_pit_mask_band(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, topo4);
  });
}

template <class T>
static int mgpu_has_depressions(const rdb200_comm *comm, const T *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                int32_t row0, int32_t height, int32_t *out, bool topo4) {
  bool any = false;
  const int rc = raster_call(Side::device, "mgpu_has_depressions: null pointer", {comm, d_band, out}, w, rows,
                             [&](Arrays &, size_t) {
                               any = mgpu_has_depressions_band(comm, d_band, w, rows, gt, gb, row0, height, topo4);
                             });
  if (rc == 0) *out = any ? 1 : 0;
  return rc;
}

template <class T>
static int mgpu_resolve_flats_epsilon(const rdb200_comm *comm, T *d_band, int32_t w, int32_t rows, T nodata, int32_t gt,
                                      int32_t gb, int32_t *seam_iterations) {
  int it = 0;
  const int rc = raster_call(Side::device, "mgpu_resolve_flats: null pointer", {comm, d_band}, w, rows,
                             [&](Arrays &, size_t) { mgpu_resolve_flats_band(comm, d_band, w, rows, nodata, gt, gb, &it); });
  if (rc == 0 && seam_iterations) *seam_iterations = it;
  return rc;
}

template <class T>
static int mgpu_d8_flow_directions_flats(const rdb200_comm *comm, T *d_band_dem, uint8_t *d_band_dirs, int32_t w, int32_t rows,
                                         T nodata, int32_t gt, int32_t gb, int32_t alter, int32_t *seam_iterations) {
  int it = 0;
  const int rc = raster_call(Side::device, "mgpu_d8_flow_directions_flats: null pointer", {comm, d_band_dem, d_band_dirs}, w, rows,
                             [&](Arrays &, size_t) {
                               mgpu_d8_flow_directions_flats_band(comm, d_band_dem, d_band_dirs, w, rows, nodata, gt, gb,
                                                                  alter != 0, &it);
                             });
  if (rc == 0 && seam_iterations) *seam_iterations = it;
  return rc;
}

// FM_x and TA_x over row bands: one exchange of the DEM's edge rows gives every owned cell its whole 3 x 3 neighbourhood,
// and a local edge row is a raster edge row exactly when it is not a ghost row, so the single-GPU kernel on the local raster
// gives the owned rows the single-GPU bits.
template <class T>
static int mgpu_fm_method(const rdb200_comm *comm, int32_t method, T *d_band_dem, float *d_band_props9, int32_t w, int32_t rows,
                          T nodata, int32_t gt, int32_t gb, double xparam) {
  return raster_call(
      Side::device, "mgpu_fm_method: null pointer", {d_band_props9, comm, d_band_dem}, w, rows,
      [&] {
        check_band_args("mgpu_fm_method", comm, d_band_dem, w, rows, gt, gb);
        if (method < 0 || method > 4) fail("unknown flow metric %d", method);
      },
      [&](Arrays &, size_t) {
        exchange_band_rows(comm, d_band_dem, sizeof(T), w, rows, gt, gb);
        fm_method_dev(method, d_band_dem, d_band_props9, w, rows, nodata, xparam);
      });
}

template <class T>
static int mgpu_terrain_attribute(const rdb200_comm *comm, int32_t attribute, T *d_band_dem, float *d_band_out, int32_t w,
                                  int32_t rows, T nodata_in, float nodata_out, float zscale, double cell_x, double cell_y,
                                  int32_t gt, int32_t gb) {
  return raster_call(
      Side::device, "mgpu_terrain_attribute: null pointer", {d_band_out, comm, d_band_dem}, w, rows,
      [&] {
        check_band_args("mgpu_terrain_attribute", comm, d_band_dem, w, rows, gt, gb);
        if (attribute < RDB200_TA_SLOPE_RISERUN || attribute > RDB200_TA_PROFILE_CURVATURE)
          fail("unknown terrain attribute %d", attribute);
        if (!(cell_x > 0) || !(cell_y > 0))
          fail("terrain attribute: cell lengths must be positive (got %g x %g)", cell_x, cell_y);
      },
      [&](Arrays &, size_t) {
        exchange_band_rows(comm, d_band_dem, sizeof(T), w, rows, gt, gb);
        terrain_attribute_dev(attribute, d_band_dem, d_band_out, w, rows, nodata_in, nodata_out, zscale, cell_x, cell_y);
      });
}

// The float32 driver checks the method as it begins; the float64 driver needs the communicator, the band and the method
// checked before kappa_G's first collective.
template <class T>
static int mgpu_fa_method(const rdb200_comm *comm, const T *d_dem, double *d_accum, int32_t w, int32_t rows, T nodata, int32_t gt,
                          int32_t gb, int32_t method, double xparam, int32_t ones, int32_t *exchange_rounds) {
  constexpr bool keyed = std::is_same_v<T, double>;
  int xr = 0;
  const int rc = raster_call(
      Side::device, "mgpu_fa: null pointer", {keyed ? (const void *)comm : d_dem, d_dem, d_accum}, w, rows,
      [&] {
        if (!keyed) return;
        check_band_args("mgpu_fa", comm, d_dem, w, rows, gt, gb);
        check_fa_method(method, xparam);
      },
      [&](Arrays &, size_t) { mgpu_fa_band(comm, d_dem, d_accum, w, rows, nodata, gt, gb, method, xparam, ones != 0, &xr); });
  if (rc == 0 && exchange_rounds) *exchange_rounds = xr;
  return rc;
}

}  // namespace rdb

using namespace rdb;

extern "C" {

int rdb200_init(int device) {
  return capi_call([&] { init_device(device); });
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
  return capi_call([&] {
    ensure_init();
    Ctx &c = ctx();
    RDB_CK(cudaStreamSynchronize(c.stream));
    c.stream = cuda_stream ? (cudaStream_t)cuda_stream : c.own_stream;
  });
}

int rdb200_get_stats(rdb200_stats *out) {
  return capi_call([&] {
    if (!out) fail("rdb200_get_stats: null pointer");
    *out = ctx().stats;
  });
}

int rdb200_set_param(const char *name, int64_t value) {
  return capi_call([&] {
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
    else if (n == "f64_band_rank_cap") p.f64_band_rank_cap = value;
    else fail("rdb200_set_param: unknown parameter '%s'", name);
  });
}

// ---- host entry points ------------------------------------------------------------------------

int rdb200_fill_depressions_d8_f32(float *dem, int32_t w, int32_t h) { return fill_depressions(Side::host, dem, w, h, false); }
int rdb200_fill_depressions_d4_f32(float *dem, int32_t w, int32_t h) { return fill_depressions(Side::host, dem, w, h, true); }
int rdb200_fill_depressions_epsilon_d8_f32(float *dem, int32_t w, int32_t h, float nodata) {
  return fill_depressions_epsilon(Side::host, dem, w, h, nodata, false);
}
int rdb200_fill_depressions_epsilon_d4_f32(float *dem, int32_t w, int32_t h, float nodata) {
  return fill_depressions_epsilon(Side::host, dem, w, h, nodata, true);
}
int rdb200_pit_mask_d8_f32(const float *dem, uint8_t *mask, int32_t w, int32_t h, float nodata) {
  return pit_mask(Side::host, dem, mask, w, h, nodata, false);
}
int rdb200_pit_mask_d4_f32(const float *dem, uint8_t *mask, int32_t w, int32_t h, float nodata) {
  return pit_mask(Side::host, dem, mask, w, h, nodata, true);
}
int rdb200_has_depressions_d8_f32(const float *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::host, dem, w, h, out, false);
}
int rdb200_has_depressions_d4_f32(const float *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::host, dem, w, h, out, true);
}
int rdb200_resolve_flats_epsilon_f32(float *dem, int32_t w, int32_t h, float nodata) {
  return resolve_flats_epsilon(Side::host, dem, w, h, nodata);
}
int rdb200_get_flat_mask_f32(const float *dem, int32_t *flat_mask, int32_t *labels, int32_t w, int32_t h, float nodata) {
  return get_flat_mask(Side::host, dem, flat_mask, labels, w, h, nodata);
}
int rdb200_d8_flow_directions_f32(const float *dem, uint8_t *dirs, int32_t w, int32_t h, float nodata) {
  return d8_flow_directions(Side::host, dem, dirs, w, h, nodata);
}
int rdb200_d8_flow_directions_flats_f32(float *dem, uint8_t *dirs, int32_t w, int32_t h, float nodata, int32_t alter) {
  return d8_flow_directions_flats(Side::host, dem, dirs, w, h, nodata, alter);
}
int rdb200_d8_flow_accum_u8_i32(const uint8_t *dirs, int32_t *area, int32_t w, int32_t h) {
  return d8_flow_accum(Side::host, dirs, area, w, h);
}
int rdb200_fm_d8_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm(Side::host, 0, dem, props, w, h, nodata);
}
int rdb200_fm_tarboton_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm(Side::host, 1, dem, props, w, h, nodata);
}
int rdb200_fm_d4_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm(Side::host, 2, dem, props, w, h, nodata);
}
int rdb200_fm_quinn_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata) {
  return fm(Side::host, 3, dem, props, w, h, nodata, 1.0);
}
int rdb200_fm_holmgren_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata, double xparam) {
  return fm(Side::host, 3, dem, props, w, h, nodata, xparam);
}
int rdb200_fm_freeman_f32(const float *dem, float *props, int32_t w, int32_t h, float nodata, double xparam) {
  return fm(Side::host, 4, dem, props, w, h, nodata, xparam);
}
int rdb200_terrain_attribute_f32(int32_t attribute, const float *dem, float *out, int32_t w, int32_t h, float nodata_in,
                                 float nodata_out, float zscale, double cell_x, double cell_y) {
  return terrain_attribute(Side::host, attribute, dem, out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
}
int rdb200_fa_d4_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata) {
  return fa_via_props(Side::host, 2, dem, accum, w, h, nodata, 0);
}
int rdb200_fa_quinn_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata) {
  return fa_via_props(Side::host, 3, dem, accum, w, h, nodata, 1.0);
}
int rdb200_fa_holmgren_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, double xparam) {
  return fa_via_props(Side::host, 3, dem, accum, w, h, nodata, xparam);
}
int rdb200_fa_freeman_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, double xparam) {
  return fa_via_props(Side::host, 4, dem, accum, w, h, nodata, xparam);
}
int rdb200_flow_accumulation_props_f64(const float *props, double *accum, int32_t w, int32_t h) {
  return flow_accumulation_props(Side::host, props, accum, w, h);
}
int rdb200_fa_d8_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, int32_t ones) {
  return fa_fused(Side::host, dem, accum, w, h, nodata, ones, false);
}
int rdb200_fa_tarboton_f32_f64(const float *dem, double *accum, int32_t w, int32_t h, float nodata, int32_t ones) {
  return fa_fused(Side::host, dem, accum, w, h, nodata, ones, true);
}

int rdb200_fill_depressions_d8_f64(double *dem, int32_t w, int32_t h) { return fill_depressions(Side::host, dem, w, h, false); }
int rdb200_fill_depressions_d4_f64(double *dem, int32_t w, int32_t h) { return fill_depressions(Side::host, dem, w, h, true); }
int rdb200_pit_mask_d8_f64(const double *dem, uint8_t *mask, int32_t w, int32_t h, double nodata) {
  return pit_mask(Side::host, dem, mask, w, h, nodata, false);
}
int rdb200_pit_mask_d4_f64(const double *dem, uint8_t *mask, int32_t w, int32_t h, double nodata) {
  return pit_mask(Side::host, dem, mask, w, h, nodata, true);
}
int rdb200_has_depressions_d8_f64(const double *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::host, dem, w, h, out, false);
}
int rdb200_has_depressions_d4_f64(const double *dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::host, dem, w, h, out, true);
}
int rdb200_resolve_flats_epsilon_f64(double *dem, int32_t w, int32_t h, double nodata) {
  return resolve_flats_epsilon(Side::host, dem, w, h, nodata);
}
int rdb200_d8_flow_directions_f64(const double *dem, uint8_t *dirs, int32_t w, int32_t h, double nodata) {
  return d8_flow_directions(Side::host, dem, dirs, w, h, nodata);
}
int rdb200_get_flat_mask_f64(const double *dem, int32_t *flat_mask, int32_t *labels, int32_t w, int32_t h, double nodata) {
  return get_flat_mask(Side::host, dem, flat_mask, labels, w, h, nodata);
}
int rdb200_d8_flow_directions_flats_f64(double *dem, uint8_t *dirs, int32_t w, int32_t h, double nodata, int32_t alter) {
  return d8_flow_directions_flats(Side::host, dem, dirs, w, h, nodata, alter);
}
int rdb200_fa_d8_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  return fa_fused(Side::host, dem, accum, w, h, nodata, ones, false);
}
int rdb200_fa_d4_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata) {
  return fa_via_props(Side::host, 2, dem, accum, w, h, nodata, 0);
}
int rdb200_fm_d8_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm(Side::host, 0, dem, props, w, h, nodata);
}
int rdb200_fm_tarboton_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm(Side::host, 1, dem, props, w, h, nodata);
}
int rdb200_fm_d4_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm(Side::host, 2, dem, props, w, h, nodata);
}
int rdb200_fm_quinn_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata) {
  return fm(Side::host, 3, dem, props, w, h, nodata, 1.0);
}
int rdb200_fm_holmgren_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata, double xparam) {
  return fm(Side::host, 3, dem, props, w, h, nodata, xparam);
}
int rdb200_fm_freeman_f64(const double *dem, float *props, int32_t w, int32_t h, double nodata, double xparam) {
  return fm(Side::host, 4, dem, props, w, h, nodata, xparam);
}
int rdb200_fa_quinn_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata) {
  return fa_via_props(Side::host, 3, dem, accum, w, h, nodata, 1.0);
}
int rdb200_fa_holmgren_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, double xparam) {
  return fa_via_props(Side::host, 3, dem, accum, w, h, nodata, xparam);
}
int rdb200_fa_freeman_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, double xparam) {
  return fa_via_props(Side::host, 4, dem, accum, w, h, nodata, xparam);
}
int rdb200_fa_tarboton_f64_f64(const double *dem, double *accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  return fa_fused(Side::host, dem, accum, w, h, nodata, ones, true);
}
int rdb200_terrain_attribute_f64(int32_t attribute, const double *dem, float *out, int32_t w, int32_t h, double nodata_in,
                                 float nodata_out, float zscale, double cell_x, double cell_y) {
  return terrain_attribute(Side::host, attribute, dem, out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
}
int rdb200_f64_order_keys(const double *dem, float *keys, int32_t w, int32_t h, double nodata, float *nodata_key,
                          int32_t *ranked) {
  return f64_order_keys(Side::host, dem, keys, w, h, nodata, nodata_key, ranked);
}

// ---- device entry points ------------------------------------------------------------------------

int rdb200_dev_fill_depressions_d8_f32(float *d_dem, int32_t w, int32_t h) {
  return fill_depressions(Side::device, d_dem, w, h, false);
}
int rdb200_dev_fill_depressions_d4_f32(float *d_dem, int32_t w, int32_t h) {
  return fill_depressions(Side::device, d_dem, w, h, true);
}
int rdb200_dev_fill_depressions_epsilon_d8_f32(float *d_dem, int32_t w, int32_t h, float nodata) {
  return fill_depressions_epsilon(Side::device, d_dem, w, h, nodata, false);
}
int rdb200_dev_fill_depressions_epsilon_d4_f32(float *d_dem, int32_t w, int32_t h, float nodata) {
  return fill_depressions_epsilon(Side::device, d_dem, w, h, nodata, true);
}
int rdb200_dev_pit_mask_d8_f32(const float *d_dem, uint8_t *d_mask, int32_t w, int32_t h, float nodata) {
  return pit_mask(Side::device, d_dem, d_mask, w, h, nodata, false);
}
int rdb200_dev_pit_mask_d4_f32(const float *d_dem, uint8_t *d_mask, int32_t w, int32_t h, float nodata) {
  return pit_mask(Side::device, d_dem, d_mask, w, h, nodata, true);
}
int rdb200_dev_has_depressions_d8_f32(const float *d_dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::device, d_dem, w, h, out, false);
}
int rdb200_dev_has_depressions_d4_f32(const float *d_dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::device, d_dem, w, h, out, true);
}
int rdb200_dev_resolve_flats_epsilon_f32(float *d_dem, int32_t w, int32_t h, float nodata) {
  return resolve_flats_epsilon(Side::device, d_dem, w, h, nodata);
}
int rdb200_dev_d8_flow_directions_f32(const float *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, float nodata) {
  return d8_flow_directions(Side::device, d_dem, d_dirs, w, h, nodata);
}
int rdb200_dev_d8_flow_directions_flats_f32(float *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, float nodata, int32_t alter) {
  return d8_flow_directions_flats(Side::device, d_dem, d_dirs, w, h, nodata, alter);
}
int rdb200_dev_d8_flow_accum_u8_i32(const uint8_t *d_dirs, int32_t *d_area, int32_t w, int32_t h) {
  return d8_flow_accum(Side::device, d_dirs, d_area, w, h);
}
int rdb200_dev_fm_d8_f32(const float *d_dem, float *d_props, int32_t w, int32_t h, float nodata) {
  return fm(Side::device, 0, d_dem, d_props, w, h, nodata);
}
int rdb200_dev_fm_tarboton_f32(const float *d_dem, float *d_props, int32_t w, int32_t h, float nodata) {
  return fm(Side::device, 1, d_dem, d_props, w, h, nodata);
}
int rdb200_dev_fm_method_f32(int32_t method, const float *d_dem, float *d_props, int32_t w, int32_t h, float nodata,
                             double xparam) {
  return fm(Side::device, method, d_dem, d_props, w, h, nodata, xparam);
}
int rdb200_dev_fa_method_f32_f64(int32_t method, const float *d_dem, double *d_accum, int32_t w, int32_t h, float nodata,
                                 double xparam) {
  return fa_via_props(Side::device, method, d_dem, d_accum, w, h, nodata, xparam);
}
int rdb200_dev_flow_accumulation_props_f64(const float *d_props, double *d_accum, int32_t w, int32_t h) {
  return flow_accumulation_props(Side::device, d_props, d_accum, w, h);
}
int rdb200_dev_fa_d8_f32_f64(const float *d_dem, double *d_accum, int32_t w, int32_t h, float nodata, int32_t ones) {
  return fa_fused(Side::device, d_dem, d_accum, w, h, nodata, ones, false);
}
int rdb200_dev_fa_tarboton_f32_f64(const float *d_dem, double *d_accum, int32_t w, int32_t h, float nodata, int32_t ones) {
  return fa_fused(Side::device, d_dem, d_accum, w, h, nodata, ones, true);
}
int rdb200_dev_terrain_attribute_f32(int32_t attribute, const float *d_dem, float *d_out, int32_t w, int32_t h, float nodata_in,
                                     float nodata_out, float zscale, double cell_x, double cell_y) {
  return terrain_attribute(Side::device, attribute, d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
}

int rdb200_dev_fill_depressions_d8_f64(double *d_dem, int32_t w, int32_t h) {
  return fill_depressions(Side::device, d_dem, w, h, false);
}
int rdb200_dev_fill_depressions_d4_f64(double *d_dem, int32_t w, int32_t h) {
  return fill_depressions(Side::device, d_dem, w, h, true);
}
int rdb200_dev_pit_mask_d8_f64(const double *d_dem, uint8_t *d_mask, int32_t w, int32_t h, double nodata) {
  return pit_mask(Side::device, d_dem, d_mask, w, h, nodata, false);
}
int rdb200_dev_pit_mask_d4_f64(const double *d_dem, uint8_t *d_mask, int32_t w, int32_t h, double nodata) {
  return pit_mask(Side::device, d_dem, d_mask, w, h, nodata, true);
}
int rdb200_dev_has_depressions_d8_f64(const double *d_dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::device, d_dem, w, h, out, false);
}
int rdb200_dev_has_depressions_d4_f64(const double *d_dem, int32_t w, int32_t h, int32_t *out) {
  return has_depressions(Side::device, d_dem, w, h, out, true);
}
int rdb200_dev_resolve_flats_epsilon_f64(double *d_dem, int32_t w, int32_t h, double nodata) {
  return resolve_flats_epsilon(Side::device, d_dem, w, h, nodata);
}
int rdb200_dev_d8_flow_directions_f64(const double *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, double nodata) {
  return d8_flow_directions(Side::device, d_dem, d_dirs, w, h, nodata);
}
int rdb200_dev_d8_flow_directions_flats_f64(double *d_dem, uint8_t *d_dirs, int32_t w, int32_t h, double nodata, int32_t alter) {
  return d8_flow_directions_flats(Side::device, d_dem, d_dirs, w, h, nodata, alter);
}
int rdb200_dev_fa_d8_f64_f64(const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  return fa_fused(Side::device, d_dem, d_accum, w, h, nodata, ones, false);
}
int rdb200_dev_fa_d4_f64_f64(const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata) {
  return fa_via_props(Side::device, 2, d_dem, d_accum, w, h, nodata, 0);
}
int rdb200_dev_fm_method_f64(int32_t method, const double *d_dem, float *d_props, int32_t w, int32_t h, double nodata,
                             double xparam) {
  return fm(Side::device, method, d_dem, d_props, w, h, nodata, xparam);
}
int rdb200_dev_fa_method_f64_f64(int32_t method, const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata,
                                 double xparam) {
  return fa_via_props(Side::device, method, d_dem, d_accum, w, h, nodata, xparam);
}
int rdb200_dev_fa_tarboton_f64_f64(const double *d_dem, double *d_accum, int32_t w, int32_t h, double nodata, int32_t ones) {
  return fa_fused(Side::device, d_dem, d_accum, w, h, nodata, ones, true);
}
int rdb200_dev_terrain_attribute_f64(int32_t attribute, const double *d_dem, float *d_out, int32_t w, int32_t h,
                                     double nodata_in, float nodata_out, float zscale, double cell_x, double cell_y) {
  return terrain_attribute(Side::device, attribute, d_dem, d_out, w, h, nodata_in, nodata_out, zscale, cell_x, cell_y);
}
int rdb200_dev_f64_order_keys(const double *d_dem, float *d_keys, int32_t w, int32_t h, double nodata, float *nodata_key,
                              int32_t *ranked) {
  return f64_order_keys(Side::device, d_dem, d_keys, w, h, nodata, nodata_key, ranked);
}

int rdb200_dev_generate_fbm_f32(float *d_dem, int32_t w, int32_t h, int32_t y0, uint32_t seed, int32_t octaves,
                                float quantum) {
  return raster_call(Side::device, "generate_fbm: null pointer", {d_dem}, w, h,
                     [&](Arrays &, size_t) { generate_fbm_dev(d_dem, w, h, y0, seed, octaves, quantum); });
}

// ---- row-band entry points ----------------------------------------------------------------------

int rdb200_mgpu_fill_depressions_d8_f32(const rdb200_comm *comm, float *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                        int32_t row0, int32_t height, int32_t *exchange_rounds) {
  return mgpu_fill(comm, d_band, w, rows, gt, gb, row0, height, exchange_rounds, false);
}
int rdb200_mgpu_fill_depressions_d4_f32(const rdb200_comm *comm, float *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                        int32_t row0, int32_t height, int32_t *exchange_rounds) {
  return mgpu_fill(comm, d_band, w, rows, gt, gb, row0, height, exchange_rounds, true);
}

int rdb200_mgpu_pit_mask_d8_f32(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows,
                                float nodata, int32_t gt, int32_t gb, int32_t row0, int32_t height) {
  return mgpu_pit_mask(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, false);
}
int rdb200_mgpu_pit_mask_d4_f32(const rdb200_comm *comm, const float *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows,
                                float nodata, int32_t gt, int32_t gb, int32_t row0, int32_t height) {
  return mgpu_pit_mask(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, true);
}
int rdb200_mgpu_has_depressions_d8_f32(const rdb200_comm *comm, const float *d_band, int32_t w, int32_t rows, int32_t gt,
                                       int32_t gb, int32_t row0, int32_t height, int32_t *out) {
  return mgpu_has_depressions(comm, d_band, w, rows, gt, gb, row0, height, out, false);
}
int rdb200_mgpu_has_depressions_d4_f32(const rdb200_comm *comm, const float *d_band, int32_t w, int32_t rows, int32_t gt,
                                       int32_t gb, int32_t row0, int32_t height, int32_t *out) {
  return mgpu_has_depressions(comm, d_band, w, rows, gt, gb, row0, height, out, true);
}

int rdb200_mgpu_fa_method_f32_f64(const rdb200_comm *comm, const float *d_dem, double *d_accum, int32_t w, int32_t rows,
                                  float nodata, int32_t gt, int32_t gb, int32_t method, double xparam, int32_t ones,
                                  int32_t *exchange_rounds) {
  return mgpu_fa_method(comm, d_dem, d_accum, w, rows, nodata, gt, gb, method, xparam, ones, exchange_rounds);
}
int rdb200_mgpu_fa_f32_f64(const rdb200_comm *comm, const float *d_dem, double *d_accum, int32_t w, int32_t rows, float nodata,
                           int32_t gt, int32_t gb, int32_t dinf, int32_t ones, int32_t *exchange_rounds) {
  return rdb200_mgpu_fa_method_f32_f64(comm, d_dem, d_accum, w, rows, nodata, gt, gb, dinf ? 1 : 0, 0.0, ones, exchange_rounds);
}

int rdb200_mgpu_fm_method_f32(const rdb200_comm *comm, int32_t method, float *d_band_dem, float *d_band_props9, int32_t w,
                              int32_t rows, float nodata, int32_t gt, int32_t gb, double xparam) {
  return mgpu_fm_method(comm, method, d_band_dem, d_band_props9, w, rows, nodata, gt, gb, xparam);
}

int rdb200_mgpu_terrain_attribute_f32(const rdb200_comm *comm, int32_t attribute, float *d_band_dem, float *d_band_out, int32_t w,
                                      int32_t rows, float nodata_in, float nodata_out, float zscale, double cell_x, double cell_y,
                                      int32_t gt, int32_t gb) {
  return mgpu_terrain_attribute(comm, attribute, d_band_dem, d_band_out, w, rows, nodata_in, nodata_out, zscale, cell_x,
                                cell_y, gt, gb);
}

int rdb200_mgpu_flow_accumulation_props_f64(const rdb200_comm *comm, float *d_band_props9, double *d_band_accum_inout, int32_t w,
                                            int32_t rows, int32_t gt, int32_t gb, int32_t *exchange_rounds) {
  int xr = 0;
  const int rc = raster_call(Side::device, "mgpu_flow_accumulation_props: null pointer", {comm, d_band_props9, d_band_accum_inout},
                             w, rows, [&](Arrays &, size_t) {
                               mgpu_flow_accumulation_props_band(comm, d_band_props9, d_band_accum_inout, w, rows, gt, gb, &xr);
                             });
  if (rc == 0 && exchange_rounds) *exchange_rounds = xr;
  return rc;
}

int rdb200_mgpu_resolve_flats_epsilon_f32(const rdb200_comm *comm, float *d_band, int32_t w, int32_t rows, float nodata,
                                          int32_t gt, int32_t gb, int32_t *seam_iterations) {
  return mgpu_resolve_flats_epsilon(comm, d_band, w, rows, nodata, gt, gb, seam_iterations);
}

int rdb200_mgpu_d8_flow_directions_flats_f32(const rdb200_comm *comm, float *d_band_dem, uint8_t *d_band_dirs, int32_t w,
                                             int32_t rows, float nodata, int32_t gt, int32_t gb, int32_t alter,
                                             int32_t *seam_iterations) {
  return mgpu_d8_flow_directions_flats(comm, d_band_dem, d_band_dirs, w, rows, nodata, gt, gb, alter, seam_iterations);
}

int rdb200_mgpu_d8_flow_accum_u8_i32(const rdb200_comm *comm, const uint8_t *d_band_dirs, int32_t *d_band_area, int32_t w,
                                     int32_t rows, int32_t gt, int32_t gb, int32_t *exchange_rounds) {
  int xr = 0;
  const int rc = raster_call(Side::device, "mgpu_d8_flow_accum: null pointer", {comm, d_band_dirs, d_band_area}, w, rows,
                             [&](Arrays &, size_t) { mgpu_d8_flow_accum_band(comm, d_band_dirs, d_band_area, w, rows, gt, gb, &xr); });
  if (rc == 0 && exchange_rounds) *exchange_rounds = xr;
  return rc;
}

// ---- float64 row bands (f64_band.cu): the float32 band drivers on kappa_G, and the double flow metrics and attributes --

int rdb200_mgpu_fill_depressions_d8_f64(const rdb200_comm *comm, double *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                        int32_t row0, int32_t height, int32_t *exchange_rounds) {
  return mgpu_fill(comm, d_band, w, rows, gt, gb, row0, height, exchange_rounds, false);
}
int rdb200_mgpu_fill_depressions_d4_f64(const rdb200_comm *comm, double *d_band, int32_t w, int32_t rows, int32_t gt, int32_t gb,
                                        int32_t row0, int32_t height, int32_t *exchange_rounds) {
  return mgpu_fill(comm, d_band, w, rows, gt, gb, row0, height, exchange_rounds, true);
}
int rdb200_mgpu_pit_mask_d8_f64(const rdb200_comm *comm, const double *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows,
                                double nodata, int32_t gt, int32_t gb, int32_t row0, int32_t height) {
  return mgpu_pit_mask(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, false);
}
int rdb200_mgpu_pit_mask_d4_f64(const rdb200_comm *comm, const double *d_band, uint8_t *d_band_mask, int32_t w, int32_t rows,
                                double nodata, int32_t gt, int32_t gb, int32_t row0, int32_t height) {
  return mgpu_pit_mask(comm, d_band, d_band_mask, w, rows, nodata, gt, gb, row0, height, true);
}
int rdb200_mgpu_has_depressions_d8_f64(const rdb200_comm *comm, const double *d_band, int32_t w, int32_t rows, int32_t gt,
                                       int32_t gb, int32_t row0, int32_t height, int32_t *out) {
  return mgpu_has_depressions(comm, d_band, w, rows, gt, gb, row0, height, out, false);
}
int rdb200_mgpu_has_depressions_d4_f64(const rdb200_comm *comm, const double *d_band, int32_t w, int32_t rows, int32_t gt,
                                       int32_t gb, int32_t row0, int32_t height, int32_t *out) {
  return mgpu_has_depressions(comm, d_band, w, rows, gt, gb, row0, height, out, true);
}

int rdb200_mgpu_resolve_flats_epsilon_f64(const rdb200_comm *comm, double *d_band, int32_t w, int32_t rows, double nodata,
                                          int32_t gt, int32_t gb, int32_t *seam_iterations) {
  return mgpu_resolve_flats_epsilon(comm, d_band, w, rows, nodata, gt, gb, seam_iterations);
}

int rdb200_mgpu_d8_flow_directions_flats_f64(const rdb200_comm *comm, double *d_band_dem, uint8_t *d_band_dirs, int32_t w,
                                             int32_t rows, double nodata, int32_t gt, int32_t gb, int32_t alter,
                                             int32_t *seam_iterations) {
  return mgpu_d8_flow_directions_flats(comm, d_band_dem, d_band_dirs, w, rows, nodata, gt, gb, alter, seam_iterations);
}

int rdb200_mgpu_fm_method_f64(const rdb200_comm *comm, int32_t method, double *d_band_dem, float *d_band_props9, int32_t w,
                              int32_t rows, double nodata, int32_t gt, int32_t gb, double xparam) {
  return mgpu_fm_method(comm, method, d_band_dem, d_band_props9, w, rows, nodata, gt, gb, xparam);
}

int rdb200_mgpu_terrain_attribute_f64(const rdb200_comm *comm, int32_t attribute, double *d_band_dem, float *d_band_out, int32_t w,
                                      int32_t rows, double nodata_in, float nodata_out, float zscale, double cell_x, double cell_y,
                                      int32_t gt, int32_t gb) {
  return mgpu_terrain_attribute(comm, attribute, d_band_dem, d_band_out, w, rows, nodata_in, nodata_out, zscale, cell_x,
                                cell_y, gt, gb);
}

int rdb200_mgpu_fa_method_f64_f64(const rdb200_comm *comm, const double *d_dem, double *d_accum, int32_t w, int32_t rows,
                                  double nodata, int32_t gt, int32_t gb, int32_t method, double xparam, int32_t ones,
                                  int32_t *exchange_rounds) {
  return mgpu_fa_method(comm, d_dem, d_accum, w, rows, nodata, gt, gb, method, xparam, ones, exchange_rounds);
}

int rdb200_mgpu_f64_order_keys(const rdb200_comm *comm, const double *d_band, float *d_band_keys, int32_t w, int32_t rows,
                               double nodata, int32_t gt, int32_t gb, float *nodata_key, int32_t *ranked) {
  float nd = 0;
  int r = 0;
  const int rc = raster_call(
      Side::device, "mgpu_f64_order_keys: null pointer", {comm, d_band, d_band_keys}, w, rows,
      [&] { check_band_args("mgpu_f64_order_keys", comm, d_band, w, rows, gt, gb); },
      [&](Arrays &, size_t) { nd = mgpu_f64_keys_dev(comm, d_band, d_band_keys, w, rows, gt, gb, nodata, nullptr, &r); });
  if (rc == 0 && nodata_key) *nodata_key = nd;
  if (rc == 0 && ranked) *ranked = r;
  return rc;
}

}  // extern "C"
