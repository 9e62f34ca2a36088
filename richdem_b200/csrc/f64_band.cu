// float64 rasters over row bands (DESIGN §0.1 "kappa over row bands", §4): the float32 band drivers on kappa_G, the key
// map every band shares (f64.cu), and the double instantiations of the flow metrics and terrain attributes on bands
// whose ghost rows were exchanged.  Every driver checks its arguments before its first collective, as its float32
// twin does, and no key of a ghost row is computed locally: a ghost value need not be in the band's own table, so the
// ghost keys are the neighbours' owned keys (mgpu_f64_keys_dev exchanges them).
#include "common.cuh"

namespace rdb {

namespace {

__global__ void __launch_bounds__(256) fill_f64_kernel(double *__restrict__ a, size_t n, double v) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) a[i] = v;
}

// the band fill's geometry (mgpu_fill_band checks the same, but only after kappa_G has communicated)
void check_fill_band(const rdb200_comm *comm, const double *d_band, int w, int hloc, int gt, int gb, int row0, int H) {
  check_band_args("mgpu_fill", comm, d_band, w, hloc, gt, gb);
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  if (w < 3 || hloc - gt - gb < 1 || hloc < 3) fail("mgpu_fill: band too small (%d x %d)", w, hloc);
  if (row0 < 0 || row0 + hloc > H) fail("mgpu_fill: rows [%d, %d) are outside the raster (%d rows)", row0, row0 + hloc, H);
}

}  // namespace

// FillDepressions<D8 / D4>: kappa_G, the float32 band fill on the keys, kappa_G^-1 of the owned rows, and one exchange
// so that the ghost rows hold the neighbours' filled edge rows, as the float32 band fill leaves them
void mgpu_fill_band(const rdb200_comm *comm, double *d_band, int w, int hloc, int gt, int gb, int row0, int H, int *xrounds,
                    bool topo4) {
  check_fill_band(comm, d_band, w, hloc, gt, gb, row0, H);
  Ctx &c = ctx();
  const size_t n = (size_t)w * hloc;
  DevBuf<float> k0(n), kf(n);
  BandKeys inv;
  mgpu_f64_keys_dev(comm, d_band, k0.p, w, hloc, gt, gb, 0.0, &inv, nullptr);
  RDB_CK(cudaMemcpyAsync(kf.p, k0.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  mgpu_fill_band(comm, kf.p, w, hloc, gt, gb, row0, H, xrounds, topo4);
  mgpu_f64_writeback_dev(comm, inv, d_band, k0.p, kf.p, w, hloc, gt, gb);
  exchange_band_rows(comm, d_band, sizeof(double), w, hloc, gt, gb);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// pit_mask<D8 / D4>: the float32 band mask on the key band, with kappa_G(nodata)
void mgpu_pit_mask_band(const rdb200_comm *comm, const double *d_band, uint8_t *d_mask, int w, int hloc, double nodata, int gt,
                        int gb, int row0, int H, bool topo4) {
  check_mask_band("mgpu_pit_mask", comm, d_band, w, hloc, gt, gb, row0, H);
  if (!d_mask) fail("mgpu_pit_mask: null pointer");
  DevBuf<float> k(static_cast<size_t>(w) * hloc);
  const float nd = mgpu_f64_keys_dev(comm, d_band, k.p, w, hloc, gt, gb, nodata, nullptr, nullptr);
  mgpu_pit_mask_band(comm, k.p, d_mask, w, hloc, nd, gt, gb, row0, H, topo4);
}

// HasDepressions<D8 / D4>: strict pits of the doubles first (no keys needed), as the float32 driver does; only if no
// rank finds one, kappa_G, the band fill on the keys and the compare of the owned rows
bool mgpu_has_depressions_band(const rdb200_comm *comm, const double *d_band, int w, int hloc, int gt, int gb, int row0, int H,
                               bool topo4) {
  check_mask_band("mgpu_has_depressions", comm, d_band, w, hloc, gt, gb, row0, H);
  Ctx &c = ctx();
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  const size_t n = (size_t)w * hloc, own = (size_t)w * (hloc - gt - gb), off = (size_t)w * gt;
  DevBuf<int> flag(1);
  RDB_CK(cudaMemsetAsync(flag.p, 0, sizeof(int), c.stream));
  {
    DevBuf<double> z(n);
    RDB_CK(cudaMemcpyAsync(z.p, d_band, n * sizeof(double), cudaMemcpyDeviceToDevice, c.stream));
    exchange_band_rows(comm, z.p, sizeof(double), w, hloc, gt, gb);
    strict_pit_dev(z.p, w, hloc, topo4, flag.p);
  }
  comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
  if (read_i32(flag.p)) return true;
  if (w < 3 || H < 3) return false;
  DevBuf<float> k0(n), l(n);
  mgpu_f64_keys_dev(comm, d_band, k0.p, w, hloc, gt, gb, 0.0, nullptr, nullptr);
  RDB_CK(cudaMemcpyAsync(l.p, k0.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  mgpu_fill_band(comm, l.p, w, hloc, gt, gb, row0, H, nullptr, topo4);
  pit_mask_compare_dev(k0.p + off, l.p + off, nullptr, own, 0.f, flag.p);
  comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
  return read_i32(flag.p) != 0;
}

// ResolveFlatsEpsilon: the float32 band flats on kappa_G return the increment mask, which the owned doubles take as
// ulps; then one exchange puts the neighbours' resolved edge rows in the ghost rows, as the float32 call leaves them
void mgpu_resolve_flats_band(const rdb200_comm *comm, double *d_band, int w, int hloc, double nodata, int gt, int gb,
                             int *seam_iters) {
  check_band_args("mgpu_resolve_flats", comm, d_band, w, hloc, gt, gb);
  Ctx &c = ctx();
  const size_t n = (size_t)w * hloc;
  DevBuf<float> k(n);
  DevBuf<int32_t> mask(n);
  const float nd = mgpu_f64_keys_dev(comm, d_band, k.p, w, hloc, gt, gb, nodata, nullptr, nullptr);
  mgpu_resolve_flats_band(comm, k.p, w, hloc, nd, gt, gb, seam_iters, mask.p);
  f64_apply_ulps_dev(d_band, mask.p, w, hloc);  // local rows 1 .. hloc-2: the owned rows, less the raster's edge rows
  exchange_band_rows(comm, d_band, sizeof(double), w, hloc, gt, gb);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// barnes_flat_resolution_d8<double> over row bands: the plain directions come from the doubles (their ghost rows hold the
// neighbours' edge rows on entry, as the band fill leaves them), the flats of those directions are resolved by the
// float32 band protocol on kappa_G, and then either d8_flow_flats (alter = 0) or the float steps of d8_flats_alter_dem on
// the owned rows, one exchange of the altered edge rows and the directions of the doubles again (alter = 1).  On return
// the ghost rows of d_dirs (and, with alter = 1, of d_band) hold the neighbours' edge rows, as in the float32 driver.
void mgpu_d8_flow_directions_flats_band(const rdb200_comm *comm, double *d_band, uint8_t *d_dirs, int w, int hloc, double nodata,
                                        int gt, int gb, bool alter, int *seam_iters) {
  const char *what = "mgpu_d8_flow_directions_flats";
  if (!d_dirs) fail("%s: null pointer", what);
  check_band_args(what, comm, d_band, w, hloc, gt, gb);
  Ctx &c = ctx();
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  const size_t n = (size_t)w * hloc;
  DevBuf<float> k(n);
  const float nd = mgpu_f64_keys_dev(comm, d_band, k.p, w, hloc, gt, gb, nodata, nullptr, nullptr);
  d8_flow_directions_dev(d_band, d_dirs, w, hloc, nodata);
  DevBuf<int32_t> mask(alter ? n : 0);
  const int iters = mgpu_dir_flats_band(comm, k.p, d_dirs, w, hloc, nd, gt, gb, alter, alter ? mask.p : nullptr);
  k.reset();
  if (alter) {
    f64_float_steps_dev(d_band, mask.p, w, hloc);  // local rows 1 .. hloc-2: the owned rows, less the raster's edge rows
    exchange_band_rows(comm, d_band, sizeof(double), w, hloc, gt, gb);
    d8_flow_directions_dev(d_band, d_dirs, w, hloc, nodata);
  }
  exchange_band_rows(comm, d_dirs, 1, w, hloc, gt, gb);
  RDB_CK(cudaStreamSynchronize(c.stream));
  if (seam_iters) *seam_iters = iters;
}

// FlowAccumulation of a double band.  Methods 0 (D8) and 2 (D4) compare elevations only: the float32 band accumulation
// on kappa_G.  The others compute with them: the double flow metric on a copy of the band whose ghost rows hold the
// neighbours' edge rows, then the band accumulation of those proportions.  The caller's ghost rows are not read.
void mgpu_fa_band(const rdb200_comm *comm, const double *d_dem, double *d_accum, int w, int hloc, double nodata, int gt, int gb,
                  int method, double xparam, bool ones, int *xrounds) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * hloc;
  if (method == 0 || method == 2) {
    DevBuf<float> k(n);
    const float nd = mgpu_f64_keys_dev(comm, d_dem, k.p, w, hloc, gt, gb, nodata, nullptr, nullptr);
    mgpu_fa_band(comm, k.p, d_accum, w, hloc, nd, gt, gb, method, 0.0, ones, xrounds);
    return;
  }
  DevBuf<float> props(9 * n);
  {
    DevBuf<double> z(n);
    RDB_CK(cudaMemcpyAsync(z.p, d_dem, n * sizeof(double), cudaMemcpyDeviceToDevice, c.stream));
    exchange_band_rows(comm, z.p, sizeof(double), w, hloc, gt, gb);
    fm_method_dev(method, z.p, props.p, w, hloc, nodata, xparam);
  }
  if (ones) {
    const size_t want = (n + 255) / 256, cap = (size_t)c.num_sms * 8;
    fill_f64_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, c.stream>>>(d_accum, n, 1.0);
    RDB_CK(cudaGetLastError());
    count_launch();
  }
  mgpu_flow_accumulation_props_band(comm, props.p, d_accum, w, hloc, gt, gb, xrounds);
}

}  // namespace rdb
