// Depression masks and depression tests: pit_mask<topo> (reference depressions/Barnes2014.hpp:593-676, app
// rd_depressions_mask) and HasDepressions<topo> (:43-104, app rd_depressions_has), on one GPU and over row bands.
//
// Both reduce to the fill this library already has.  Let L be the Priority-Flood fill of Z (NoData an ordinary value,
// as in FillDepressions) with the topology's neighbourhood.  The reference pops cells in non-decreasing level, and the
// first cell to discover an interior cell c has level min over c's neighbours n of L(n), so L(c) = max(Z(c), that
// level).  pit_mask writes 1 where Z(c) is below its discoverer's level, i.e. where Z(c) < L(c); 0 where Z(c) is above
// it; nothing where they are equal and nothing on the raster's edge; and 3 on every cell that is NoData (Z == nodata),
// edge cells included.  The output starts as resize() leaves it, all 0 (common/Array2D.hpp:852-872), so the mask is
//     3 if Z == nodata,  else 1 if Z < L,  else 0
// cell by cell, whatever order the reference's queues took.  HasDepressions returns true as soon as it discovers a cell
// lower than the cell that discovers it.  That happens iff some cell has Z < L: with no such event every cell is reached
// along a path that never descends, so L == Z everywhere; and the first such event finds a cell that no path at or
// below its own height connects to the edge (the flood would have reached it from that path first), so its Z < L.
//
// Hot path: one fill of a scratch copy of Z (the caller's raster is not modified) and one fused pass over Z and L that
// writes the uint8 mask and raises a device "any depression" flag (4 + 4 + 1 B per cell).  HasDepressions first runs a
// stencil pass that looks for a strict pit (below), and fills only when it finds none.
#include "common.cuh"

namespace rdb {

namespace {

constexpr int PIT_ROWS = 64;  // rows one block of the strict-pit pass walks down

// mask[i] = 3 / 1 / 0 as above (mask may be null: flag only); *any = 1 if some Z < L.  The water surface L is 4-byte
// aligned float data like Z, so when the three pointers allow it four cells move per load.
__global__ void __launch_bounds__(256) pit_mask_kernel(const float *__restrict__ Z, const float *__restrict__ L,
                                                       uint8_t *__restrict__ mask, size_t n, size_t n4, float nodata,
                                                       int *__restrict__ any) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int found = 0;
  for (size_t q = t; q < n4; q += stride) {
    const float4 z = reinterpret_cast<const float4 *>(Z)[q];
    const float4 l = reinterpret_cast<const float4 *>(L)[q];
    const int p0 = z.x < l.x, p1 = z.y < l.y, p2 = z.z < l.z, p3 = z.w < l.w;
    found |= p0 | p1 | p2 | p3;
    if (mask) {
      uchar4 m;
      m.x = z.x == nodata ? 3 : p0;
      m.y = z.y == nodata ? 3 : p1;
      m.z = z.z == nodata ? 3 : p2;
      m.w = z.w == nodata ? 3 : p3;
      reinterpret_cast<uchar4 *>(mask)[q] = m;
    }
  }
  for (size_t i = 4 * n4 + t; i < n; i += stride) {
    const float z = Z[i];
    const int p = z < L[i];
    found |= p;
    if (mask) mask[i] = z == nodata ? 3 : p;
  }
  if (__syncthreads_or(found) && threadIdx.x == 0) *any = 1;
}

// Strict pits.  *flag = 1 if some interior cell (1 <= x <= W-2, 1 <= y <= H-2) is strictly lower than each of its 8
// (D8) or 4 (D4: W, N, E, S, the reference's d4x / d4y of common/constants.hpp) neighbours, every value compared as the
// fill sees it (NoData cells at their NoData value, +-inf as themselves; a NaN neighbour makes no pit).
//
// Such a cell c is a depression for the reference: c is not on the edge, so some neighbour p discovers it, and p's
// level is at least Z(p) > Z(c) -- HasDepressions returns true there (Z(c) < Z(p) is exactly its test), and
// L(c) >= min over neighbours of Z(n) > Z(c).  So a pit found here never turns a "false" into "true".  The converse
// does not hold -- an enclosed flat-bottomed basin has no strict pit -- which is why a "no" from this pass still needs
// the fill.  The reference does not look at NoData in HasDepressions, and neither does this test: a NoData cell that is
// a strict pit is a depression to it like any other.
//
// One thread per column walks PIT_ROWS rows of a block's strip with a three-row window in registers; the left and right
// neighbours are the adjacent threads' loads (L1 hits).  Blocks stop early once another block has found a pit.
// T is float, or double for the float64 entry points (f64.cu), which compare their doubles directly here.
template <bool TOPO4, class T>
__global__ void __launch_bounds__(256) strict_pit_kernel(const T *__restrict__ Z, int W, int H, int *flag) {
  const int x = 1 + blockIdx.x * blockDim.x + threadIdx.x;
  const int strips = (H - 2 + PIT_ROWS - 1) / PIT_ROWS;
  int found = 0;
  if (x <= W - 2) {
    for (int s = blockIdx.y; s < strips && !found; s += gridDim.y) {
      if (*(volatile int *)flag) break;
      const int y0 = 1 + s * PIT_ROWS, y1 = y0 + PIT_ROWS < H - 1 ? y0 + PIT_ROWS : H - 1;
      const T *r = Z + (size_t)(y0 - 1) * W + x;
      T ul = r[-1], uc = r[0], ur = r[1];
      r += W;
      T cl = r[-1], cc = r[0], cr = r[1];
      for (int y = y0; y < y1; y++) {
        r += W;
        const T dl = r[-1], dc = r[0], dr = r[1];
        bool pit = cc < cl && cc < cr && cc < uc && cc < dc;
        if (!TOPO4) pit = pit && cc < ul && cc < ur && cc < dl && cc < dr;
        found |= pit;
        ul = cl, uc = cc, ur = cr;
        cl = dl, cc = dc, cr = dr;
      }
    }
  }
  if (__syncthreads_or(found) && threadIdx.x == 0) *flag = 1;
}

int read_flag(const int *d_flag) {
  Ctx &c = ctx();
  int *h = (int *)c.pinned;
  RDB_CK(cudaMemcpyAsync(h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  return *h;
}

}  // namespace

// mask (may be null) and *d_any (device; OR-ed into) of rows already filled: Z and L of n cells
void pit_mask_compare_dev(const float *d_z, const float *d_l, uint8_t *d_mask, size_t n, float nodata, int *d_any) {
  Ctx &c = ctx();
  if (n == 0) return;
  const bool vec = ((uintptr_t)d_z & 15) == 0 && ((uintptr_t)d_l & 15) == 0 && ((uintptr_t)d_mask & 3) == 0;
  const size_t n4 = vec ? n / 4 : 0;
  const size_t work = vec ? n4 + (n & 3) : n;
  const size_t want = (work + 255) / 256, cap = (size_t)c.num_sms * 8;
  pit_mask_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, c.stream>>>(d_z, d_l, d_mask, n, n4, nodata, d_any);
  RDB_CK(cudaGetLastError());
  count_launch();
}

// strict-pit pass over a w x h raster whose first and last rows and columns are not tested; OR-ed into *d_flag
template <class T>
void strict_pit_dev(const T *d_z, int w, int h, bool topo4, int *d_flag) {
  Ctx &c = ctx();
  if (w < 3 || h < 3) return;
  const int strips = (h - 2 + PIT_ROWS - 1) / PIT_ROWS;
  dim3 blk(256), grd((unsigned)((w - 2 + 255) / 256), (unsigned)(strips < 65535 ? strips : 65535));
  if (topo4) strict_pit_kernel<true, T><<<grd, blk, 0, c.stream>>>(d_z, w, h, d_flag);
  else strict_pit_kernel<false, T><<<grd, blk, 0, c.stream>>>(d_z, w, h, d_flag);
  RDB_CK(cudaGetLastError());
  count_launch();
}
template void strict_pit_dev(const float *, int, int, bool, int *);
template void strict_pit_dev(const double *, int, int, bool, int *);

// L = the fill of d_dem, in a scratch copy (the fill relaxes its water surface in the raster it is handed)
static void fill_copy_dev(const float *d_dem, float *d_l, int w, int h, bool topo4) {
  Ctx &c = ctx();
  RDB_CK(cudaMemcpyAsync(d_l, d_dem, (size_t)w * h * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  fill_depressions_dev(d_l, w, h, topo4);
}

void pit_mask_dev(const float *d_dem, uint8_t *d_mask, int w, int h, float nodata, bool topo4) {
  const size_t n = (size_t)w * h;
  DevBuf<float> l(n);
  DevBuf<int> any(1);
  RDB_CK(cudaMemsetAsync(any.p, 0, sizeof(int), ctx().stream));
  fill_copy_dev(d_dem, l.p, w, h, topo4);
  pit_mask_compare_dev(d_dem, l.p, d_mask, n, nodata, any.p);
  ctx().stats.cells = (int64_t)n;
}

// pit_mask of a double raster: pit_mask of its keys, with kappa(nodata)
void pit_mask_dev(const double *d_z, uint8_t *d_mask, int w, int h, double nodata, bool topo4) {
  const size_t n = (size_t)w * h;
  DevBuf<float> key(n);
  const float nd = f64_keys_dev(d_z, key.p, n, nodata, nullptr, nullptr);
  pit_mask_dev(key.p, d_mask, w, h, nd, topo4);
}

// the strict-pit pass on d_z into a zeroed *d_flag: a strict pit answers HasDepressions alone
template <class T>
static bool strict_pit_found(const T *d_z, int w, int h, bool topo4, int *d_flag) {
  RDB_CK(cudaMemsetAsync(d_flag, 0, sizeof(int), ctx().stream));
  strict_pit_dev(d_z, w, h, topo4, d_flag);
  return read_flag(d_flag) != 0;
}

// HasDepressions when no strict pit was found: whether the fill of d_dem raises a cell (OR-ed into *d_flag)
static bool fill_raises(const float *d_dem, int w, int h, bool topo4, int *d_flag) {
  const size_t n = (size_t)w * h;
  DevBuf<float> l(n);
  fill_copy_dev(d_dem, l.p, w, h, topo4);
  pit_mask_compare_dev(d_dem, l.p, nullptr, n, 0.f, d_flag);
  ctx().stats.cells = (int64_t)n;
  return read_flag(d_flag) != 0;
}

bool has_depressions_dev(const float *d_dem, int w, int h, bool topo4) {
  DevBuf<int> flag(1);
  if (strict_pit_found(d_dem, w, h, topo4, flag.p)) return true;
  if (w < 3 || h < 3) return false;  // every cell is an edge cell
  return fill_raises(d_dem, w, h, topo4, flag.p);
}

// HasDepressions of a double raster: strict pits of the doubles (no keys needed), then the fill of the keys
bool has_depressions_dev(const double *d_z, int w, int h, bool topo4) {
  DevBuf<int> flag(1);
  if (strict_pit_found(d_z, w, h, topo4, flag.p)) return true;
  if (w < 3 || h < 3) return false;
  DevBuf<float> key((size_t)w * h);
  f64_keys_dev(d_z, key.p, (size_t)w * h, 0.0, nullptr, nullptr);
  return fill_raises(key.p, w, h, topo4, flag.p);
}

// ---- row bands ---------------------------------------------------------------------------------------------------
// The band fill runs on a copy of the local raster (mgpu_fill_band ignores the ghost rows on entry), so d_band is not
// modified; the compare then runs on the owned rows.  A raster without interior cells is its own fill (no band fill:
// every rank sees the same width and height, so all skip it together).
void check_mask_band(const char *what, const rdb200_comm *comm, const void *d_band, int w, int hloc, int gt, int gb, int row0,
                     int H) {
  check_band_args(what, comm, d_band, w, hloc, gt, gb);
  if (row0 < 0 || row0 + hloc > H) fail("%s: rows [%d, %d) are outside the raster (%d rows)", what, row0, row0 + hloc, H);
  if (w >= 3 && H >= 3 && hloc < 3) fail("%s: band too small (%d x %d); the band fill needs three local rows", what, w, hloc);
}

void mgpu_pit_mask_band(const rdb200_comm *comm, const float *d_band, uint8_t *d_mask, int w, int hloc, float nodata, int gt,
                        int gb, int row0, int H, bool topo4) {
  check_mask_band("mgpu_pit_mask", comm, d_band, w, hloc, gt, gb, row0, H);
  if (!d_mask) fail("mgpu_pit_mask: null pointer");
  Ctx &c = ctx();
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  const size_t n = (size_t)w * hloc, own = (size_t)w * (hloc - gt - gb), off = (size_t)w * gt;
  DevBuf<float> l(n);
  DevBuf<int> any(1);
  RDB_CK(cudaMemsetAsync(any.p, 0, sizeof(int), c.stream));
  RDB_CK(cudaMemcpyAsync(l.p, d_band, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  if (w >= 3 && H >= 3) mgpu_fill_band(comm, l.p, w, hloc, gt, gb, row0, H, nullptr, topo4);
  pit_mask_compare_dev(d_band + off, l.p + off, d_mask + off, own, nodata, any.p);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// 1. strict pits of the owned rows, on a copy whose ghost rows hold the neighbours' edge rows (a local edge row is a
//    ghost row or a raster edge row, neither of which this rank tests); 2. one OR (MAX) all-reduce; 3. only if no rank
//    found one, the band fill and the compare of the owned rows, and a second all-reduce.
bool mgpu_has_depressions_band(const rdb200_comm *comm, const float *d_band, int w, int hloc, int gt, int gb, int row0, int H,
                               bool topo4) {
  check_mask_band("mgpu_has_depressions", comm, d_band, w, hloc, gt, gb, row0, H);
  Ctx &c = ctx();
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  const size_t n = (size_t)w * hloc, own = (size_t)w * (hloc - gt - gb), off = (size_t)w * gt;
  DevBuf<float> l(n);
  DevBuf<int> flag(1);
  RDB_CK(cudaMemsetAsync(flag.p, 0, sizeof(int), c.stream));
  RDB_CK(cudaMemcpyAsync(l.p, d_band, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  exchange_band_rows(comm, l.p, sizeof(float), w, hloc, gt, gb);
  strict_pit_dev(l.p, w, hloc, topo4, flag.p);
  comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
  if (read_flag(flag.p)) return true;
  if (w < 3 || H < 3) return false;
  mgpu_fill_band(comm, l.p, w, hloc, gt, gb, row0, H, nullptr, topo4);
  pit_mask_compare_dev(d_band + off, l.p + off, nullptr, own, 0.f, flag.p);
  comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
  return read_flag(flag.p) != 0;
}

}  // namespace rdb
