// Per-cell flow-direction / flow-proportion kernels (pure 3x3 stencils, HBM-bound):
//   d8_flow_directions  (reference flowmet/d8_flowdirs.hpp:96-123)      4 B in, 1 B out per cell
//   FM_D8               (reference flowmet/OCallaghan1984.hpp:13-84)    4 B in, 36 B out
//   FM_Tarboton         (reference flowmet/Tarboton1997.hpp:14-149)     4 B in, 36 B out
//   FM_D4               (reference flowmet/OCallaghan1984.hpp:13-77,89-91)
//   FM_Holmgren / FM_Quinn / FM_Freeman (reference flowmet/Holmgren1994.hpp:13-83, Quinn1991.hpp:12-16,
//                        Freeman1991.hpp:13-80)                         4 B in, 36 B out
// Neighbour reads go through the read-only path; a warp covers 32 consecutive cells of a row so
// the three row segments it touches are fetched once from HBM and re-used from L1/L2.
#include "flowmet.cuh"

namespace rdb {

namespace {

// d8_FlowDir, flowmet/d8_flowdirs.hpp:32-74; T is float, or double for rdb200_d8_flow_directions_f64
template <class T>
__global__ void d8_flowdirs_kernel(const T *__restrict__ dem, uint8_t *__restrict__ dirs, int W, int H, T nodata) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const size_t i = (size_t)y * W + x;
    const T e = __ldg(dem + i);
    uint8_t d;
    if (e == nodata) {  // :117-118
      d = 255;
    } else if (x == 0 || y == 0 || x == W - 1 || y == H - 1) {  // :36-54
      if (x == 0 && y == 0) d = 2;
      else if (x == 0 && y == H - 1) d = 8;
      else if (x == W - 1 && y == 0) d = 4;
      else if (x == W - 1 && y == H - 1) d = 6;
      else if (x == 0) d = 1;
      else if (x == W - 1) d = 5;
      else if (y == 0) d = 3;
      else d = 7;
    } else {
      T minimum = e;
      int flowdir = 0;
#pragma unroll
      for (int n = 1; n <= 8; n++) {  // :63-71 (NoData neighbours are NOT skipped here)
        const T ne = __ldg(dem + (size_t)(y + d8dy(n)) * W + (x + d8dx(n)));
        if (ne < minimum || (ne == minimum && flowdir > 0 && (flowdir & 1) == 0 && (n & 1) == 1)) {
          minimum = ne;
          flowdir = n;
        }
      }
      d = (uint8_t)flowdir;
    }
    dirs[i] = d;
  }
}

// Rolling-window variant (flowdirs_rolling = 1, W % 4 == 0): a thread owns 4 columns and walks down a
// chunk of rows keeping three DEM rows in registers, so every row is fetched once per block (one
// float4 per thread, the two halo columns by shuffle) instead of nine scalar loads per cell; the
// direction bytes leave as uchar4.  Same per-cell rule as above.
constexpr int kDirRows = 64;

__global__ void __launch_bounds__(256) d8_flowdirs_rolling_kernel(const float *__restrict__ dem, uint8_t *__restrict__ dirs,
                                                                   int W, int H, float nodata) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int xc = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const bool col_in = xc < W;
  const int y0 = blockIdx.y * kDirRows;
  float d[3][6];  // rows y-1, y, y+1 ; columns xc-1 .. xc+4
  auto load_row = [&](int gy, float(&o)[6]) {
    const bool rin = gy >= 0 && gy < H;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rin && col_in) m = __ldg(reinterpret_cast<const float4 *>(dem + (size_t)gy * W + xc));
    float left = __shfl_up_sync(full, m.w, 1), right = __shfl_down_sync(full, m.x, 1);
    if (lane == 0) left = (rin && col_in && xc > 0) ? __ldg(dem + (size_t)gy * W + xc - 1) : 0.f;
    if (lane == 31) right = (rin && xc + 4 < W) ? __ldg(dem + (size_t)gy * W + xc + 4) : 0.f;
    o[0] = left; o[1] = m.x; o[2] = m.y; o[3] = m.z; o[4] = m.w; o[5] = right;
  };
  load_row(y0 - 1, d[0]);
  load_row(y0, d[1]);
  for (int y = y0; y < y0 + kDirRows && y < H; y++) {  // uniform across the block
    load_row(y + 1, d[2]);
    if (col_in) {
      uint8_t out[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int x = xc + k;
        const float e = d[1][k + 1];
        int dd;
        if (e == nodata) {
          dd = 255;
        } else if (x == 0 || y == 0 || x == W - 1 || y == H - 1) {
          if (x == 0 && y == 0) dd = 2;
          else if (x == 0 && y == H - 1) dd = 8;
          else if (x == W - 1 && y == 0) dd = 4;
          else if (x == W - 1 && y == H - 1) dd = 6;
          else if (x == 0) dd = 1;
          else if (x == W - 1) dd = 5;
          else if (y == 0) dd = 3;
          else dd = 7;
        } else {
          // neighbours n = 1..8 : W, NW, N, NE, E, SE, S, SW
          const float ne[9] = {0.f, d[1][k], d[0][k], d[0][k + 1], d[0][k + 2], d[1][k + 2], d[2][k + 2], d[2][k + 1], d[2][k]};
          float minimum = e;
          int flowdir = 0;
#pragma unroll
          for (int n = 1; n <= 8; n++) {
            if (ne[n] < minimum || (ne[n] == minimum && flowdir > 0 && (flowdir & 1) == 0 && (n & 1) == 1)) {
              minimum = ne[n];
              flowdir = n;
            }
          }
          dd = flowdir;
        }
        out[k] = (uint8_t)dd;
      }
      *reinterpret_cast<uchar4 *>(dirs + (size_t)y * W + xc) = make_uchar4(out[0], out[1], out[2], out[3]);
    }
#pragma unroll
    for (int k = 0; k < 6; k++) {
      d[0][k] = d[1][k];
      d[1][k] = d[2][k];
    }
  }
}

// materialised proportions: 256 cells per block staged through shared memory so the 36 B/cell
// AoS output leaves as coalesced float4 stores
// MODE: 0 FM_D8, 1 FM_Tarboton, 2 FM_D4, 3 FM_Holmgren (FM_Quinn = exponent 1), 4 FM_Freeman
enum : int { FM_MODE_D8 = 0, FM_MODE_DINF = 1, FM_MODE_D4 = 2, FM_MODE_HOLMGREN = 3, FM_MODE_FREEMAN = 4 };

// T: float, or double for the rdb200_fm_*_f64 entry points (8 B in per cell instead of 4)
template <int MODE, class T>
__global__ void __launch_bounds__(256) fm_props_kernel(const T *__restrict__ dem, float *__restrict__ props,
                                                        int W, int H, T nodata, double xparam, int tfilter) {
  constexpr bool DINF = MODE == FM_MODE_DINF;
  __shared__ __align__(16) float s[256 * 9];
  const size_t n = (size_t)W * H;
  const size_t base = (size_t)blockIdx.x * 256;
  const size_t i = base + threadIdx.x;
  float p[9];
#pragma unroll
  for (int k = 0; k < 9; k++) p[k] = kNoFlowGen;
  if (i < n) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    if (DINF) {
      float rmax = 0;
      const int nm = fm_tarboton_cell(dem, x, y, W, H, nodata, &rmax, tfilter != 0);
      if (nm == kCodeNoData) {
        p[0] = kNoDataGen;
      } else if (nm > 0) {
        p[0] = kHasFlowGen;
        const int nn = nwrap(nm + 1);
        float p1 = 0, p2 = 0;
        int n1 = 0, n2 = 0;  // slots to write
        if (rmax == 0.0f) {
          n1 = nm;
          p1 = 1.0f;
        } else if (rmax == kDang) {
          n1 = nn;
          p1 = 1.0f;
        } else {
          tarboton_props(rmax, &p1, &p2);
          n1 = nm;
          n2 = nn;
        }
#pragma unroll
        for (int k = 1; k <= 8; k++) {
          if (k == n1) p[k] = p1;
          if (k == n2) p[k] = p2;
        }
      }
    } else if (MODE == FM_MODE_D4) {
      const int c = fm_d4_cell(dem, x, y, W, H, nodata);
      if (c == kCodeNoData) {
        p[0] = kNoDataGen;
      } else if (c > 0) {
        p[0] = kHasFlowGen;
#pragma unroll
        for (int k = 1; k <= 4; k++)
          if (k == c) p[k] = 1.0f;
      }
    } else if (MODE == FM_MODE_HOLMGREN || MODE == FM_MODE_FREEMAN) {
      fm_mfd_cell<MODE == FM_MODE_HOLMGREN>(dem, x, y, W, H, nodata, xparam, p);
    } else {
      const int c = fm_d8_cell(dem, x, y, W, H, nodata);
      if (c == kCodeNoData) {
        p[0] = kNoDataGen;
      } else if (c > 0) {
        p[0] = kHasFlowGen;
#pragma unroll
        for (int k = 1; k <= 8; k++)
          if (k == c) p[k] = 1.0f;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 9; k++) s[threadIdx.x * 9 + k] = p[k];
  __syncthreads();
  const size_t cells_here = (base + 256 <= n) ? 256 : (n > base ? n - base : 0);
  const size_t floats_here = cells_here * 9;
  float *out = props + base * 9;  // 256*36 B per block keeps float4 alignment
  if (cells_here == 256) {
    const float4 *s4 = reinterpret_cast<const float4 *>(s);
    float4 *o4 = reinterpret_cast<float4 *>(out);
    for (int k = threadIdx.x; k < 256 * 9 / 4; k += 256) __stcs(o4 + k, s4[k]);
  } else {
    for (size_t k = threadIdx.x; k < floats_here; k += 256) out[k] = s[k];
  }
}

}  // namespace

void d8_flow_directions_dev(const float *d_dem, uint8_t *d_dirs, int w, int h, float nodata) {
  Ctx &c = ctx();
  if (c.params.flowdirs_rolling && (w & 3) == 0 && ((uintptr_t)d_dem & 15) == 0 && ((uintptr_t)d_dirs & 3) == 0) {
    dim3 blk(256), grd((unsigned)((w / 4 + 255) / 256), (unsigned)((h + kDirRows - 1) / kDirRows));
    d8_flowdirs_rolling_kernel<<<grd, blk, 0, c.stream>>>(d_dem, d_dirs, w, h, nodata);
  } else {
    dim3 blk(128), grd((w + 127) / 128, h < 16384 ? h : 16384);
    d8_flowdirs_kernel<float><<<grd, blk, 0, c.stream>>>(d_dem, d_dirs, w, h, nodata);
  }
  RDB_CK(cudaGetLastError());
  count_launch();
}

// the same rule on doubles, compared as doubles (one 8 B load per cell and neighbour, 1 B out)
void d8_flow_directions_dev(const double *d_dem, uint8_t *d_dirs, int w, int h, double nodata) {
  Ctx &c = ctx();
  dim3 blk(128), grd((w + 127) / 128, h < 16384 ? h : 16384);
  d8_flowdirs_kernel<double><<<grd, blk, 0, c.stream>>>(d_dem, d_dirs, w, h, nodata);
  RDB_CK(cudaGetLastError());
  count_launch();
}

template <int MODE, class T>
static void fm_launch(const T *d_dem, float *d_props, int w, int h, T nodata, double xparam) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  fm_props_kernel<MODE, T><<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d_dem, d_props, w, h, nodata, xparam,
                                                                           (int)c.params.flowmet_tarboton_filter);
  RDB_CK(cudaGetLastError());
  count_launch();
}

template <class T>
void fm_method_dev(int method, const T *d_dem, float *d_props, int w, int h, T nodata, double xparam) {
  switch (method) {
    case 0: fm_launch<FM_MODE_D8>(d_dem, d_props, w, h, nodata, 0.0); break;
    case 1: fm_launch<FM_MODE_DINF>(d_dem, d_props, w, h, nodata, 0.0); break;
    case 2: fm_launch<FM_MODE_D4>(d_dem, d_props, w, h, nodata, 0.0); break;
    case 3: fm_launch<FM_MODE_HOLMGREN>(d_dem, d_props, w, h, nodata, xparam); break;
    case 4: fm_launch<FM_MODE_FREEMAN>(d_dem, d_props, w, h, nodata, xparam); break;
    default: fail("unknown flow metric %d", method);
  }
}
template void fm_method_dev(int, const float *, float *, int, int, float, double);
template void fm_method_dev(int, const double *, float *, int, int, double, double);  // reference templates with E = double

}  // namespace rdb
